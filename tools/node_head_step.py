"""Device time of the node heads and their losses, forward + backward, captured in a CUDA graph, against the same head
and loss as the reference runs them in eager torch (GraphGym's MLP with F.normalize, then
graphgps/loss/weighted_cross_entropy.py's bincount / nonzero / unique weights or the masked cross-entropy).

    python tools/node_head_step.py [--iters 200] [--out results/node_head_step.json]

Shapes: PATTERN (inductive_node, L 3, d 64, C 2), VOC (L 3, d 96, C 21), COCO (L 3, d 96, C 81) and actor (node, L 1,
d 64, C 5, the train mask).  Prints the card's name and power limit with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import graphgps_b200  # noqa: E402

DEV = "cuda:0"
SHAPES = {   # name: (head, N, d, C, L, loss)
    "PATTERN": ("inductive_node", 32 * 118, 64, 2, 3, "weighted_cross_entropy"),
    "VOC": ("inductive_node", 32 * 480, 96, 21, 3, "weighted_cross_entropy"),
    "COCO": ("inductive_node", 32 * 480, 96, 81, 3, "weighted_cross_entropy"),
    "actor": ("node", 7600, 64, 5, 1, "cross_entropy"),
}


def reference_step(ours, x, y, mask, loss_fun):
    """The reference's head and loss in eager torch, on ours' parameters."""
    lins = [m for m in ours.modules() if isinstance(m, nn.Linear)]
    h = x
    for i, lin in enumerate(lins):
        h = lin(h)
        if i < len(lins) - 1:
            h = F.normalize(torch.relu(h), p=2, dim=1)
    pred, true = (h[mask], y[mask]) if mask is not None else (h, y)
    if loss_fun == "weighted_cross_entropy":   # weighted_cross_entropy.py
        V = true.size(0)
        n_classes = pred.shape[1]
        label_count = torch.bincount(true)
        label_count = label_count[label_count.nonzero(as_tuple=True)].squeeze()
        cluster_sizes = torch.zeros(n_classes, device=pred.device).long()
        cluster_sizes[torch.unique(true)] = label_count
        weight = (V - cluster_sizes).float() / V
        weight *= (cluster_sizes > 0).float()
        loss = F.nll_loss(F.log_softmax(pred, dim=-1), true, weight=weight)
    else:
        loss = F.nll_loss(F.log_softmax(pred, dim=-1), true)
    loss.backward()


def time_ms(fn, iters):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def measure(name, iters):
    head_kind, N, d, C, L, loss_fun = SHAPES[name]
    torch.manual_seed(0)
    cls = graphgps_b200.NodeHead if head_kind == "node" else graphgps_b200.InductiveNodeHead
    head = cls(d, C, layers_post_mp=L).to(DEV).train()
    x = torch.randn(N, d, device=DEV).requires_grad_(True)
    y = torch.randint(0, C, (N,), device=DEV)
    mask = (torch.rand(N, device=DEV) < 0.6) if head_kind == "node" else None
    data = type("B", (), {})()
    data.y, data.split, data.train_mask = y, "train", mask
    fn = graphgps_b200.weighted_cross_entropy if loss_fun == "weighted_cross_entropy" else graphgps_b200.cross_entropy

    def ours():
        data.x = x
        pred, true = head(data)
        loss, _ = fn(pred, true)
        loss.backward()

    ours()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ours()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ours()
    captured = time_ms(g.replay, iters)
    eager = time_ms(ours, iters)
    ref = time_ms(lambda: reference_step(head, x, y, mask, loss_fun), iters)
    return {"shape": name, "N": N, "d": d, "C": C, "L": L, "ours_captured_us": captured * 1e3,
            "ours_eager_us": eager * 1e3, "reference_eager_us": ref * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("node_head_step.py needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    res = {"card": card, "results": [measure(n, args.iters) for n in SHAPES]}
    for r in res["results"]:
        print(f"{r['shape']:8s} ours captured {r['ours_captured_us']:8.1f} us  eager {r['ours_eager_us']:8.1f} us  "
              f"reference eager {r['reference_eager_us']:8.1f} us")
    print("card:", card)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
