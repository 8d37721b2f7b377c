"""Cost of an L-layer SAN2 stack, forward + backward in training mode, at the shipped SAN configs' shapes.

    python tools/san2_step.py [--steps K] [--warmup W] [--rounds R] [--only zinc,coco]

Two legs, alternated round by round in the same process on the same GPU:
  * lib:   graphgps_b200.SAN2Layer x L (fp32-grade), captured into one CUDA graph per step and replayed;
  * torch: the reference's composition in eager torch fp32 - tests/san2_oracle.py's san2_forward per layer (pyg_softmax
           per set, the learned float64 gamma), with the complement edge set rebuilt in every layer by a per-graph loop
           with one host sync per graph, as the reference's negate_edge_index does (graphgps/utils.py:12-65).
Each leg's time is the median over rounds of the mean ms per step, from CUDA events around K steps.  The table also
gives the library's kernel launches per step, the card name and its power limit.
"""
import argparse
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import graphgps_b200  # noqa: E402
from graphgps_b200 import _call, _lib  # noqa: E402
from graphgps_b200.batch import GraphBatch  # noqa: E402
from graphgps_b200.graph import graph_of  # noqa: E402
from san2_oracle import san2_forward  # noqa: E402
from san_oracle import dataset_sizes, san_batch  # noqa: E402
from san_step import negate_edge_index_eager, power_limit, timed  # noqa: E402

DEV = "cuda:0"
# name, kind, graphs per batch, L, d, heads, dropout (configs/SAN/*.yaml shapes)
CONFIGS = [
    ("zinc", "mol", 32, 10, 56, 8, 0.0),
    ("pattern", "sbm", 16, 4, 80, 10, 0.0),
    ("molpcba", "mol", 512, 5, 304, 4, 0.2),
    ("coco", "knn", 8, 4, 88, 8, 0.0),
]


def setup(cfg):
    name, kind, B, L, d, H, p = cfg
    torch.manual_seed(0)
    emb = nn.Embedding(1, d)
    seq = nn.Sequential(*[graphgps_b200.SAN2Layer(0.1, d, d, H, True, emb, p) for _ in range(L)]).to(DEV)
    sb = san_batch(kind, dataset_sizes(kind, B, 0), d, 0).to(DEV)
    b = GraphBatch(x=sb.x, edge_index=sb.edge_index, edge_attr=sb.edge_attr, batch=sb.batch, num_graphs=B)
    graph_of(b).nmax
    x = sb.x.clone().requires_grad_(True)
    e = sb.edge_attr.clone().requires_grad_(True)
    ct = torch.randn(sb.x.shape, device=DEV)
    params = list(seq.parameters())

    def lib_step():
        b.x, b.edge_attr = x, e
        out = seq(b).x
        return torch.autograd.grad((out * ct).sum(), [x, e] + params)

    lib = _lib.load()
    lib_step()
    torch.cuda.synchronize()
    c0 = lib.gps_launch_count()
    lib_step()
    torch.cuda.synchronize()
    launches = lib.gps_launch_count() - c0
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            lib_step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, capture_error_mode="thread_local"):
        lib_step()
    torch.cuda.synchronize()

    # torch leg: the same parameters as leaves (fp32, gamma float64 as the reference keeps it), eager
    named = dict(seq.named_parameters())
    state = {k: v.detach().clone().requires_grad_(v.is_floating_point() and k in named)
             for k, v in seq.state_dict().items()}
    for li in range(1, L):
        state[f"{li}.attention.fake_edge_emb.weight"] = state["0.attention.fake_edge_emb.weight"]
    leaves = [t for t in state.values() if t.requires_grad]
    ei, bt = sb.edge_index, sb.batch

    def torch_step():
        h = x
        for li in range(L):
            fake = negate_edge_index_eager(ei, bt)
            masks = None
            if p > 0:
                masks = ((torch.rand(h.shape[0], d, device=DEV) >= p).float() / (1 - p),
                         (torch.rand(h.shape[0], 2 * d, device=DEV) >= p).float() / (1 - p))
            h = san2_forward(state, h, e, ei, fake, H, True, masks, f"{li}.")
        return torch.autograd.grad((h * ct).sum(), [x, e] + leaves)

    def replay():
        # The graph holds raw addresses of the layers' parameters (gamma included), their gradients and of the batch's
        # graph structure: this closure keeps all of them (seq, b, x, e, ct) alive for as long as the graph is replayed
        graph.replay()
        return seq, b, x, e, ct

    return replay, torch_step, launches, sb.x.shape[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("san2_step.py times the H100 path and needs a GPU")
    name = torch.cuda.get_device_name(0)
    print(f"card: {name}, power limit {power_limit()}")
    print(f"{'config':10s} {'N':>6s} {'L':>3s} {'lib ms/step':>12s} {'torch ms/step':>14s} {'launches/step':>14s}")
    for cfg in CONFIGS:
        if args.only and cfg[0] not in args.only.split(","):
            continue
        _call._drop_counters.clear()
        lib_fn, torch_fn, launches, N = setup(cfg)
        for _ in range(args.warmup):
            lib_fn()
            torch_fn()
        torch.cuda.synchronize()
        lt, tt = [], []
        for _ in range(args.rounds):
            lt.append(timed(lib_fn, args.steps))
            tt.append(timed(torch_fn, max(1, args.steps // 2)))
        lt.sort()
        tt.sort()
        print(f"{cfg[0]:10s} {N:6d} {cfg[3]:3d} {lt[len(lt) // 2]:12.3f} {tt[len(tt) // 2]:14.2f} {launches:14d}",
              flush=True)
        del lib_fn, torch_fn
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
