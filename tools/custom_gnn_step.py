"""Cost of an L-layer CustomGNN stack (GatedGCN or GINE), forward + backward in training mode, at the LRGB shapes.

    python tools/custom_gnn_step.py [--steps K] [--warmup W] [--rounds R] [--only NAME,...]

Two legs, alternated round by round in the same process on the same GPU:
  * lib:   graphgps_b200.GatedGCNLayer / GINEConvLayer x L (fp32-grade), captured into one CUDA graph per step and
           replayed;
  * torch: the same stack composed in eager torch fp32 (tests/custom_gnn_oracle.py's modules: nn.Linear, index_add
           scatters, nn.BatchNorm1d), with the same parameters.
Batches come from graphgps_b200.batch.make_batch on the ShapeSpecs below (published mean sizes of the LRGB datasets:
peptides ~151 nodes / ~307 directed edges per graph, pcqm-contact ~30 / ~61, VOC / COCO superpixels ~479 / ~2 710).
Each leg's time is the median over rounds of the mean ms per step, from CUDA events around K steps.  The table also
gives the library's kernel launches per step, the card name and its power limit.
"""
import argparse
import os
import subprocess
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import graphgps_b200  # noqa: E402
from graphgps_b200 import _call, _lib  # noqa: E402
from graphgps_b200.batch import ShapeSpec, make_batch  # noqa: E402
from graphgps_b200.graph import graph_of  # noqa: E402
from custom_gnn_oracle import oracle_layer, run_stack  # noqa: E402

DEV = "cuda:0"
# spanning tree plus extra undirected edges per node, stored both ways: 2 (n - 1 + extra n) directed edges per graph
PEPTIDES = ShapeSpec("peptides", 128, 0, 1, 150.94, 30.0, 20, 450, 0.0232, True)
PCQM_CONTACT = ShapeSpec("pcqm-contact", 256, 0, 1, 30.14, 5.0, 5, 60, 0.048, True)
SUPERPIXELS = ShapeSpec("superpixels", 32, 0, 1, 479.40, 30.0, 300, 520, 1.83, True)
# name, layer, shape, L, d (configs/GatedGCN, configs/GINE; peptides-func / -struct and VOC / COCO share their shapes)
CONFIGS = [
    ("peptides-GatedGCN", "gatedgcn", PEPTIDES, 5, 138),
    ("pcqm-contact-GatedGCN", "gatedgcn", PCQM_CONTACT, 5, 138),
    ("superpixels-GatedGCN", "gatedgcn", SUPERPIXELS, 8, 108),
    ("peptides-GINE", "gine", PEPTIDES, 5, 208),
    ("pcqm-contact-GINE", "gine", PCQM_CONTACT, 5, 208),
    ("superpixels-GINE", "gine", SUPERPIXELS, 8, 166),
]


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20)
        return r.stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def setup(cfg):
    name, kind, spec, L, d = cfg
    torch.manual_seed(0)
    if kind == "gatedgcn":
        seq = nn.Sequential(*[graphgps_b200.GatedGCNLayer(d, d, 0.0, True) for _ in range(L)])
    else:
        seq = nn.Sequential(*[graphgps_b200.GINEConvLayer(d, d, 0.0, True) for _ in range(L)])
    seq = seq.to(DEV).train()
    b = make_batch(spec, seed=1, dim=d)
    b.x, b.edge_attr, b.edge_index, b.batch = (t.to(DEV) for t in (b.x, b.edge_attr, b.edge_index, b.batch))
    graph_of(b)
    x = b.x.clone().requires_grad_(True)
    e = b.edge_attr.clone().requires_grad_(True)
    ct = torch.randn(b.x.shape, device=DEV)
    params = list(seq.parameters())

    def lib_step():
        b.x, b.edge_attr = x, e
        out = seq(b).x
        return torch.autograd.grad((out * ct).sum(), [x, e] + params)

    lib = _lib.load()
    lib_step()
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

    def replay():
        # The graph holds raw addresses of the layers' parameters, buffers and weight planes and of the batch's graph
        # structure: this closure keeps all of them (seq, b) alive for as long as the graph is replayed
        graph.replay()
        return seq, b

    # torch leg: the same parameters in the eager fp32 composition
    ref = nn.Sequential(*[oracle_layer(kind, d) for _ in range(L)]).to(DEV).train()
    ref.load_state_dict(seq.state_dict())
    leaves = list(ref.parameters())
    ei = b.edge_index

    def torch_step():
        h, _ = run_stack(list(ref), x, e, ei)
        # (the last GatedGCN layer's bn_edge_e does not reach the loss)
        return torch.autograd.grad((h * ct).sum(), [x, e] + leaves, allow_unused=True)

    return replay, torch_step, launches, b.x.shape[0], ei.shape[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    print(f"card: {torch.cuda.get_device_name(0)}, power limit {power_limit()}")
    print(f"{'config':22s} {'N':>6s} {'E':>7s} {'L':>3s} {'d':>4s} {'lib ms/step':>12s} {'torch ms/step':>14s} "
          f"{'launches/step':>14s}")
    for cfg in CONFIGS:
        if args.only and cfg[0] not in args.only.split(","):
            continue
        _call._drop_counters.clear()
        lib_fn, torch_fn, launches, N, E = setup(cfg)
        for _ in range(args.warmup):
            lib_fn()
            torch_fn()
        torch.cuda.synchronize()
        lt, tt = [], []
        for _ in range(args.rounds):
            lt.append(timed(lib_fn, args.steps))
            tt.append(timed(torch_fn, args.steps))
        lt.sort()
        tt.sort()
        print(f"{cfg[0]:22s} {N:6d} {E:7d} {cfg[3]:3d} {cfg[4]:4d} {lt[len(lt) // 2]:12.3f} {tt[len(tt) // 2]:14.3f} "
              f"{launches:14d}", flush=True)
        del lib_fn, torch_fn
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
