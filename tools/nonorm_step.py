"""Step time of the GCN+Transformer configs' layer stack with and without BatchNorm (GPSLayer(..., batch_norm=False)).

    python tools/nonorm_step.py [--shapes webkb,chameleon,squirrel,actor] [--precisions fp32,bf16] [--steps 50]
                                [--rounds 5] [--profile actor]

A step is the forward + backward of a 2-layer GCN+Transformer GPSStack (gt.layers = 2, GELU, dropout 0.2, attn_dropout
as the config: 0.5 at chameleon, else 0.0) on one seeded single-graph node-level batch (tests/nonorm_util.py shapes),
recorded once into a CUDA graph and replayed.  batch_norm=True and batch_norm=False (same weights) are timed
alternately in one process: each round replays every variant `steps` times between two CUDA events.  Prints the median
ms/step of each variant over the rounds, the GPU name and its power limit.

--profile SHAPE: instead, one torch.profiler capture of 5 eager fp32 steps of each variant at SHAPE and the kernels that
take most of the GPU time."""
import argparse
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import graphgps_b200  # noqa: E402
from graphgps_b200.graph import graph_of  # noqa: E402
from nonorm_util import NODE_SHAPES, node_shape_batch  # noqa: E402


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        out = ""
    return name, out or "unknown"


def stacks(shape, precision, dev):
    s = NODE_SHAPES[shape]
    torch.manual_seed(0)
    kw = dict(act="gelu", dropout=0.2, attn_dropout=s.attn_dropout, precision=precision)
    bn = graphgps_b200.GPSStack(2, s.d, "GCN", "Transformer", s.heads, **kw)
    none = graphgps_b200.GPSStack(2, s.d, "GCN", "Transformer", s.heads, batch_norm=False, **kw)
    none.load_state_dict(bn.state_dict(), strict=False)
    return {"batch_norm": bn.to(dev).train(), "none": none.to(dev).train()}


def time_shape(shape, precision, steps, rounds, dev):
    b = node_shape_batch(shape, seed=1).to(dev)
    graph_of(b)
    ct = torch.randn_like(b.x)
    caps = {k: st.capture(b, ct) for k, st in stacks(shape, precision, dev).items()}
    for c in caps.values():
        for _ in range(5):
            c.replay()
    torch.cuda.synchronize()
    times = {k: [] for k in caps}
    for _ in range(rounds):
        for k, c in caps.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                c.replay()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / steps)
    return b, {k: statistics.median(v) for k, v in times.items()}, times


def launches(shape, dev):
    """gps_launch_count delta of one eager fp32 fwd+bwd of each 2-layer stack."""
    lib = graphgps_b200._lib.load()
    b = node_shape_batch(shape, seed=1).to(dev)
    graph_of(b)
    out = {}
    for k, st in stacks(shape, "fp32", dev).items():
        for i in range(2):
            c0 = lib.gps_launch_count()
            x = b.x.clone().requires_grad_(True)
            o = st(graphgps_b200.GraphBatch(x=x, edge_index=b.edge_index, edge_attr=b.edge_attr, batch=b.batch,
                                            num_graphs=1, _gps_b200_graph=b.__dict__["_gps_b200_graph"]))
            o.x.sum().backward()
            torch.cuda.synchronize()
            out[k] = lib.gps_launch_count() - c0
    return out


def profile(shape, dev, top=12):
    from torch.profiler import ProfilerActivity, profile as tprof
    b = node_shape_batch(shape, seed=1).to(dev)
    graph_of(b)
    for k, st in stacks(shape, "fp32", dev).items():
        def step():
            x = b.x.clone().requires_grad_(True)
            o = st(graphgps_b200.GraphBatch(x=x, edge_index=b.edge_index, edge_attr=b.edge_attr, batch=b.batch,
                                            num_graphs=1, _gps_b200_graph=b.__dict__["_gps_b200_graph"]))
            o.x.sum().backward()
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        with tprof(activities=[ProfilerActivity.CUDA]) as p:
            for _ in range(5):
                step()
            torch.cuda.synchronize()
        rows = [e for e in p.key_averages() if e.self_device_time_total > 0]
        tot = sum(e.self_device_time_total for e in rows)
        rows.sort(key=lambda e: -e.self_device_time_total)
        print(f"\n{shape} fp32 {k}: GPU time per step {tot / 5 / 1e3:.3f} ms (5 eager steps, kernels by self time)")
        for e in rows[:top]:
            print(f"  {e.self_device_time_total / tot * 100:5.1f} %  {e.self_device_time_total / 5 / 1e3:8.3f} ms/step"
                  f"  x{e.count // 5:<3d} {e.key[:110]}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="webkb,chameleon,squirrel,actor")
    ap.add_argument("--precisions", default="fp32,bf16")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", default=None, choices=sorted(NODE_SHAPES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/nonorm_step.py needs a CUDA device")
    dev = "cuda:0"
    gpu, power = gpu_info()
    print(f"GPU: {gpu}, power limit {power}")
    if args.profile:
        profile(args.profile, dev)
        return
    print(f"2-layer GCN+Transformer GPSStack fwd+bwd, GELU, dropout 0.2; CUDA-graph replay, median of {args.rounds} "
          f"alternating rounds x {args.steps} steps")
    print(f"{'shape':10s} {'N':>5s} {'E':>7s} {'d':>3s} {'prec':5s} {'batch_norm ms':>14s} {'none ms':>9s} {'none/bn':>8s}"
          "  round spread (min-max) bn | none")
    for shape in args.shapes.split(","):
        for prec in args.precisions.split(","):
            b, med, t = time_shape(shape, prec, args.steps, args.rounds, dev)
            s = NODE_SHAPES[shape]
            print(f"{shape:10s} {s.N:5d} {s.E:7d} {s.d:3d} {prec:5s} {med['batch_norm']:14.4f} {med['none']:9.4f} "
                  f"{med['none'] / med['batch_norm']:8.3f}  {min(t['batch_norm']):.4f}-{max(t['batch_norm']):.4f} | "
                  f"{min(t['none']):.4f}-{max(t['none']):.4f}", flush=True)
    for shape in args.shapes.split(","):
        print(f"launches per fwd+bwd of the 2-layer stack @ {shape}: {launches(shape, dev)}")
    print(f"GPU: {gpu}, power limit {power}")


if __name__ == "__main__":
    main()
