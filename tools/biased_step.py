"""Cost of the BiasedTransformer attention bias on a 10-layer GPSLayer stack.

    python tools/biased_step.py [--steps 100] [--rounds 7] [--layers 10] [--workload zinc-gine]

A step is the fp32-grade forward + backward of a GINE+BiasedTransformer GPSStack (dropout 0.0, attn_dropout 0.5, BatchNorm, as
zinc-GPSwGraphormer.yaml builds it) on one seeded synthetic batch, recorded once into a CUDA graph and replayed, against
the same stack as GINE+Transformer.  The attention bias is [num_graphs * heads, Nmax, Nmax] with std 2 and needs its
gradient.  The two variants are timed alternately in one process: each round replays every variant `steps` times
between two CUDA events.  Prints the median ms/step of each variant over the rounds, the difference, the kernel
launches of one eager step, the GPU name and its power limit."""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import graphgps_b200  # noqa: E402
from graphgps_b200 import _lib  # noqa: E402
from graphgps_b200.graph import graph_of  # noqa: E402


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        out = ""
    return name, out or "unknown"


def eager_launches(lib, stack, bb, ct_x):
    """Kernel launches of one eager fwd+bwd step (its autograd graph is gone when this returns, before any capture)."""
    eb = bb.clone()
    eb.__dict__["_gps_b200_graph"] = graph_of(bb)
    eb.x.requires_grad_(True)
    if getattr(eb, "attn_bias", None) is not None:
        eb.attn_bias.requires_grad_(True)
    torch.cuda.synchronize()
    n0 = lib.gps_launch_count()
    stack(eb).x.backward(ct_x)
    torch.cuda.synchronize()
    return lib.gps_launch_count() - n0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="zinc-gine", choices=sorted(graphgps_b200.SHAPES))
    ap.add_argument("--layers", type=int, default=10)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/biased_step.py needs a CUDA device")
    dev = "cuda:0"
    spec = graphgps_b200.SHAPES[args.workload]
    d, heads = spec.dim, spec.heads
    torch.manual_seed(0)
    kw = dict(dropout=0.0, attn_dropout=0.5)
    plain = graphgps_b200.GPSStack(args.layers, d, "GINE", "Transformer", heads, **kw)
    biased = graphgps_b200.GPSStack(args.layers, d, "GINE", "BiasedTransformer", heads, **kw)
    biased.load_state_dict(plain.state_dict(), strict=True)
    b = graphgps_b200.make_batch(args.workload, seed=1).to(dev)
    gs = graph_of(b)
    g = torch.Generator(device="cpu").manual_seed(2)
    bias = (2.0 * torch.randn(b.num_graphs * heads, gs.nmax, gs.nmax, generator=g)).to(dev)
    ct_x = torch.randn_like(b.x)
    lib = _lib.load()

    steps, launches = {}, {}
    for name, stack, with_bias in (("Transformer", plain, False), ("BiasedTransformer", biased, True)):
        stack = stack.to(dev).train()
        bb = b.clone()
        if with_bias:
            bb.attn_bias = bias
        launches[name] = eager_launches(lib, stack, bb, ct_x)
        for p in stack.parameters():
            p.grad = None
        steps[name] = stack.capture(bb, ct_x)
    for s in steps.values():
        for _ in range(10):
            s.replay()
    torch.cuda.synchronize()

    times = {k: [] for k in steps}
    for _ in range(args.rounds):
        for name, s in steps.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                s.replay()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.steps)
    gpu, power = gpu_info()
    med = {k: statistics.median(v) for k, v in times.items()}
    print(f"{args.workload} fp32: {args.layers} GINE layers, N={b.num_nodes} E={b.num_edges} "
          f"B={b.num_graphs} Nmax={gs.nmax} d={d} heads={heads}; fwd+bwd, CUDA-graph replay, "
          f"{args.rounds} alternating rounds x {args.steps} steps")
    for k in ("Transformer", "BiasedTransformer"):
        print(f"  {k:17s} ms/step median {med[k]:.4f}  launches/step {launches[k]}  rounds "
              + " ".join(f"{t:.4f}" for t in times[k]))
    d_ms = med["BiasedTransformer"] - med["Transformer"]
    print(f"  difference {d_ms:+.4f} ms/step ({(med['BiasedTransformer'] / med['Transformer'] - 1) * 100:+.1f} %)")
    print(f"  GPU: {gpu}, power limit {power}")


if __name__ == "__main__":
    main()
