"""Cost of the GENConv local model: a GENConv+Transformer GPSLayer against GINE+Transformer.

    python tools/genconv_step.py [--workloads zinc-gine pcqm4m-small] [--steps 100] [--rounds 7] [--layers 1]

A step is the fp32-grade forward + backward of a GPSStack (dropout 0.0, BatchNorm) on one seeded synthetic batch of
the workload's BASELINE shape, recorded once into a CUDA graph and replayed.  The two variants are timed alternately in
one process: each round replays each variant `steps` times between two CUDA events; the median ms/step over the rounds
is printed with the kernel launches of one eager step.  Then torch.profiler times the GENConv message-passing kernels
(k_genconv_*) of one eager step and reports their achieved bytes/s against algorithmic bytes: every tensor they read or
write, counted once (forward: x, edge_attr, agg, lse, u and u's bf16 hi/lo planes; backward, destination pass: x,
edge_attr, agg, lse, g_u, grad_edge_attr).  The source-ordered pass is GINE's k_gine_bwd_src and is not counted.  Prints
the GPU name and its power limit."""
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


def eager_step(stack, bb, ct_x):
    eb = bb.clone()
    eb.__dict__["_gps_b200_graph"] = graph_of(bb)
    eb.x.requires_grad_(True)
    eb.edge_attr.requires_grad_(True)
    stack(eb).x.backward(ct_x)


def genconv_kernel_times(stack, bb, ct_x):
    """(forward us, backward us) of the k_genconv_* kernels of one eager step."""
    from torch.profiler import ProfilerActivity, profile
    eager_step(stack, bb, ct_x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eager_step(stack, bb, ct_x)
        torch.cuda.synchronize()
    fwd = bwd = 0.0
    for ev in prof.events():
        if ev.device_type.name != "CUDA" or "k_genconv_" not in ev.name:
            continue
        t = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        if "bwd" in ev.name:
            bwd += t
        else:
            fwd += t
    return fwd, bwd


def genconv_bytes(N, E, d, layers):
    f = 4 * (4 * N * d + E * d) + 2 * 2 * N * d
    b = 4 * (4 * N * d + 2 * E * d)
    return f * layers, b * layers


def run(workload, args, dev, lib):
    spec = graphgps_b200.SHAPES[workload]
    d, heads = spec.dim, spec.heads
    torch.manual_seed(0)
    stacks = {loc: graphgps_b200.GPSStack(args.layers, d, loc, "Transformer", heads).to(dev).train()
              for loc in ("GINE", "GENConv")}
    b = graphgps_b200.make_batch(workload, seed=1).to(dev)
    ct_x = torch.randn_like(b.x)
    steps, launches, cap = {}, {}, {}
    for name, stack in stacks.items():
        torch.cuda.synchronize()
        n0 = lib.gps_launch_count()
        eager_step(stack, b, ct_x)
        torch.cuda.synchronize()
        launches[name] = lib.gps_launch_count() - n0
        for p in stack.parameters():
            p.grad = None
        cap[name] = b.clone()   # a captured step reads this batch's tensors on every replay: keep it referenced
        graph_of(cap[name])
        steps[name] = stack.capture(cap[name], ct_x)
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
    med = {k: statistics.median(v) for k, v in times.items()}
    print(f"{workload} fp32: {args.layers} layer(s) x+Transformer, N={b.num_nodes} E={b.num_edges} B={b.num_graphs} "
          f"d={d} heads={heads}; fwd+bwd, CUDA-graph replay, {args.rounds} alternating rounds x {args.steps} steps")
    for k in ("GINE", "GENConv"):
        print(f"  {k:7s} ms/step median {med[k]:.4f}  launches/step {launches[k]}  rounds "
              + " ".join(f"{t:.4f}" for t in times[k]))
    print(f"  GENConv - GINE {med['GENConv'] - med['GINE']:+.4f} ms/step "
          f"({(med['GENConv'] / med['GINE'] - 1) * 100:+.1f} %)")
    for p in stacks["GENConv"].parameters():
        p.grad = None
    fus, bus = genconv_kernel_times(stacks["GENConv"], b, ct_x)
    fb, bb_ = genconv_bytes(b.num_nodes, b.num_edges, d, args.layers)
    print(f"  GENConv kernels (eager, profiler): forward {fus:.1f} us, {fb / 1e6:.2f} MB algorithmic, "
          f"{fb / max(fus, 1e-9) / 1e3:.0f} GB/s;  backward {bus:.1f} us, {bb_ / 1e6:.2f} MB, "
          f"{bb_ / max(bus, 1e-9) / 1e3:.0f} GB/s")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["zinc-gine", "pcqm4m-small"])
    ap.add_argument("--layers", type=int, default=1)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/genconv_step.py needs a CUDA device")
    lib = _lib.load()
    for w in args.workloads:
        run(w, args, "cuda:0", lib)
    gpu, power = gpu_info()
    print(f"  GPU: {gpu}, power limit {power}")


if __name__ == "__main__":
    main()
