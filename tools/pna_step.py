"""Cost of the PNA local model: a PNA+Transformer GPSLayer against GINE+Transformer.

    python tools/pna_step.py [--workloads zinc-gine pcqm4m-small] [--steps 100] [--rounds 7] [--layers 1]

A step is the fp32-grade forward + backward of a GPSStack (dropout 0.0, BatchNorm) on one seeded synthetic batch of
the workload's BASELINE shape, recorded once into a CUDA graph and replayed; PNA reads the batch's edge_attr cut to its
first min(128, d) columns.  The two variants are timed alternately in one process: each round replays each variant
`steps` times between two CUDA events; the median ms/step over the rounds is printed with the kernel launches of one
eager step.  Then torch.profiler times the PNA message-passing kernels (k_pna_fwd, k_pna_bwd_*) of one eager step and
reports their achieved bytes/s against algorithmic bytes: every tensor they read or write, counted once (forward:
P_dst | P_src, q, x, Z's bf16 hi/lo planes, the argmax; backward: g_Z, the argmax, the upstream g_x, g_q with its planes,
g_P_dst | g_P_src with their planes, g_x).  The edge fold (k_pna_fold / k_pna_unfold) is timed separately.  Prints the
GPU name and its power limit."""
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


def pna_kernel_times(stack, bb, ct_x):
    """(forward us, backward us, fold us) of the k_pna_* kernels of one eager step."""
    from torch.profiler import ProfilerActivity, profile
    eager_step(stack, bb, ct_x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eager_step(stack, bb, ct_x)
        torch.cuda.synchronize()
    fwd = bwd = fold = 0.0
    for ev in prof.events():
        if ev.device_type.name != "CUDA" or "k_pna_" not in ev.name:
            continue
        t = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        if "fold" in ev.name:
            fold += t
        elif "bwd" in ev.name:
            bwd += t
        else:
            fwd += t
    return fwd, bwd, fold


def pna_bytes(N, E, d, layers):
    f = 4 * (2 * N * d + E * d + N * d) + 4 * 4 * N * d + 4 * N * d
    b = 4 * (4 * N * d + N * d + E * d + 2 * N * d + N * d) + 4 * N * d + 4 * E * d + 4 * 2 * N * d
    return f * layers, b * layers


def run(workload, args, dev, lib):
    spec = graphgps_b200.SHAPES[workload]
    d, heads = spec.dim, spec.heads
    torch.manual_seed(0)
    stacks = {loc: graphgps_b200.GPSStack(args.layers, d, loc, "Transformer", heads, pna_degrees=[0, 1, 2, 1]
                                          if loc == "PNA" else None).to(dev).train()
              for loc in ("GINE", "PNA")}
    b = graphgps_b200.make_batch(workload, seed=1).to(dev)
    bp = b.clone()
    bp.edge_attr = b.edge_attr[:, :min(128, d)].contiguous()
    batches = {"GINE": b, "PNA": bp}
    ct_x = torch.randn_like(b.x)
    steps, launches, cap = {}, {}, {}
    for name, stack in stacks.items():
        torch.cuda.synchronize()
        n0 = lib.gps_launch_count()
        eager_step(stack, batches[name], ct_x)
        torch.cuda.synchronize()
        launches[name] = lib.gps_launch_count() - n0
        for p in stack.parameters():
            p.grad = None
        cap[name] = batches[name].clone()   # a captured step reads this batch's tensors on every replay: keep it referenced
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
    for k in ("GINE", "PNA"):
        print(f"  {k:7s} ms/step median {med[k]:.4f}  launches/step {launches[k]}  rounds "
              + " ".join(f"{t:.4f}" for t in times[k]))
    print(f"  PNA - GINE {med['PNA'] - med['GINE']:+.4f} ms/step "
          f"({(med['PNA'] / med['GINE'] - 1) * 100:+.1f} %)")
    for p in stacks["PNA"].parameters():
        p.grad = None
    fus, bus, folds = pna_kernel_times(stacks["PNA"], bp, ct_x)
    fb, bb_ = pna_bytes(b.num_nodes, b.num_edges, d, args.layers)
    print(f"  PNA kernels (eager, profiler): forward {fus:.1f} us, {fb / 1e6:.2f} MB algorithmic, "
          f"{fb / max(fus, 1e-9) / 1e3:.0f} GB/s;  backward {bus:.1f} us, {bb_ / 1e6:.2f} MB, "
          f"{bb_ / max(bus, 1e-9) / 1e3:.0f} GB/s;  fold + unfold {folds:.1f} us")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["zinc-gine", "pcqm4m-small"])
    ap.add_argument("--layers", type=int, default=1)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/pna_step.py needs a CUDA device")
    lib = _lib.load()
    for w in args.workloads:
        run(w, args, "cuda:0", lib)
    gpu, power = gpu_info()
    print(f"  GPU: {gpu}, power limit {power}")


if __name__ == "__main__":
    main()
