"""Cost of the EquivStableLapPE edge gate (GPSLayer(..., equivstable_pe=True)) on one GPSLayer step.

    python tools/eslappe_step.py [--precision fp32|bf16] [--steps 200] [--rounds 5] [--workload pcqm4m-small]

A step is the forward + backward of one GatedGCN+Transformer layer (dropout 0.0, attn_dropout 0.5, as bench.py runs
the pcqm4m-small workload) on one seeded synthetic batch, recorded once into a CUDA graph and replayed.  The layer with
the PE (k = d, as the pcqm4m-GPS-ESLapPE config produces it) and the same layer without it are timed alternately in
one process: each round replays every variant `steps` times between two CUDA events.  Prints the median ms/step of
each variant over the rounds, the difference, the GPU name and its power limit."""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import graphgps_b200  # noqa: E402
from graphgps_b200.graph import graph_of  # noqa: E402


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        out = ""
    return name, out or "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="pcqm4m-small", choices=sorted(graphgps_b200.SHAPES))
    ap.add_argument("--precision", default="fp32", choices=["fp32", "bf16"])
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/eslappe_step.py needs a CUDA device")
    dev = "cuda:0"
    spec = graphgps_b200.SHAPES[args.workload]
    d, heads = spec.dim, spec.heads
    torch.manual_seed(0)
    off = graphgps_b200.GPSLayer(d, "CustomGatedGCN", "Transformer", heads, dropout=0.0, attn_dropout=0.5,
                                 precision=args.precision)
    on = graphgps_b200.GPSLayer(d, "CustomGatedGCN", "Transformer", heads, dropout=0.0, attn_dropout=0.5,
                                precision=args.precision, equivstable_pe=True)
    missing = on.load_state_dict(off.state_dict(), strict=False).missing_keys
    assert all(k.startswith("local_model.mlp_r_ij.") for k in missing)
    b = graphgps_b200.make_batch(args.workload, seed=1).to(dev)
    g = torch.Generator(device="cpu").manual_seed(2)
    pe = torch.randn(b.num_nodes, d, generator=g)
    pe = (pe / pe.norm(dim=1, keepdim=True) * (0.3 + 1.8 * torch.rand(b.num_nodes, 1, generator=g))).to(dev)
    ct_x, ct_e = torch.randn_like(b.x), torch.randn_like(b.edge_attr)

    steps = {}
    for name, layer, with_pe in (("off", off, False), ("on", on, True)):
        layer = layer.to(dev).train()
        bb = b.clone()
        if with_pe:
            bb.pe_EquivStableLapPE = pe
        graph_of(bb)
        steps[name] = graphgps_b200.GPSStack.from_layers([layer]).capture(bb, ct_x, ct_e)
    for s in steps.values():
        for _ in range(20):
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
    print(f"{args.workload} {args.precision}: N={b.num_nodes} E={b.num_edges} d={d} k={d}; CUDA-graph replay, "
          f"{args.rounds} alternating rounds x {args.steps} steps")
    for k in ("off", "on"):
        print(f"  equivstable_pe={k:3s}  ms/step median {med[k]:.4f}  rounds " + " ".join(f"{t:.4f}" for t in times[k]))
    print(f"  difference {med['on'] - med['off']:+.4f} ms/step ({(med['on'] / med['off'] - 1) * 100:+.1f} %)")
    print(f"  GPU: {gpu}, power limit {power}")


if __name__ == "__main__":
    main()
