"""Cost of the BigBird global model: a captured 3-layer GINE+BigBird GPSStack at the shipped shape.

    python tools/bigbird_step.py [--steps 100] [--rounds 7] [--layers 3]

The shipped config (zinc-GPS-BigBird.yaml): make_batch("zinc-gine", dim=56), 8 heads, block size 3, 3 random blocks,
BatchNorm, dropout 0.0.  It is timed alternately in one process with GINE+None at the same width and with
GINE+Transformer at d = 64 / 8 heads.  A step is the fp32-grade forward + backward of the stack, recorded once into a
CUDA graph and replayed; each round replays each variant `steps` times between two CUDA events, and the median ms/step
over the rounds is printed with the kernel launches of one eager step, the GPU name and its power limit."""
import argparse
import os
import statistics
import subprocess
import sys
import types

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


def bigbird_cfg():
    return types.SimpleNamespace(attention_type="block_sparse", chunk_size_feed_forward=0, is_decoder=False,
                                 add_cross_attention=False, hidden_act="relu", max_position_embeddings=128,
                                 use_bias=False, num_random_blocks=3, block_size=3, layer_norm_eps=1e-6)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=3)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bigbird_step.py needs a CUDA device")
    lib = _lib.load()
    dev = "cuda:0"
    torch.manual_seed(0)
    variants = {
        "GINE+BigBird d=56": (56, 8, "BigBird", dict(bigbird_cfg=bigbird_cfg())),
        "GINE+None d=56": (56, 8, "None", {}),
        "GINE+Transformer d=64": (64, 8, "Transformer", {}),
    }
    steps, launches, keep = {}, {}, {}
    for name, (d, heads, glob, kw) in variants.items():
        stack = graphgps_b200.GPSStack(args.layers, d, "GINE", glob, heads, **kw).to(dev).train()
        b = graphgps_b200.make_batch("zinc-gine", seed=1, dim=d).to(dev)
        graph_of(b)
        ct_x = torch.randn_like(b.x)
        eager_step(stack, b, ct_x)   # warm: block lists, plans, workspaces
        torch.cuda.synchronize()
        n0 = lib.gps_launch_count()
        eager_step(stack, b, ct_x)
        torch.cuda.synchronize()
        launches[name] = lib.gps_launch_count() - n0
        for p in stack.parameters():
            p.grad = None
        steps[name] = stack.capture(b, ct_x)
        keep[name] = (stack, b, ct_x)
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
    b = keep["GINE+BigBird d=56"][1]
    print(f"zinc-gine fp32: {args.layers} layers, N={b.num_nodes} E={b.num_edges} B={b.num_graphs}; fwd+bwd, CUDA-graph "
          f"replay, {args.rounds} alternating rounds x {args.steps} steps")
    for k in variants:
        med = statistics.median(times[k])
        print(f"  {k:22s} ms/step median {med:.4f}  launches/eager step {launches[k]}  rounds "
              + " ".join(f"{t:.4f}" for t in times[k]))
    gpu, power = gpu_info()
    print(f"  GPU: {gpu}, power limit {power}")


if __name__ == "__main__":
    main()
