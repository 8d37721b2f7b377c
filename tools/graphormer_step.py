"""Cost of the Graphormer layer: a captured stack forward + backward against the same stack run eagerly in torch.

    python tools/graphormer_step.py [--steps 20] [--rounds 5]
    python tools/graphormer_step.py --profile      # kernel breakdown of one eager actor-Graphormer step (separate run)

Shapes (dropout as the shipped configs, training mode):
  zinc-Graphormer   12 layers, 256 ZINC-sized graphs with a graph token each, d 80, 8 heads, attn_bias
  actor-Graphormer  2 layers, one graph of 7 600 nodes, d 64, 4 heads, attn_bias [4, 7600, 7600]
A step is the forward + backward of the stack (gradients of x, attn_bias and every parameter), recorded once into a
CUDA graph and replayed, in fp32-grade and in bf16.  The torch arm is the reference's composition (to_dense_batch, the
layer's own nn.MultiheadAttention / LayerNorm / Linear modules, fp32) run eagerly on the same GPU.  Each round times
every arm `steps` times between two CUDA events; the median ms/step over the rounds is printed with the GPU name and
its power limit."""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

import graphgps_b200  # noqa: E402
from graphgps_b200.batch import GraphBatch  # noqa: E402
from graphgps_b200.graph import graph_of  # noqa: E402
from graphormer_oracle import graphormer_batch, random_bias  # noqa: E402

SHAPES = {
    "zinc-Graphormer": dict(layers=12, d=80, heads=8, p=(0.1, 0.1, 0.1), token=True),
    "actor-Graphormer": dict(layers=2, d=64, heads=4, p=(0.2, 0.2, 0.2), token=False),
}


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        out = ""
    return name, out or "unknown"


def sizes_of(shape):
    if shape == "actor-Graphormer":
        return [7600]
    g = torch.Generator().manual_seed(3)
    return (torch.randint(10, 38, (256,), generator=g) + 1).tolist()


def torch_layer(layer, x, batch, counts, attn_bias):
    """The reference's forward (graphormer_layer.py:39-49) on the layer's own torch modules."""
    B, nmax = len(counts), max(counts)
    h = layer.input_norm(x)
    pos = torch.arange(x.shape[0], device=x.device) - torch.repeat_interleave(
        torch.cumsum(torch.tensor([0] + counts[:-1], device=x.device), 0), torch.tensor(counts, device=x.device))
    dense = h.new_zeros(B, nmax, h.shape[1]).index_put((batch, pos), h)
    real = torch.zeros(B, nmax, dtype=torch.bool, device=x.device).index_put((batch, pos),
                                                                             torch.ones_like(batch, dtype=torch.bool))
    a = layer.attention(dense, dense, dense, ~real, attn_mask=attn_bias)[0][real]
    x1 = layer.dropout(a) + x
    return layer.mlp(x1) + x1


def build(shape, precision):
    cfg = SHAPES[shape]
    torch.manual_seed(0)
    layers = nn.Sequential(*[graphgps_b200.GraphormerLayer(cfg["d"], cfg["heads"], *cfg["p"], precision=precision)
                             for _ in range(cfg["layers"])]).cuda()
    sizes = sizes_of(shape)
    bb = graphormer_batch(sizes, cfg["d"], 1, cfg["token"])
    b = GraphBatch(x=bb.x.cuda(), edge_index=bb.edge_index.cuda(), edge_attr=None, batch=bb.batch.cuda(),
                   num_graphs=len(sizes))
    b.attn_bias = random_bias(sizes, cfg["heads"], 1).cuda().requires_grad_(True)
    graph_of(b).nmax
    return layers, b, sizes


def lib_step(layers, b, x, ct):
    b.x = x
    out = layers(b).x
    return torch.autograd.grad((out * ct).sum(), [x, b.attn_bias] + list(layers.parameters()))


def torch_step(layers, b, x, ct, counts):
    h = x
    for layer in layers:
        h = torch_layer(layer, h, b.batch, counts, b.attn_bias)
    return torch.autograd.grad((h * ct).sum(), [x, b.attn_bias] + list(layers.parameters()))


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/graphormer_step.py needs a CUDA device")
    name, plim = gpu_info()
    print(f"GPU: {name}, power limit {plim}")
    if args.profile:
        return profile()
    for shape in SHAPES:
        arms = {}
        for precision in ("fp32", "bf16"):
            layers, b, sizes = build(shape, precision)
            x = b.x.clone().requires_grad_(True)
            ct = torch.randn_like(x)
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(3):
                    lib_step(layers, b, x, ct)
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                lib_step(layers, b, x, ct)
            arms[f"library {precision} (captured)"] = g.replay
        tl, tb, sizes = build(shape, "fp32")
        tx = tb.x.clone().requires_grad_(True)
        tct = torch.randn_like(tx)
        arms["torch fp32 (eager)"] = lambda: torch_step(tl, tb, tx, tct, sizes)
        for fn in arms.values():
            fn()
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, fn in arms.items():
                times[k].append(timed(fn, args.steps))
        print(f"{shape}: {SHAPES[shape]['layers']} layers, N {sum(sizes)}, {len(sizes)} graphs")
        base = statistics.median(times["torch fp32 (eager)"])
        for k, v in times.items():
            m = statistics.median(v)
            print(f"  {k:28s} {m:9.3f} ms/step  (torch / this = {base / m:5.2f}x)")
        del arms
        torch.cuda.empty_cache()


def profile():
    from torch.profiler import ProfilerActivity, profile as tprof
    layers, b, sizes = build("actor-Graphormer", "fp32")
    x = b.x.clone().requires_grad_(True)
    ct = torch.randn_like(x)
    for _ in range(3):
        lib_step(layers, b, x, ct)
    torch.cuda.synchronize()
    with tprof(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            lib_step(layers, b, x, ct)
        torch.cuda.synchronize()
    rows = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0) > 0:
            rows[e.key] = getattr(e, "self_device_time_total", getattr(e, "self_cuda_time_total", 0))
    total = sum(rows.values())
    print(f"actor-Graphormer, 2 layers, fp32, 5 eager steps: GPU time {total / 5e3:.3f} ms/step")
    for k, v in sorted(rows.items(), key=lambda kv: -kv[1])[:15]:
        print(f"  {100 * v / total:5.1f}%  {v / 5e3:8.3f} ms/step  {k[:110]}")
    bwd = sum(v for k, v in rows.items() if "k_attn_bwd" in k or "k_attn_delta" in k)
    print(f"attention backward (k_attn_delta + k_attn_bwd): {100 * bwd / max(total, 1):.1f}% of GPU time")


if __name__ == "__main__":
    main()
