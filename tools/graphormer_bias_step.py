"""Cost of Graphormer's attention-bias encoder: forward + backward of graphgps_b200.BiasEncoder against the reference's
composition restated in eager torch, and the encoder's share of a captured zinc-Graphormer step.

    python tools/graphormer_bias_step.py [--steps 20] [--rounds 5]

Shapes (num_spatial_types 20):
  zinc-Graphormer  256 ZINC-sized graphs of 10..37 nodes (159 k pairs), 8 heads, 4 edge types, graph token
  actor            one graph of 7 600 nodes (57.8 M pairs), 4 heads, no shortest_path_types, no graph token
A step is the encoder's forward and the backward into its parameters from a fixed cotangent of attn_bias.  The library
arm is recorded once into a CUDA graph and replayed; the torch arm is the reference's forward (graphormer_encoder.py:
140-183: embedding lookups, to_dense_adj's scatter, permute, bmm over the path positions, sum, F.pad) on the same
parameters, run eagerly, with Nmax and the graph count given (to_dense_adj's own host reads are not timed).  The step
share runs BiasEncoder + 12 GraphormerLayers (d 80, dropout 0.1) forward + backward, captured, against the same 12
layers fed a constant attn_bias.  Each round times every arm `steps` times between two CUDA events; the median ms/step
over the rounds is printed with the GPU name and its power limit."""
import argparse
import os
import statistics
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import graphgps_b200  # noqa: E402
from graphgps_b200.batch import GraphBatch  # noqa: E402
from graphgps_b200.graph import graph_of  # noqa: E402
from graphormer_oracle import graphormer_batch  # noqa: E402
from graphormer_step import gpu_info, timed  # noqa: E402

S = 20
SHAPES = {
    "zinc-Graphormer": dict(heads=8, T=4, token=True),
    "actor": dict(heads=4, T=0, token=False),
}


def sizes_of(shape):
    if shape == "actor":
        return [7600]
    g = torch.Generator().manual_seed(3)
    return torch.randint(10, 38, (256,), generator=g).tolist()


def pairs(sizes, T, seed):
    """graphormer_pre_processing's collated attributes in its pair order (i * n + j per graph), random types."""
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(seed)
    gis, off = [], 0
    for n in sizes:
        a = torch.arange(n, device=dev)
        gis.append(torch.stack([a.repeat_interleave(n), a.repeat(n)]) + off)
        off += n
    gi = torch.cat(gis, 1)
    P = gi.shape[1]
    data = types.SimpleNamespace(graph_index=gi, spatial_types=torch.randint(0, S + 1, (P,), device=dev, generator=g),
                                 batch=torch.repeat_interleave(torch.arange(len(sizes), device=dev),
                                                               torch.tensor(sizes, device=dev)))
    if T:
        data.shortest_path_types = torch.randint(0, T, (P, S), device=dev, generator=g)
    return data


def to_dense_adj(edge_index, batch, edge_attr, B, nmax):
    """torch_geometric.utils.to_dense_adj with the batch size and Nmax given."""
    num_nodes = torch.zeros(B, dtype=torch.int64, device=batch.device).index_add_(0, batch, torch.ones_like(batch))
    cum = torch.cat([num_nodes.new_zeros(1), num_nodes.cumsum(0)])
    idx0 = batch[edge_index[0]]
    idx1 = edge_index[0] - cum[batch][edge_index[0]]
    idx2 = edge_index[1] - cum[batch][edge_index[1]]
    idx = (idx0 * nmax + idx1) * nmax + idx2
    out = edge_attr.new_zeros((B * nmax * nmax,) + tuple(edge_attr.shape[1:])).index_add(0, idx, edge_attr)
    return out.view((B, nmax, nmax) + tuple(edge_attr.shape[1:]))


def torch_encoder(enc, data, B, nmax):
    """The reference's BiasEncoder.forward (graphormer_encoder.py:140-183) on enc's parameters."""
    H = enc.num_heads
    bias = to_dense_adj(data.graph_index, data.batch, F.embedding(data.spatial_types, enc.spatial_encoder.weight), B,
                        nmax).permute(0, 3, 1, 2)
    if hasattr(data, "shortest_path_types"):
        e = to_dense_adj(data.graph_index, data.batch, F.embedding(data.shortest_path_types, enc.edge_encoder.weight), B,
                         nmax)
        sd = to_dense_adj(data.graph_index, data.batch, data.spatial_types, B, nmax).float().clamp(min=1.0).unsqueeze(1)
        _, N, _, D, _ = e.shape
        e = e.permute(3, 0, 1, 2, 4).reshape(D, -1, H)
        e = torch.bmm(e, enc.edge_dis_encoder.weight.reshape(-1, H, H))
        e = e.reshape(D, B, N, N, H).permute(1, 2, 3, 0, 4).sum(-2).permute(0, 3, 1, 2) / sd
        bias = bias + e
    if enc.use_graph_token:
        bias = F.pad(bias, (1, 0, 1, 0))
        bias[:, :, 1:, 0] = enc.graph_token
        bias[:, :, 0, :] = enc.graph_token
    Bb, Hh, N, _ = bias.shape
    return bias.reshape(Bb * Hh, N, N)


def capture(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def report(title, arms, steps, rounds, base_key):
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(timed(fn, steps))
    print(title)
    med = {k: statistics.median(v) for k, v in times.items()}
    for k, m in med.items():
        ratio = f"  ({base_key} / this = {med[base_key] / m:6.2f}x)" if base_key else ""
        print(f"  {k:44s} {m:9.3f} ms/step{ratio}")
    return med


def encoder_arms(shape):
    cfg = SHAPES[shape]
    torch.manual_seed(0)
    enc = graphgps_b200.BiasEncoder(cfg["heads"], S, cfg["T"], cfg["token"]).cuda()
    sizes = sizes_of(shape)
    data = pairs(sizes, cfg["T"], 1)
    params = list(enc.parameters())
    with torch.no_grad():
        out = enc(data).attn_bias   # the one host read per batch, before capture
        ct = torch.randn_like(out)
        B, nmax = len(sizes), max(sizes)
        err = float((torch_encoder(enc, data, B, nmax) - out).abs().max())
    del out, data.attn_bias

    def lib_step():
        out = enc(data).attn_bias
        del data.attn_bias   # a batch holding the last step's output would keep its autograd graph alive
        return torch.autograd.grad((out * ct).sum(), params, allow_unused=True)

    def torch_step():
        return torch.autograd.grad((torch_encoder(enc, data, B, nmax) * ct).sum(), params, allow_unused=True)

    return {"library (captured)": capture(lib_step), "torch fp32 (eager)": torch_step}, sizes, data, err


def step_share(steps, rounds):
    """zinc-Graphormer: BiasEncoder + 12 GraphormerLayers, captured, against the 12 layers alone."""
    torch.manual_seed(0)
    enc = graphgps_b200.BiasEncoder(8, S, 4, True).cuda()
    layers = nn.Sequential(*[graphgps_b200.GraphormerLayer(80, 8, 0.1, 0.1, 0.1) for _ in range(12)]).cuda()
    sizes = sizes_of("zinc-Graphormer")
    data = pairs(sizes, 4, 1)
    bb = graphormer_batch([n + 1 for n in sizes], 80, 1, True)
    b = GraphBatch(x=bb.x.cuda(), edge_index=bb.edge_index.cuda(), edge_attr=None, batch=bb.batch.cuda(),
                   num_graphs=len(sizes))
    graph_of(b).nmax
    with torch.no_grad():
        const_bias = enc(data).attn_bias.clone().requires_grad_(True)
    del data.attn_bias
    x = b.x.clone().requires_grad_(True)
    ct = torch.randn_like(x)
    lp = list(layers.parameters())
    ep = list(enc.parameters())

    def full():
        b.x, b.attn_bias = x, enc(data).attn_bias
        out = layers(b).x
        del data.attn_bias   # drop the batches' references to this step's autograd graph
        b.x, b.attn_bias = x, None
        return torch.autograd.grad((out * ct).sum(), [x] + lp + ep)

    def layers_only():
        b.x, b.attn_bias = x, const_bias
        out = layers(b).x
        b.x = x
        return torch.autograd.grad((out * ct).sum(), [x, const_bias] + lp)

    med = report("zinc-Graphormer step: 12 GraphormerLayers (d 80, 8 heads, dropout 0.1), forward + backward, fp32",
                 {"BiasEncoder + 12 layers (captured)": capture(full),
                  "12 layers, constant attn_bias (captured)": capture(layers_only)}, steps, rounds, None)
    return med


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/graphormer_bias_step.py needs a CUDA device")
    name, plim = gpu_info()
    print(f"GPU: {name}, power limit {plim}")
    enc_ms = {}
    for shape in SHAPES:
        arms, sizes, data, err = encoder_arms(shape)
        cfg = SHAPES[shape]
        P = data.spatial_types.numel()
        med = report(f"{shape}: BiasEncoder forward + backward, {len(sizes)} graphs, {P} pairs, H {cfg['heads']}, "
                     f"T {cfg['T']}, graph token {cfg['token']} (max |library - torch| of attn_bias {err:.1e})",
                     arms, args.steps, args.rounds, "torch fp32 (eager)")
        enc_ms[shape] = med
        del arms, data
        torch.cuda.empty_cache()
    med = step_share(args.steps, args.rounds)
    full, layers = med["BiasEncoder + 12 layers (captured)"], med["12 layers, constant attn_bias (captured)"]
    enc = enc_ms["zinc-Graphormer"]
    print(f"  encoder share of the captured step: (full - layers) / full = {100 * (full - layers) / full:.1f}%; "
          f"encoder alone / full = {100 * enc['library (captured)'] / full:.1f}%")
    print(f"  with the torch encoder instead: layers + torch encoder = {layers + enc['torch fp32 (eager)']:.3f} ms, "
          f"torch encoder share {100 * enc['torch fp32 (eager)'] / (layers + enc['torch fp32 (eager)']):.1f}%")


if __name__ == "__main__":
    main()
