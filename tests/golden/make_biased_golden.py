"""Generates tests/golden/biased/*.pt: GPSLayer(..., 'BiasedTransformer', ...) fixtures from the REFERENCE ITSELF (its
own layer files run verbatim under oracle/ref_shim.py, fp64), next to the fixtures of tests/golden/make_golden.py.

    python tests/golden/make_biased_golden.py [REFERENCE_LAYER_DIR]

The fixtures live in a subdirectory because tests/util.py::golden_names() feeds every tests/golden/*.pt to tests that
build other layers.  Each holds what a make_golden.py fixture holds (config, inputs, reference state_dict, cotangents,
fp64 outputs / gradients / running statistics stored as fp32) plus the attention bias `attn_bias` [B*H, Nmax, Nmax] and
its gradient `grad_attn_bias`.  reference_live_GINE_BiasedTransformer.pt is the reference_live-style case (fp64 inputs,
weights, bias, outputs and gradients) that pins the oracle at 1e-10 / 1e-9.

Graphormer's initial bias (embeddings with std 0.02) barely moves the softmax, so a transposed, offset or wrong-head
bias would pass a 1e-3 parity test.  The biases here have std 2 (tests/biased_util.py::make_bias): asymmetric, different
per head and graph, a graph-token case and a shortest-path lookup case; padded entries hold 30.  Cotangents are random
and the BatchNorm affines non-trivial: under training BatchNorm with default affines, (out.x ** 2).sum() is nearly
constant and its attn_bias gradient nearly 0.  The norm of each case's grad_attn_bias is printed.  Every fixture stays
below 1 MB.
"""
import os
import sys
import zlib

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from biased_util import make_bias  # noqa: E402
from graphgps_b200.batch import make_batch  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402

OUT = os.path.join(HERE, "biased")

# name, local, shape, d, heads, act, num_graphs, training, batch_norm, bias kind
CASES = [
    ("gine_biased_relu", "GINE", "zinc-gine", 64, 4, "relu", 7, True, True, "random"),
    ("gine_biased_eval", "GINE", "zinc-gine", 64, 4, "relu", 6, False, True, "random"),
    ("gine_biased_gelu", "GINE", "zinc-gine", 64, 4, "gelu", 6, True, True, "random"),
    ("gatedgcn_biased_relu", "CustomGatedGCN", "zinc-gatedgcn", 64, 4, "relu", 4, True, True, "random"),
    ("none_biased_relu", "None", "zinc-gine", 64, 4, "relu", 6, True, True, "random"),
    ("gine_biased_nonorm", "GINE", "zinc-gine", 64, 4, "relu", 6, True, False, "random"),
    ("gine_biased_graph_token", "GINE", "zinc-gine", 64, 4, "relu", 6, True, True, "graph_token"),
    ("gine_biased_spd", "GINE", "zinc-gine", 64, 4, "relu", 6, True, True, "spd"),
]
LIVE_NAME = "reference_live_GINE_BiasedTransformer"


def run_case(ref, name, local, shape, d, heads, act, B, training, batch_norm, kind):
    seed = zlib.crc32(name.encode()) % (2 ** 31)
    torch.manual_seed(seed)
    layer = ref.GPSLayer(d, local, "BiasedTransformer", heads, act=act, batch_norm=batch_norm)
    with torch.no_grad():   # non-trivial BatchNorm affine + running stats so they are actually exercised
        for m in layer.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.3, 0.3)
                m.running_mean.uniform_(-0.2, 0.2)
                m.running_var.uniform_(0.6, 1.4)
    batch = make_batch(shape, seed=11, dim=d, num_graphs=B)
    bias = make_bias(batch.batch, B, heads, seed % 1000, kind, batch.edge_index)
    state = {k: v.clone() for k, v in layer.state_dict().items()}
    fix = {"config": dict(name=name, local=local, glob="BiasedTransformer", d=d, heads=heads, act=act,
                          training=training, batch_norm=batch_norm, bias_kind=kind),
           "x": batch.x.clone(), "edge_index": batch.edge_index.clone(), "edge_attr": batch.edge_attr.clone(),
           "batch": batch.batch.clone(), "num_graphs": B, "state": state, "attn_bias": bias}
    layer = layer.double()
    layer.train(training)
    b = batch.clone()
    b.x = b.x.double().requires_grad_(True)
    b.edge_attr = b.edge_attr.double().requires_grad_(True)
    b.attn_bias = bias.double().requires_grad_(True)
    x_in, e_in, ab_in = b.x, b.edge_attr, b.attn_bias
    out = layer(b)
    g = torch.Generator().manual_seed(5)
    ct_x = torch.randn(out.x.shape, generator=g)
    fix["ct_x"] = ct_x
    fix["out_x"] = out.x.detach().float()
    loss = (out.x * ct_x.double()).sum()
    if local == "CustomGatedGCN":
        ct_e = torch.randn(out.edge_attr.shape, generator=g)
        fix["ct_e"] = ct_e
        fix["out_e"] = out.edge_attr.detach().float()
        loss = loss + (out.edge_attr * ct_e.double()).sum()
    if training:
        loss.backward()
        fix["grad_x"] = x_in.grad.float()
        if local in ("CustomGatedGCN", "GINE"):
            fix["grad_e"] = e_in.grad.float()
        fix["grad_attn_bias"] = ab_in.grad.float()
        fix["grad_params"] = {n: p.grad.float() for n, p in layer.named_parameters() if p.grad is not None}
    fix["state_after"] = {k: v.detach().float() if v.is_floating_point() else v.clone()
                          for k, v in layer.state_dict().items() if "running" in k or "num_batches" in k}
    return fix


def run_live_case(ref):
    """The reference layer in fp64 on seeded inputs (GINE, d = 32, 4 heads, 7 zinc-shaped graphs), attn_bias gradient
    included."""
    torch.manual_seed(3)
    R = ref.GPSLayer(32, "GINE", "BiasedTransformer", 4)
    b = make_batch("zinc-gine", seed=5, dim=32, num_graphs=7, dtype=torch.float64)
    bias = make_bias(b.batch, 7, 4, 6).double()
    state = {k: v.clone() for k, v in R.state_dict().items()}
    R = R.double()
    fix = {"local": "GINE", "glob": "BiasedTransformer", "state": state, "x": b.x.clone(),
           "edge_index": b.edge_index.clone(), "edge_attr": b.edge_attr.clone(), "batch": b.batch.clone(),
           "num_graphs": 7, "attn_bias": bias.clone()}
    b.x.requires_grad_(True)
    b.edge_attr.requires_grad_(True)
    b.attn_bias = bias.requires_grad_(True)
    x_in = b.x
    o = R(b)
    ct = torch.randn(o.x.shape, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    fix["ct_x"] = ct
    (o.x * ct).sum().backward()
    fix["out_x"] = o.x.detach().clone()
    fix["grad_x"] = x_in.grad.clone()
    fix["grad_attn_bias"] = bias.grad.clone()
    fix["grad_params"] = {n: p.grad.clone() for n, p in R.named_parameters() if p.grad is not None}
    return fix


def main():
    args = sys.argv[1:]
    ref = load_reference(args[0] if args else None)
    os.makedirs(OUT, exist_ok=True)
    for case in CASES:
        fix = run_case(ref, *case)
        path = os.path.join(OUT, case[0] + ".pt")
        torch.save(fix, path)
        gb = fix.get("grad_attn_bias")
        print(case[0], "N", fix["x"].shape[0], "Nmax", fix["attn_bias"].shape[-1],
              "|grad_attn_bias|", "%.4g" % float(gb.norm()) if gb is not None else "-",
              f"{os.path.getsize(path)/1e3:.0f} kB")
    fix = run_live_case(ref)
    path = os.path.join(OUT, LIVE_NAME + ".pt")
    torch.save(fix, path)
    print(LIVE_NAME, "|grad_attn_bias| %.4g" % float(fix["grad_attn_bias"].norm()), f"{os.path.getsize(path)/1e3:.0f} kB")


if __name__ == "__main__":
    main()
