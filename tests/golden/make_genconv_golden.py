"""Generates tests/golden/genconv/*.pt: GPSLayer(dim_h, 'GENConv', ...) fixtures from the REFERENCE's own gps_layer.py
run verbatim under oracle/ref_shim.py in fp64, with tests/genconv_oracle.py's GENConvMP installed as PyG's GENConv.

    python tests/golden/make_genconv_golden.py [REFERENCE_LAYER_DIR]

The fixtures live in a subdirectory because tests/util.py::golden_names() feeds every tests/golden/*.pt to tests that
build other layers.  Each holds what a make_golden.py fixture holds (config, inputs, reference state_dict, cotangents,
fp64 outputs / gradients / running statistics stored as fp32, grad_e = the edge_attr gradient), plus attn_bias and its
gradient for the BiasedTransformer case.  reference_live_GENConv_Transformer.pt keeps everything in fp64 and pins the
oracle at 1e-10 / 1e-9.

The batches (genconv_oracle.genconv_batch) hold self-loop edges, duplicated edges, a hub with 40 in-edges, an isolated
node and a node whose messages are all 1e-7.  x and edge_attr are scaled by 3 so that the messages of one segment spread
over several units per channel: with near-uniform softmax weights a mean or sum aggregation would pass a 1e-3 test.
Cotangents are random, and the BatchNorm affines and running statistics (local_model.mlp.1 included) non-trivial.
Every fixture stays below 1 MB.
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
from genconv_oracle import genconv_batch, shim_genconv  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402

OUT = os.path.join(HERE, "genconv")

# name, global, shape, d, heads, act, num_graphs, training, batch_norm
CASES = [
    ("genconv_transformer_relu", "Transformer", "zinc-gine", 64, 4, "relu", 6, True, True),
    ("genconv_transformer_gelu", "Transformer", "zinc-gine", 64, 4, "gelu", 6, True, True),
    ("genconv_transformer_eval", "Transformer", "zinc-gine", 64, 4, "relu", 6, False, True),
    ("genconv_transformer_nonorm", "Transformer", "zinc-gine", 64, 4, "relu", 6, True, False),
    ("genconv_biased_relu", "BiasedTransformer", "zinc-gine", 64, 4, "relu", 6, True, True),
    ("genconv_performer_relu", "Performer", "zinc-gine", 32, 4, "relu", 4, True, True),
    ("genconv_none_relu", "None", "zinc-gine", 64, 4, "relu", 6, True, True),
]
LIVE_NAME = "reference_live_GENConv_Transformer"


def _prepare(layer):
    with torch.no_grad():
        for m in layer.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.3, 0.3)
                m.running_mean.uniform_(-0.2, 0.2)
                m.running_var.uniform_(0.6, 1.4)


def run_case(ref, name, glob, shape, d, heads, act, B, training, batch_norm, dtype=torch.float32):
    seed = zlib.crc32(name.encode()) % (2 ** 31)
    torch.manual_seed(seed)
    with shim_genconv():
        layer = ref.GPSLayer(d, "GENConv", glob, heads, act=act, batch_norm=batch_norm)
    _prepare(layer)
    batch = genconv_batch(shape, 11, d, B, dtype)
    state = {k: v.clone() for k, v in layer.state_dict().items()}
    fix = {"config": dict(name=name, local="GENConv", glob=glob, d=d, heads=heads, act=act, training=training,
                          batch_norm=batch_norm),
           "x": batch.x.clone(), "edge_index": batch.edge_index.clone(), "edge_attr": batch.edge_attr.clone(),
           "batch": batch.batch.clone(), "num_graphs": batch.num_graphs, "state": state}
    bias = None
    if glob == "BiasedTransformer":
        bias = make_bias(batch.batch, batch.num_graphs, heads, seed % 1000).to(dtype)
        fix["attn_bias"] = bias
    layer = layer.double()
    layer.train(training)
    b = batch.clone()
    b.x = b.x.double().requires_grad_(True)
    b.edge_attr = b.edge_attr.double().requires_grad_(True)
    x_in, e_in = b.x, b.edge_attr
    if bias is not None:
        b.attn_bias = bias.double().requires_grad_(True)
    out = layer(b)
    g = torch.Generator().manual_seed(5)
    ct_x = torch.randn(out.x.shape, generator=g, dtype=torch.float64).to(dtype)
    fix["ct_x"] = ct_x
    keep = (lambda t: t.detach().clone()) if dtype == torch.float64 else (lambda t: t.detach().float())
    fix["out_x"] = keep(out.x)
    if training or dtype == torch.float64:
        (out.x * ct_x.double()).sum().backward()
        fix["grad_x"] = keep(x_in.grad)
        fix["grad_e"] = keep(e_in.grad)
        if bias is not None:
            fix["grad_attn_bias"] = keep(b.attn_bias.grad)
        fix["grad_params"] = {n: keep(p.grad) for n, p in layer.named_parameters() if p.grad is not None}
    fix["state_after"] = {k: (keep(v) if v.is_floating_point() else v.clone())
                          for k, v in layer.state_dict().items() if "running" in k or "num_batches" in k}
    return fix


def main():
    args = sys.argv[1:]
    ref = load_reference(args[0] if args else None)
    os.makedirs(OUT, exist_ok=True)
    for case in CASES:
        fix = run_case(ref, *case)
        path = os.path.join(OUT, case[0] + ".pt")
        torch.save(fix, path)
        ge = fix.get("grad_e")
        print(case[0], "N", fix["x"].shape[0], "E", fix["edge_index"].shape[1],
              "|grad_e| %.4g" % float(ge.norm()) if ge is not None else "-", f"{os.path.getsize(path)/1e3:.0f} kB")
    fix = run_case(ref, LIVE_NAME, "Transformer", "zinc-gine", 32, 4, "relu", 5, True, True, dtype=torch.float64)
    path = os.path.join(OUT, LIVE_NAME + ".pt")
    torch.save(fix, path)
    print(LIVE_NAME, f"{os.path.getsize(path)/1e3:.0f} kB")


if __name__ == "__main__":
    main()
