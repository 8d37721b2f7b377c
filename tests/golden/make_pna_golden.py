"""Generates tests/golden/pna/*.pt: GPSLayer(dim_h, 'PNA', ...) fixtures from the REFERENCE's own gps_layer.py run
verbatim under oracle/ref_shim.py in fp64, with tests/pna_oracle.py's PNAConvMP installed as PyG's PNAConv.

    python tests/golden/make_pna_golden.py [REFERENCE_LAYER_DIR]

The fixtures live in a subdirectory because tests/util.py::golden_names() feeds every tests/golden/*.pt to tests that
build other layers.  Each holds what a make_golden.py fixture holds (config with pna_degrees, inputs, reference
state_dict, cotangents, fp64 outputs / gradients / running statistics stored as fp32, grad_e = the edge_attr gradient),
plus attn_bias and its gradient for the BiasedTransformer case.  reference_live_PNA_Transformer.pt keeps everything in
fp64 and pins the oracle at 1e-10 / 1e-9.

The batches (pna_oracle.pna_batch) hold self-loop edges, duplicated edges, an exact duplicate (a tie in every channel),
a hub with 40 in-edges and an isolated node; edge_attr is min(128, d) wide.  pna_d160 has de = 128 < d: its state_dict
alone would pass 1 MB, so it stores the seed of pna_oracle.seeded_state instead ("state_seed") and the gradients of
edge_encoder, pre_nns, lin and post's bias only.  Every fixture stays below 1 MB.
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
from oracle.ref_shim import load_reference  # noqa: E402
from pna_oracle import pna_batch, seeded_state, shim_pna  # noqa: E402

OUT = os.path.join(HERE, "pna")
DEGREES = [0, 3, 11, 9, 4, 1]

# name, global, shape, d, heads, act, num_graphs, training, batch_norm
CASES = [
    ("pna_transformer_relu", "Transformer", "zinc-gine", 64, 4, "relu", 6, True, True),
    ("pna_transformer_gelu", "Transformer", "zinc-gine", 64, 4, "gelu", 6, True, True),
    ("pna_transformer_eval", "Transformer", "zinc-gine", 64, 4, "relu", 6, False, True),
    ("pna_transformer_nonorm", "Transformer", "zinc-gine", 64, 4, "relu", 6, True, False),
    ("pna_biased_relu", "BiasedTransformer", "zinc-gine", 64, 4, "relu", 4, True, True),
    ("pna_performer_relu", "Performer", "zinc-gine", 32, 4, "relu", 4, True, True),
    ("pna_none_relu", "None", "zinc-gine", 64, 4, "relu", 6, True, True),
    ("pna_d160_none", "None", "zinc-gine", 160, 4, "relu", 2, True, True),
]
LIVE_NAME = "reference_live_PNA_Transformer"
# the gradients pna_d160_none keeps: the edge path (edge_encoder, pre_nns), lin and post's bias
LARGE_GRADS = ("local_model.edge_encoder.", "local_model.pre_nns.", "local_model.lin.", "local_model.post_nns.0.0.bias")


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
    with shim_pna():
        layer = ref.GPSLayer(d, "PNA", glob, heads, act=act, pna_degrees=DEGREES, batch_norm=batch_norm)
    _prepare(layer)
    large = d > 128
    if large:
        layer.load_state_dict(seeded_state(layer, seed), strict=True)
    batch = pna_batch(shape, 11, d, B, dtype)
    fix = {"config": dict(name=name, local="PNA", glob=glob, d=d, heads=heads, act=act, training=training,
                          batch_norm=batch_norm, pna_degrees=DEGREES),
           "x": batch.x.clone(), "edge_index": batch.edge_index.clone(), "edge_attr": batch.edge_attr.clone(),
           "batch": batch.batch.clone(), "num_graphs": batch.num_graphs}
    if large:
        fix["state_seed"] = seed
    else:
        fix["state"] = {k: v.clone() for k, v in layer.state_dict().items()}
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
        fix["grad_params"] = {n: keep(p.grad) for n, p in layer.named_parameters()
                              if p.grad is not None and (not large or n.startswith(LARGE_GRADS))}
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
