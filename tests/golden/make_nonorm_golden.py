"""Generates tests/golden/nonorm/*.pt: GPSLayer(..., batch_norm=False) fixtures from the REFERENCE ITSELF (its own
layer files run verbatim under oracle/ref_shim.py, fp64), next to the fixtures of tests/golden/make_golden.py.

    python tests/golden/make_nonorm_golden.py [REFERENCE_LAYER_DIR]

The fixtures live in a subdirectory because tests/util.py::golden_names() feeds every tests/golden/*.pt to tests that
build BatchNorm layers.  Each holds what a make_golden.py fixture holds (config, inputs, reference state_dict,
cotangents, fp64 outputs / gradients / running statistics stored as fp32); config["batch_norm"] is False.  The
single-graph cases are node-level batches (the whole graph is the batch, as the GCN+Transformer configs train) drawn
by tests/nonorm_util.py::node_graph; the WebKB-sized one also has a self loop, a duplicate edge and an isolated node.
reference_live_GCN_Transformer.pt is the reference_live-style case (fp64 inputs, weights, outputs and gradients) that
pins the oracle at 1e-10 / 1e-9.  Every fixture stays below 1 MB.
"""
import os
import sys
import zlib

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from graphgps_b200.batch import make_batch  # noqa: E402
from nonorm_util import LIVE_NAME, node_graph, with_edge_cases  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "nonorm")

# name, local, global, batch, d, heads, act, training.  batch: ("node", N, E) = one directed graph, or
# (shape, num_graphs) = a multi-graph batch of a make_batch shape
CASES = [
    ("gcn_transformer_gelu_webkb", "GCN", "Transformer", ("node-edge-cases", 183, 325), 64, 4, "gelu", True),
    ("gcn_transformer_gelu_hd24", "GCN", "Transformer", ("node", 96, 240), 96, 4, "gelu", True),
    ("gcn_none_gelu", "GCN", "None", ("node", 150, 400), 64, 4, "gelu", True),
    ("gatedgcn_transformer_relu", "CustomGatedGCN", "Transformer", ("zinc-gatedgcn", 5), 48, 4, "relu", True),
    ("gine_transformer_gelu", "GINE", "Transformer", ("zinc-gine", 5), 48, 4, "gelu", True),
    ("none_transformer_gelu", "None", "Transformer", ("node", 120, 300), 32, 2, "gelu", True),
    ("gatedgcn_performer_relu", "CustomGatedGCN", "Performer", ("zinc-gatedgcn", 5), 48, 2, "relu", True),
    ("gatedgcn_transformer_eval", "CustomGatedGCN", "Transformer", ("zinc-gatedgcn", 5), 48, 4, "relu", False),
    ("gcn_transformer_gelu_multigraph", "GCN", "Transformer", ("zinc-gine", 6), 64, 4, "gelu", True),
]


def case_batch(spec, d, seed, dtype=torch.float32):
    if spec[0] in ("node", "node-edge-cases"):
        b = node_graph(spec[1], spec[2], d, seed=seed, dtype=dtype)
        return with_edge_cases(b, seed) if spec[0] == "node-edge-cases" else b
    return make_batch(spec[0], seed=11, dim=d, num_graphs=spec[1], dtype=dtype)


def run_case(ref, name, local, glob, spec, d, heads, act, training):
    torch.manual_seed(zlib.crc32(name.encode()) % (2 ** 31))
    layer = ref.GPSLayer(d, local, glob, heads, act=act, batch_norm=False)
    assert not any(k.startswith(("norm1_local.", "norm1_attn.", "norm2.")) for k in layer.state_dict())
    with torch.no_grad():
        for m in layer.modules():   # GatedGCN's own BatchNorms: non-trivial affine + running stats
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.3, 0.3)
                m.running_mean.uniform_(-0.2, 0.2)
                m.running_var.uniform_(0.6, 1.4)
        if local == "GCN":
            layer.local_model.bias.uniform_(-0.3, 0.3)   # PyG initialises it to zero
    state = {k: v.clone() for k, v in layer.state_dict().items()}
    batch = case_batch(spec, d, zlib.crc32(name.encode()) % 1000)
    fix = {"config": dict(name=name, local=local, glob=glob, d=d, heads=heads, act=act, training=training,
                          batch_norm=False),
           "x": batch.x.clone(), "edge_index": batch.edge_index.clone(), "edge_attr": batch.edge_attr.clone(),
           "batch": batch.batch.clone(), "num_graphs": batch.num_graphs, "state": state}
    layer = layer.double()
    layer.train(training)
    b = batch.clone()
    b.x = b.x.double().requires_grad_(True)
    b.edge_attr = b.edge_attr.double().requires_grad_(True)
    x_in, e_in = b.x, b.edge_attr
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
        if e_in.grad is not None:
            fix["grad_e"] = e_in.grad.float()
        fix["grad_params"] = {n: p.grad.float() for n, p in layer.named_parameters() if p.grad is not None}
    fix["state_after"] = {k: v.detach().float() if v.is_floating_point() else v.clone()
                          for k, v in layer.state_dict().items() if "running" in k or "num_batches" in k}
    return fix


def run_live_case(ref):
    """The reference GCN+Transformer layer in fp64 (d = 32, 4 heads, GELU) on one directed node-level graph."""
    torch.manual_seed(3)
    R = ref.GPSLayer(32, "GCN", "Transformer", 4, act="gelu", batch_norm=False)
    with torch.no_grad():
        R.local_model.bias.uniform_(-0.3, 0.3)
    state = {k: v.clone() for k, v in R.state_dict().items()}
    R = R.double()
    b = with_edge_cases(node_graph(140, 420, 32, seed=4, dtype=torch.float64), 4)
    fix = {"local": "GCN", "glob": "Transformer", "act": "gelu", "state": state, "x": b.x.clone(),
           "edge_index": b.edge_index.clone(), "edge_attr": b.edge_attr.clone(), "batch": b.batch.clone(),
           "num_graphs": 1}
    b.x.requires_grad_(True)
    x_in = b.x
    o = R(b)
    (o.x ** 2).sum().backward()
    fix["out_x"] = o.x.detach().clone()
    fix["grad_x"] = x_in.grad.clone()
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
        print(case[0], "N", fix["x"].shape[0], "E", fix["edge_index"].shape[1], f"{os.path.getsize(path)/1e3:.0f} kB")
    path = os.path.join(OUT, LIVE_NAME + ".pt")
    torch.save(run_live_case(ref), path)
    print(LIVE_NAME, f"{os.path.getsize(path)/1e3:.0f} kB")


if __name__ == "__main__":
    main()
