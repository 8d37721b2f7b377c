"""Generates tests/golden/*.pt from the REFERENCE ITSELF (its own layer files run verbatim under
oracle/ref_shim.py, fp64), so the fixtures pin both the oracle and the CUDA path without the reference.

    python tests/golden/make_golden.py [REFERENCE_LAYER_DIR] [names...]

REFERENCE_LAYER_DIR is graphgps/layer of a GraphGPS checkout (default: oracle/_ref).  Every fixture stays below
1 MB: the sizes below are chosen for that (parameters and their gradients dominate).

Each fixture holds: config, inputs (x, edge_index, edge_attr, batch), the module state_dict (fp32),
the cotangents used for the backward pass, and the reference's outputs / input gradients /
parameter gradients / updated BatchNorm running statistics (computed in fp64, stored as fp32).
"""
import os
import zlib
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from graphgps_b200.batch import make_batch, batch_from_lists  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

CASES = [
    # name, local, global, shape, d, heads, act, num_graphs, training
    ("gatedgcn_transformer_relu", "CustomGatedGCN", "Transformer", "zinc-gatedgcn", 64, 4, "relu", 6, True),
    ("gatedgcn_transformer_gelu", "CustomGatedGCN", "Transformer", "pcqm4m-small", 48, 4, "gelu", 12, True),
    ("gatedgcn_transformer_hd76", "CustomGatedGCN", "Transformer", "pcqm4m-small", 76, 1, "relu", 6, True),
    ("gine_transformer_relu", "GINE", "Transformer", "zinc-gine", 64, 4, "relu", 6, True),
    ("gatedgcn_none_relu", "CustomGatedGCN", "None", "zinc-gatedgcn", 32, 4, "relu", 5, True),
    ("none_transformer_relu", "None", "Transformer", "zinc-gine", 32, 2, "relu", 5, True),
    ("gine_none_gelu", "GINE", "None", "zinc-gine", 32, 4, "gelu", 5, True),
    ("gatedgcn_transformer_eval", "CustomGatedGCN", "Transformer", "zinc-gatedgcn", 64, 4, "relu", 6, False),
    ("gatedgcn_performer_relu", "CustomGatedGCN", "Performer", "zinc-gatedgcn", 48, 2, "relu", 6, True),
    ("code2_gatedgcn_transformer", "CustomGatedGCN", "Transformer", "code2", 32, 4, "relu", 3, True),
    # GCN: the aggregation is PyG's GCNConv (third party) as restated in oracle/ref_shim.py; the composition is the
    # reference's own gps_layer.py
    ("gcn_transformer_relu", "GCN", "Transformer", "zinc-gine", 64, 4, "relu", 6, True),
    ("gcn_transformer_hd76", "GCN", "Transformer", "pcqm4m-small", 76, 1, "gelu", 8, True),
]

# tests/golden/reference_live/<local>_<glob>.pt: the reference layer (fp64, seed 3, d=32, 4 heads) on one seeded
# zinc-shaped batch; tests/test_oracle.py::test_oracle_equals_reference_live holds the oracle to it at 1e-9
LIVE_CASES = [("CustomGatedGCN", "Transformer"), ("GINE", "Transformer"), ("CustomGatedGCN", "Performer"),
              ("None", "Transformer"), ("GINE", "None"), ("GCN", "Transformer"), ("GCN", "None")]


def run_live_case(ref, local, glob):
    torch.manual_seed(3)
    R = ref.GPSLayer(32, local, glob, 4)
    state = {k: v.clone() for k, v in R.state_dict().items()}   # fp32 init: stored exactly
    R = R.double()
    b = make_batch("zinc-gatedgcn", seed=5, dim=32, num_graphs=7, dtype=torch.float64)
    fix = {"local": local, "glob": glob, "state": state, "x": b.x.clone(), "edge_index": b.edge_index.clone(),
           "edge_attr": b.edge_attr.clone(), "batch": b.batch.clone(), "num_graphs": 7}
    b.x.requires_grad_(True)
    b.edge_attr.requires_grad_(True)
    x_in = b.x
    o = R(b)
    (o.x ** 2).sum().backward()
    fix["out_x"] = o.x.detach().clone()
    fix["grad_x"] = x_in.grad.clone()
    fix["grad_params"] = {n: p.grad.clone() for n, p in R.named_parameters() if p.grad is not None}
    return fix


def run_case(ref, name, local, glob, shape, d, heads, act, B, training):
    torch.manual_seed(zlib.crc32(name.encode()) % (2 ** 31))
    layer = ref.GPSLayer(d, local, glob, heads, act=act)
    # non-trivial BatchNorm affine + running stats so they are actually exercised
    with torch.no_grad():
        for m in layer.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.3, 0.3)
                m.running_mean.uniform_(-0.2, 0.2)
                m.running_var.uniform_(0.6, 1.4)
        if local == "GCN":
            layer.local_model.bias.uniform_(-0.3, 0.3)   # PyG initialises it to zero
    state = {k: v.clone() for k, v in layer.state_dict().items()}
    batch = make_batch(shape, seed=11, dim=d, num_graphs=B)
    fix = {"config": dict(name=name, local=local, glob=glob, d=d, heads=heads, act=act, training=training),
           "x": batch.x.clone(), "edge_index": batch.edge_index.clone(), "edge_attr": batch.edge_attr.clone(),
           "batch": batch.batch.clone(), "num_graphs": B, "state": state}
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


def main():
    args = sys.argv[1:]
    layer_dir = args.pop(0) if args and os.path.isdir(args[0]) else None
    ref = load_reference(layer_dir)
    only = set(args)   # optional: regenerate just the named fixtures
    for case in CASES:
        if only and case[0] not in only:
            continue
        fix = run_case(ref, *case)
        path = os.path.join(HERE, case[0] + ".pt")
        torch.save(fix, path)
        print(case[0], "N", fix["x"].shape[0], "E", fix["edge_index"].shape[1], f"{os.path.getsize(path)/1e3:.0f} kB")
    os.makedirs(os.path.join(HERE, "reference_live"), exist_ok=True)
    for local, glob in LIVE_CASES:
        name = f"{local}_{glob}"
        if only and name not in only:
            continue
        path = os.path.join(HERE, "reference_live", name + ".pt")
        torch.save(run_live_case(ref, local, glob), path)
        print("reference_live", name, f"{os.path.getsize(path)/1e3:.0f} kB")


if __name__ == "__main__":
    main()
