"""Generates tests/golden/custom_gnn/*.pt: fixtures of CustomGNN's GatedGCNLayer and GINEConvLayer made by running the
REFERENCE's own gatedgcn_layer.py and gine_conv_layer.py unmodified in fp64, loaded by oracle/ref_shim.load_reference().

    python tests/golden/make_custom_gnn_golden.py [CASE ...]

Each fixture holds the config, the batch (x, edge_attr, edge_index, batch, num_graphs), the state_dict of the layer
stack before the call, the cotangents of the last layer's batch.x (and, GatedGCN, batch.edge_attr), the outputs, every
gradient and the BatchNorm buffers after the call (running statistics updated in training mode), stored as fp32.
reference_live keeps fp64, pins tests/custom_gnn_oracle.py at 1e-10 / 1e-9 and holds `init_state` / `init_state_gine`,
the state_dicts of both layers right after construction from torch.manual_seed(INIT_SEED).  Dropout is 0 in every
fixture.
"""
import os
import sys
import zlib

import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle.ref_shim import load_reference  # noqa: E402
from custom_gnn_oracle import SanBatch, edge_case_batch, no_edge_batch, san_batch  # noqa: E402

OUT = os.path.join(HERE, "custom_gnn")
INIT_SEED = 2468
INIT_D = 24


def classes():
    load_reference()
    return (sys.modules["graphgps.layer.gatedgcn_layer"].GatedGCNLayer,
            sys.modules["graphgps.layer.gine_conv_layer"].GINEConvLayer)


# name, kind, d, act, residual, training, layers, batch kind, graph sizes
CASES = [
    ("gatedgcn_peptides_d138", "gatedgcn", 138, "relu", True, True, 1, "chain", [14, 10]),
    ("gatedgcn_voc_d108", "gatedgcn", 108, "relu", True, True, 1, "knn", [12, 10]),
    ("gatedgcn_gelu_d108", "gatedgcn", 108, "gelu", True, True, 1, "chain", [24]),
    ("gatedgcn_nores_d108", "gatedgcn", 108, "relu", False, True, 1, "chain", [20, 18]),
    ("gatedgcn_eval_d138", "gatedgcn", 138, "relu", True, False, 1, "chain", [22]),
    ("gatedgcn_stack3_d37", "gatedgcn", 37, "gelu", True, True, 3, "chain", [40, 33]),
    ("gatedgcn_edge_cases_d20", "gatedgcn", 20, "relu", True, True, 1, "edge_cases", None),
    ("gatedgcn_no_edges_d20", "gatedgcn", 20, "relu", True, True, 1, "no_edges", None),
    ("gine_peptides_d208", "gine", 208, None, True, True, 1, "chain", [12, 10]),
    ("gine_voc_d166", "gine", 166, None, True, True, 1, "knn", [14, 12]),
    ("gine_nores_d166", "gine", 166, None, False, True, 1, "chain", [24]),
    ("gine_eval_d208", "gine", 208, None, True, False, 1, "chain", [20]),
    ("gine_stack2_d37", "gine", 37, None, True, True, 2, "chain", [30, 22]),
    ("gine_edge_cases_d21", "gine", 21, None, True, True, 1, "edge_cases", None),
    ("gine_no_edges_d21", "gine", 21, None, True, True, 1, "no_edges", None),
]
LIVE = ("reference_live", "gatedgcn", 12, "gelu", True, True, 2, "edge_cases", None)
LIVE_GINE = ("reference_live_gine", "gine", 13, None, True, True, 2, "edge_cases", None)


def _prepare(layer, g):
    """Non-trivial BatchNorm affine parameters and running statistics, and a non-zero GINE eps."""
    with torch.no_grad():
        for name in ("bn_node_x", "bn_edge_e"):
            bn = getattr(layer, name, None)
            if bn is None:
                continue
            bn.weight.uniform_(0.5, 1.5, generator=g)
            bn.bias.uniform_(-0.3, 0.3, generator=g)
            bn.running_mean.uniform_(-0.5, 0.5, generator=g)
            bn.running_var.uniform_(0.5, 2.0, generator=g)
        if hasattr(layer, "model"):
            layer.model.eps.fill_(0.25)


def make_batch(kind, sizes, d, seed, dtype):
    if kind == "edge_cases":
        return edge_case_batch(d, seed, dtype)
    if kind == "no_edges":
        return no_edge_batch(d, seed, dtype)
    return san_batch(kind, sizes, d, seed, dtype)


def build(Gated, Gine, kind, d, act, residual):
    if kind == "gatedgcn":
        return Gated(d, d, dropout=0.0, residual=residual, act=act)
    return Gine(d, d, dropout=0.0, residual=residual)


def run_case(Gated, Gine, name, kind, d, act, residual, training, layers, bkind, sizes, dtype=torch.float32):
    seed = zlib.crc32(name.encode()) % (2 ** 31)
    torch.manual_seed(seed)
    stack = nn.Sequential(*[build(Gated, Gine, kind, d, act, residual) for _ in range(layers)])
    g = torch.Generator().manual_seed(seed)
    for layer in stack:
        _prepare(layer, g)
    b = make_batch(bkind, sizes, d, seed % 1000, dtype)
    state = {k: v.clone() for k, v in stack.state_dict().items()}
    fix = {"config": dict(name=name, kind=kind, d=d, act=act, residual=residual, training=training, layers=layers),
           "x": b.x.clone(), "edge_attr": b.edge_attr.clone(), "edge_index": b.edge_index.clone(),
           "batch": b.batch.clone(), "num_graphs": b.num_graphs, "state": state}
    stack = stack.double()
    stack.train(training)
    x_in = b.x.double().clone().requires_grad_(True)
    e_in = b.edge_attr.double().clone().requires_grad_(True)
    data = SanBatch(x_in, e_in, b.edge_index, b.batch, b.num_graphs)
    out = stack(data)
    gen = torch.Generator().manual_seed(5)
    ct_x = torch.randn(out.x.shape, generator=gen, dtype=torch.float64)
    loss = (out.x * ct_x).sum()
    ct_e = None
    if kind == "gatedgcn":
        ct_e = torch.randn(out.edge_attr.shape, generator=gen, dtype=torch.float64)
        loss = loss + (out.edge_attr * ct_e).sum()
    loss.backward()
    keep = (lambda t: t.detach().clone()) if dtype == torch.float64 else (lambda t: t.detach().float())
    fix["ct_x"] = ct_x.to(dtype)
    fix["ct_e"] = ct_e.to(dtype) if ct_e is not None else None
    fix["out_x"] = keep(out.x)
    fix["out_e"] = keep(out.edge_attr) if kind == "gatedgcn" else None
    fix["grad_x"] = keep(x_in.grad)
    fix["grad_edge_attr"] = keep(e_in.grad) if e_in.grad is not None else torch.zeros_like(b.edge_attr)
    fix["grad_params"] = {n: keep(p.grad) for n, p in stack.named_parameters()}
    # the buffers after the call (the parameters are unchanged)
    fix["state_after"] = {k: keep(v) if v.is_floating_point() else v.clone() for k, v in stack.state_dict().items()
                          if k.rsplit(".", 1)[-1] in ("running_mean", "running_var", "num_batches_tracked")}
    return fix


def main():
    only = sys.argv[1:]
    Gated, Gine = classes()
    os.makedirs(OUT, exist_ok=True)
    for case in CASES:
        if only and case[0] not in only:
            continue
        fix = run_case(Gated, Gine, *case)
        path = os.path.join(OUT, case[0] + ".pt")
        torch.save(fix, path)
        print(case[0], "N", fix["x"].shape[0], "E", fix["edge_index"].shape[1], f"{os.path.getsize(path)/1e3:.0f} kB")
    if only and LIVE[0] not in only:
        return
    fix = run_case(Gated, Gine, *LIVE, dtype=torch.float64)
    fix["gine"] = run_case(Gated, Gine, *LIVE_GINE, dtype=torch.float64)
    fix["init_seed"], fix["init_d"] = INIT_SEED, INIT_D
    torch.manual_seed(INIT_SEED)
    fix["init_state"] = {k: v.clone() for k, v in Gated(INIT_D, INIT_D, 0.1, True).state_dict().items()}
    torch.manual_seed(INIT_SEED)
    fix["init_state_gine"] = {k: v.clone() for k, v in Gine(INIT_D, INIT_D, 0.1, True).state_dict().items()}
    path = os.path.join(OUT, LIVE[0] + ".pt")
    torch.save(fix, path)
    print(LIVE[0], f"{os.path.getsize(path)/1e3:.0f} kB")


if __name__ == "__main__":
    main()
