"""Generates tests/golden/san/*.pt: SANLayer fixtures from the REFERENCE's own san_layer.py and graphgps/utils.py
(negate_edge_index) run verbatim in fp64, loaded by path after oracle/ref_shim.load_reference().  Their third-party
imports come from stubs defined here:
  * torch_scatter.scatter(src, index, dim=0, out=out, reduce='add'): out.index_add_ (san_layer.py:75,81,85,87);
  * torch_geometric.utils.scatter(src, index, dim=0, dim_size, reduce) for 'sum' and 'mul' with torch_scatter's
    semantics: the output starts at 0 for 'sum' and at 1 for 'mul', so positions no index touches keep 1 - the
    reading under which negate_edge_index (utils.py:56) yields the complement;
  * torch_geometric.utils.remove_self_loops and degree; yacs.config.CfgNode.
They are installed only while the two files load, so ref_shim's own stubs stay as they are.

    python tests/golden/make_san_golden.py [REFERENCE_ROOT] [CASE ...]

Each fixture holds the config, the batch (x, edge_attr, edge_index, batch, num_graphs), the state_dict of the layer (or
of the layer stack), the cotangent, the output and every gradient, stored as fp32; reference_live keeps fp64, pins
tests/san_oracle.py at 1e-10 / 1e-9, and holds `init_state`, the reference layer's state_dict right after
construction from torch.manual_seed(INIT_SEED), and `fake_pairs`, negate_edge_index's output for its batch.  Dropout
is 0 in every fixture.
"""
import importlib.util
import os
import sys
import types
import zlib

import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle.ref_shim import load_reference  # noqa: E402
from san_oracle import SanBatch, dataset_sizes, san_batch  # noqa: E402

OUT = os.path.join(HERE, "san")
INIT_SEED = 4321


# ----------------------------------------------------------------------------- stubs
def _ts_scatter(src, index, dim=0, out=None, dim_size=None, reduce="sum"):
    assert dim == 0 and out is not None and reduce in ("add", "sum")
    return out.index_add_(0, index, src)


def _pyg_scatter(src, index, dim=0, dim_size=None, reduce="sum"):
    assert dim == 0
    size = (dim_size if dim_size is not None else int(index.max()) + 1,) + tuple(src.shape[1:])
    if reduce == "sum":
        return torch.zeros(size, dtype=src.dtype, device=src.device).index_add_(0, index, src)
    if reduce == "mul":
        out = torch.ones(size, dtype=src.dtype, device=src.device)
        return out.scatter_reduce_(0, index, src, reduce="prod", include_self=True)
    raise NotImplementedError(reduce)


def _remove_self_loops(edge_index, edge_attr=None):
    keep = edge_index[0] != edge_index[1]
    return edge_index[:, keep], (edge_attr[keep] if edge_attr is not None else None)


def _degree(index, num_nodes=None, dtype=None):
    n = num_nodes if num_nodes is not None else (int(index.max()) + 1 if index.numel() else 0)
    return torch.zeros(n, dtype=dtype or torch.float).index_add_(0, index, torch.ones(index.numel(), dtype=dtype or torch.float))


def load_san(ref_root=None):
    """The reference's san_layer module (its negate_edge_index bound from graphgps/utils.py), loaded verbatim."""
    ref_root = ref_root or "/root/reference"
    load_reference()
    saved = {k: sys.modules.get(k) for k in ("torch_scatter", "torch_geometric.utils", "yacs", "yacs.config")}
    utils = types.ModuleType("torch_geometric.utils")
    utils.__dict__.update(sys.modules["torch_geometric.utils"].__dict__)
    utils.scatter, utils.remove_self_loops, utils.degree = _pyg_scatter, _remove_self_loops, _degree
    yacs_config = types.ModuleType("yacs.config")
    yacs_config.CfgNode = dict
    try:
        sys.modules["torch_scatter"] = types.SimpleNamespace(scatter=_ts_scatter)
        sys.modules["torch_geometric.utils"] = utils
        sys.modules["yacs"] = types.ModuleType("yacs")
        sys.modules["yacs.config"] = yacs_config
        mods = {}
        for name, rel in (("graphgps.utils", "graphgps/utils.py"), ("graphgps.layer.san_layer",
                                                                     "graphgps/layer/san_layer.py")):
            spec = importlib.util.spec_from_file_location(name, os.path.join(ref_root, rel))
            m = importlib.util.module_from_spec(spec)
            sys.modules[name] = m
            spec.loader.exec_module(m)
            mods[name] = m
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return mods["graphgps.layer.san_layer"], mods["graphgps.utils"]


# ----------------------------------------------------------------------------- cases
def edge_case_batch(d, seed, dtype=torch.float32):
    """Three graphs: 6 nodes with a self loop, a duplicated edge, a one-way (directed) edge and an isolated node; a
    one-node graph; 4 nodes with a self loop on the last."""
    src = [0, 1, 1, 2, 2, 3, 0, 4, 2, 6, 7, 8, 9, 10, 10]
    dst = [1, 0, 2, 1, 2, 0, 1, 3, 1, 6, 8, 7, 8, 9, 10]
    ei = torch.tensor([src, dst], dtype=torch.int64)   # node 5 isolated, node 6 alone with its self loop
    batch = torch.tensor([0] * 6 + [1] + [2] * 4, dtype=torch.int64)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(11, d, generator=g, dtype=torch.float64).to(dtype)
    e = torch.randn(ei.shape[1], d, generator=g, dtype=torch.float64).to(dtype)
    return SanBatch(x, e, ei, batch, 3)


# name, d, heads, gamma, kind, sizes, training, layers, weight scale of Q/K/E/Q_2/K_2
CASES = [
    ("zinc_hd7", 56, 8, 1e-5, "mol", dataset_sizes("mol", 6, 1), True, 1, 1.0),
    ("pattern_dense_hd6", 24, 4, 1e-1, "sbm", [50, 40], True, 1, 1.0),
    ("coco_hd11_knn", 44, 4, 1e-6, "knn", [200], True, 1, 1.0),
    ("molhiv_hd16_eval", 64, 4, 1e-5, "mol", dataset_sizes("mol", 4, 2), False, 1, 1.0),
    ("peptides_hd21", 84, 4, 1e-1, "chain", [70], True, 1, 1.0),
    ("molpcba_hd76", 76, 1, 1e-5, "mol", [20, 18], True, 1, 1.0),
    ("saturate_hd8", 32, 4, 1e-1, "mol", dataset_sizes("mol", 4, 3), True, 1, 4.0),
    ("edge_cases_hd6", 24, 4, 1e-1, "edge_cases", None, True, 1, 1.0),
    ("two_layer_shared_hd6", 24, 4, 1e-1, "mol", dataset_sizes("mol", 3, 4), True, 2, 1.0),
]
LIVE = ("reference_live", 16, 2, 1e-1, "edge_cases", None, True, 2, 1.5)


def _prepare(layer, wscale, g):
    with torch.no_grad():
        for bn in (layer.batch_norm1_h, layer.batch_norm2_h):
            bn.weight.uniform_(0.5, 1.5, generator=g)
            bn.bias.uniform_(-0.3, 0.3, generator=g)
            bn.running_mean.uniform_(-0.5, 0.5, generator=g)
            bn.running_var.uniform_(0.5, 2.0, generator=g)
        att = layer.attention
        for lin in (att.Q, att.K, att.E, att.Q_2, att.K_2):
            lin.weight.mul_(wscale)


def run_case(san, name, d, heads, gamma, kind, sizes, training, layers, wscale, dtype=torch.float32):
    seed = zlib.crc32(name.encode()) % (2 ** 31)
    torch.manual_seed(seed)
    emb = nn.Embedding(1, d)
    stack = nn.Sequential(*[san.SANLayer(gamma, d, d, heads, True, emb, dropout=0.0) for _ in range(layers)])
    g = torch.Generator().manual_seed(seed)
    for layer in stack:
        _prepare(layer, wscale, g)
    b = edge_case_batch(d, seed % 1000, dtype) if kind == "edge_cases" else san_batch(kind, sizes, d, seed % 1000, dtype)
    state = {k: v.clone() for k, v in (stack[0] if layers == 1 else stack).state_dict().items()}
    fix = {"config": dict(name=name, d=d, heads=heads, gamma=gamma, kind=kind, training=training, layers=layers),
           "x": b.x.clone(), "edge_attr": b.edge_attr.clone(), "edge_index": b.edge_index.clone(),
           "batch": b.batch.clone(), "num_graphs": b.num_graphs, "state": state}
    stack = stack.double()
    stack.train(training)
    data = SanBatch(b.x.double().clone().requires_grad_(True), b.edge_attr.double().clone().requires_grad_(True),
                    b.edge_index, b.batch, b.num_graphs)
    x_in, e_in = data.x, data.edge_attr
    out = stack(data).x
    ct = torch.randn(out.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    (out * ct).sum().backward()
    keep = (lambda t: t.detach().clone()) if dtype == torch.float64 else (lambda t: t.detach().float())
    fix["ct"] = ct.to(dtype)
    fix["out"] = keep(out)
    fix["grad_x"] = keep(x_in.grad)
    fix["grad_edge_attr"] = keep(e_in.grad)
    named = (stack[0] if layers == 1 else stack).named_parameters()
    fix["grad_params"] = {n: keep(p.grad) for n, p in named}
    return fix


def main():
    args = sys.argv[1:]
    names = {c[0] for c in CASES} | {LIVE[0]}
    ref_root = args[0] if args and args[0] not in names else None
    only = [a for a in args if a in names]
    san, utils = load_san(ref_root)
    os.makedirs(OUT, exist_ok=True)
    for case in CASES:
        if only and case[0] not in only:
            continue
        fix = run_case(san, *case)
        path = os.path.join(OUT, case[0] + ".pt")
        torch.save(fix, path)
        print(case[0], "N", fix["x"].shape[0], "E", fix["edge_index"].shape[1], f"{os.path.getsize(path)/1e3:.0f} kB")
    if only and LIVE[0] not in only:
        return
    fix = run_case(san, *LIVE, dtype=torch.float64)
    fix["fake_pairs"] = utils.negate_edge_index(fix["edge_index"], fix["batch"])
    torch.manual_seed(INIT_SEED)
    fix["init_seed"] = INIT_SEED
    emb = nn.Embedding(1, 56)
    fix["init_state"] = {k: v.clone() for k, v in san.SANLayer(0.1, 56, 56, 8, True, emb, 0.2).state_dict().items()}
    path = os.path.join(OUT, LIVE[0] + ".pt")
    torch.save(fix, path)
    print(LIVE[0], f"{os.path.getsize(path)/1e3:.0f} kB")


if __name__ == "__main__":
    main()
