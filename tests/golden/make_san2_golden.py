"""Generates tests/golden/san2/*.pt: SAN2Layer fixtures from the REFERENCE's own san2_layer.py and graphgps/utils.py
(negate_edge_index) run verbatim in fp64, loaded by path after oracle/ref_shim.load_reference().  Their third-party
imports come from stubs: those of make_san_golden.py (torch_scatter.scatter, torch_geometric.utils.scatter /
remove_self_loops / degree, yacs.config.CfgNode) and, with torch_scatter's semantics,
  * torch_scatter.scatter_max(src, index, dim=0, dim_size): the per-segment max, 0 for a segment no index touches (the
    reference reads only the values, san2_layer.py:28, so the argmax is not formed);
  * torch_scatter.scatter_add(src, index, dim=0, dim_size): the per-segment sum from 0;
  * torch_geometric.utils.num_nodes.maybe_num_nodes(index, num_nodes): num_nodes, else index.max() + 1 (0 when empty).
They are installed only while the two files load, so ref_shim's own stubs stay as they are.

    python tests/golden/make_san2_golden.py [REFERENCE_ROOT] [CASE ...]

Each fixture holds the config, the batch (x, edge_attr, edge_index, batch, num_graphs), the state_dict of the layer (or
of the layer stack; attention.gamma float64, set to the case's gamma), the cotangent, the output and every gradient,
stored as fp32 (gamma's gradient as fp64); `max_score` is the largest |score| of the first layer.  reference_live keeps
fp64, pins tests/san2_oracle.py at 1e-10 / 1e-9, and holds `init_state`, the reference layer's state_dict right after
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
sys.path.insert(0, HERE)
from oracle.ref_shim import load_reference  # noqa: E402
from make_san_golden import _degree, _prepare, _pyg_scatter, _remove_self_loops, _ts_scatter  # noqa: E402
from san_oracle import SanBatch, dataset_sizes, san_batch  # noqa: E402
from san2_oracle import scores  # noqa: E402

OUT = os.path.join(HERE, "san2")
INIT_SEED = 4321


# ----------------------------------------------------------------------------- stubs
def _seg_shape(src, index, dim, dim_size):
    assert dim == 0
    n = dim_size if dim_size is not None else (int(index.max()) + 1 if index.numel() else 0)
    return (n,) + tuple(src.shape[1:]), index.view((-1,) + (1,) * (src.dim() - 1)).expand_as(src)


def _scatter_max(src, index, dim=0, dim_size=None):
    size, idx = _seg_shape(src, index, dim, dim_size)
    out = torch.zeros(size, dtype=src.dtype, device=src.device)
    return out.scatter_reduce(0, idx, src, reduce="amax", include_self=False), None


def _scatter_add(src, index, dim=0, dim_size=None):
    size, _ = _seg_shape(src, index, dim, dim_size)
    return torch.zeros(size, dtype=src.dtype, device=src.device).index_add(0, index, src)


def _maybe_num_nodes(index, num_nodes=None):
    if num_nodes is not None:
        return num_nodes
    return int(index.max()) + 1 if index.numel() > 0 else 0


def load_san2(ref_root=None):
    """The reference's san2_layer module (its negate_edge_index bound from graphgps/utils.py), loaded verbatim."""
    ref_root = ref_root or "/root/reference"
    load_reference()
    keys = ("torch_scatter", "torch_geometric.utils", "torch_geometric.utils.num_nodes", "yacs", "yacs.config")
    saved = {k: sys.modules.get(k) for k in keys}
    utils = types.ModuleType("torch_geometric.utils")
    utils.__dict__.update(sys.modules["torch_geometric.utils"].__dict__)
    utils.scatter, utils.remove_self_loops, utils.degree = _pyg_scatter, _remove_self_loops, _degree
    num_nodes = types.ModuleType("torch_geometric.utils.num_nodes")
    num_nodes.maybe_num_nodes = _maybe_num_nodes
    utils.num_nodes = num_nodes
    yacs_config = types.ModuleType("yacs.config")
    yacs_config.CfgNode = dict
    try:
        sys.modules["torch_scatter"] = types.SimpleNamespace(scatter=_ts_scatter, scatter_max=_scatter_max,
                                                             scatter_add=_scatter_add)
        sys.modules["torch_geometric.utils"] = utils
        sys.modules["torch_geometric.utils.num_nodes"] = num_nodes
        sys.modules["yacs"] = types.ModuleType("yacs")
        sys.modules["yacs.config"] = yacs_config
        mods = {}
        for name, rel in (("graphgps.utils", "graphgps/utils.py"),
                          ("graphgps.layer.san2_layer", "graphgps/layer/san2_layer.py")):
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
    return mods["graphgps.layer.san2_layer"], mods["graphgps.utils"]


# ----------------------------------------------------------------------------- cases
def edge_case_batch(d, seed, dtype=torch.float32):
    """Five graphs: 6 nodes with a self loop, a duplicated edge, a one-way edge, a node without in-edges (4) and an
    isolated node (5); a one-node graph with a self loop; 4 nodes with a self loop on the last; a complete 3-node graph
    (no fake pairs); a one-node graph without edges (no term at all)."""
    src = [0, 1, 1, 2, 2, 3, 0, 4, 2, 6, 7, 8, 9, 10, 10, 11, 12, 11, 13, 12, 13]
    dst = [1, 0, 2, 1, 2, 0, 1, 3, 1, 6, 8, 7, 8, 9, 10, 12, 11, 13, 11, 13, 12]
    ei = torch.tensor([src, dst], dtype=torch.int64)
    batch = torch.tensor([0] * 6 + [1] + [2] * 4 + [3] * 3 + [4], dtype=torch.int64)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(15, d, generator=g, dtype=torch.float64).to(dtype)
    e = torch.randn(ei.shape[1], d, generator=g, dtype=torch.float64).to(dtype)
    return SanBatch(x, e, ei, batch, 5)


# name, d, heads, gamma (the value attention.gamma is set to), kind, sizes, training, layers, weight scale of
# Q/K/E/Q_2/K_2
CASES = [
    ("zinc_hd7", 56, 8, 0.5, "mol", dataset_sizes("mol", 6, 1), True, 1, 1.0),
    ("cluster_hd6", 48, 8, 0.5, "sbm", [30, 24], True, 1, 1.0),
    ("pattern_dense_hd8", 40, 5, 0.5, "sbm", [36, 28], True, 1, 1.0),
    ("coco_hd11_knn", 44, 4, 0.5, "knn", [200], True, 1, 1.0),
    ("peptides_hd21", 84, 4, 0.5, "chain", [70], True, 1, 1.0),
    ("molpcba_hd76", 76, 1, 0.5, "mol", [20, 18], True, 1, 1.0),
    ("molhiv_hd16_eval", 64, 4, 0.5, "mol", dataset_sizes("mol", 4, 2), False, 1, 1.0),
    ("edge_cases_hd6", 24, 4, 0.5, "edge_cases", None, True, 1, 1.0),
    ("no_clamp_hd8", 32, 4, 0.5, "mol", dataset_sizes("mol", 4, 3), True, 1, 5.0),
    ("gamma_2p5_hd7", 28, 4, 2.5, "mol", dataset_sizes("mol", 4, 7), True, 1, 1.0),
    ("gamma_zero_hd7", 28, 4, 0.0, "mol", dataset_sizes("mol", 4, 8), True, 1, 1.0),
    ("two_layer_shared_hd6", 24, 4, 0.3, "mol", dataset_sizes("mol", 3, 4), True, 2, 1.0),
]
LIVE = ("reference_live", 16, 2, 0.7, "edge_cases", None, True, 2, 1.5)


def run_case(san2, name, d, heads, gamma, kind, sizes, training, layers, wscale, dtype=torch.float32):
    seed = zlib.crc32(("san2/" + name).encode()) % (2 ** 31)
    torch.manual_seed(seed)
    emb = nn.Embedding(1, d)
    # the constructor's gamma is ignored by the reference: 0.1 here, the learned value set below
    stack = nn.Sequential(*[san2.SAN2Layer(0.1, d, d, heads, True, emb, dropout=0.0) for _ in range(layers)])
    g = torch.Generator().manual_seed(seed)
    for layer in stack:
        _prepare(layer, wscale, g)
        with torch.no_grad():
            layer.attention.gamma.fill_(gamma)
    b = edge_case_batch(d, seed % 1000, dtype) if kind == "edge_cases" else san_batch(kind, sizes, d, seed % 1000, dtype)
    mod = stack[0] if layers == 1 else stack
    state = {k: v.clone() for k, v in mod.state_dict().items()}
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
    with torch.no_grad():   # the first layer's scores, from its own projections
        att = stack[0].attention
        x0 = x_in.detach()
        fake = san2.negate_edge_index(b.edge_index, b.batch) if b.edge_index.numel() else None
        t, u = scores(att.Q(x0), att.K(x0), att.Q_2(x0), att.K_2(x0), att.E(e_in.detach()),
                      att.E_2(att.fake_edge_emb.weight)[0], b.edge_index, fake, heads)
        fix["max_score"] = float(max(t.abs().max(), u.abs().max() if u.numel() else 0.0))
    keep = (lambda t: t.detach().clone()) if dtype == torch.float64 else (lambda t: t.detach().float())
    fix["ct"] = ct.to(dtype)
    fix["out"] = keep(out)
    fix["grad_x"] = keep(x_in.grad)
    fix["grad_edge_attr"] = keep(e_in.grad)
    fix["grad_params"] = {n: (p.grad.detach().clone() if n.endswith("attention.gamma") else keep(p.grad))
                          for n, p in mod.named_parameters()}
    return fix


def main():
    args = sys.argv[1:]
    names = {c[0] for c in CASES} | {LIVE[0]}
    ref_root = args[0] if args and args[0] not in names else None
    only = [a for a in args if a in names]
    san2, utils = load_san2(ref_root)
    os.makedirs(OUT, exist_ok=True)
    for case in CASES:
        if only and case[0] not in only:
            continue
        fix = run_case(san2, *case)
        path = os.path.join(OUT, case[0] + ".pt")
        torch.save(fix, path)
        print(case[0], "N", fix["x"].shape[0], "E", fix["edge_index"].shape[1], f"max |score| {fix['max_score']:.1f}",
              f"{os.path.getsize(path)/1e3:.0f} kB")
    if only and LIVE[0] not in only:
        return
    fix = run_case(san2, *LIVE, dtype=torch.float64)
    fix["fake_pairs"] = utils.negate_edge_index(fix["edge_index"], fix["batch"])
    torch.manual_seed(INIT_SEED)
    fix["init_seed"] = INIT_SEED
    emb = nn.Embedding(1, 56)
    fix["init_state"] = {k: v.clone() for k, v in san2.SAN2Layer(0.1, 56, 56, 8, True, emb, 0.2).state_dict().items()}
    path = os.path.join(OUT, LIVE[0] + ".pt")
    torch.save(fix, path)
    print(LIVE[0], f"{os.path.getsize(path)/1e3:.0f} kB")


if __name__ == "__main__":
    main()
