"""Generates tests/golden/graphormer_bias/*.pt: BiasEncoder fixtures from the REFERENCE's own graphormer_encoder.py, run
verbatim (loaded by path) for both graphormer_pre_processing and BiasEncoder.  Its PyG imports are stubbed here:

  * torch_geometric.graphgym.config.cfg: only cfg.posenc_GraphormerBias.{num_in_degrees, num_out_degrees,
    node_degrees_only} are read;
  * register_node_encoder: the identity decorator;
  * to_networkx(data): a networkx DiGraph on nodes 0 .. n-1 with one edge per edge_index column.  Shortest-path
    tie-breaking may differ from PyG's; the fixture stores the preprocessed attributes as the inputs, so it does not
    matter;
  * to_dense_adj(edge_index, batch, edge_attr): PyG's algorithm (batch size batch.max() + 1, per-graph node offsets from
    the node counts, graph of a pair = batch[edge_index[0]], sum-scatter into [B, Nmax, Nmax, ...]);
  * networkx's all-pairs nx.shortest_path returns the dict of networkx 2.x, which the reference iterates.

    python tests/golden/make_graphormer_bias_golden.py [REFERENCE_ENCODER_FILE]

Each graph is preprocessed on its own and the batch collated as PyG does (graph_index offset by the node count).  Each
fixture holds the config, the inputs (spatial_types, graph_index, shortest_path_types when the graphs have edge
attributes, batch, ptr), the reference state_dict, the cotangent, the output and the four gradients (None for a
parameter the output does not depend on), stored as fp32; reference_live keeps fp64 and pins
tests/graphormer_bias_oracle.py at 1e-10.  reference_live also holds `init_state`, the reference encoder's state_dict
right after construction from torch.manual_seed(INIT_SEED).
"""
import importlib.util
import os
import sys
import types
import zlib

import networkx as nx
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "graphormer_bias")
REF = "/root/reference/graphgps/encoder/graphormer_encoder.py"
INIT_SEED = 4321


def _to_networkx(data):
    g = nx.DiGraph()
    g.add_nodes_from(range(data.num_nodes))
    for u, v in data.edge_index.t().tolist():
        g.add_edge(u, v)
    return g


def _to_dense_adj(edge_index, batch, edge_attr):
    B = int(batch.max()) + 1 if batch.numel() else 1
    num_nodes = torch.zeros(B, dtype=torch.int64).index_add_(0, batch, torch.ones_like(batch))
    cum = torch.zeros(B + 1, dtype=torch.int64)
    cum[1:] = torch.cumsum(num_nodes, 0)
    idx0 = batch[edge_index[0]]
    idx1 = edge_index[0] - cum[batch][edge_index[0]]
    idx2 = edge_index[1] - cum[batch][edge_index[1]]
    n = int(num_nodes.max())
    idx = idx0 * n * n + idx1 * n + idx2
    adj = torch.zeros((B * n * n,) + tuple(edge_attr.shape[1:]), dtype=edge_attr.dtype)
    adj = adj.index_add(0, idx, edge_attr)
    return adj.view((B, n, n) + tuple(edge_attr.shape[1:]))


def load_encoder(path=REF):
    cfg = types.SimpleNamespace(posenc_GraphormerBias=types.SimpleNamespace(num_in_degrees=64, num_out_degrees=64,
                                                                            node_degrees_only=False))
    mods = {
        "torch_geometric": {},
        "torch_geometric.graphgym": {},
        "torch_geometric.graphgym.config": {"cfg": cfg},
        "torch_geometric.graphgym.register": {"register_node_encoder": lambda name: (lambda cls: cls)},
        "torch_geometric.utils": {"to_dense_adj": _to_dense_adj, "to_networkx": _to_networkx},
    }
    for name, attrs in mods.items():
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        m.__path__ = []
        sys.modules[name] = m
    spec = importlib.util.spec_from_file_location("graphgps.encoder.graphormer_encoder", path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    # networkx >= 3.5 returns all-pairs shortest paths as a generator; the reference iterates the dict of networkx 2.x
    m.nx = types.SimpleNamespace(DiGraph=nx.DiGraph, shortest_path=lambda graph: dict(nx.shortest_path(graph)))
    return m


# ------------------------------------------------------------------------------------------------------------ graphs
def molecule(n, T, g):
    """An undirected molecule-like graph: a random tree with two ring closures, both directions of a bond sharing one
    type in [0, T)."""
    und = [(int(torch.randint(0, v, (1,), generator=g)), v) for v in range(1, n)]
    for _ in range(2 if n > 5 else 0):
        u, v = sorted(torch.randperm(n, generator=g)[:2].tolist())
        if (u, v) not in und:
            und.append((u, v))
    edges, types_ = [], []
    for u, v in und:
        t = int(torch.randint(0, T, (1,), generator=g))
        edges += [(u, v), (v, u)]
        types_ += [t, t]
    return n, edges, types_


def directed(n, T, g):
    """Edges only from lower to higher index: every pair (i, j) with j < i is unreachable."""
    edges = [(v, v + 1) for v in range(n - 1)] + [(v, v + 3) for v in range(0, n - 3, 2)]
    return n, edges, torch.randint(0, T, (len(edges),), generator=g).tolist()


def path(n, T, g):
    edges = [(v, v + 1) for v in range(n - 1)] + [(v + 1, v) for v in range(n - 1)]
    return n, edges, torch.randint(0, T, (len(edges),), generator=g).tolist()


def collate(enc, graphs, S, with_edges):
    sts, gis, spts, batch = [], [], [], []
    off = 0
    for b, (n, edges, types_) in enumerate(graphs):
        d = types.SimpleNamespace(num_nodes=n, edge_index=torch.tensor(edges, dtype=torch.int64).reshape(-1, 2).t())
        if with_edges:
            d.edge_attr = torch.tensor(types_, dtype=torch.int64)
        d = enc.graphormer_pre_processing(d, S)
        sts.append(d.spatial_types)
        gis.append(d.graph_index + off)
        if with_edges:
            spts.append(d.shortest_path_types)
        batch.append(torch.full((n,), b, dtype=torch.int64))
        off += n
    ptr = torch.zeros(len(graphs) + 1, dtype=torch.int64)
    ptr[1:] = torch.cumsum(torch.tensor([gr[0] for gr in graphs]), 0)
    return (torch.cat(sts), torch.cat(gis, 1), torch.cat(spts) if with_edges else None, torch.cat(batch), ptr)


# name, heads, S, T, graph token, edge attributes, graphs (kind, n)
CASES = [
    ("zinc_token", 8, 20, 4, True, True, [("mol", n) for n in (24, 19, 30, 12, 27, 21)]),
    ("zinc_no_token", 8, 20, 4, False, True, [("mol", n) for n in (17, 23, 14, 26)]),
    ("spatial_only", 4, 20, 0, False, False, [("mol", n) for n in (40, 33)]),
    ("directed_unreachable", 4, 6, 3, True, True, [("dir", 14), ("mol", 9)]),
    ("long_path", 4, 8, 3, False, True, [("path", 30), ("mol", 7)]),
    ("one_node", 8, 20, 4, True, True, [("mol", 1), ("mol", 11), ("mol", 1)]),
    ("largest_not_first", 4, 20, 4, True, True, [("mol", 8), ("mol", 29), ("path", 13)]),
]
LIVE = ("reference_live", 3, 5, 3, True, True, [("mol", 6), ("path", 9), ("dir", 7), ("mol", 1)])
KINDS = {"mol": molecule, "dir": directed, "path": path}


def run_case(enc, name, heads, S, T, token, with_edges, graph_specs, dtype=torch.float32):
    seed = zlib.crc32(name.encode()) % (2 ** 31)
    g = torch.Generator().manual_seed(seed)
    graphs = [KINDS[k](n, max(T, 1), g) for k, n in graph_specs]
    st, gi, spt, batch, ptr = collate(enc, graphs, S, with_edges)
    torch.manual_seed(seed)
    mod = enc.BiasEncoder(heads, S, T, token)
    with torch.no_grad():   # O(1) parameters so every term is visible against the others
        for p in mod.parameters():
            p.normal_(std=1.0)
    fix = {"config": dict(name=name, heads=heads, num_spatial_types=S, num_edge_types=T, use_graph_token=token,
                          sizes=[gr[0] for gr in graphs]),
           "spatial_types": st, "graph_index": gi, "batch": batch, "ptr": ptr, "num_graphs": len(graphs),
           "state": {k: v.clone() for k, v in mod.state_dict().items()}}
    if spt is not None:
        fix["shortest_path_types"] = spt
    mod = mod.double()
    data = types.SimpleNamespace(spatial_types=st, graph_index=gi, batch=batch)
    if spt is not None:
        data.shortest_path_types = spt
    out = mod(data).attn_bias
    ct = torch.randn(out.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    (out * ct).sum().backward()
    keep = (lambda t: t.detach().clone()) if dtype == torch.float64 else (lambda t: t.detach().float())
    fix["ct"] = ct.to(dtype)
    fix["out"] = keep(out)
    fix["grad_params"] = {n: None if p.grad is None else keep(p.grad) for n, p in mod.named_parameters()}
    return fix


def main():
    enc = load_encoder(sys.argv[1] if len(sys.argv) > 1 else REF)
    os.makedirs(OUT, exist_ok=True)
    for case in CASES:
        fix = run_case(enc, *case)
        p = os.path.join(OUT, case[0] + ".pt")
        torch.save(fix, p)
        print(case[0], "pairs", fix["spatial_types"].numel(), "out", list(fix["out"].shape),
              f"{os.path.getsize(p) / 1e3:.0f} kB")
    fix = run_case(enc, *LIVE, dtype=torch.float64)
    torch.manual_seed(INIT_SEED)
    fix["init_seed"] = INIT_SEED
    fix["init_state"] = {k: v.clone() for k, v in enc.BiasEncoder(8, 20, 4, True).state_dict().items()}
    fix["init_state_no_token"] = {k: v.clone() for k, v in enc.BiasEncoder(4, 20, 0, False).state_dict().items()}
    p = os.path.join(OUT, LIVE[0] + ".pt")
    torch.save(fix, p)
    print(LIVE[0], f"{os.path.getsize(p) / 1e3:.0f} kB")


if __name__ == "__main__":
    main()
