"""Generates tests/golden/graph_head/*.pt: graph-prediction head fixtures from the REFERENCE's own
graphgps/head/san_graph.py, graphgps/head/graphormer_graph.py and graphgps/pooling/graph_token.py, run verbatim (loaded
by path).  Their PyG imports are stubbed here, after PyG 2.x's source:

  * torch_geometric.graphgym.cfg: only cfg.model.graph_pooling and cfg.gnn.act are read, at construction;
  * torch_geometric.graphgym.register: register_head / register_pooling decorators, pooling_dict with
    global_mean_pool / global_add_pool restated as index sums over batch.max() + 1 graphs (size=None: the mean divides
    by the count clamped to 1) and graph_token from the reference's file, act_dict = {relu: nn.ReLU, gelu: nn.GELU};
  * torch_geometric.utils.to_dense_batch: [B, Nmax, d] zero-filled, each graph's rows in order, and its mask.

    python tests/golden/make_graph_head_golden.py [REFERENCE_GRAPHGPS_DIR]

Each fixture holds the config, the graph offsets ptr (batch.batch follows from them) and num_graphs, the reference
state_dict (float32), pred and the parameter gradients under a cotangent of pred.  The reference runs in float64 on
the float32 parameters.  x and the cotangent are tests/inductive_edge_oracle.py's hashed_x, exact in bf16, each stored
as its seed with an exact checksum; grad_x is stored where it stays small and otherwise taken from
tests/graph_head_oracle.py, which is pinned to the reference.  So every fixture stays under 1 MB.  reference_live
keeps float64, pins the oracle at 1e-10, and holds `init_state` and `init_state_graphormer`, the reference heads' state_dicts right after construction from torch.manual_seed(INIT_SEED).
"""
import importlib.util
import os
import sys
import types
import zlib

import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from inductive_edge_oracle import hashed_x  # noqa: E402
OUT = os.path.join(HERE, "graph_head")
REF = "/root/reference/graphgps"
INIT_SEED = 1357
GRAD_X_MAX = 120_000   # elements of grad_x a fixture stores


def _size(batch):
    return int(batch.max()) + 1 if batch.numel() else 0


def global_add_pool(x, batch, size=None):
    B = _size(batch) if size is None else size
    return x.new_zeros(B, x.shape[1]).index_add_(0, batch, x)


def global_mean_pool(x, batch, size=None):
    B = _size(batch) if size is None else size
    s = x.new_zeros(B, x.shape[1]).index_add_(0, batch, x)
    n = torch.bincount(batch, minlength=B).clamp(min=1).to(x.dtype)
    return s / n.unsqueeze(1)


def to_dense_batch(x, batch):
    B = _size(batch)
    n = torch.bincount(batch, minlength=B)
    ptr = torch.zeros(B + 1, dtype=torch.int64)
    ptr[1:] = torch.cumsum(n, 0)
    nmax = int(n.max()) if B else 0
    pos = torch.arange(batch.numel()) - ptr[batch]
    out = x.new_zeros(B, nmax, x.shape[1])
    out[batch, pos] = x
    mask = torch.zeros(B, nmax, dtype=torch.bool)
    mask[batch, pos] = True
    return out, mask


CFG = types.SimpleNamespace(model=types.SimpleNamespace(graph_pooling="mean"), gnn=types.SimpleNamespace(act="relu"))


def load_heads(ref=REF):
    """The reference's SANGraphHead and GraphormerHead classes (and the stubbed registry they read)."""
    register = types.ModuleType("torch_geometric.graphgym.register")
    register.pooling_dict = {"mean": global_mean_pool, "add": global_add_pool}
    register.act_dict = {"relu": nn.ReLU, "gelu": nn.GELU}
    register.head_dict = {}

    def register_pooling(name):
        def deco(fn):
            register.pooling_dict[name] = fn
            return fn
        return deco

    register.register_pooling = register_pooling
    register.register_head = lambda name: (lambda cls: cls)
    mods = {"torch_geometric": {}, "torch_geometric.graphgym": {"cfg": CFG, "register": register},
            "torch_geometric.utils": {"to_dense_batch": to_dense_batch}}
    for name, attrs in mods.items():
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        m.__path__ = []
        sys.modules[name] = m
    sys.modules["torch_geometric.graphgym.register"] = register
    sys.modules["torch_geometric"].graphgym = sys.modules["torch_geometric.graphgym"]
    sys.modules["torch_geometric"].utils = sys.modules["torch_geometric.utils"]
    out = {}
    for mod, rel in (("graph_token", "pooling/graph_token.py"), ("san_graph", "head/san_graph.py"),
                     ("graphormer_graph", "head/graphormer_graph.py")):
        spec = importlib.util.spec_from_file_location("graphgps." + rel[:-3].replace("/", "."), os.path.join(ref, rel))
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        out[mod] = m
    return out["san_graph"].SANGraphHead, out["graphormer_graph"].GraphormerHead


def build_head(classes, kind, d, dout, L, pooling, act):
    CFG.model.graph_pooling, CFG.gnn.act = pooling, act
    san, graphormer = classes
    return san(d, dout, L) if kind == "san_graph" else graphormer(d, dout)


def run_case(classes, name, kind, d, dout, L, pooling, act, sizes, dtype=torch.float32):
    seed = zlib.crc32(name.encode()) % (2 ** 31)
    torch.manual_seed(seed)
    head = build_head(classes, kind, d, dout, L, pooling, act)
    if kind == "graphormer_graph":   # LayerNorm starts at (1, 0): give it values a test can see
        with torch.no_grad():
            head.ln.weight.uniform_(0.5, 1.5)
            head.ln.bias.uniform_(-0.5, 0.5)
    if dtype != torch.float64:
        head.float()   # the stored float32 parameters are the ones the reference runs on
    head.double()
    N = sum(sizes)
    x = hashed_x(N, d, seed)
    batch = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes, dtype=torch.int64))
    ptr = torch.zeros(len(sizes) + 1, dtype=torch.int64)
    ptr[1:] = torch.cumsum(torch.tensor(sizes, dtype=torch.int64), 0)
    fix = {"config": dict(name=name, kind=kind, d=d, dout=dout, L=L, pooling=pooling, act=act, sizes=list(sizes)),
           "x_seed": seed, "x_shape": (N, d), "x_sum": float(x.sum()), "x_sumsq": float((x * x).sum()),
           "ptr": ptr, "num_graphs": len(sizes),
           "state": {k: v.detach().to(dtype).clone() for k, v in head.state_dict().items()}}
    xr = x.clone().requires_grad_(True)
    y = torch.randn(len(sizes), dout, dtype=torch.float64)
    pred, label = head(types.SimpleNamespace(x=xr, batch=batch, y=y))
    assert label is y and pred.shape == (len(sizes), dout)
    ct = hashed_x(len(sizes), dout, seed + 1)
    (pred * ct).sum().backward()
    keep = (lambda t: t.detach().clone()) if dtype == torch.float64 else (lambda t: t.detach().float())
    fix.update(ct_seed=seed + 1, ct_sum=float(ct.sum()), pred=keep(pred),
               grads={k: keep(p.grad) for k, p in head.named_parameters()})
    if N * d <= GRAD_X_MAX or dtype == torch.float64:
        fix["grad_x"] = keep(xr.grad)
    return fix


def graph_sizes(B, lo, hi, seed):
    return torch.randint(lo, hi + 1, (B,), generator=torch.Generator().manual_seed(seed)).tolist()


# name, kind, dim_in, dim_out, L, pooling, act, graph sizes
CASES = [
    ("pcqm4m_d304_mean", "san_graph", 304, 1, 2, "mean", "relu", graph_sizes(256, 1, 51, 1)),
    ("pcqm4m_deep_d256_gelu_mean", "san_graph", 256, 1, 3, "mean", "gelu", graph_sizes(256, 1, 51, 2)),
    ("zinc_d64_add", "san_graph", 64, 1, 2, "add", "relu", graph_sizes(32, 9, 37, 3)),
    ("molpcba_san_d304_add_out128", "san_graph", 304, 128, 2, "add", "relu", graph_sizes(512, 5, 40, 4)),
    ("zinc_san_d56_add", "san_graph", 56, 1, 2, "add", "relu", graph_sizes(32, 9, 37, 5)),
    ("molhiv_d72_mean", "san_graph", 72, 1, 2, "mean", "relu", graph_sizes(64, 6, 60, 6)),
    ("zinc_vn_d64_token", "san_graph", 64, 1, 2, "graph_token", "relu", graph_sizes(32, 10, 38, 7)),
    ("zinc_graphormer_d80_token", "graphormer_graph", 80, 1, 0, "graph_token", "relu", graph_sizes(256, 10, 38, 8)),
    # GraphormerHead at d % 8 == 4 with empty graphs in the middle: their rows are zero after the LayerNorm (pred = b)
    ("graphormer_edge_d76_token", "graphormer_graph", 76, 3, 0, "graph_token", "relu", [5, 0, 12, 1, 0, 40, 3, 70, 2]),
    # one-node graphs, an empty graph in the middle, a graph across several 64-row chunks; L = 0 and L = 3
    ("edge_cases_L0_add", "san_graph", 20, 3, 0, "add", "relu", [1, 1, 5, 0, 3, 1, 150, 0, 2, 1]),
    ("edge_cases_L3_mean", "san_graph", 24, 5, 3, "mean", "gelu", [1, 0, 70, 1, 1, 0, 0, 9, 200, 1]),
    ("edge_cases_token", "san_graph", 12, 2, 1, "graph_token", "relu", [1, 0, 4, 1, 0, 90, 3]),
    ("one_large_graph", "san_graph", 64, 1, 2, "mean", "relu", [20000]),
]
LIVE = ("reference_live", "san_graph", 40, 3, 2, "mean", "gelu", [6, 1, 0, 9, 70, 2, 7])


def main():
    classes = load_heads(sys.argv[1] if len(sys.argv) > 1 else REF)
    os.makedirs(OUT, exist_ok=True)
    for case in CASES:
        fix = run_case(classes, *case)
        p = os.path.join(OUT, case[0] + ".pt")
        torch.save(fix, p)
        print(case[0], "graphs", fix["num_graphs"], "nodes", fix["x_shape"][0], "grad_x" in fix,
              f"{os.path.getsize(p) / 1e3:.0f} kB")
    fix = run_case(classes, *LIVE, dtype=torch.float64)
    fix["init_seed"] = INIT_SEED
    torch.manual_seed(INIT_SEED)
    fix["init_state"] = {k: v.clone() for k, v in build_head(classes, "san_graph", 304, 1, 2, "mean",
                                                             "relu").state_dict().items()}
    torch.manual_seed(INIT_SEED)
    fix["init_state_graphormer"] = {k: v.clone() for k, v in build_head(classes, "graphormer_graph", 80, 1, 0,
                                                                        "graph_token", "relu").state_dict().items()}
    p = os.path.join(OUT, LIVE[0] + ".pt")
    torch.save(fix, p)
    print(LIVE[0], f"{os.path.getsize(p) / 1e3:.0f} kB")


if __name__ == "__main__":
    main()
