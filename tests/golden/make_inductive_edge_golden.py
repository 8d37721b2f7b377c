"""Generates tests/golden/inductive_edge/*.pt: link-prediction head fixtures from the REFERENCE's own
graphgps/head/inductive_edge.py, run verbatim (loaded by path).  Its PyG imports are stubbed here, after PyG 2.x's
source:

  * torch_geometric.graphgym.config.cfg: only cfg.model.edge_decoding ('dot') and cfg.gnn.layers_post_mp (1) are read;
  * torch_geometric.graphgym.register.register_head: the identity decorator;
  * torch_geometric.graphgym.models.layer.new_layer_config / MLP / Linear for one layer: MLP.model is a Sequential
    holding one GraphGym Linear, whose `model` is a torch_geometric.nn.Linear(dim_in, dim_out, bias=True) (here an
    nn.Linear: same parameter names and shapes); both apply themselves to batch.x;
  * Batch.to_data_list(): per graph, x[n0:n1], the graph's labeled pairs with the node offset n0 subtracted from
    edge_index_labeled (PyG's __inc__ offsets every attribute whose name contains "index") and its edge_label.

    python tests/golden/make_inductive_edge_golden.py [REFERENCE_HEAD_FILE]

Batches are contact-shaped: graphs of 15 to 50 nodes, each positive (i, j) joined by two structured negatives (i, k)
and (j, k') of the same graph, the graph's pairs in a random order.  A positive's target is drawn only among nodes
whose score <y_i, y_j> lies at least 1 % of the score spread of row i away from every other candidate's, so the
fixtures have no near-ties and the ranks are the same in fp32 and bf16.  Each fixture holds the config, the inputs
(x, edge_index_labeled, edge_label, batch, ptr), the reference state_dict, the cotangent of pred, pred, grad_x,
grad_weight, grad_bias and the reference's eval stats.  x is tests/inductive_edge_oracle.py's hashed_x, exact in bf16,
stored as its seed with an exact checksum, and the two 256-graph batches leave grad_x out (the tests take it from the
oracle, which is pinned to the reference), so every fixture stays well under 1 MB; reference_live keeps fp64 and pins
tests/inductive_edge_oracle.py at 1e-10, and holds `init_state`, the reference head's state_dict right after
construction from torch.manual_seed(INIT_SEED).
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
OUT = os.path.join(HERE, "inductive_edge")
REF = "/root/reference/graphgps/head/inductive_edge.py"
INIT_SEED = 2468
MARGIN = 1e-2


class _GymLinear(nn.Module):
    def __init__(self, layer_config, **kwargs):
        super().__init__()
        self.model = nn.Linear(layer_config.dim_in, layer_config.dim_out, bias=layer_config.has_bias)

    def forward(self, batch):
        if isinstance(batch, torch.Tensor):
            return self.model(batch)
        batch.x = self.model(batch.x)
        return batch


class _GymMLP(nn.Module):
    def __init__(self, layer_config, **kwargs):
        super().__init__()
        assert layer_config.num_layers == 1
        self.model = nn.Sequential(_GymLinear(layer_config))

    def forward(self, batch):
        if isinstance(batch, torch.Tensor):
            return self.model(batch)
        batch.x = self.model(batch.x)
        return batch


def _new_layer_config(dim_in, dim_out, num_layers, has_act, has_bias, cfg):
    return types.SimpleNamespace(dim_in=dim_in, dim_out=dim_out, num_layers=num_layers, has_act=has_act,
                                 has_bias=has_bias)


class Batch:
    """x, edge_index_labeled (global node ids), edge_label, and the per-graph node and pair counts."""

    def __init__(self, x, eli, label, sizes, npairs):
        self.x, self.edge_index_labeled, self.edge_label = x, eli, label
        self.sizes, self.npairs = sizes, npairs

    def to_data_list(self):
        out, n0, p0 = [], 0, 0
        for n, p in zip(self.sizes, self.npairs):
            out.append(types.SimpleNamespace(x=self.x[n0:n0 + n], edge_index_labeled=self.edge_index_labeled[:, p0:p0 + p] - n0,
                                             edge_label=self.edge_label[p0:p0 + p], num_nodes=n))
            n0, p0 = n0 + n, p0 + p
        return out


def load_head(path=REF):
    cfg = types.SimpleNamespace(model=types.SimpleNamespace(edge_decoding="dot"),
                                gnn=types.SimpleNamespace(layers_post_mp=1))
    mods = {
        "torch_geometric": {},
        "torch_geometric.graphgym": {},
        "torch_geometric.graphgym.config": {"cfg": cfg},
        "torch_geometric.graphgym.register": {"register_head": lambda name: (lambda cls: cls), "head_dict": {}},
        "torch_geometric.graphgym.models": {},
        "torch_geometric.graphgym.models.layer": {"new_layer_config": _new_layer_config, "MLP": _GymMLP,
                                                  "Linear": _GymLinear},
    }
    for name, attrs in mods.items():
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        m.__path__ = []
        sys.modules[name] = m
    spec = importlib.util.spec_from_file_location("graphgps.head.inductive_edge", path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


# ------------------------------------------------------------------------------------------------------------ batches
def contact_pairs(y, sizes, n_pos, g):
    """Labeled pairs per graph: n_pos[b] positives whose targets are clear of every other candidate by MARGIN of the
    row's score spread, two negatives per positive, shuffled within the graph."""
    eli, lab, npairs, n0 = [], [], [], 0
    for n, m in zip(sizes, n_pos):
        pairs, labels, used = [], [], set()
        yg = y[n0:n0 + n]
        for _ in range(m if n > 0 else 0):
            for _try in range(50):
                i = int(torch.randint(0, n, (1,), generator=g))
                s = yg @ yg[i]
                ss, order = s.sort()
                step = torch.full((n + 1,), float("inf"), dtype=s.dtype)
                step[1:n] = ss[1:] - ss[:-1]
                gap = torch.empty_like(s)
                gap[order] = torch.minimum(step[:n], step[1:])   # distance to the nearest other score
                ok = gap > MARGIN * (float(s.max() - s.min()) if n > 1 else 1.0)
                if n > 1:
                    ok[i] = False   # no self contacts
                cand = [j for j in ok.nonzero().flatten().tolist() if (i, j) not in used]
                if cand:
                    j = cand[int(torch.randint(0, len(cand), (1,), generator=g))]
                    break
            else:
                continue
            used.add((i, j))
            pairs.append((i, j))
            labels.append(1)
            for a in (i, j):   # the structured negatives
                k = int(torch.randint(0, n, (1,), generator=g))
                pairs.append((a, k))
                labels.append(1 if (a, k) in used else 0)
        perm = torch.randperm(len(pairs), generator=g).tolist()
        eli += [(pairs[p][0] + n0, pairs[p][1] + n0) for p in perm]
        lab += [labels[p] for p in perm]
        npairs.append(len(pairs))
        n0 += n
    return (torch.tensor(eli, dtype=torch.int64).reshape(-1, 2).t().contiguous(), torch.tensor(lab, dtype=torch.int64),
            npairs)


def run_case(m, name, d, sizes, pos_range, dtype=torch.float32):
    seed = zlib.crc32(name.encode()) % (2 ** 31)
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    head = m.GNNInductiveEdgeHead(d, 1).double()
    x = hashed_x(sum(sizes), d, seed)   # stored as its seed and checksum
    with torch.no_grad():
        y = head.layer_post_mp(x)
    n_pos = [int(torch.randint(pos_range[0], pos_range[1] + 1, (1,), generator=g)) for _ in sizes]
    eli, label, npairs = contact_pairs(y, sizes, n_pos, g)
    batch = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes, dtype=torch.int64))
    ptr = torch.zeros(len(sizes) + 1, dtype=torch.int64)
    ptr[1:] = torch.cumsum(torch.tensor(sizes, dtype=torch.int64), 0)
    fix = {"config": dict(name=name, d=d, sizes=list(sizes)),
           "x_seed": seed, "x_shape": tuple(x.shape), "x_sum": float(x.sum()), "x_sumsq": float((x * x).sum()),
           "edge_index_labeled": eli, "edge_label": label, "batch": batch, "ptr": ptr,
           "num_graphs": len(sizes),
           "state": {k: v.detach().to(dtype).clone() for k, v in head.state_dict().items()}}
    xr = x.clone().requires_grad_(True)
    head.train()
    pred, lab = head(Batch(xr, eli, label, sizes, npairs))
    assert torch.equal(lab, label)
    ct = torch.randn(pred.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    (pred * ct).sum().backward()
    keep = (lambda t: t.detach().clone()) if dtype == torch.float64 else (lambda t: t.detach().float())
    lin = head.layer_post_mp.model[0].model
    fix.update(ct=ct.to(dtype), pred=keep(pred), grad_weight=keep(lin.weight.grad), grad_bias=keep(lin.bias.grad))
    if len(sizes) < 256 or dtype == torch.float64:   # the 256-graph batches' grad_x comes from the pinned oracle
        fix["grad_x"] = keep(xr.grad)
    head.eval()
    with torch.no_grad():
        _, _, stats = head(Batch(x.clone(), eli, label, sizes, npairs))
    fix["stats"] = {k: float(v) for k, v in stats.items()}
    return fix


def contact_sizes(B, seed):
    return torch.randint(15, 51, (B,), generator=torch.Generator().manual_seed(seed)).tolist()


# name, d, graph sizes, positives per graph [lo, hi]
CASES = [
    ("contact_d138", 138, contact_sizes(256, 1), (0, 12)),
    ("contact_d208", 208, contact_sizes(256, 2), (0, 12)),
    ("no_positives_d64", 64, [23, 31, 17, 40, 28, 19, 35, 26], (0, 1)),
    ("tiny_graphs_d20", 20, [1, 2, 1, 18, 2, 1, 25, 2], (1, 3)),
    ("large_graph_d40", 40, [3000, 21, 34], (20, 40)),
]
LIVE = ("reference_live", 12, [6, 1, 9, 2, 7, 12], (0, 4))


def main():
    m = load_head(sys.argv[1] if len(sys.argv) > 1 else REF)
    os.makedirs(OUT, exist_ok=True)
    for case in CASES:
        fix = run_case(m, *case)
        p = os.path.join(OUT, case[0] + ".pt")
        torch.save(fix, p)
        print(case[0], "nodes", fix["x_shape"][0], "pairs", fix["edge_label"].numel(), "positives",
              int((fix["edge_label"] == 1).sum()), fix["stats"], f"{os.path.getsize(p) / 1e3:.0f} kB")
    fix = run_case(m, *LIVE, dtype=torch.float64)
    torch.manual_seed(INIT_SEED)
    fix["init_seed"] = INIT_SEED
    fix["init_state"] = {k: v.clone() for k, v in m.GNNInductiveEdgeHead(138, 1).state_dict().items()}
    p = os.path.join(OUT, LIVE[0] + ".pt")
    torch.save(fix, p)
    print(LIVE[0], fix["stats"], f"{os.path.getsize(p) / 1e3:.0f} kB")


if __name__ == "__main__":
    main()
