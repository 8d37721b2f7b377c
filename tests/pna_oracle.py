"""TEST INFRASTRUCTURE - CPU restatements (pure torch) of the PNA local model and the GPSLayer that uses it.

graphgps/layer/gps_layer.py (paths relative to the reference checkout) builds, for local_gnn_type == 'PNA' (:75-90),
    pygnn.PNAConv(dim_h, dim_h, aggregators=['mean', 'max', 'sum'], scalers=['identity'],
                  deg=torch.from_numpy(np.array(pna_degrees)), edge_dim=min(128, dim_h), towers=1, pre_layers=1,
                  post_layers=1, divide_input=False)
and calls it as local_model(h, edge_index, edge_attr), then dropout_local, the residual h + . and norm1_local
(:183-194); batch.edge_attr is not updated.  PyG is not installed here, so PNAConv is restated from PyG 2.2's published
pna_conv.py, aggr/scaler.py (DegreeScalerAggregation), aggr/multi.py (MultiAggregation), aggr/basic.py and
torch_scatter's scatter_max.  Assumptions taken from them (de = min(128, d)):
  * parameters: edge_encoder = Linear(de, d); pre_nns[0] = Sequential(Linear(3d, d)); post_nns[0] =
    Sequential(Linear(4d, d)); lin = Linear(d, d), all with bias: state_dict keys edge_encoder.{weight,bias},
    pre_nns.0.0.{weight,bias}, post_nns.0.0.{weight,bias}, lin.{weight,bias}.  PyG's Linear without initialisers draws
    as torch.nn.Linear does;
  * DegreeScalerAggregation keeps the average degrees as a Python dict (no buffers).  It computes them as
    float(sum_k k deg[k]) / int(sum deg), so an empty or all-zero histogram raises ZeroDivisionError; with
    scalers=['identity'] they never enter the arithmetic;
  * message(x_i, x_j, edge_attr) = pre_nns[0](cat[x_i, x_j, edge_encoder(edge_attr)]) for edge j -> i (x_i the target);
    no activation (pre_layers = 1), no self loops are added, and duplicate edges are ordinary edges;
  * aggregation: cat[mean, max, sum] per target and channel over its in-edges (MultiAggregation, mode 'cat'); a node
    without in-edges gets 0 in all three.  max is torch_scatter's scatter_max: it updates on a strictly greater value
    in edge order, so the first maximising edge is the argmax, and its backward sends the whole gradient to that edge
    (torch.scatter_reduce('amax') would split it between tied edges instead);
  * forward(x, edge_index, edge_attr): out = lin(post_nns[0](cat[x, aggregation])), no activation (post_layers = 1).
    The forward takes three tensors, so a fourth positional argument (equivstable_pe=True) fails.

Two independent restatements: PNAConvMP (message passing with an explicit first-wins argmax; installed as the shim's
PNAConv so that the reference's gps_layer.py runs verbatim with PNA) and PNAConvLoop (a per-node loop, the local model of
the oracle layer).  tests/test_pna.py holds them to each other at 1e-12 and the oracle layer to the reference layer's
stored fp64 outputs at 1e-10 / 1e-9.
"""
from __future__ import annotations

import contextlib
import sys

import torch
import torch.nn as nn

from biased_oracle import OracleGPSLayerBiased
from oracle.gps_oracle import OracleGPSLayer


class _PNAParams(nn.Module):
    """Parameters of PyG 2.2 PNAConv with the options the reference passes."""

    def __init__(self, in_channels, out_channels, aggregators, scalers, deg, edge_dim=None, towers=1, pre_layers=1,
                 post_layers=1, divide_input=False, **kw):
        super().__init__()
        assert in_channels == out_channels and list(aggregators) == ["mean", "max", "sum"]
        assert list(scalers) == ["identity"] and towers == 1 and pre_layers == 1 and post_layers == 1
        assert not divide_input and edge_dim is not None and not kw
        d = out_channels
        deg = deg.to(torch.float)
        num_nodes = int(deg.sum())
        bins = torch.arange(deg.numel())
        self.avg_deg = {"lin": float((bins * deg).sum()) / num_nodes,                # ZeroDivisionError as in 2.2
                        "log": float(((bins + 1).log() * deg).sum()) / num_nodes,
                        "exp": float((bins.exp() * deg).sum()) / num_nodes}
        self.edge_encoder = nn.Linear(edge_dim, d)
        self.pre_nns = nn.ModuleList([nn.Sequential(nn.Linear(3 * d, d))])
        self.post_nns = nn.ModuleList([nn.Sequential(nn.Linear(4 * d, d))])
        self.lin = nn.Linear(d, d)

    def forward(self, x, edge_index, edge_attr):
        return self.lin(self.post_nns[0](torch.cat([x, self.aggregate(x, edge_index, edge_attr)], -1)))


class PNAConvMP(_PNAParams):
    """Message passing: one product per edge, index_add_ for sum and mean, and the first maximising edge of each
    (target, channel) found as the smallest edge id among the maximisers; the max is gathered from that edge alone."""

    def aggregate(self, x, edge_index, edge_attr):
        N, d = x.shape
        src, dst = edge_index[0], edge_index[1]
        E = src.numel()
        m = self.pre_nns[0](torch.cat([x[dst], x[src], self.edge_encoder(edge_attr)], -1))
        cnt = torch.zeros(N, dtype=m.dtype).index_add_(0, dst, torch.ones(E, dtype=m.dtype))
        s = torch.zeros(N, d, dtype=m.dtype).index_add_(0, dst, m)
        mean = s / cnt.clamp(min=1)[:, None]
        idx = dst[:, None].expand(-1, d)
        top = torch.full((N, d), -torch.inf, dtype=m.dtype).scatter_reduce(0, idx, m.detach(), "amax")
        cand = torch.where(m.detach() == top[dst], torch.arange(E)[:, None].expand(-1, d), E)
        arg = torch.full((N, d), E, dtype=torch.int64).scatter_reduce(0, idx, cand, "amin")
        mx = torch.cat([m, m.new_zeros(1, d)]).gather(0, arg)   # arg == E: no in-edges -> 0
        return torch.cat([mean, mx, s], -1)


class PNAConvLoop(_PNAParams):
    """Per node: its in-edges' messages from the three column blocks of the pre weight, then mean / sum over them and,
    per channel, the first edge at the maximum (argmax of a 0/1 mask returns the first index)."""

    def aggregate(self, x, edge_index, edge_attr):
        N, d = x.shape
        W, b = self.pre_nns[0][0].weight, self.pre_nns[0][0].bias
        enc = self.edge_encoder
        rows = []
        for i in range(N):
            k = torch.nonzero(edge_index[1] == i).flatten()
            if k.numel() == 0:
                rows.append(x.new_zeros(3 * d))
                continue
            m = (x[i] @ W[:, :d].t() + x[edge_index[0, k]] @ W[:, d:2 * d].t()
                 + (edge_attr[k] @ enc.weight.t() + enc.bias) @ W[:, 2 * d:].t() + b)
            first = (m.detach() == m.detach().max(0).values).to(torch.int8).argmax(0)
            rows.append(torch.cat([m.mean(0), m.gather(0, first[None]).squeeze(0), m.sum(0)]))
        return torch.stack(rows) if rows else x.new_zeros(0, 3 * d)


PNA_KW = dict(aggregators=["mean", "max", "sum"], scalers=["identity"], towers=1, pre_layers=1, post_layers=1,
              divide_input=False)


def pna_conv(cls, d, deg):
    return cls(d, d, deg=torch.as_tensor(deg), edge_dim=min(128, d), **PNA_KW)


def pna_oracle_layer(dim_h, global_model_type, num_heads, pna_degrees=(1, 2, 3), **kw):
    """OracleGPSLayer (or its BiasedTransformer subclass) with the PNAConvLoop local model; same state_dict keys as the
    reference layer.  Parameters are not drawn in the reference's order: load a state_dict to compare."""
    cls = OracleGPSLayerBiased if global_model_type == "BiasedTransformer" else OracleGPSLayer
    layer = cls(dim_h, "GCN", global_model_type, num_heads, **kw)
    layer.local_model = pna_conv(PNAConvLoop, dim_h, pna_degrees)
    layer.local_gnn_type = "PNA"
    return layer


@contextlib.contextmanager
def shim_pna():
    """Installs PNAConvMP as PNAConv in the reference shim's torch_geometric.nn for the duration of the block."""
    pygnn = sys.modules["torch_geometric.nn"]
    old = pygnn.PNAConv
    pygnn.PNAConv = PNAConvMP
    try:
        yield
    finally:
        pygnn.PNAConv = old


def pna_batch(shape, seed, d, num_graphs, dtype=torch.float32):
    """gat_oracle.gat_batch (self-loop edges, duplicated edges with attributes of their own, a hub with 40 in-edges, an
    isolated node, a trailing graph) with edge attributes of width min(128, d), plus one exact duplicate: the last edge
    repeats edge `tie_edge(b)` (same source, destination and attribute row), so that their messages tie in every
    channel and the first-wins rule decides where the max gradient goes."""
    from gat_oracle import gat_batch
    b = gat_batch(shape, seed, d, num_graphs, dtype=dtype)
    de = min(128, d)
    b.edge_attr = b.edge_attr[:, :de].contiguous()
    k = tie_edge(b)
    b.edge_index = torch.cat([b.edge_index, b.edge_index[:, k:k + 1]], 1)
    b.edge_attr = torch.cat([b.edge_attr, b.edge_attr[k:k + 1]])
    return b


def tie_edge(b):
    """The edge pna_batch duplicates: the first in-edge of node 1 of graph 0 (in-degree >= 2 in the batches used)."""
    t = int(b.ptr[0]) + 1
    return int(torch.nonzero(b.edge_index[1] == t).flatten()[0])


def seeded_state(layer, seed):
    """A full state_dict for `layer` drawn from `seed` alone (Linear weights U(+-1/sqrt(fan_in)), biases likewise,
    BatchNorm affines and running statistics away from their defaults), for fixtures too large to store it."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, v in layer.state_dict().items():
        if not v.is_floating_point():
            out[k] = v.clone()
            continue
        u = torch.rand(v.shape, generator=g, dtype=torch.float64)
        if "running_var" in k:
            t = 0.6 + 0.8 * u
        elif "running_mean" in k:
            t = 0.4 * u - 0.2
        elif k.startswith("norm") and k.endswith(".weight"):
            t = 0.5 + u
        else:
            fan = v.shape[-1] if v.dim() > 1 else v.shape[0]
            t = (2 * u - 1) / fan ** 0.5
        out[k] = t.to(v.dtype)
    return out
