"""TEST INFRASTRUCTURE - CPU restatements (pure torch) of the GAT local model and the GPSLayer that uses it.

graphgps/layer/gps_layer.py (paths relative to the reference checkout) builds, for local_gnn_type == 'GAT' (:70-74),
    pygnn.GATConv(in_channels=dim_h, out_channels=dim_h // num_heads, heads=num_heads, edge_dim=dim_h)
and calls it as local_model(h, edge_index, edge_attr), then dropout_local, the residual h + . and norm1_local
(:183-194); batch.edge_attr is not updated.  PyG is not installed here, so GATConv is restated from PyG 2.2's published
source.  Assumptions taken from it:
  * defaults concat=True, negative_slope=0.2, dropout=0.0, add_self_loops=True, fill_value='mean', bias=True;
  * parameters att_src, att_dst, att_edge [1, H, C]; bias [H*C]; lin_src.weight and lin_edge.weight [H*C, d] without
    bias; lin_dst is the same module as lin_src, so state_dict() holds lin_src.weight and lin_dst.weight while
    named_parameters() yields lin_src.weight only;
  * initialisation: glorot for lin_src, lin_edge and the three att_* (fan (H, C) for att_*), zeros for bias;
  * self loops: remove_self_loops, then add_self_loops(fill_value='mean'): one loop (i, i) per node whose attribute is
    scatter(edge_attr, target, reduce='mean'), 0 for a node without remaining in-edges;
  * softmax(alpha, target): alpha - segment max (detached), exp, / (segment sum + 1e-16);
  * leaky_relu at exactly 0 takes the negative slope in its derivative (torch).

Two independent restatements: GATConvMP (message passing with explicit self-loop removal / addition and PyG's softmax;
installed as the shim's GATConv so that the reference's gps_layer.py runs verbatim with GAT) and GATConvDense (a dense
per-graph masked softmax over (target, edge-slot) pairs, the local model of the oracle layer).  tests/test_gat.py holds
them to each other at 1e-12 and the oracle layer to the reference layer's stored fp64 outputs at 1e-10 / 1e-9.
"""
from __future__ import annotations

import contextlib
import math
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

from biased_oracle import OracleGPSLayerBiased
from oracle.gps_oracle import OracleGPSLayer


def glorot_(t):
    a = math.sqrt(6.0 / (t.size(-2) + t.size(-1)))
    with torch.no_grad():
        t.uniform_(-a, a)
    return t


class _GATParams(nn.Module):
    """Parameters in PyG 2.2 GATConv's registration order."""

    def __init__(self, in_channels, out_channels, heads=1, edge_dim=None, **kw):
        super().__init__()
        assert edge_dim is not None and kw.get("concat", True) and kw.get("dropout", 0.0) == 0.0
        assert kw.get("add_self_loops", True) and kw.get("fill_value", "mean") == "mean" and kw.get("bias", True)
        assert kw.get("negative_slope", 0.2) == 0.2
        self.in_channels, self.out_channels, self.heads = in_channels, out_channels, heads
        H, C = heads, out_channels
        self.lin_src = nn.Linear(in_channels, H * C, bias=False)
        self.lin_dst = self.lin_src
        self.att_src = nn.Parameter(torch.empty(1, H, C))
        self.att_dst = nn.Parameter(torch.empty(1, H, C))
        self.lin_edge = nn.Linear(edge_dim, H * C, bias=False)
        self.att_edge = nn.Parameter(torch.empty(1, H, C))
        self.bias = nn.Parameter(torch.empty(H * C))
        for t in (self.lin_src.weight, self.lin_edge.weight, self.att_src, self.att_dst, self.att_edge):
            glorot_(t)
        nn.init.zeros_(self.bias)

    def scores(self, x):
        H, C = self.heads, self.out_channels
        y = self.lin_src(x).view(-1, H, C)
        return y, (y * self.att_src).sum(-1), (y * self.att_dst).sum(-1)


class GATConvMP(_GATParams):
    """Message passing: remove / add self loops, per-edge scores, PyG softmax over each target's segment."""

    def forward(self, x, edge_index, edge_attr):
        N, H, C = x.shape[0], self.heads, self.out_channels
        y, a_src, a_dst = self.scores(x)
        keep = edge_index[0] != edge_index[1]                           # remove_self_loops
        ei, ea = edge_index[:, keep], edge_attr[keep]
        cnt = torch.zeros(N, dtype=x.dtype).index_add_(0, ei[1], torch.ones(ei.shape[1], dtype=x.dtype))
        loop_attr = torch.zeros(N, ea.shape[1], dtype=ea.dtype).index_add_(0, ei[1], ea) / cnt.clamp(min=1)[:, None]
        loops = torch.arange(N, dtype=ei.dtype)
        ei = torch.cat([ei, torch.stack([loops, loops])], 1)            # add_self_loops(fill_value='mean')
        ea = torch.cat([ea, loop_attr], 0)
        a_edge = (self.lin_edge(ea).view(-1, H, C) * self.att_edge).sum(-1)
        z = F.leaky_relu(a_src[ei[0]] + a_dst[ei[1]] + a_edge, 0.2)
        idx = ei[1][:, None].expand(-1, H)
        zmax = torch.full((N, H), -math.inf, dtype=z.dtype).scatter_reduce(0, idx, z.detach(), "amax")
        ex = (z - zmax[ei[1]]).exp()
        den = torch.zeros(N, H, dtype=z.dtype).index_add_(0, ei[1], ex) + 1e-16
        alpha = ex / den[ei[1]]
        out = torch.zeros(N, H, C, dtype=y.dtype).index_add_(0, ei[1], alpha[..., None] * y[ei[0]])
        return out.reshape(N, H * C) + self.bias


class GATConvDense(_GATParams):
    """Dense per graph: slots = the graph's non-self edges then one loop per node; a [H, n, slots] score matrix masked to
    -inf where the slot does not end at the row's node, torch.softmax over the slots, then alpha @ Y[slot source]."""

    ptr = None   # node offsets of the graphs (set by the oracle layer per call); None = one graph

    def forward(self, x, edge_index, edge_attr):
        N, H, C = x.shape[0], self.heads, self.out_channels
        y, a_src, a_dst = self.scores(x)
        ptr = self.ptr if self.ptr is not None else torch.tensor([0, N])
        outs = []
        for g in range(len(ptr) - 1):
            s, e = int(ptr[g]), int(ptr[g + 1])
            n = e - s
            if n == 0:
                continue
            sel = (edge_index[1] >= s) & (edge_index[1] < e) & (edge_index[0] != edge_index[1])
            src, dst, ea = edge_index[0, sel] - s, edge_index[1, sel] - s, edge_attr[sel]
            inc = torch.zeros(n, src.shape[0], dtype=x.dtype)          # incidence: target x edge
            inc[dst, torch.arange(src.shape[0])] = 1.0
            deg = inc.sum(1, keepdim=True)
            loop_attr = torch.where(deg > 0, inc @ ea / deg.clamp(min=1), torch.zeros_like(inc @ ea))
            slot_src = torch.cat([src, torch.arange(n)])
            slot_dst = torch.cat([dst, torch.arange(n)])
            slot_attr = torch.cat([ea, loop_attr])
            a_edge = (self.lin_edge(slot_attr).view(-1, H, C) * self.att_edge).sum(-1)            # [slots, H]
            z = F.leaky_relu(a_src[s:e][slot_src] + a_dst[s:e][slot_dst] + a_edge, 0.2).t()        # [H, slots]
            mask = slot_dst[None, :] == torch.arange(n)[:, None]                                    # [n, slots]
            scores = torch.where(mask[None], z[:, None, :], torch.full((), -math.inf, dtype=z.dtype))
            alpha = torch.softmax(scores, dim=-1)                                                   # [H, n, slots]
            yv = y[s:e][slot_src].permute(1, 0, 2)                                                  # [H, slots, C]
            outs.append((alpha @ yv).permute(1, 0, 2).reshape(n, H * C))
        out = torch.cat(outs) if outs else y.new_zeros(0, H * C)
        return out + self.bias


def gat_oracle_layer(dim_h, global_model_type, num_heads, **kw):
    """OracleGPSLayer (or its BiasedTransformer subclass) with the GATConvDense local model; same state_dict keys as the
    reference layer.  Parameters are not drawn in the reference's order: load a state_dict to compare."""
    cls = OracleGPSLayerBiased if global_model_type == "BiasedTransformer" else OracleGPSLayer
    layer = cls(dim_h, "GCN", global_model_type, num_heads, **kw)
    layer.local_model = GATConvDense(dim_h, dim_h // num_heads, heads=num_heads, edge_dim=dim_h)
    layer.local_gnn_type = "GAT"
    fwd = layer.forward

    def forward(batch):
        n = torch.bincount(batch.batch, minlength=batch.num_graphs)
        layer.local_model.ptr = torch.cat([torch.zeros(1, dtype=torch.int64), n.cumsum(0)])
        try:
            return fwd(batch)
        finally:
            layer.local_model.ptr = None

    layer.forward = forward
    return layer


@contextlib.contextmanager
def shim_gatconv():
    """Installs GATConvMP as GATConv in the reference shim's torch_geometric.nn for the duration of the block."""
    pygnn = sys.modules["torch_geometric.nn"]
    old = pygnn.GATConv
    pygnn.GATConv = GATConvMP
    try:
        yield
    finally:
        pygnn.GATConv = old


def gat_batch(shape, seed, d, num_graphs, dtype=torch.float32):
    """A make_batch batch plus the structures GAT treats specially: self-loop edges on three nodes, four duplicated
    edges (with attributes of their own), a hub with 40 in-edges (two of them duplicates), and a trailing 3-node graph
    whose last node is isolated."""
    from graphgps_b200.batch import GraphBatch, make_batch
    b = make_batch(shape, seed=seed, dim=d, num_graphs=num_graphs, dtype=dtype)
    g = torch.Generator().manual_seed(seed + 101)
    ptr = b.ptr
    ei = [b.edge_index]
    n0 = int(ptr[1] - ptr[0])
    ei.append(torch.tensor([[0, 1, n0 - 1], [0, 1, n0 - 1]]))                         # self loops, graph 0
    E = b.edge_index.shape[1]
    dup = torch.randint(0, E, (4,), generator=g)
    ei.append(b.edge_index[:, dup])                                                    # duplicates
    s1, e1 = int(ptr[1]), int(ptr[2])
    srcs = torch.arange(s1 + 1, e1).repeat(40)[:40]
    srcs[-2:] = srcs[:2]
    ei.append(torch.stack([srcs, torch.full_like(srcs, s1)]))                           # hub: node 0 of graph 1
    N = int(ptr[-1])
    ei.append(torch.tensor([[N], [N + 1]]))                                            # trailing graph: 0 -> 1, 2 isolated
    edge_index = torch.cat(ei, 1)
    extra = edge_index.shape[1] - E
    edge_attr = torch.cat([b.edge_attr, torch.randn(extra, d, generator=g).to(dtype)])
    x = torch.cat([b.x, torch.randn(3, d, generator=g).to(dtype)])
    batch = torch.cat([b.batch, torch.full((3,), num_graphs, dtype=torch.int64)])
    new_ptr = torch.cat([ptr, ptr[-1:] + 3])
    return GraphBatch(x=x, edge_index=edge_index, edge_attr=edge_attr, batch=batch, num_graphs=num_graphs + 1,
                      ptr=new_ptr)
