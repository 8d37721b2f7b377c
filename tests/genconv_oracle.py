"""TEST INFRASTRUCTURE - CPU restatements (pure torch) of the GENConv local model and the GPSLayer that uses it.

graphgps/layer/gps_layer.py (paths relative to the reference checkout) builds, for local_gnn_type == 'GENConv' (:60-61),
    pygnn.GENConv(dim_h, dim_h)
and calls it as local_model(h, edge_index, edge_attr), then dropout_local, the residual h + . and norm1_local
(:183-194); batch.edge_attr is not updated.  PyG is not installed here, so GENConv is restated from PyG 2.2's published
gen_conv.py, aggr/basic.py::SoftmaxAggregation and utils/softmax.py.  Assumptions taken from them:
  * defaults aggr='softmax', t=1.0, learn_t=False, msg_norm=False, norm='batch', num_layers=2, expansion=2, eps=1e-7,
    bias=False, edge_dim=None; with in_channels == out_channels there is no lin_src, lin_dst, lin_edge or lin_aggr_out;
  * t is a Python float, so SoftmaxAggregation holds no parameter and skips the multiplication by t;
  * mlp = Linear(d, 2d, bias=False), BatchNorm1d(2d), ReLU(), Dropout(0.0), Linear(2d, d, bias=False): state_dict keys
    mlp.0.weight, mlp.1.{weight, bias, running_mean, running_var, num_batches_tracked}, mlp.4.weight.  The MLP's ReLU
    does not follow gnn.act;
  * message(x_j, edge_attr) = relu(x_j + edge_attr) + eps (edge_attr must have d columns); ReLU's derivative at 0 is 0;
  * softmax(src, index): src - segment max (detached), exp, / (segment sum + 1e-16); the aggregation is
    sum_k alpha_k m_k per target and channel (a node without in-edges gets 0).  No self loops are added, and existing
    self loops and duplicate edges are ordinary edges;
  * forward: out = aggregation + x (x_dst), return mlp(out).

Two independent restatements: GENConvMP (message passing with PyG's scatter softmax; installed as the shim's GENConv so
that the reference's gps_layer.py runs verbatim with GENConv) and GENConvLoop (a per-node loop with torch.softmax over
the node's in-edges, the local model of the oracle layer).  tests/test_genconv.py holds them to each other at 1e-12 and
the oracle layer to the reference layer's stored fp64 outputs at 1e-10 / 1e-9.
"""
from __future__ import annotations

import contextlib
import math
import sys

import torch
import torch.nn as nn

from biased_oracle import OracleGPSLayerBiased
from oracle.gps_oracle import OracleGPSLayer

MSG_EPS = 1e-7


class _GENParams(nn.Module):
    """Parameters of PyG 2.2 GENConv(in, out) with the defaults the reference uses."""

    def __init__(self, in_channels, out_channels, **kw):
        super().__init__()
        assert in_channels == out_channels and kw.get("edge_dim") is None
        assert kw.get("aggr", "softmax") == "softmax" and kw.get("t", 1.0) == 1.0 and not kw.get("learn_t", False)
        assert not kw.get("msg_norm", False) and kw.get("norm", "batch") == "batch" and not kw.get("bias", False)
        assert kw.get("num_layers", 2) == 2 and kw.get("expansion", 2) == 2 and kw.get("eps", MSG_EPS) == MSG_EPS
        d = out_channels
        self.in_channels, self.out_channels, self.eps = in_channels, out_channels, MSG_EPS
        self.mlp = nn.Sequential(nn.Linear(d, 2 * d, bias=False), nn.BatchNorm1d(2 * d), nn.ReLU(), nn.Dropout(0.0),
                                 nn.Linear(2 * d, d, bias=False))

    def messages(self, x, edge_index, edge_attr):
        assert edge_attr is not None and edge_attr.shape[-1] == x.shape[-1]
        return (x[edge_index[0]] + edge_attr).relu() + self.eps


class GENConvMP(_GENParams):
    """Message passing: PyG's scatter softmax over each target's segment, per channel."""

    def aggregate(self, x, edge_index, edge_attr):
        N, d = x.shape
        m = self.messages(x, edge_index, edge_attr)
        dst = edge_index[1]
        idx = dst[:, None].expand(-1, d)
        mmax = torch.full((N, d), -math.inf, dtype=m.dtype).scatter_reduce(0, idx, m.detach(), "amax")
        ex = (m - mmax[dst]).exp()
        den = torch.zeros(N, d, dtype=m.dtype).index_add_(0, dst, ex) + 1e-16
        alpha = ex / den[dst]
        return torch.zeros(N, d, dtype=m.dtype).index_add_(0, dst, m * alpha)

    def forward(self, x, edge_index, edge_attr=None, size=None):
        assert size is None
        return self.mlp(self.aggregate(x, edge_index, edge_attr) + x)


class GENConvLoop(_GENParams):
    """Per node: gather the node's in-edges, torch.softmax over them per channel, alpha-weighted sum of the messages."""

    def aggregate(self, x, edge_index, edge_attr):
        N, d = x.shape
        rows = []
        for i in range(N):
            k = torch.nonzero(edge_index[1] == i).flatten()
            if k.numel() == 0:
                rows.append(x.new_zeros(d))
                continue
            m = (x[edge_index[0, k]] + edge_attr[k]).relu() + self.eps
            rows.append((torch.softmax(m, dim=0) * m).sum(0))
        return torch.stack(rows) if rows else x.new_zeros(0, d)

    def forward(self, x, edge_index, edge_attr=None, size=None):
        assert size is None
        return self.mlp(self.aggregate(x, edge_index, edge_attr) + x)


def genconv_oracle_layer(dim_h, global_model_type, num_heads, **kw):
    """OracleGPSLayer (or its BiasedTransformer subclass) with the GENConvLoop local model; same state_dict keys as the
    reference layer.  Parameters are not drawn in the reference's order: load a state_dict to compare."""
    cls = OracleGPSLayerBiased if global_model_type == "BiasedTransformer" else OracleGPSLayer
    layer = cls(dim_h, "GCN", global_model_type, num_heads, **kw)
    layer.local_model = GENConvLoop(dim_h, dim_h)
    layer.local_gnn_type = "GENConv"
    return layer


@contextlib.contextmanager
def shim_genconv():
    """Installs GENConvMP as GENConv in the reference shim's torch_geometric.nn for the duration of the block."""
    pygnn = sys.modules["torch_geometric.nn"]
    old = pygnn.GENConv
    pygnn.GENConv = GENConvMP
    try:
        yield
    finally:
        pygnn.GENConv = old


def genconv_batch(shape, seed, d, num_graphs, dtype=torch.float32, scale=3.0):
    """gat_oracle.gat_batch (self-loop edges, duplicated edges, a hub with 40 in-edges, an isolated node) with x and
    edge_attr scaled by `scale`, so that the messages of one segment spread over several units per channel, and one node
    (node 2 of graph 0) whose in-edges all have x_src + e <= 0 in every channel: its messages are all 1e-7."""
    from gat_oracle import gat_batch
    b = gat_batch(shape, seed, d, num_graphs, dtype=dtype)
    b.x = b.x * scale
    b.edge_attr = b.edge_attr * scale
    g = torch.Generator().manual_seed(seed + 202)
    t = int(b.ptr[0]) + 2
    k = torch.nonzero(b.edge_index[1] == t).flatten()
    assert k.numel() > 0
    src = b.edge_index[0, k]
    b.edge_attr[k] = -b.x[src] - 0.25 - torch.rand(k.numel(), d, generator=g).to(dtype)
    return b


def dead_node(b):
    """The node genconv_batch gives all-1e-7 messages."""
    return int(b.ptr[0]) + 2
