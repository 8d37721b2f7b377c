"""Float64 restatement of CustomGNN's two message-passing layers, and batches with LRGB-like shapes.

  * GatedGCNLayer (gatedgcn_layer.py:45-136, no EquivStableLapPE): Ax..Ex, Ce; e_ij = Dx_i + Ex_j + Ce per edge j -> i;
    sigma = sigmoid(e_ij); x = Ax + scatter_sum(sigma Bx_j) / (scatter_sum(sigma) + 1e-6) over the destination;
    x = act(bn_node_x(x)), e = act(bn_edge_e(e_ij)), dropout, then the residual when set.
  * GINEConvLayer (gine_conv_layer.py:102-113): GINEConv(nn.0, ReLU, nn.2) with eps from its buffer:
    nn((1 + eps) x + scatter_sum(relu(x_j + e_ij))), then relu, dropout and the residual when set.
BatchNorm is nn.BatchNorm1d's: batch statistics (biased variance) in training, which also update the running ones
(unbiased variance, momentum 0.1), the running ones in eval.  Dropout masks (the library's, 0 or 1/(1-p)) can be
injected in place of F.dropout.  The modules carry the reference's parameter names, so a fixture's state loads strictly.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from san_oracle import SanBatch, san_batch  # noqa: F401  (re-exported for the tests)

_ACT = {"relu": F.relu, "gelu": F.gelu}


class OracleGatedGCN(nn.Module):
    def __init__(self, d, act="relu", residual=True):
        super().__init__()
        for n in "ABCDE":
            setattr(self, n, nn.Linear(d, d))
        self.bn_node_x = nn.BatchNorm1d(d)
        self.bn_edge_e = nn.BatchNorm1d(d)
        self.act, self.residual = act, residual

    def forward(self, x, e, edge_index, mask_x=None, mask_e=None):
        src, dst = edge_index[0], edge_index[1]
        Ax, Bx, Dx, Ex, Ce = self.A(x), self.B(x), self.D(x), self.E(x), self.C(e)
        e_ij = Dx[dst] + Ex[src] + Ce
        sigma = torch.sigmoid(e_ij)
        num = torch.zeros_like(Ax).index_add(0, dst, sigma * Bx[src])
        den = torch.zeros_like(Ax).index_add(0, dst, sigma)
        h = Ax + num / (den + 1e-6)
        h = _ACT[self.act](self.bn_node_x(h))
        ee = _ACT[self.act](self.bn_edge_e(e_ij))
        if mask_x is not None:
            h = h * mask_x
        if mask_e is not None:
            ee = ee * mask_e
        if self.residual:
            h, ee = x + h, e + ee
        return h, ee


class _GINE(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.nn = nn.Sequential(nn.Linear(d, d), nn.ReLU(), nn.Linear(d, d))
        self.register_buffer("eps", torch.Tensor([0.0]))


class OracleGINE(nn.Module):
    def __init__(self, d, residual=True):
        super().__init__()
        self.model = _GINE(d)
        self.residual = residual

    def forward(self, x, e, edge_index, mask_x=None):
        src, dst = edge_index[0], edge_index[1]
        agg = torch.zeros_like(x).index_add(0, dst, F.relu(x[src] + e))
        h = F.relu(self.model.nn((1 + self.model.eps) * x + agg))
        if mask_x is not None:
            h = h * mask_x
        return (x + h if self.residual else h), e


def oracle_layer(kind, d, act="relu", residual=True):
    return OracleGatedGCN(d, act, residual) if kind == "gatedgcn" else OracleGINE(d, residual)


def run_stack(layers, x, e, edge_index, masks=None):
    """Runs the layers in order, edge_attr chaining (GINE passes it through); masks: per layer (mask_x, mask_e)."""
    for i, layer in enumerate(layers):
        mx, me = masks[i] if masks else (None, None)
        if isinstance(layer, OracleGatedGCN):
            x, e = layer(x, e, edge_index, mx, me)
        else:
            x, e = layer(x, e, edge_index, mx)
    return x, e


def edge_case_batch(d, seed, dtype=torch.float32):
    """Three graphs: 6 nodes with a self loop, a duplicated edge, a one-way edge and an isolated node; a one-node
    graph; 4 nodes with a self loop on the last."""
    src = [0, 1, 1, 2, 2, 3, 0, 4, 2, 6, 7, 8, 9, 10, 10]
    dst = [1, 0, 2, 1, 2, 0, 1, 3, 1, 6, 8, 7, 8, 9, 10]
    ei = torch.tensor([src, dst], dtype=torch.int64)
    batch = torch.tensor([0] * 6 + [1] + [2] * 4, dtype=torch.int64)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(11, d, generator=g, dtype=torch.float64).to(dtype)
    e = torch.randn(ei.shape[1], d, generator=g, dtype=torch.float64).to(dtype)
    return SanBatch(x, e, ei, batch, 3)


def no_edge_batch(d, seed, dtype=torch.float32):
    """Two graphs of 3 and 2 nodes and no edges at all."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(5, d, generator=g, dtype=torch.float64).to(dtype)
    return SanBatch(x, torch.zeros(0, d, dtype=dtype), torch.zeros(2, 0, dtype=torch.int64),
                    torch.tensor([0, 0, 0, 1, 1]), 2)
