"""Plain float64 torch references of the message-passing stages (csrc/scatter.cu, csrc/eslap.cu), one function per
stage and direction, for the stage tests in tests/test_message_passing*.py.

Each forward follows the lines of oracle/gps_oracle.py (OracleGatedGCN, OracleGINE, OracleGCN) and
tests/eslappe_oracle.py (OracleGatedGCNESLapPE); tests/test_message_passing.py ties them to those modules.  Every
backward is torch.autograd.grad of the matching forward with the caller's upstream gradients: no backward formula is
derived by hand here.  Edge j -> i: src = edge_index[0] = j, dst = edge_index[1] = i.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

ACTS = {"relu": torch.relu, "gelu": F.gelu}


def _grads(outputs, inputs, grad_outputs):
    gs = torch.autograd.grad(outputs, inputs, grad_outputs, allow_unused=True)
    return [torch.zeros_like(t) if g is None else g for t, g in zip(inputs, gs)]


def _leaf(t):
    return t.detach().double().requires_grad_(True)


# ---------------------------------------------------------------------------------------------------- GatedGCN
def gatedgcn_sums(Bx, e_ij, src, dst, rho=None):
    """num_i = sum_j sigma_ij Bx_j, den_i = sum_j sigma_ij with sigma = sigmoid(e_ij) [* rho_e] (gatedgcn_layer.py:97-123)"""
    sigma = torch.sigmoid(e_ij)
    if rho is not None:
        sigma = sigma * rho.reshape(-1, 1)
    num = torch.zeros_like(Bx).index_add_(0, dst, sigma * Bx[src])
    den = torch.zeros_like(Bx).index_add_(0, dst, sigma)
    return num, den


def gatedgcn_forward(Ax, Bx, Dx, Ex, Ce, src, dst, rho=None):
    """x~ = Ax + num / (den + 1e-6) and e_ij = Dx_i + Ex_j + Ce_ij.  Returns (xt, e_ij, num, den)."""
    e_ij = Dx[dst] + Ex[src] + Ce
    num, den = gatedgcn_sums(Bx, e_ij, src, dst, rho)
    return Ax + num / (den + 1e-6), e_ij, num, den


def gatedgcn_backward(Ax, Bx, Dx, Ex, Ce, src, dst, g_xt, g_e, rho=None):
    """Gradients of <g_xt, x~> + <g_e, e_ij>: g_Bx, g_Dx, g_Ex, g_e (total, w.r.t. e_ij), g_num, g_den."""
    Bx, Dx, Ex, Ce = (_leaf(t) for t in (Bx, Dx, Ex, Ce))
    rho = None if rho is None else rho.detach().double()
    xt, e_ij, num, den = gatedgcn_forward(Ax.detach().double(), Bx, Dx, Ex, Ce, src, dst, rho)
    gB, gD, gE, gC, gnum, gden = _grads([xt, e_ij], [Bx, Dx, Ex, Ce, num, den], [g_xt.double(), g_e.double()])
    return {"g_Bx": gB, "g_Dx": gD, "g_Ex": gE, "g_e": gC, "g_num": gnum, "g_den": gden}


# ---------------------------------------------------------------------------------------------------- EquivStableLapPE
def eslap_forward(pe, src, dst, w1, b1, w2, b2, act):
    """r_e = sum_c (PE_i - PE_j)^2, rho_e = mlp_r_ij(r_e) = sigmoid(w2 . act(w1 r + b1) + b2)  (gatedgcn_layer.py:29-35,
    101-104).  w1 = mlp_r_ij.0.weight [d,1], b1 [d], w2 = mlp_r_ij.2.weight [1,d], b2 [1].  Returns (r [E], rho [E])."""
    r = ((pe[dst] - pe[src]) ** 2).sum(dim=-1, keepdim=True)
    h = ACTS[act](F.linear(r, w1, b1))
    return r.reshape(-1), torch.sigmoid(F.linear(h, w2, b2)).reshape(-1)


def eslap_backward(pe, src, dst, w1, b1, w2, b2, act, Bx, ehat, g_num, g_den):
    """What the gate receives from the GatedGCN backward: the gradients of <g_num, num> + <g_den, den> (num, den of
    gatedgcn_sums with e_ij = ehat) w.r.t. pe and mlp_r_ij.  Returns grad_pe, gw1, gb1, gw2, gb2."""
    pe, w1, b1, w2, b2 = (_leaf(t) for t in (pe, w1, b1, w2, b2))
    _, rho = eslap_forward(pe, src, dst, w1, b1, w2, b2, act)
    num, den = gatedgcn_sums(Bx.double(), ehat.double(), src, dst, rho)
    g = _grads([num, den], [pe, w1, b1, w2, b2], [g_num.double(), g_den.double()])
    return dict(zip(("grad_pe", "gw1", "gb1", "gw2", "gb2"), g))


# ---------------------------------------------------------------------------------------------------- GINE
def gine_forward(x, e, src, dst, eps):
    """out_i = (1 + eps) x_i + sum_j relu(x_j + e_ij)  (OracleGINE before its nn)"""
    msg = (x[src] + e).relu()
    return torch.zeros_like(x).index_add_(0, dst, msg) + (1 + eps) * x


def gine_backward(x, e, src, dst, eps, g_out, add=None):
    """g_x, g_e of <g_out, out>; `add` [N,d] (another gradient path into x) is added to g_x."""
    x, e = _leaf(x), _leaf(e)
    g_x, g_e = _grads([gine_forward(x, e, src, dst, eps)], [x, e], [g_out.double()])
    if add is not None:
        g_x = g_x + add.double()
    return g_x, g_e


# ---------------------------------------------------------------------------------------------------- GCN
def gcn_dinv(src, dst, N):
    """(1 + #{j -> i, j != i})^-1/2: existing self loops are replaced by one unit loop (add_remaining_self_loops)"""
    keep = src != dst
    deg = torch.ones(N, dtype=torch.float64, device=dst.device)
    return deg.index_add_(0, dst[keep], torch.ones_like(deg[:1]).expand(int(keep.sum()))).rsqrt()


def gcn_aggregate(Y, src, dst):
    """A_hat Y = D^-1/2 (A' + I) D^-1/2 Y  (OracleGCN without lin and bias)"""
    dinv = gcn_dinv(src, dst, Y.shape[0]).to(Y.device)
    keep = src != dst
    s, t = src[keep], dst[keep]
    agg = (dinv * dinv).unsqueeze(1) * Y
    return agg.index_add(0, t, (dinv[s] * dinv[t]).unsqueeze(1) * Y[s])


def gcn_forward(Y, bias, x, src, dst, keep=None, p=0.0):
    """x_loc = x + dropout(bias + A_hat Y); keep: the 0/1 keep-mask of the dropout (scale 1 / (1 - p))"""
    h = gcn_aggregate(Y, src, dst) + bias
    if keep is not None:
        h = h * keep / (1.0 - p)
    return x + h


def gcn_backward(Y, src, dst, g_h):
    """gradient of <g_h, A_hat Y> w.r.t. Y"""
    Y = _leaf(Y)
    return _grads([gcn_aggregate(Y, src, dst)], [Y], [g_h.double()])[0]
