"""TEST INFRASTRUCTURE - float64 restatement of the PNA stages (csrc/pna.cu) with elementwise fp32 error bounds.

The stages take the layer's operands: Y = [P_dst | P_src] (the node projections, [N, >= 2d]), q = e F^T + c [E, d]
(the edge term) and x.  For edge k from j to i, m_k = Y[i, :d] + Y[j, d:2d] + q[k].  With u = 2^-24 and n the
in-degree of i:
  * m_k: two fp32 additions, |err| <= 2u (|Y_i| + |Y_j| + |q_k|) =: b_k;
  * sum: n - 1 more additions in order, |err| <= sum_k b_k + (n - 1) u sum_k |m_k| (+ the same again for slack);
  * mean = sum / n: the sum's bound / n + u |mean|;
  * max: the chosen message is the fp32 value of some m_k that the kernel saw as largest, so it lies within
    max_k b_k of the fp64 maximum; the argmax may pick any edge of the near-tied set {k : m_k >= max - 2 max b};
  * backward, given the kernel's argmax: g_m = g_mean / n + g_sum + [k = arg] g_max, |err| <= 3u (|g_mean| / n +
    |g_sum| + |g_max|); the in- and out-edge sums add (count - 1) u sum |g_m|.
Bounds carry a factor 2 of slack.
"""
from __future__ import annotations

import torch

U = 2.0 ** -24


def messages(Y, q, ei, d):
    src, dst = ei[0], ei[1]
    m = Y[dst, :d] + Y[src, d:2 * d] + q
    b = 2 * U * (Y[dst, :d].abs() + Y[src, d:2 * d].abs() + q.abs())
    return m, b


def aggregate(x, Y, q, ei):
    """Z = [x | mean | max | sum] and the near-tied sets' lower threshold, fp64; the bounds on Z."""
    N, d = x.shape
    src, dst = ei[0], ei[1]
    m, b = messages(Y, q, ei, d)
    n = torch.zeros(N, dtype=m.dtype).index_add_(0, dst, torch.ones_like(dst, dtype=m.dtype))
    idx = dst[:, None].expand(-1, d)
    s = torch.zeros(N, d, dtype=m.dtype).index_add_(0, dst, m)
    sa = torch.zeros(N, d, dtype=m.dtype).index_add_(0, dst, m.abs())
    sb = torch.zeros(N, d, dtype=m.dtype).index_add_(0, dst, b)
    mx = torch.full((N, d), -torch.inf, dtype=m.dtype).scatter_reduce(0, idx, m, "amax")
    bmax = torch.zeros(N, d, dtype=m.dtype).scatter_reduce(0, idx, b, "amax")
    has = (n > 0)[:, None]
    mx = torch.where(has, mx, torch.zeros_like(mx))
    nn_ = n.clamp(min=1)[:, None]
    mean = s / nn_
    b_sum = 2 * (sb + (nn_ - 1) * U * sa)
    b_mean = b_sum / nn_ + 2 * U * mean.abs()
    Z = torch.cat([x, mean, mx, s], 1)
    B = torch.cat([torch.zeros_like(x), b_mean, 2 * bmax, b_sum], 1)
    return Z, B, m, b, bmax


def argmax_ok(arg, m, ei, mx, bmax):
    """Every chosen edge is an in-edge of its node whose message lies within 4 max b of the segment maximum; nodes
    without in-edges carry -1."""
    N, d = mx.shape
    n = torch.bincount(ei[1], minlength=N)
    if not bool((arg[n == 0] == -1).all()):
        return False
    a = arg[n > 0].long()
    if a.numel() == 0:
        return True
    if bool((a < 0).any()):
        return False
    nodes = torch.nonzero(n > 0).flatten()
    if not bool((ei[1][a] == nodes[:, None]).all()):
        return False
    chosen = m.gather(0, a)
    return bool((chosen >= mx[nodes] - 4 * bmax[nodes]).all())


def backward(gZ, arg, ei, N, d, add=None):
    """g_q [E, d], gY [N, 2d] (g_P_dst | g_P_src), g_x [N, d] given the kernel's argmax, and their bounds."""
    src, dst = ei[0], ei[1]
    E = src.numel()
    n = torch.bincount(dst, minlength=N).to(gZ.dtype).clamp(min=1)[:, None]
    gmean, gmax, gsum = gZ[:, d:2 * d], gZ[:, 2 * d:3 * d], gZ[:, 3 * d:]
    is_arg = arg.long()[dst] == torch.arange(E)[:, None]
    gq = (gmean / n + gsum)[dst] + torch.where(is_arg, gmax[dst], torch.zeros_like(gmax[dst]))
    bq = 6 * U * ((gmean / n).abs() + gsum.abs() + gmax.abs())[dst]
    gd = torch.zeros(N, d, dtype=gZ.dtype).index_add_(0, dst, gq)
    gs = torch.zeros(N, d, dtype=gZ.dtype).index_add_(0, src, gq)
    ad = torch.zeros(N, d, dtype=gZ.dtype).index_add_(0, dst, gq.abs())
    as_ = torch.zeros(N, d, dtype=gZ.dtype).index_add_(0, src, gq.abs())
    bd = torch.zeros(N, d, dtype=gZ.dtype).index_add_(0, dst, bq)
    bs = torch.zeros(N, d, dtype=gZ.dtype).index_add_(0, src, bq)
    cd = torch.bincount(dst, minlength=N).to(gZ.dtype)[:, None]
    cs = torch.bincount(src, minlength=N).to(gZ.dtype)[:, None]
    gY = torch.cat([gd, gs], 1)
    bY = torch.cat([2 * (bd + cd * U * ad), 2 * (bs + cs * U * as_)], 1)
    gx = gZ[:, :d] + (add if add is not None else 0)
    bx = 2 * U * gx.abs()
    return gq, bq, gY, bY, gx, bx


def fold(Wpre, bpre, Wenc, benc):
    """F = W_e W_enc and c = W_e b_enc + b_pre (W_e = Wpre[:, 2d:]) with |err| <= 2 d u sum |terms|."""
    d = Wpre.shape[0]
    We = Wpre[:, 2 * d:]
    F = We @ Wenc
    c = We @ benc + bpre
    bF = 2 * d * U * (We.abs() @ Wenc.abs())
    bc = 2 * d * U * (We.abs() @ benc.abs() + bpre.abs())
    return F, bF, c, bc


def unfold(Wpre, Wenc, benc, gF, gc):
    """The fold's backward and its bounds: g_W_e = g_F W_enc^T + g_c b_enc^T, g_W_enc = W_e^T g_F, g_b_enc = W_e^T g_c,
    g_b_pre = g_c."""
    d, de = gF.shape
    We = Wpre[:, 2 * d:]
    gWe = gF @ Wenc.t() + gc[:, None] * benc[None, :]
    bWe = 2 * (de + 1) * U * (gF.abs() @ Wenc.abs().t() + (gc.abs()[:, None] * benc.abs()[None, :]))
    gWenc = We.t() @ gF
    bWenc = 2 * d * U * (We.abs().t() @ gF.abs())
    gbenc = We.t() @ gc
    bbenc = 2 * d * U * (We.abs().t() @ gc.abs())
    return gWe, bWe, gWenc, bWenc, gbenc, bbenc
