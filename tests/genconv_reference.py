"""fp64 restatement of the GENConv stages the library exports (genconv.cu) and elementwise bounds on their fp32 error.

aggregate(x, edge_index, edge_attr) = (agg, lse, u) as gps_genconv_aggregate_forward: m_k = relu(x[src_k] + e_k) + 1e-7,
agg_i = sum_k softmax_k(m) m_k over i's in-edges per channel (0 without in-edges), lse_i = log sum_k exp(m_k) (0 without
in-edges), u = agg + x.  The backward stage is torch.autograd of u: g_e = d(u . g_u)/d e and g_x = d(u . g_u)/d x + add.
"""
import math

import torch


def aggregate(x, edge_index, edge_attr):
    N, d = x.shape
    src, dst = edge_index[0], edge_index[1]
    m = (x[src] + edge_attr).relu() + 1e-7
    idx = dst[:, None].expand(-1, d)
    mmax = torch.full((N, d), -math.inf, dtype=x.dtype).scatter_reduce(0, idx, m.detach(), "amax")
    ex = (m - mmax[dst]).exp()
    den = torch.zeros(N, d, dtype=x.dtype).index_add_(0, dst, ex)
    agg = torch.zeros(N, d, dtype=x.dtype).index_add_(0, dst, m * ex / (den[dst] + 1e-16))
    has = torch.bincount(dst, minlength=N)[:, None] > 0
    lse = torch.where(has, mmax + den.clamp(min=1e-300).log(), torch.zeros_like(den))
    return agg, lse, agg + x


def error_bounds(x, edge_index, edge_attr, g_u, add=None, K=4.0, u=2.0 ** -24):
    """Elementwise bounds on |library - exact| of agg, lse, u, g_e and g_x, from the fp64 intermediates.  Each sum of n
    terms gets K n u sum|terms| (n = the node's in-degree for the online softmax, out-degree + 2 for g_x).  The message
    errors e_m (the fp32 add and the + 1e-7) are carried through exp: the weight of edge k has a relative error of
    e_m_k + max_j e_m_j + K (n + 2) u (its exp, the subtraction of the running max, up to n rescales), which moves agg by
    sum_k alpha_k eps_k |m_k - agg|.  alpha = exp(m - lse) in the backward carries e_m and lse's error.  The sign of
    x_src + e is exact in fp32, so the ReLU masks agree.  All arguments float64."""
    with torch.no_grad():
        N, d = x.shape
        src, dst = edge_index[0], edge_index[1]
        pre = x[src] + edge_attr
        m = pre.relu() + 1e-7
        e_m = 2 * u * (x[src].abs() + edge_attr.abs() + 1e-7)
        idx = dst[:, None].expand(-1, d)
        ones = torch.ones(src.shape[0], dtype=x.dtype)
        deg = torch.zeros(N, dtype=x.dtype).index_add_(0, dst, ones)[:, None]
        outd = torch.zeros(N, dtype=x.dtype).index_add_(0, src, ones)[:, None]
        agg, lse, _ = aggregate(x, edge_index, edge_attr)
        has = deg > 0
        mmax = torch.full((N, d), -math.inf, dtype=x.dtype).scatter_reduce(0, idx, m, "amax")
        mmax = torch.where(has, mmax, torch.zeros_like(mmax))
        emax = torch.zeros(N, d, dtype=x.dtype).scatter_reduce(0, idx, e_m, "amax")
        alpha = (m - lse[dst]).exp()
        eps = e_m + emax[dst] + K * (deg[dst] + 2) * u
        seg = lambda t: torch.zeros(N, d, dtype=x.dtype).index_add_(0, dst, t)
        b_agg = seg(alpha * (eps * (m - agg[dst]).abs() + e_m)) + K * deg * u * (seg(alpha * m) + agg.abs())
        b_lse = torch.where(has, emax + K * (deg + 2) * u + K * u * (lse.abs() + mmax.abs() + 1), torch.zeros_like(lse))
        b_u = b_agg + K * u * (agg.abs() + x.abs())
        # backward, dst ordered: g_e = g_u alpha (1 + m - agg) [pre > 0]
        gu = g_u[dst]
        fac = 1 + m - agg[dst]
        e_alpha = e_m + b_lse[dst] + K * u * (m.abs() + lse[dst].abs() + 1)
        e_fac = e_m + b_agg[dst] + K * u * (1 + m.abs() + agg[dst].abs())
        mask = (pre > 0).to(x.dtype)
        b_ge = mask * gu.abs() * alpha * (e_alpha * fac.abs() + e_fac + K * u * fac.abs())
        ge = mask * gu * alpha * fac
        # src ordered: g_x = g_u + sum_out g_e + add
        segs = lambda t: torch.zeros(N, d, dtype=x.dtype).index_add_(0, src, t)
        a = add.abs() if add is not None else torch.zeros_like(x)
        b_gx = segs(b_ge) + K * (outd + 2) * u * (g_u.abs() + segs(ge.abs()) + a)
        return dict(agg=b_agg, lse=b_lse, u=b_u, g_e=b_ge, g_x=b_gx)
