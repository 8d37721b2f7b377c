"""fp64 restatement of the GAT stages the library exports (gat.cu); each backward is torch.autograd of its forward.

fold(W_edge, att_edge, H) = v [H, d], v[h] = W_edge[hC:(h+1)C, :]^T att_edge[h]
aggregate(Y, edge_index, edge_attr, v, att_src, att_dst, bias, H) = GATConv's output [N, d] (bias included) given
Y = x lin_src^T: a_edge = e . v[h] is GATConv's (lin_edge(e) * att_edge).sum(-1) by linearity, and the added self
loop's score is the mean of the remaining in-edges' scores (the loop attribute is their mean).
"""
import math

import torch
import torch.nn.functional as F


def fold(W_edge, att_edge, H):
    d = W_edge.shape[1]
    C = W_edge.shape[0] // H
    return torch.einsum("hck,hc->hk", W_edge.view(H, C, d), att_edge.reshape(H, C))


def scores(Y, edge_index, edge_attr, v, att_src, att_dst, H):
    """a_src, a_dst, a_self, lse [N, H], a_edge [E, H] (a_edge of removed self loops included), as gps_gat_forward."""
    N, d = Y.shape
    C = d // H
    y = Y.view(N, H, C)
    a_src = (y * att_src.reshape(1, H, C)).sum(-1)
    a_dst = (y * att_dst.reshape(1, H, C)).sum(-1)
    a_edge = edge_attr @ v.t()
    keep = edge_index[0] != edge_index[1]
    src, dst, ae = edge_index[0, keep], edge_index[1, keep], a_edge[keep]
    cnt = torch.zeros(N, dtype=Y.dtype).index_add_(0, dst, torch.ones(dst.shape[0], dtype=Y.dtype))
    a_self = torch.zeros(N, H, dtype=Y.dtype).index_add_(0, dst, ae) / cnt.clamp(min=1)[:, None]
    loops = torch.arange(N)
    src, dst = torch.cat([src, loops]), torch.cat([dst, loops])
    z = F.leaky_relu(a_src[src] + a_dst[dst] + torch.cat([ae, a_self]), 0.2)
    idx = dst[:, None].expand(-1, H)
    zmax = torch.full((N, H), -math.inf, dtype=z.dtype).scatter_reduce(0, idx, z.detach(), "amax")
    ex = (z - zmax[dst]).exp()
    den = torch.zeros(N, H, dtype=z.dtype).index_add_(0, dst, ex)
    lse = zmax + den.log()
    return dict(a_src=a_src, a_dst=a_dst, a_self=a_self, lse=lse, a_edge=a_edge, src=src, dst=dst, z=z, ex=ex, den=den)


def aggregate(Y, edge_index, edge_attr, v, att_src, att_dst, bias, H):
    N, d = Y.shape
    C = d // H
    s = scores(Y, edge_index, edge_attr, v, att_src, att_dst, H)
    alpha = s["ex"] / (s["den"][s["dst"]] + 1e-16)
    out = torch.zeros(N, H, C, dtype=Y.dtype).index_add_(0, s["dst"], alpha[..., None] * Y.view(N, H, C)[s["src"]])
    return out.reshape(N, d) + bias


def chunk(rows, num_sms=132):
    """Rows per block of the library's fixed-chunk column sums (gat.cu gat_chunk) and the number of blocks."""
    c = max(32, -(-rows // num_sms))
    return c, -(-rows // c) if rows else 0


def error_bounds(Y, edge_index, edge_attr, v, att_src, att_dst, bias, x, g_h, H, K=4.0, u=2.0 ** -24):
    """Elementwise bounds on |library - exact| of every stage output, from the fp64 intermediates of the same
    computation: each sum of n terms gets K n u sum|terms| (n = its actual length: C for a head's dot product, d for an
    edge score, the in- or out-degree + 1 for a segment, the chunk length + chunk count for a column sum), and the
    errors of the scores are carried through exp: an absolute error e on z - lse is a relative error e on alpha.  A
    LeakyReLU whose pre-activation lies within its error of 0 may take either slope; its slot gets the difference.
    All arguments are float64 (v: the library's fold), g_h the cotangent of the aggregation output."""
    with torch.no_grad():
        N, d = Y.shape
        C = d // H
        E = edge_attr.shape[0]
        y, gh = Y.view(N, H, C), g_h.view(N, H, C)
        ats, atd = att_src.reshape(1, H, C), att_dst.reshape(1, H, C)
        a_src, a_dst = (y * ats).sum(-1), (y * atd).sum(-1)
        e_src = K * C * u * (y.abs() * ats.abs()).sum(-1)
        e_dst = K * C * u * (y.abs() * atd.abs()).sum(-1)
        a_edge = edge_attr @ v.t()
        e_edge = K * d * u * (edge_attr.abs() @ v.abs().t())
        keep = edge_index[0] != edge_index[1]
        eid = torch.nonzero(keep).flatten()
        src, dst = edge_index[0, keep], edge_index[1, keep]
        ones = torch.ones(src.shape[0], dtype=Y.dtype)
        deg = torch.zeros(N, dtype=Y.dtype).index_add_(0, dst, ones)
        outd = torch.zeros(N, dtype=Y.dtype).index_add_(0, src, ones)
        dinv = 1.0 / deg.clamp(min=1)[:, None]
        a_self = torch.zeros(N, H, dtype=Y.dtype).index_add_(0, dst, a_edge[eid]) * dinv
        e_self = (torch.zeros(N, H, dtype=Y.dtype).index_add_(0, dst, e_edge[eid] + K * u * a_edge[eid].abs())
                  * dinv * (1 + K * deg[:, None] * u) + K * u * a_self.abs())
        loops = torch.arange(N)
        s_src, s_dst = torch.cat([src, loops]), torch.cat([dst, loops])
        ae = torch.cat([a_edge[eid], a_self])
        pre = a_src[s_src] + a_dst[s_dst] + ae
        e_pre = e_src[s_src] + e_dst[s_dst] + torch.cat([e_edge[eid], e_self]) + 2 * K * u * (
            a_src[s_src].abs() + a_dst[s_dst].abs() + ae.abs())
        z = torch.nn.functional.leaky_relu(pre, 0.2)
        lam = torch.where(pre > 0, 1.0, 0.2).to(Y.dtype)
        flip = pre.abs() <= e_pre
        idx = s_dst[:, None].expand(-1, H)
        zmax = torch.full((N, H), -math.inf, dtype=Y.dtype).scatter_reduce(0, idx, z, "amax")
        ex = (z - zmax[s_dst]).exp()
        den = torch.zeros(N, H, dtype=Y.dtype).index_add_(0, s_dst, ex)
        lse = zmax + den.log()
        emax = torch.zeros(N, H, dtype=Y.dtype).scatter_reduce(0, idx, e_pre, "amax")
        e_lse = emax + K * (deg[:, None] + 3) * u + K * u * lse.abs()
        alpha = (z - lse[s_dst]).exp()
        e_alpha = e_pre + e_lse[s_dst] + K * u * (z.abs() + lse[s_dst].abs() + 2)   # relative error of alpha
        n_dst = (deg + 3)[:, None, None]
        n_src = (outd + 3)[:, None, None]
        # forward: x_loc = x + sum alpha Y[src] + bias
        ay = alpha[..., None] * y[s_src].abs()
        sum_ay = torch.zeros(N, H, C, dtype=Y.dtype).index_add_(0, s_dst, ay)
        sum_ay_e = torch.zeros(N, H, C, dtype=Y.dtype).index_add_(0, s_dst, ay * e_alpha[..., None])
        b_xloc = (sum_ay_e + K * n_dst * u * (sum_ay + x.view(N, H, C).abs() + bias.view(1, H, C).abs())).reshape(N, d)
        # backward, destination side
        ga = (gh[s_dst] * y[s_src]).sum(-1)
        e_ga = K * C * u * (gh[s_dst].abs() * y[s_src].abs()).sum(-1)
        delta = torch.zeros(N, H, dtype=Y.dtype).index_add_(0, s_dst, alpha * ga)
        e_delta = torch.zeros(N, H, dtype=Y.dtype).index_add_(0, s_dst, alpha * (e_alpha * ga.abs() + e_ga)) + \
            K * (deg[:, None] + 1) * u * torch.zeros(N, H, dtype=Y.dtype).index_add_(0, s_dst, alpha * ga.abs())
        gdiff = ga - delta[s_dst]
        gz = alpha * gdiff * lam
        e_gz = lam * (alpha * e_alpha * gdiff.abs() + alpha * (e_ga + e_delta[s_dst]) +
                      K * u * alpha * (ga.abs() + delta[s_dst].abs()))
        e_gz = e_gz + torch.where(flip, 0.8 * alpha * gdiff.abs(), torch.zeros_like(gz))
        gad = torch.zeros(N, H, dtype=Y.dtype).index_add_(0, s_dst, gz)
        e_gad = torch.zeros(N, H, dtype=Y.dtype).index_add_(0, s_dst, e_gz) + \
            K * (deg[:, None] + 1) * u * torch.zeros(N, H, dtype=Y.dtype).index_add_(0, s_dst, gz.abs())
        ne = src.shape[0]
        gz_e, gz_s, e_gz_e, e_gz_s = gz[:ne], gz[ne:], e_gz[:ne], e_gz[ne:]
        share = gz_s * dinv
        gae = gz_e + share[dst]
        e_gae = e_gz_e + (e_gz_s * dinv)[dst] + K * u * (gz_e.abs() + share[dst].abs())
        # backward, source side: gY
        G = torch.zeros(N, H, dtype=Y.dtype).index_add_(0, s_src, gz)
        e_G = torch.zeros(N, H, dtype=Y.dtype).index_add_(0, s_src, e_gz) + \
            K * (outd[:, None] + 1) * u * torch.zeros(N, H, dtype=Y.dtype).index_add_(0, s_src, gz.abs())
        ag = alpha[..., None] * gh[s_dst].abs()
        sum_ag = torch.zeros(N, H, C, dtype=Y.dtype).index_add_(0, s_src, ag)
        sum_ag_e = torch.zeros(N, H, C, dtype=Y.dtype).index_add_(0, s_src, ag * e_alpha[..., None])
        b_gY = (sum_ag_e + K * n_src * u * (sum_ag + (G[..., None] * ats).abs() + (gad[..., None] * atd).abs())
                + e_G[..., None] * ats.abs() + e_gad[..., None] * atd.abs()).reshape(N, d)
        # grad_edge_attr (0 on removed self loops, checked exactly)
        b_gea = torch.zeros(E, d, dtype=Y.dtype)
        b_gea[eid] = e_gae @ v.abs() + K * H * u * (gae.abs() @ v.abs())
        # column sums
        ce, pe = chunk(E)
        cn, pn = chunk(N)
        ea = edge_attr[eid].abs()
        b_gv = e_gae.t() @ ea + K * (ce + pe) * u * (gae.abs().t() @ ea)
        Yh = Y.abs().view(N, H, C)
        b_gas = ((e_G[..., None] * Yh).sum(0) + K * (cn + pn) * u * (G.abs()[..., None] * Yh).sum(0)).reshape(d)
        b_gad = ((e_gad[..., None] * Yh).sum(0) + K * (cn + pn) * u * (gad.abs()[..., None] * Yh).sum(0)).reshape(d)
        b_gb = K * (cn + pn) * u * g_h.abs().sum(0)
        return dict(a_self=e_self, lse=e_lse, xloc=b_xloc, gY=b_gY, grad_edge_attr=b_gea, g_v=b_gv, g_att_src=b_gas,
                    g_att_dst=b_gad, g_bias=b_gb)
