"""float64 references of the Performer stages (csrc/performer.cu, csrc/performer_quad.cu) on the packed layout.

A (node, head) row is r = n * H + h: Q, K, V, O are [N*H, 64], feature maps [N*H, m], gmax [B*H].  The reference
(performer_layer.py:119-144,200-205) runs on the zero-padded dense batch [B, H, Nmax, .] and masks only v, so the padded
rows of a graph with n < Nmax are written out here as that batch does: they have dd = 0 and diag = 0, so they put 0 into
the key max and add (Nmax - n) k'_pad, k'_pad = ratio (exp(-gmax) + eps), to sum_n k'.

Each backward is torch.autograd.grad of its forward; gmax is an explicit output of `features` and an input of
`attention`, so an upstream gradient of it can be fed in.  `ties="first"` replaces torch.amax's even split of the
gradient among tied maxima by the kernels' rule (all of it to the lowest index; the dense batch's flat (row, feature)
order puts the real rows before the padded ones)."""
import torch

DH = 64
EPS = 1e-4


def layout(ptr):
    """node -> graph, node -> position in its graph, B, Nmax"""
    ptr = ptr.long()
    n = ptr[1:] - ptr[:-1]
    B = n.numel()
    batch = torch.repeat_interleave(torch.arange(B, device=ptr.device), n)
    pos = torch.arange(batch.numel(), device=ptr.device) - ptr[:-1][batch]
    return batch, pos, B, int(n.max()) if B else 0


def to_dense(x, ptr, H):
    """[N*H, c] -> [B, H, Nmax, c] with zero padded rows"""
    batch, pos, B, Nmax = layout(ptr)
    N, c = batch.numel(), x.shape[1]
    out = x.new_zeros(B, Nmax, H, c).index_put((batch, pos), x.view(N, H, c))
    return out.transpose(1, 2)


def to_packed(xd, ptr):
    batch, pos, _, _ = layout(ptr)
    return xd.transpose(1, 2)[batch, pos].reshape(-1, xd.shape[-1])


def _amax(x, dims, ties):
    if ties == "split":
        return torch.amax(x, dim=dims)
    flat = x.flatten(start_dim=x.dim() - len(dims))          # the reduced dims are trailing
    return flat.gather(-1, flat.argmax(-1, keepdim=True)).squeeze(-1)


def features(dd_q, dd_k, Q, K, ptr, H, m, ties="split"):
    """dd [N*H, >= m] (columns < m used), Q, K [N*H, 64] -> q', k' [N*H, m], gmax [B*H]"""
    dd_q, dd_k = dd_q[:, :m], dd_k[:, :m]
    ratio, dn2 = m ** -0.5, DH ** -0.5
    diag_q = (Q ** 2).sum(-1, keepdim=True) / 2.0 * dn2
    diag_k = (K ** 2).sum(-1, keepdim=True) / 2.0 * dn2
    fq = ratio * (torch.exp(dd_q - diag_q - _amax(dd_q, (-1,), ties).unsqueeze(-1)) + EPS)
    batch, _, B, _ = layout(ptr)
    gmax = _amax(to_dense(dd_k, ptr, H), (-2, -1), ties)      # [B, H]: over the graph's rows and its padded rows
    fk = ratio * (torch.exp(dd_k - diag_k - gmax[batch].reshape(-1, 1)) + EPS)
    return fq, fk, gmax.reshape(-1)


def attention(qf, kf, V, gmax, ptr, H, Nmax, form):
    """q', k' [N*H, m], V [N*H, 64], gmax [B*H] -> O [N*H, 64], den [N*H].  form 0: q'.(sum k'^T v) / q'.(sum k'),
    form 1: sum_j (q'.k'_j) v_j / sum_j (q'.k'_j); both with the padded rows' k'_pad in the denominator."""
    m = qf.shape[1]
    ratio = m ** -0.5
    _, _, B, _ = layout(ptr)
    n = (ptr[1:] - ptr[:-1]).to(qf.dtype)
    kpad = ratio * (torch.exp(-gmax.view(B, H)) + EPS) * (Nmax - n).unsqueeze(1)          # [B, H]
    qd, kd, vd = (to_dense(t, ptr, H) for t in (qf, kf, V))
    if form == 0:
        ksum = kd.sum(2) + kpad.unsqueeze(-1)
        den = torch.einsum("bhnj,bhj->bhn", qd, ksum)
        num = torch.einsum("bhnj,bhje->bhne", qd, torch.einsum("bhnj,bhne->bhje", kd, vd))
    else:
        s = torch.einsum("bhij,bhkj->bhik", qd, kd)
        den = s.sum(-1) + kpad.unsqueeze(-1) * qd.sum(-1)
        num = torch.einsum("bhik,bhke->bhie", s, vd)
    real = to_dense(torch.ones(qf.shape[0], 1, dtype=qf.dtype, device=qf.device), ptr, H)[..., 0]
    den = den + (1 - real)                                    # padded query rows: 0 / 1, never read
    O = num / den.unsqueeze(-1)
    return to_packed(O, ptr), to_packed(den.unsqueeze(-1), ptr)[:, 0]


def features_backward(dd_q, dd_k, Q, K, ptr, H, m, g_fq, g_fk, g_gmax, ties="split"):
    """-> g_dd_q, g_dd_k [N*H, m], g_Q, g_K [N*H, 64] (the diag paths)"""
    leaves = [t.detach().clone().requires_grad_(True) for t in (dd_q[:, :m], dd_k[:, :m], Q, K)]
    out = features(*leaves, ptr, H, m, ties)
    return torch.autograd.grad(out, leaves, [g_fq[:, :m], g_fk[:, :m], g_gmax])


def attention_backward(qf, kf, V, gmax, ptr, H, Nmax, form, gO):
    """-> g_qf, g_kf [N*H, m], gV [N*H, 64], g_gmax [B*H]"""
    leaves = [t.detach().clone().requires_grad_(True) for t in (qf, kf, V, gmax)]
    O, _ = attention(*leaves, ptr, H, Nmax, form)
    return torch.autograd.grad(O, leaves, gO)
