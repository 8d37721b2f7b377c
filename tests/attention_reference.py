"""Float64 restatement of the softmax attention stages (csrc/attention.cu, csrc/attention_tc.cu) and a numpy replica of
their dropout stream, for the stage tests.

  * attention(): dense per-graph softmax(q k^T / sqrt(hd) + bias) v in float64, each graph's rows attending to its own
    rows only (to_dense_batch -> nn.MultiheadAttention with a key padding mask), with an optional explicit keep mask on
    the probabilities as nn.MultiheadAttention applies its dropout: the softmax weights are dropped and scaled by
    1 / (1 - p), the denominators are not.  Returns O and the log-sum-exp of the undropped scores; the backward is
    autograd of it.
  * philox4x32_10(): Philox4x32-10 as csrc/common.cuh states it, vectorised over numpy uint64 arrays.
  * attention_keep(): the kernels' keep decision of (query i, key jl of its graph, head h): the Philox draw at key
    = seed, counter hi = offset + 16 + h (GPS_SITE_ATTN_P + head), counter lo = (i << 20) | (jl >> 2), component
    jl & 3; keep iff bits >= uint32(float32(p) * 2^32).
  * fwd_bounds() / bwd_bounds(): per-element error bounds of the kernels' fp32 arithmetic, stated from the unit
    roundoff u = 2^-24, the dot-product length hd, the key count n of the row's graph, the score magnitudes and, for
    the tensor-core forward, the bf16 operand splits.
"""
import numpy as np
import torch

SITE_ATTN_P = 16
U32 = np.uint64(0xFFFFFFFF)
U = 2.0 ** -24            # fp32 unit roundoff
# relative error of one product term a * b whose operands went through the wgmma operand planes: fp32-grade
# (hi*hi + hi*lo + lo*hi of 8-bit bf16 halves: each operand kept to 2^-17, the dropped lo*lo below that) and bf16
# (one round-to-nearest bf16 per operand)
U_TERM = {0: 3 * 2.0 ** -16, 1: 2 * 2.0 ** -8}


# ------------------------------------------------------------------------------------------------ Philox4x32-10
def philox4x32_10(key, ctr_hi, ctr_lo):
    """Philox4x32-10 of counter (ctr_lo low word, ctr_lo high word, ctr_hi low word, ctr_hi high word) under key
    (low word, high word); arguments broadcast.  Returns uint32 [..., 4]."""
    key, ctr_hi, ctr_lo = (np.asarray(x, dtype=np.uint64) for x in (key, ctr_hi, ctr_lo))
    key, ctr_hi, ctr_lo = np.broadcast_arrays(key, ctr_hi, ctr_lo)
    c0, c1 = ctr_lo & U32, ctr_lo >> np.uint64(32)
    c2, c3 = ctr_hi & U32, ctr_hi >> np.uint64(32)
    k0, k1 = key & U32, key >> np.uint64(32)
    M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
    for _ in range(10):
        p0, p1 = M0 * c0, M1 * c2                 # 32 x 32 -> 64-bit products: exact in uint64
        hi0, lo0 = p0 >> np.uint64(32), p0 & U32
        hi1, lo1 = p1 >> np.uint64(32), p1 & U32
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + W0) & U32, (k1 + W1) & U32
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.uint32)


def keep_threshold(p):
    """The kernels' keep threshold: uint32(min(float32(p) * 2^32, 2^32 - 1)) in float32 arithmetic."""
    x = float(np.float32(p)) * 2.0 ** 32         # exact: a power-of-two scaling of a float32
    return min(int(x), 0xFFFFFFFF)


def attention_keep(seed, offset, p, rows, n, h):
    """bool [len(rows), n]: the keep decision of query rows `rows` (global node indices) against the n keys of their
    graph (local indices 0..n-1), head h, at dropout offset `offset` (the host offset plus the device one)."""
    rows = np.asarray(rows, dtype=np.uint64)
    if n == 0 or len(rows) == 0:
        return np.ones((len(rows), n), dtype=bool)
    quads = np.arange((n + 3) // 4, dtype=np.uint64)
    lo = (rows[:, None] << np.uint64(20)) | quads[None, :]
    bits = philox4x32_10(np.uint64(seed), np.uint64(offset + SITE_ATTN_P + h), lo)   # [rows, quads, 4]
    return bits.reshape(len(rows), -1)[:, :n] >= np.uint32(keep_threshold(p))


def keep_masks(ptr, H, p, seed, offset, device="cpu"):
    """Per graph, bool [H, n, n] keep masks of the attention probabilities (None for p == 0: nothing dropped)."""
    if p == 0:
        return None
    out = []
    for g in range(len(ptr) - 1):
        s, e = int(ptr[g]), int(ptr[g + 1])
        rows = np.arange(s, e)
        out.append(torch.from_numpy(np.stack([attention_keep(seed, offset, p, rows, e - s, h) for h in range(H)]))
                   .to(device))
    return out


def dropout_mask(rows, cols, p, seed, offset, site):
    """gps_dropout_mask: float 1 / 0 [rows, cols], four consecutive flat elements per Philox draw at counter
    (offset + site, flat index / 4)."""
    n4 = rows * cols // 4
    bits = philox4x32_10(np.uint64(seed), np.uint64(offset + site), np.arange(n4, dtype=np.uint64)).reshape(rows, cols)
    return (bits >= np.uint32(keep_threshold(p))).astype(np.float32)


# ------------------------------------------------------------------------------------------------ float64 attention
def _graphs(ptr):
    for g in range(len(ptr) - 1):
        s, e = int(ptr[g]), int(ptr[g + 1])
        if e > s:
            yield g, s, e


def _heads(t, s, e, H, hd):
    return t[s:e].reshape(e - s, H, hd).transpose(0, 1)   # [H, n, hd]


def attention(Q, K, V, ptr, H, hd, bias=None, keep=None, p=0.0):
    """Float64 dense per-graph attention.  Q, K, V [N, H*hd]; bias [B*H, nmax, nmax] or None; keep a list of per-graph
    bool [H, n, n] or None.  Returns O [N, H*hd] and lse [N, H] (of the undropped, biased scores)."""
    N, D = Q.shape[0], H * hd
    O = Q.new_zeros(N, D)
    lse = Q.new_zeros(N, H)
    outs, lses, idx = [], [], []
    for g, s, e in _graphs(ptr):
        n = e - s
        q, k, v = (_heads(t, s, e, H, hd) for t in (Q, K, V))
        sc = q @ k.transpose(1, 2) / hd ** 0.5
        if bias is not None:
            sc = sc + bias[g * H:(g + 1) * H, :n, :n]
        w = torch.softmax(sc, -1)
        if keep is not None:
            w = w * keep[g].to(w.dtype) / (1.0 - p)
        outs.append((w @ v).transpose(0, 1).reshape(n, D))
        lses.append(torch.logsumexp(sc, -1).transpose(0, 1))
        idx.append(torch.arange(s, e, device=Q.device))
    if idx:
        idx = torch.cat(idx)
        O = O.index_copy(0, idx, torch.cat(outs))
        lse = lse.index_copy(0, idx, torch.cat(lses))
    return O, lse


def padded_planes(QKV, H, hd, extra=0):
    """[N, 3*H*hd] fp32 -> bf16 hi / lo planes [2, N, 3*H*hd_pad + extra] (hd_pad = hd rounded up to 16) in the
    per-head padded layout the wgmma attention reads, column (which * H + h) * hd_pad + k: pad columns zero, the extra
    pitch columns NaN (never read).  Returns the planes and their pitch."""
    N = QKV.shape[0]
    hp = (hd + 15) // 16 * 16
    x = torch.zeros(N, 3 * H, hp, device=QKV.device)
    x[:, :, :hd] = QKV.reshape(N, 3 * H, hd)
    x = x.reshape(N, 3 * H * hp)
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    ld = 3 * H * hp + extra
    buf = torch.full((2, N, ld), float("nan"), dtype=torch.bfloat16, device=QKV.device)
    buf[0, :, :3 * H * hp] = hi
    buf[1, :, :3 * H * hp] = lo
    return buf, ld


# ------------------------------------------------------------------------------------------------ error bounds
def _stats(Q, K, V, ptr, H, hd, bias, keep, p, g, s, e):
    """Per graph [H, n, n]: scores, probabilities, dropped probabilities, |q| |k| dot magnitudes."""
    n = e - s
    q, k = _heads(Q, s, e, H, hd), _heads(K, s, e, H, hd)
    scale = hd ** -0.5
    sc = q @ k.transpose(1, 2) * scale
    a = q.abs() @ k.abs().transpose(1, 2) * scale
    if bias is not None:
        b = bias[g * H:(g + 1) * H, :n, :n]
        sc, a = sc + b, a + b.abs()
    P = torch.softmax(sc, -1)
    Pd = P * keep[g].to(P.dtype) / (1.0 - p) if keep is not None else P
    return sc, a, P, Pd


def fwd_bounds(Q, K, V, ptr, H, hd, bias=None, keep=None, p=0.0, tc_precision=None):
    """Per-element bounds on |O - O_ref| [N, D] and |lse - lse_ref| [N, H] of the fp32 forward (CUDA core:
    tc_precision None; wgmma: 0 = fp32-grade, 1 = bf16).  Inputs float64 (the values the kernel read).

    e_ij, the relative error of one probability, is the score's error (fp32 dot of hd terms, or the operand splits
    on the tensor cores, times the |q||k| magnitude a_ij) plus the exp argument's rounding; E_i adds the online max
    rescales (their arguments telescope to at most twice the largest |score|).  O sums n dropped-probability-weighted
    rows in fp32 and divides by l, itself an n-term sum."""
    N, D = Q.shape[0], H * hd
    bO = Q.new_zeros(N, D)
    blse = Q.new_zeros(N, H)
    u_dot = 0.0 if tc_precision is None else U_TERM[tc_precision]
    u_pv = 0.0 if tc_precision is None else U_TERM[tc_precision]
    for g, s, e in _graphs(ptr):
        n = e - s
        sc, a, P, Pd = _stats(Q, K, V, ptr, H, hd, bias, keep, p, g, s, e)
        m = sc.max(-1, keepdim=True).values
        eij = (u_dot + (hd + 4) * U) * a + U * ((sc - m).abs() + 16)
        Ei = U * (2 * sc.abs().amax(-1, keepdim=True) + 4 * n)
        rel_l = (P * eij).sum(-1, keepdim=True) + Ei + (n + 2) * U          # [H, n, 1]
        v = _heads(V, s, e, H, hd).abs()
        o = (Pd @ _heads(V, s, e, H, hd)).abs()
        term = (Pd * (eij + Ei + u_pv + (n + 2) * U)) @ v + o * rel_l       # [H, n, hd]
        bO[s:e] = 2 * term.transpose(0, 1).reshape(n, D)
        lse = torch.logsumexp(sc, -1, keepdim=True)
        bl = rel_l + 3 * U * (m.abs() + (lse - m).abs()) + 2.0 ** -21
        blse[s:e] = 2 * bl.squeeze(-1).transpose(0, 1)
    return bO, blse


def bwd_bounds(Q, K, V, dO, ptr, H, hd, bias=None, keep=None, p=0.0, O_err=None, lse_err=None):
    """Per-element bounds on |dQ|, |dK|, |dV| errors [N, D] (and |grad_bias| errors [B*H, nmax, nmax] when bias is
    given: None otherwise) of the fp32 backward fed O and lse that differ from the float64 ones by at most O_err
    [N, D] and lse_err [N, H] (None: the fp32 rounding of exact values).

    p_ij = exp(s_ij - lse_i) carries the score error, the lse input's error and the exp rounding (e_ij); dP_ij =
    dO_i . V_j and delta_i = dO_i . O_i are hd-term fp32 dots (delta also carries O's error); dS = P (dP k - delta);
    dQ, dK, dV sum n terms each."""
    N, D = Q.shape[0], H * hd
    bq, bk, bv = (Q.new_zeros(N, D) for _ in range(3))
    gb = None if bias is None else torch.zeros_like(bias)
    scale = hd ** -0.5
    for g, s, e in _graphs(ptr):
        n = e - s
        sc, a, P, Pd = _stats(Q, K, V, ptr, H, hd, bias, keep, p, g, s, e)
        lse = torch.logsumexp(sc, -1, keepdim=True)
        le = U * lse.abs() if lse_err is None else lse_err[s:e].transpose(0, 1).unsqueeze(-1) + U * lse.abs()
        eij = (hd + 4) * U * a + U * (sc.abs() + lse.abs() + 16) + le
        q, k, v, go = (_heads(t, s, e, H, hd) for t in (Q, K, V, dO))
        o = P.detach() @ v if keep is None else Pd @ v
        oe = U * o.abs() if O_err is None else _heads(O_err, s, e, H, hd) + U * o.abs()
        ks = keep[g].to(P.dtype) / (1.0 - p) if keep is not None else torch.ones_like(P)
        dP = go @ v.transpose(1, 2)
        bdp = (hd + 2) * U * (go.abs() @ v.abs().transpose(1, 2))
        delta = (go * o).sum(-1, keepdim=True)
        bdl = (hd + 8) * U * (go.abs() * o.abs()).sum(-1, keepdim=True) + (go.abs() * oe).sum(-1, keepdim=True)
        dS = P * (dP * ks - delta)
        bds = P * (eij * (dP * ks - delta).abs() + bdp * ks + bdl + 2 * U * ((dP * ks).abs() + delta.abs()))
        acc = (n + 2) * U
        bq[s:e] = 2 * (scale * ((bds + dS.abs() * acc) @ k.abs())).transpose(0, 1).reshape(n, D)
        bk[s:e] = 2 * (scale * ((bds + dS.abs() * acc).transpose(1, 2) @ q.abs())).transpose(0, 1).reshape(n, D)
        bv[s:e] = 2 * ((Pd * (eij + acc)).transpose(1, 2) @ go.abs()).transpose(0, 1).reshape(n, D)
        if gb is not None:
            gb[g * H:(g + 1) * H, :n, :n] = 2 * bds
    return bq, bk, bv, gb
