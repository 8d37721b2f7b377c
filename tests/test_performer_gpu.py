"""GPU: every Performer kernel of csrc/performer.cu and csrc/performer_quad.cu, called through its stage entry point,
against the float64 stage references of tests/performer_reference.py: the C4 (pcqm4m-medium-performer, H = 16), zinc
and code2 (H = 4) shapes, a MalNet-like batch of two graphs of thousands of nodes, the padding extremes (one 200-node
graph among graphs of 1-3 nodes; equal sizes, so no padded rows; B = 1; empty graphs between non-empty ones; single
nodes), feature widths m = 257, 266, 272, both attention forms on every batch, and hand-built dd cases: a key max that
comes from the padded rows, a key max of -0.0 in a graph without padding, and exact ties.

Every output buffer starts as NaN, and the feature-padding columns m..271 of the dd inputs start as NaN (or +inf, which
a max would not skip): they must come out 0 and never be read.  The upstream gradients g_fq, g_fk and of gmax are drawn
at random, so the arg-max terms of the stabilisers are O(1) instead of hidden by the eps-cancellation.  Bounds are
elementwise, from the fp64 reference, with no relative-L2 fallback:
  * feature maps: the roundings of diag and of dd - diag - max, and 2 + 1.2 |x| ulps for __expf(x);
  * sums over keys and features: gamma_K times the same sums evaluated on |inputs| (K = the longest chain of roundings),
    with the reciprocal's derivative taken positive, plus the relative errors of the denominator and of k'_pad;
  * arg-max indices, gmax, and the zeros in the padding: exact.
Two runs of each backward give the same bits.  The worst error as a fraction of its bound is printed (pytest -s)."""
import ctypes as C

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import make_batch
from graphgps_b200.graph import GraphStructure
from oracle.gps_oracle import gaussian_orthogonal_random_matrix
import performer_reference as R
from util import _nan, _stream

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F64 = torch.float64
U = 2.0 ** -24
MP, DH = 272, 64
DN = DH ** -0.25
INT_MAX = 2 ** 31 - 1
WORST = {}


def gamma(k):
    return k * U / (1 - k * U)


def check(name, got, ref, bound):
    got, ref = got.double(), ref.double()
    assert not bool(torch.isnan(got).any()), f"{name}: NaN in the output (an element never written)"
    err = (got - ref).abs()
    frac = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
    WORST[name] = max(WORST.get(name, 0.0), frac)
    assert frac <= 1.0, f"{name}: error {frac:.3g} x its bound (max err {float(err.max()):.3g})"


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):
        print(f"worst error / bound  {k:36s} {WORST[k]:.3e}")


def _sizes(shape, seed=2):
    ptr = make_batch(shape, seed=seed, dim=8).ptr
    return (ptr[1:] - ptr[:-1]).tolist()


# name -> (graph sizes, H)
SHAPES = {
    "c4": (lambda: _sizes("pcqm4m-medium-performer"), 16),
    "zinc": (lambda: _sizes("zinc-gatedgcn"), 4),
    "code2": (lambda: _sizes("code2"), 4),
    "malnet": (lambda: [4100, 2500], 1),
    "pad200": (lambda: [200] + [1 + k % 3 for k in range(45)], 2),
    "equal": (lambda: [13] * 24, 4),           # no padded rows: gmax starts at -inf; N = 312, not a multiple of 16
    "equal16": (lambda: [16] * 8, 1),          # N = 128
    "b1": (lambda: [37], 16),
    "empty": (lambda: [5, 0, 3, 0, 0, 8, 1], 2),
    "single": (lambda: [1] * 20, 4),
}
_GRAPHS = {}


class Batch:
    """the graph structure of a batch of graphs of the given sizes (no edges: the Performer reads graph_ptr only)"""

    def __init__(self, sizes, H):
        self.sizes, self.H = sizes, H
        self.ptr = torch.tensor([0] + list(sizes), device=DEV).cumsum(0)
        self.B, self.N, self.Nmax = len(sizes), int(self.ptr[-1]), max(sizes)
        batch = torch.repeat_interleave(torch.arange(self.B, device=DEV), torch.tensor(sizes, device=DEV))
        self.gs = GraphStructure(torch.zeros(2, 0, dtype=torch.int64, device=DEV), batch, self.B)
        self.batch, self.pos, _, _ = R.layout(self.ptr)
        self.row_graph = self.batch.repeat_interleave(H)                       # graph of row r = n H + h
        self.row_bh = self.row_graph * H + torch.arange(self.N * H, device=DEV) % H
        self.npad = (self.Nmax - (self.ptr[1:] - self.ptr[:-1])).to(F64)

    @property
    def desc(self):
        return C.byref(self.gs.desc)

    def seg_sum(self, rows):
        """[N*H] -> [B*H] per (graph, head)"""
        return torch.zeros(self.B * self.H, dtype=F64, device=DEV).index_add_(0, self.row_bh, rows.double())


def _batch(name):
    if name not in _GRAPHS:
        f, H = SHAPES[name]
        _GRAPHS[name] = Batch(f(), H)
    return _GRAPHS[name]


def _projection(m, seed=0):
    return gaussian_orthogonal_random_matrix(m, DH, generator=torch.Generator().manual_seed(seed)).to(DEV)


def _inputs(b, m, seed=0, pad="nan"):
    """Q, K [N*H, 64] and dd = (x 64^-1/4) P^T rounded to fp32 in [N*H, 272] buffers with `pad` in columns m.."""
    g = torch.Generator().manual_seed(seed)
    NH = b.N * b.H
    Q, K = ((torch.randn(NH, DH, generator=g) * 0.7).to(DEV) for _ in range(2))
    P = _projection(m, seed)
    dd = []
    for x in (Q, K):
        t = torch.full((NH, MP), float(pad), device=DEV)
        t[:, :m] = ((x.double() * DN) @ P.double().t()).float()
        dd.append(t)
    return Q, K, dd[0], dd[1], P


def _prep(b, m, P):
    lib = _lib.load()
    Pn, nmax = _nan(MP, DH), torch.full((1,), -1, dtype=torch.int32, device=DEV)
    gmax, argk = _nan(b.B * b.H), torch.full((b.B * b.H,), -1, dtype=torch.int32, device=DEV)
    _lib.check(lib.gps_performer_prep(b.desc, b.H, DH, m, P.data_ptr(), Pn.data_ptr(), nmax.data_ptr(), gmax.data_ptr(),
                                      argk.data_ptr(), _stream()), "performer prep")
    return Pn, nmax, gmax, argk


def _features_fwd(b, m, Q, K, ddq, ddk, P):
    lib = _lib.load()
    Pn, nmax, gmax, argk = _prep(b, m, P)
    fq, fk = ddq.clone(), ddk.clone()
    argq = torch.full((b.N * b.H,), -1, dtype=torch.int32, device=DEV)
    _lib.check(lib.gps_performer_features_forward(b.desc, b.H, DH, m, fq.data_ptr(), fk.data_ptr(), Q.data_ptr(),
                                                  K.data_ptr(), gmax.data_ptr(), argq.data_ptr(), argk.data_ptr(),
                                                  _stream()), "performer features forward")
    return dict(fq=fq, fk=fk, gmax=gmax, argq=argq, argk=argk, nmax=nmax)


def _feature_bound(b, m, Q, K, ddq, ddk, stab_q, stab_k):
    """elementwise bound on q', k' [N*H, m] computed from fp32 inputs: the roundings of diag (gamma_65 + 5u), of the
    two subtractions, __expf (2 + 1.2 |x| ulps), + eps, and ratio (3u)"""
    ratio = m ** -0.5
    out = []
    for x, dd, stab in ((Q, ddq, stab_q), (K, ddk, stab_k)):
        diag = (x.double() ** 2).sum(-1, keepdim=True) / 2.0 * DH ** -0.5
        d64 = dd[:, :m].double()
        arg = d64 - diag - stab.unsqueeze(1)
        dx = (gamma(65) + 5 * U) * diag + U * ((d64 - diag).abs() + arg.abs())
        e = torch.exp(arg)
        f = ratio * (e + R.EPS)
        out.append(ratio * e * (dx + (3 + 1.2 * arg.abs()) * U) + 4 * U * f)
    return out


def _ref_argk(b, ddk, gmax_ref, m):
    """lowest flat index r * 272 + j of an element equal to its (graph, head)'s max; INT_MAX when none is"""
    eq = ddk[:, :m].double() == gmax_ref[b.row_bh].unsqueeze(1)
    r, j = eq.nonzero(as_tuple=True)
    out = torch.full((b.B * b.H,), INT_MAX, dtype=torch.int64, device=DEV)
    return out.scatter_reduce_(0, b.row_bh[r], r * MP + j, "amin")


FEATURE_CASES = [(s, 266) for s in SHAPES] + [(s, m) for s in ("c4", "pad200", "empty", "equal16") for m in (257, 272)]


def _ids(c):
    return f"{c[0]}-m{c[1]}"


def test_prep():
    for name in ("c4", "empty", "equal", "b1"):
        b = _batch(name)
        for m in (257, 266, 272):
            P = _projection(m)
            Pn, nmax, gmax, argk = _prep(b, m, P)
            dn = torch.tensor(64.0).pow(-0.25).float().item()
            want = torch.zeros(MP, DH, device=DEV)
            want[:m] = P * dn
            assert float((Pn - want).abs().max()) <= 2 * U * float(want.abs().max()), (name, m)
            assert torch.equal(Pn[m:], torch.zeros(MP - m, DH, device=DEV))
            assert int(nmax) == b.Nmax
            padded = (b.npad > 0).repeat_interleave(b.H)
            assert torch.equal(gmax, torch.where(padded, 0.0, float("-inf")).float())
            assert bool((argk == INT_MAX).all())


@pytest.mark.parametrize("pad", ["nan", "inf"])
@pytest.mark.parametrize("case", FEATURE_CASES, ids=_ids)
def test_features_forward(case, pad):
    name, m = case
    b = _batch(name)
    Q, K, ddq, ddk, P = _inputs(b, m, seed=1, pad=pad)
    got = _features_fwd(b, m, Q, K, ddq, ddk, P)
    fq, fk, gmax = R.features(ddq.double(), ddk.double(), Q.double(), K.double(), b.ptr, b.H, m, ties="first")
    _check_features(b, m, Q, K, ddq, ddk, got, fq, fk, gmax, "features_fwd")


def _check_features(b, m, Q, K, ddq, ddk, got, fq, fk, gmax, tag):
    assert torch.equal(got["gmax"].double(), gmax), f"{tag}: gmax"
    assert torch.equal(got["argq"].long(), ddq[:, :m].argmax(1)), f"{tag}: argq"
    assert torch.equal(got["argk"].long(), _ref_argk(b, ddk, gmax, m)), f"{tag}: argk"
    bq, bk = _feature_bound(b, m, Q, K, ddq, ddk, ddq[:, :m].double().amax(1), gmax[b.row_bh])
    check(f"{tag} q'", got["fq"][:, :m], fq, bq)
    check(f"{tag} k'", got["fk"][:, :m], fk, bk)
    for t in ("fq", "fk"):
        assert torch.equal(got[t][:, m:], torch.zeros_like(got[t][:, m:])), f"{tag}: {t} padding columns not zero"


def _features_bwd(b, m, form, fwd, Q, K, g_fq, g_fk, up, pad="nan"):
    """up: ggmax [B*H] (form 0) or gmrow [N*H] (form 1), the upstream gradient of gmax"""
    lib = _lib.load()
    gq, gk = g_fq.clone(), g_fk.clone()
    gq[:, m:], gk[:, m:] = float(pad), float(pad)
    gQ, gK = _nan(*Q.shape), _nan(*K.shape)
    ggmax = up.clone() if form == 0 else None
    gmrow = up.clone() if form == 1 else _nan(b.N * b.H)
    _lib.check(lib.gps_performer_features_backward(b.desc, b.H, DH, m, form, gq.data_ptr(), gk.data_ptr(),
                                                   fwd["fq"].data_ptr(), fwd["fk"].data_ptr(), Q.data_ptr(),
                                                   K.data_ptr(), gQ.data_ptr(), gK.data_ptr(), fwd["argq"].data_ptr(),
                                                   fwd["argk"].data_ptr(), _lib.ptr(ggmax), gmrow.data_ptr(),
                                                   _stream()), "performer features backward")
    return gq, gk, gQ, gK


def _features_bwd_bound(b, m, Q, K, fwd, fq, fk, bq, bk, g_fq, g_fk, g_gmax_terms):
    """bounds on g_dd_q, g_dd_k, gQ, gK.  t_j = g_j ratio (f_j / ratio - eps) from the fp32 f (error bf):
    |dt| <= |g| (bf + 4u f) + 2u |t|;  S = sum_j t_j: sum |dt| + gamma_m sum |t|;  the arg-max element takes -S; the
    key arg-max also the (graph, head) total sum_r (-S_r) + upstream: sum |dS_r| + gamma_(n+2) sum |terms|"""
    ratio = m ** -0.5
    out = []
    for x, f, bf, g in ((Q, fq, bq, g_fq), (K, fk, bk, g_fk)):
        g = g[:, :m].double()
        t = g * (f - ratio * R.EPS)
        dt = g.abs() * (bf + 4 * U * f) + 2 * U * t.abs()
        S = t.sum(1)
        dS = dt.sum(1) + gamma(m) * t.abs().sum(1)
        out.append([t, dt, dS, S, x])
    # queries: -S at argq (one more rounding)
    tq, dtq, dSq, Sq, _ = out[0]
    bq_dd = dtq.clone()
    ar = torch.arange(b.N * b.H, device=DEV)
    aq = fwd["argq"].long()
    bq_dd[ar, aq] += dSq + U * (Sq.abs() + tq[ar, aq].abs())
    # keys: the (graph, head) total sum_r (-S_r) (+ pad terms) + upstream, added at argk
    tk, dtk, dSk, Sk, _ = out[1]
    bk_dd = dtk.clone()
    n = b.seg_sum(torch.ones_like(Sk))
    tot_b = b.seg_sum(dSk) + gamma(n + 3) * (b.seg_sum(Sk.abs()) + g_gmax_terms)
    ak = fwd["argk"].long()
    has = ak != INT_MAX
    rk, jk = ak[has] // MP, ak[has] % MP
    bk_dd[rk, jk] += tot_b[has] + U * tk[rk, jk].abs()
    gb = [DH ** -0.5 * x.double().abs() * (dS + 4 * U * S.abs()).unsqueeze(1) for (_, _, dS, S, x) in out]
    return bq_dd, bk_dd, gb[0], gb[1]


def _random_grads(b, m, seed):
    g = torch.Generator().manual_seed(seed)
    NH = b.N * b.H
    g_fq, g_fk = (torch.randn(NH, MP, generator=g).to(DEV) for _ in range(2))
    rows = torch.randn(NH, generator=g).to(DEV)
    return g_fq, g_fk, rows


@pytest.mark.parametrize("form", [0, 1])
@pytest.mark.parametrize("case", FEATURE_CASES, ids=_ids)
def test_features_backward(case, form):
    name, m = case
    b = _batch(name)
    Q, K, ddq, ddk, P = _inputs(b, m, seed=2)
    fwd = _features_fwd(b, m, Q, K, ddq, ddk, P)
    g_fq, g_fk, rows = _random_grads(b, m, seed=3)
    up = rows[:b.B * b.H].contiguous() if form == 0 else rows
    g_gmax = up.double() if form == 0 else b.seg_sum(rows)
    gq, gk, gQ, gK = _features_bwd(b, m, form, fwd, Q, K, g_fq, g_fk, up)
    _check_features_bwd(b, m, Q, K, ddq, ddk, fwd, g_fq, g_fk, up, form, g_gmax, gq, gk, gQ, gK, "features_bwd")


def _check_features_bwd(b, m, Q, K, ddq, ddk, fwd, g_fq, g_fk, up, form, g_gmax, gq, gk, gQ, gK, tag):
    args = (ddq.double(), ddk.double(), Q.double(), K.double(), b.ptr, b.H, m)
    fq, fk, _ = R.features(*args, ties="first")
    ref = R.features_backward(*args, g_fq.double(), g_fk.double(), g_gmax, ties="first")
    gm = fwd["gmax"].double()
    bq, bk = _feature_bound(b, m, Q, K, ddq, ddk, ddq[:, :m].double().amax(1), gm[b.row_bh])
    up_abs = up.double().abs() if form == 0 else b.seg_sum(up.abs())
    bounds = _features_bwd_bound(b, m, Q, K, fwd, fwd["fq"][:, :m].double(), fwd["fk"][:, :m].double(), bq, bk,
                                 g_fq, g_fk, up_abs)
    for nm, got, want, bd in zip(("g_dd_q", "g_dd_k", "g_Q", "g_K"), (gq[:, :m], gk[:, :m], gQ, gK), ref, bounds):
        check(f"{tag} {nm}", got, want, bd)
    for t in (gq, gk):
        assert torch.equal(t[:, m:], torch.zeros_like(t[:, m:])), f"{tag}: padding columns of g_dd not zero"


# ------------------------------------------------------------------------------------------------ attention
class _PosRecip(torch.autograd.Function):
    """1 / x with the derivative taken positive: evaluated on |inputs|, autograd then sums |each term| of the backward"""

    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return 1.0 / x

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return g / x ** 2


def _attention_abs(b, qf, kf, Vabs, t, form):
    """R.attention on |V| with kpad = ratio (exp(t) + eps) npad, t = -gmax, and a positive reciprocal derivative"""
    m = qf.shape[1]
    kpad = m ** -0.5 * (torch.exp(t.view(b.B, b.H)) + R.EPS) * b.npad.unsqueeze(1)
    qd, kd, vd = (R.to_dense(x, b.ptr, b.H) for x in (qf, kf, Vabs))
    if form == 0:
        ksum = kd.sum(2) + kpad.unsqueeze(-1)
        den = torch.einsum("bhnj,bhj->bhn", qd, ksum)
        num = torch.einsum("bhnj,bhje->bhne", qd, torch.einsum("bhnj,bhne->bhje", kd, vd))
    else:
        s = torch.einsum("bhij,bhkj->bhik", qd, kd)
        den = s.sum(-1) + kpad.unsqueeze(-1) * qd.sum(-1)
        num = torch.einsum("bhik,bhke->bhie", s, vd)
    real = R.to_dense(torch.ones(qf.shape[0], 1, dtype=F64, device=DEV), b.ptr, b.H)[..., 0]
    O = num * _PosRecip.apply(den + (1 - real)).unsqueeze(-1)
    return R.to_packed(O, b.ptr)


def _attn_inputs(b, m, seed):
    """q', k' from the fp64 feature maps of realistic dd, rounded to fp32 with zero padding columns; V; gmax"""
    Q, K, ddq, ddk, _ = _inputs(b, m, seed=seed)
    fq, fk, gmax = R.features(ddq.double(), ddk.double(), Q.double(), K.double(), b.ptr, b.H, m)
    qf, kf = torch.zeros(b.N * b.H, MP, device=DEV), torch.zeros(b.N * b.H, MP, device=DEV)
    qf[:, :m], kf[:, :m] = fq.float(), fk.float()
    V = torch.randn(b.N * b.H, DH, generator=torch.Generator().manual_seed(seed + 7)).to(DEV)
    return qf, kf, V, gmax.float()


def _eps(b, m, gmax):
    """relative errors: K roundings on the longest chain, k'_pad (__expf, + eps, ratio, npad), the denominator, O"""
    K = m + b.Nmax + 16
    e_kpad = (6 + 1.2 * float(gmax.abs().max() if gmax.numel() else 0)) * U
    e_den = gamma(K) + e_kpad
    e_O = gamma(K) + e_den + U
    e_bwd = gamma(K + DH + 16) + 3 * e_den + 2 * e_O + 2 * e_kpad
    return e_den, e_O, e_bwd


def _attn_fwd(b, m, form, nmax, qf, kf, V, gmax):
    lib = _lib.load()
    O, den = _nan(b.N * b.H, DH), _nan(b.N * b.H)
    _lib.check(lib.gps_performer_attention_forward(b.desc, b.H, DH, m, form, nmax.data_ptr(), qf.data_ptr(),
                                                   kf.data_ptr(), V.data_ptr(), gmax.data_ptr(), O.data_ptr(),
                                                   den.data_ptr() if form == 1 else 0, _stream()), "attention fwd")
    return O, den


def _nmax(b):
    return torch.tensor([b.Nmax], dtype=torch.int32, device=DEV)


ATTN_CASES = [(s, 266) for s in SHAPES] + [(s, m) for s in ("c4", "pad200", "empty") for m in (257, 272)]


@pytest.mark.parametrize("form", [0, 1])
@pytest.mark.parametrize("case", ATTN_CASES, ids=_ids)
def test_attention_forward(case, form):
    name, m = case
    b = _batch(name)
    qf, kf, V, gmax = _attn_inputs(b, m, seed=4)
    O, den = _attn_fwd(b, m, form, _nmax(b), qf, kf, V, gmax)
    args = (qf[:, :m].double(), kf[:, :m].double(), V.double(), gmax.double())
    O_ref, den_ref = R.attention(*args, b.ptr, b.H, b.Nmax, form)
    e_den, e_O, _ = _eps(b, m, gmax)
    O_abs = _attention_abs(b, args[0], args[1], args[2].abs(), -args[3], form)
    check(f"attn_fwd form{form} O", O, O_ref, e_O * O_abs)
    if form == 1:
        check("attn_fwd form1 den", den, den_ref, e_den * den_ref)


def _attn_bwd(b, m, form, nmax, qf, kf, V, gmax, O, den, gO):
    lib = _lib.load()
    NH = b.N * b.H
    g_qf, g_kf, gV = _nan(NH, MP), _nan(NH, MP), _nan(NH, DH)
    gden, ggmax, gmrow = _nan(NH), _nan(b.B * b.H), _nan(NH)
    _lib.check(lib.gps_performer_attention_backward(b.desc, b.H, DH, m, form, nmax.data_ptr(), qf.data_ptr(),
                                                    kf.data_ptr(), V.data_ptr(), gmax.data_ptr(), O.data_ptr(),
                                                    den.data_ptr(), gO.data_ptr(), gden.data_ptr(), g_qf.data_ptr(),
                                                    g_kf.data_ptr(), gV.data_ptr(), ggmax.data_ptr(), gmrow.data_ptr(),
                                                    _stream()), "attention bwd")
    return g_qf, g_kf, gV, (ggmax if form == 0 else gmrow)


@pytest.mark.parametrize("form", [0, 1])
@pytest.mark.parametrize("case", ATTN_CASES, ids=_ids)
def test_attention_backward(case, form):
    name, m = case
    b = _batch(name)
    qf, kf, V, gmax = _attn_inputs(b, m, seed=5)
    nmax = _nmax(b)
    O, den = _attn_fwd(b, m, form, nmax, qf, kf, V, gmax)
    gO = torch.randn(b.N * b.H, DH, generator=torch.Generator().manual_seed(6)).to(DEV)
    g_qf, g_kf, gV, gg = _attn_bwd(b, m, form, nmax, qf, kf, V, gmax, O, den, gO)
    args = [qf[:, :m].double(), kf[:, :m].double(), V.double(), gmax.double()]
    ref = R.attention_backward(*args, b.ptr, b.H, b.Nmax, form, gO.double())
    _, _, e_bwd = _eps(b, m, gmax)
    leaves = [args[0].clone().requires_grad_(True), args[1].clone().requires_grad_(True),
              args[2].abs().requires_grad_(True), (-args[3]).requires_grad_(True)]
    ab = torch.autograd.grad(_attention_abs(b, *leaves, form), leaves, gO.double().abs())
    g_gmax = gg.double() if form == 0 else b.seg_sum(gg)
    for nm, got, want, a in zip(("g_qf", "g_kf", "gV", "g_gmax"), (g_qf[:, :m], g_kf[:, :m], gV, g_gmax), ref, ab):
        check(f"attn_bwd form{form} {nm}", got, want, e_bwd * a)
    for t in (g_qf, g_kf):
        assert torch.equal(t[:, m:], torch.zeros_like(t[:, m:])), "padding columns of g_qf / g_kf not zero"


# ------------------------------------------------------------------------------------------------ hand-built dd
def _hand_case(kind, b, m):
    Q, K, ddq, ddk, P = _inputs(b, m, seed=8, pad=0.0)      # padding 0, as the dd product writes it
    if kind == "pad_max":           # every real key dd < 0: the max of each padded graph is its padded rows' 0
        ddk[:, :m] = -ddk[:, :m].abs() - 0.25
    elif kind == "neg_zero":        # no padded rows, every dd <= 0, and the max is -0.0 (gmax starts at -inf)
        ddk[:, :m] = -ddk[:, :m].abs() - 0.25
        ddk[b.H + 1, 5] = -0.0      # node 1, head 1 (H > 1) of graph 0
        ddk[0, 3] = -0.0            # node 0, head 0
    elif kind == "ties":            # features 3 and 11 tie at the max of every row, as two equal rows of P would make them
        for t in (ddq, ddk):
            t[:, 11] = t[:, 3] = t[:, :m].amax(1) + 0.5
        ddk[0, 11] = ddk[0, 3] = float(ddk[:, :m].max()) + 1.0
        ddk[b.H] = ddk[0]           # node 1 duplicates node 0 (head 0): (graph 0, head 0) has four tied maxima
        K[b.H] = K[0]
    return Q, K, ddq, ddk, P


HAND = [("pad_max", "pad200"), ("pad_max", "empty"), ("neg_zero", "equal"), ("neg_zero", "b1"), ("ties", "c4"),
        ("ties", "equal16")]


@pytest.mark.parametrize("form", [0, 1])
@pytest.mark.parametrize("kind,name", HAND)
def test_hand_built_dd(kind, name, form):
    b = _batch(name)
    m = 266
    Q, K, ddq, ddk, P = _hand_case(kind, b, m)
    got = _features_fwd(b, m, Q, K, ddq, ddk, P)
    fq, fk, gmax = R.features(ddq.double(), ddk.double(), Q.double(), K.double(), b.ptr, b.H, m, ties="first")
    _check_features(b, m, Q, K, ddq, ddk, got, fq, fk, gmax, f"hand_{kind}")
    if kind == "pad_max":
        padded = (b.npad > 0).repeat_interleave(b.H)
        assert bool((got["argk"][padded] == INT_MAX).all()) and bool((got["gmax"][padded] == 0).all())
    if kind == "neg_zero":
        assert float(got["gmax"][0]) == 0.0 and int(got["argk"][0]) == 3
        assert float(got["gmax"][1]) == 0.0 and int(got["argk"][1]) == (b.H + 1) * MP + 5
    if kind == "ties":
        assert bool((got["argq"] == 3).all()) and int(got["argk"][0]) == 3
    g_fq, g_fk, rows = _random_grads(b, m, seed=9)
    up = rows[:b.B * b.H].contiguous() if form == 0 else rows
    g_gmax = up.double() if form == 0 else b.seg_sum(rows)
    gq, gk, gQ, gK = _features_bwd(b, m, form, got, Q, K, g_fq, g_fk, up, pad=0.0)
    _check_features_bwd(b, m, Q, K, ddq, ddk, got, g_fq, g_fk, up, form, g_gmax, gq, gk, gQ, gK, f"hand_{kind}")
    if kind == "ties":
        # torch.amax splits a tied max's gradient evenly; the kernels give all of it to the lowest index: the totals
        # agree and the reference's share of the higher index moves to the lower one
        split = R.features_backward(ddq.double(), ddk.double(), Q.double(), K.double(), b.ptr, b.H, m,
                                    g_fq.double(), g_fk.double(), g_gmax)
        tot = (gq[:, 3] + gq[:, 11]).double()
        check("hand_ties query total", tot, split[0][:, 3] + split[0][:, 11], 1e-5 * (1 + tot.abs()))
        ktot = (gk[0, 3] + gk[0, 11] + gk[b.H, 3] + gk[b.H, 11]).double()
        want = split[1][0, 3] + split[1][0, 11] + split[1][b.H, 3] + split[1][b.H, 11]
        check("hand_ties key total", ktot, want, 1e-5 * (1 + ktot.abs()))


def test_attention_with_padded_rows_dominating():
    """pad200: every small graph's denominator is mostly (200 - n) k'_pad"""
    b = _batch("pad200")
    qf, kf, _, gmax = _attn_inputs(b, 266, seed=4)
    kpad = 266 ** -0.5 * (torch.exp(-gmax.double().view(b.B, b.H)) + R.EPS) * b.npad.unsqueeze(1)
    ksum = torch.zeros(b.B * b.H, 266, dtype=F64, device=DEV).index_add_(0, b.row_bh, kf[:, :266].double()).sum(1)
    assert bool((266 * kpad.reshape(-1)[b.H:] > 5 * ksum[b.H:]).all())    # the premise the pad200 cases rely on


# ------------------------------------------------------------------------------------------------ reproducibility
@pytest.mark.parametrize("form", [0, 1])
@pytest.mark.parametrize("name", ["c4", "code2", "malnet", "pad200"])
def test_backward_is_bitwise_reproducible(name, form):
    b, m = _batch(name), 266
    Q, K, ddq, ddk, P = _inputs(b, m, seed=10)
    fwd = _features_fwd(b, m, Q, K, ddq, ddk, P)
    V = torch.randn(b.N * b.H, DH, generator=torch.Generator().manual_seed(11)).to(DEV)
    O, den = _attn_fwd(b, m, form, fwd["nmax"], fwd["fq"], fwd["fk"], V, fwd["gmax"])
    gO = torch.randn(b.N * b.H, DH, generator=torch.Generator().manual_seed(12)).to(DEV)

    def run():
        g_qf, g_kf, gV, gg = _attn_bwd(b, m, form, fwd["nmax"], fwd["fq"], fwd["fk"], V, fwd["gmax"], O, den, gO)
        gq, gk, gQ, gK = _features_bwd(b, m, form, fwd, Q, K, g_qf, g_kf, gg)
        return [gq, gk, gQ, gK, gV]

    r1, r2 = run(), run()
    for k, (x, y) in enumerate(zip(r1, r2)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), f"output {k} differs between two runs"


@pytest.mark.parametrize("shape,heads", [("pcqm4m-medium-performer", 16), ("code2", 4)])
def test_layer_backward_is_bitwise_reproducible(shape, heads):
    """a Performer layer without normalisation (no BatchNorm statistics atomics): two backward passes give the same
    bits for every gradient, in the pairwise form (C4: mean 14 nodes per graph) and the context form (code2: 125)"""
    torch.manual_seed(0)
    b = make_batch(shape, seed=1).to(DEV)
    d = b.x.shape[1]
    layer = graphgps_b200.GPSLayer(d, "None", "Performer", heads, batch_norm=False).to(DEV)
    ct = torch.randn(b.x.shape, generator=torch.Generator().manual_seed(2)).to(DEV)

    def run():
        layer.zero_grad(set_to_none=True)
        bb = b.clone()
        x_in = bb.x.requires_grad_(True)
        out = layer(bb)
        (out.x * ct).sum().backward()
        return [out.x.detach(), x_in.grad] + [p.grad for p in layer.parameters()]

    r1, r2 = run(), run()
    assert len(r1) == 2 + len(list(layer.parameters()))
    for k, (x, y) in enumerate(zip(r1, r2)):
        assert x is not None and torch.equal(x.view(torch.int32), y.view(torch.int32)), f"tensor {k} differs"
