"""GPU: the row-wise BatchNorm stages (csrc/elementwise.cu) and the dropout-gradient pass (k_dropmul, layer.cu) stage by
stage, through gps_rowwise_stage, which builds each BatchNorm view with the layers' own bn_view_at.

Exact cases.  z, mean, gamma, beta, residuals and gradients are small integers times 2^-3, the backward's invstd is a
power of two and the dropout probabilities 0.5 and 0.75 keep with scales 2 and 4 (x * s exact, so an FMA contraction of
x * s + r cannot change the bits).  Then every step must equal a float32 host replay bit for bit: the apply
(z - mean) * invstd, the fmaf with gamma and beta (replayed exactly by _fma32), ReLU, dropout, the residual, the planes,
both backward sums and the backward apply.  The training forward finalises mean / invstd from the producer's float64
sums with a double formula: save_mean / save_invstd must equal its float64 replay bit for bit (with the constants
(double)1e-5f and 0.1f), the running statistics must be within 1 ulp of a float32 replay (contraction may fuse) and
num_batches_tracked must go up by exactly 1 per BatchNorm per call.  GELU and p = 0.1 get stated per-element bounds.

Random cases at the layer's shapes compare with torch.nn.functional.batch_norm in float64 (training and eval) and the
composite R + mask * act(BN(z)) with its float64 autograd, within per-element bounds derived from the float32 chains
below.  Inputs keep column means within 4 standard deviations of zero: the variance is finalised as E[z^2] - mean^2 in
float64, whose relative error grows with K = (mean^2 + var) / var, and the bounds carry K (K <= 17 here).

Reproducibility.  Every partial a CTA adds to the float64 sums is a float32 value, and the float64 atomics add them in
any order.  The sum is exact, hence order-free, while the non-zero partials of a column span fewer than 29 binary orders
(24 bits each in 53), less the few bits the running total grows by; the random cases' partials are sums of same-signed
terms of similar size (positive outputs, gradients with a positive column mean), so they do, and two runs of each
must give the same bits.

Sentinels.  Outputs start as NaN inside wider buffers, planes as 0xFFFF, and every saved, running, gradient and sums
vector sits inside a guard region that must stay untouched."""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from graphgps_b200 import _lib
from util import _stream

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

OPS = _lib.ROWWISE
RELU, GELU = _lib.ACT["relu"], _lib.ACT["gelu"]
U = 2.0 ** -24                 # unit roundoff of float32
EPS32 = np.float32(1e-5)       # kBnEps
EPS64 = float(EPS32)           # (double)kBnEps, as the statistics finalisation adds it
MOM = np.float32(0.1)          # kBnMomentum
SEED, OFFSET, OFFSET_DEV = 0x5EED1234, 4096, 8192
SITE_GCN_X, SITE_GCN_E, SITE_LOCAL, SITE_FF2 = 1, 2, 3, 6
SITE_CG_X, SITE_CG_E = 15, 4095
G = 4                          # guard elements on each side of a vector (16 bytes: float4 alignment kept)
SENT16 = -1                    # 0xFFFF as int16
NUM_SMS = 132


# ---------------------------------------------------------------------------------------------------- geometry
def row_geom(rows, d, nstat):
    """(RY, CTAs) of elementwise.cu row_geom: a CTA is d/4 x RY threads, a thread strides over rows."""
    C4 = d // 4
    RY = 1 if C4 >= 256 else 256 // C4
    cap = NUM_SMS * 8
    if nstat > 0:
        RY = 1 if C4 >= 1024 else min(16, 1024 // C4)
        smem_cap = 48 * 1024 // (nstat * C4 * 16)
        # the shared-memory cap never binds for the one- and two-statistic ops: 1024 / C4 < 1536 / C4
        assert RY <= max(1, smem_cap)
        cap = NUM_SMS // 2
    blocks = min(cap, -(-max(rows, 1) // (RY * 4)))
    return RY, blocks


def stats_chain(rows, d):
    """Longest float32 addition chain of a column sum before the float64 atomics: the rows one thread walks, then the
    RY - 1 additions of the CTA's threads."""
    RY, blocks = row_geom(rows, d, 2)
    return -(-rows // (RY * blocks)) + RY - 1


# ---------------------------------------------------------------------------------------------------- buffers
def _ints(g, *shape, lo=-8, hi=8):
    return (torch.randint(lo, hi + 1, shape, generator=g).float() * 0.125).to(DEV)


class Guarded:
    """A device vector of n elements inside a sentinel guard of G elements on each side."""

    def __init__(self, n, dtype=torch.float32, init=None):
        self.buf = torch.full((n + 2 * G,), float("nan"), dtype=dtype, device=DEV)
        self.v = self.buf[G:G + n]
        if init is not None:
            self.v.copy_(init)

    def ptr(self):
        return self.v.data_ptr()

    def check(self, name):
        assert torch.isnan(self.buf[:G]).all() and torch.isnan(self.buf[-G:]).all(), f"{name} written outside [0, n)"


class Mat:
    """A [rows, d] device matrix of pitch ld (> d: NaN guard columns on the right) inside a NaN guard row block; or,
    ld = d, a contiguous one inside a flat guard."""

    def __init__(self, rows, d, ld=None, init=None):
        self.rows, self.d, self.ld = rows, d, ld or d
        self.buf = torch.full(((rows + 2) * self.ld,), float("nan"), device=DEV)
        self.v = self.buf[self.ld:self.ld + rows * self.ld].view(rows, self.ld)[:, :d]
        if init is not None:
            self.v.copy_(init)

    def ptr(self):
        return self.v.data_ptr()

    def check(self, name):
        full = self.buf.view(self.rows + 2, self.ld)
        assert torch.isnan(full[0]).all() and torch.isnan(full[-1]).all(), f"{name}: rows outside [0, rows) written"
        assert torch.isnan(full[1:-1, self.d:]).all(), f"{name}: columns past d written"


class PlanesBuf:
    """bf16 hi / lo planes of a [rows, d] output: pitch d + 8 (guard columns), a guard row, 0xFFFF sentinels."""

    def __init__(self, rows, d, lo=True):
        self.rows, self.d, self.ld, self.lo = rows, d, (d + 7) // 8 * 8 + 8, lo
        self.buf = torch.full((2, rows + 1, self.ld), SENT16, dtype=torch.int16, device=DEV)

    def struct(self):
        return _lib.GpsPlanes(self.buf[0].data_ptr(), self.buf[1].data_ptr() if self.lo else 0, self.ld)

    def check(self, v):
        """hi = bf16(v), lo = bf16(v - hi) (round to nearest even, as __floats2bfloat162_rn), nothing else touched."""
        rows, d = self.rows, self.d
        v = v.contiguous()
        hi = v.bfloat16()
        lo = (v - hi.float()).bfloat16()
        assert (self.buf[:, rows] == SENT16).all() and (self.buf[:, :, d:] == SENT16).all(), "planes written past [rows, d)"
        assert torch.equal(self.buf[0, :rows, :d], hi.view(torch.int16)), "hi plane differs from bf16(out)"
        if self.lo:
            assert torch.equal(self.buf[1, :rows, :d], lo.view(torch.int16)), "lo plane differs from bf16(out - hi)"
        else:
            assert (self.buf[1] == SENT16).all(), "lo plane written with lo = NULL"


class Bn:
    """One BatchNorm: gamma, beta, running statistics, num_batches_tracked, gradients, saved [mean | invstd] and float64
    sums, each inside its guard."""

    def __init__(self, d, gen, train, random=False):
        self.d, self.train = d, train
        if random:
            self.w = Guarded(d, init=(torch.rand(d, generator=gen) + 0.5).to(DEV))
            self.b = Guarded(d, init=torch.randn(d, generator=gen).to(DEV))
            self.rm = Guarded(d, init=torch.randn(d, generator=gen).to(DEV))
            self.rv = Guarded(d, init=(torch.rand(d, generator=gen) + 0.5).to(DEV))
        else:
            self.w = Guarded(d, init=_ints(gen, d))
            self.b = Guarded(d, init=_ints(gen, d))
            self.rm = Guarded(d, init=_ints(gen, d))
            # eval: rv + eps rounds to a power of four in float32, so rsqrtf gives a power of two exactly
            k = torch.randint(-2, 2, (d,), generator=gen).double()
            rv = torch.from_numpy((np.float32(4.0) ** k.numpy().astype(np.float32)) - EPS32)
            assert (torch.from_numpy(rv.numpy() + EPS32) == torch.from_numpy(np.float32(4.0) ** k.numpy().astype(np.float32))).all()
            self.rv = Guarded(d, init=rv.to(DEV))
        self.nbt = torch.tensor([-7, 5, -7], dtype=torch.int64, device=DEV)
        self.gw = Guarded(d)
        self.gb = Guarded(d)
        self.saved = Guarded(2 * d)
        self.sums = Guarded(2 * d, dtype=torch.float64)

    def struct(self):
        m = _lib.GpsBatchNorm(self.w.ptr(), self.b.ptr(), self.rm.ptr(), self.rv.ptr(), self.nbt[1:].data_ptr(),
                              self.gw.ptr(), self.gb.ptr())
        return _lib.GpsRowwiseBn(m, self.saved.ptr(), self.sums.ptr(), 1 if self.train else 0, 0)

    def snapshot(self):
        return {k: getattr(self, k).buf.clone() for k in ("w", "b", "rm", "rv", "gw", "gb", "saved", "sums")} | {
            "nbt": self.nbt.clone()}

    def check_guards(self):
        for k in ("w", "b", "rm", "rv", "gw", "gb", "saved", "sums"):
            getattr(self, k).check(k)
        assert self.nbt[0] == -7 and self.nbt[2] == -7, "num_batches_tracked neighbours written"

    def mean_invstd(self):
        return self.saved.v[:self.d], self.saved.v[self.d:]


def stage(op, rows, d, *, x, ldx=0, x2=None, g=None, ldg=0, R=None, R2=None, out=None, ldo=0, out2=None, planes=None,
          bns=(), act=-1, p=0.0, site=0, p2=0.0, site2=0, accumulate=False, offset_dev=None, stats=None, E=0):
    a = _lib.GpsRowwiseArgs()
    a.rows, a.E, a.d = rows, E, d
    a.x, a.ldx, a.x2 = _ptr(x), ldx, _ptr(x2)
    a.g, a.ldg, a.R, a.R2 = _ptr(g), ldg, _ptr(R), _ptr(R2)
    a.out, a.ldo, a.out2 = _ptr(out), ldo, _ptr(out2)
    if planes is not None:
        a.planes = planes.struct()
    for i, b in enumerate(bns):
        a.bn[i] = b.struct()
    a.act, a.p, a.site, a.p2, a.site2, a.accumulate = act, p, site, p2, site2, int(accumulate)
    a.seed, a.offset, a.offset_dev = SEED, OFFSET, _ptr(offset_dev)
    a.stats = _ptr(stats)
    rc = _lib.load().gps_rowwise_stage(C.byref(a), OPS[op], _stream())
    torch.cuda.synchronize()
    return rc


def _ptr(t):
    if t is None:
        return 0
    return t.ptr() if hasattr(t, "ptr") else t.data_ptr()


def _call(op, rows, d, **kw):
    _lib.check(stage(op, rows, d, **kw), op)


# ---------------------------------------------------------------------------------------------------- replays
def _fma32(a, b, c):
    """fmaf(a, b, c) for float32 tensors, correctly rounded: a * b is exact in float64, and the double rounding of
    a * b + c (to float64, then float32) is corrected where float64 lands on a float32 midpoint."""
    p = a.double() * b.double()
    cd = c.double()
    s = p + cd
    bb = s - p
    e = (p - (s - bb)) + (cd - bb)          # s + e == p + c exactly (TwoSum)
    r = s.float()
    rd = r.double()
    up = torch.nextafter(r, torch.full_like(r, float("inf"))).double()
    dn = torch.nextafter(r, torch.full_like(r, float("-inf"))).double()
    r = torch.where((s == (rd + up) / 2) & (e > 0), up.float(), r)
    r = torch.where((s == (rd + dn) / 2) & (e < 0), dn.float(), r)
    return r


def _keep_scale(p):
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))


def _mask(rows, d, p, site, offset=OFFSET):
    m = torch.empty(rows, d, device=DEV)
    _lib.check(_lib.load().gps_dropout_mask(m.data_ptr(), rows, d, p, SEED, offset, site, _stream()), "gps_dropout_mask")
    return m


def _ulp(x):
    x32 = x.float().abs()
    return (torch.nextafter(x32, torch.full_like(x32, float("inf"))) - x32).double()


def _first(mask):
    idx = mask.nonzero()
    return tuple(idx[0].tolist()) if idx.numel() else None


def _assert_equal(got, want, what):
    bad = got != want
    assert not bad.any(), f"{what}: {int(bad.sum())} elements differ from the float32 replay, first {_first(bad)}"


def _assert_within(got, ref, bound, what):
    err = (got.double() - ref.double()).abs()
    bad = ~(err <= bound)
    assert not bad.any(), (f"{what}: {int(bad.sum())} elements off their bound, first {_first(bad)}, "
                           f"worst {float((err / (bound + 1e-300)).max()):.3g} x bound")


def finalise64(sums, n):
    """The statistics finalisation replayed in float64 (BnRegs::load, mode 1): (mean, invstd, unbiased var) as float32,
    for both ways the compiler may evaluate s1 * inv_n - mu * mu (one fma, or two roundings)."""
    d = sums.numel() // 2
    s0, s1 = sums[:d].double().cpu(), sums[d:].double().cpu()
    inv_n = 1.0 / float(n if n > 0 else 1)
    unbias = float(n) / float(n - 1) if n > 1 else 1.0
    mu = s0 * inv_n
    mm = mu * mu
    plain = s1 * inv_n - mm
    fused = torch.tensor([float(Fraction(float(a)) * Fraction(inv_n) - Fraction(float(b))) for a, b in
                          zip(s1.tolist(), mm.tolist())], dtype=torch.float64)
    res = []
    for vv in (fused, plain):
        vv = vv.clamp_min(0.0)
        res.append((mu.float(), (1.0 / torch.sqrt(vv + EPS64)).float(), (vv * unbias).float()))
    return res


def _running32(old, new):
    """(1 - 0.1f) * old + 0.1f * new in float32, unfused."""
    one_m = np.float32(1.0) - MOM
    return torch.from_numpy(one_m * old.cpu().numpy() + MOM * new.cpu().numpy())


def check_finalised(bn, before, n, calls=1):
    """Mode 1: save_mean / save_invstd bitwise the float64 formula, running statistics within 1 ulp of the float32
    update, num_batches_tracked + calls."""
    d = bn.d
    variants = finalise64(before["sums"][G:G + 2 * d], n)
    m, s = bn.mean_invstd()
    m, s = m.cpu(), s.cpu()
    _assert_equal(m, variants[0][0], "save_mean")
    ok = (s == variants[0][1]) | (s == variants[1][1])
    assert ok.all(), f"save_invstd differs from the float64 formula at {int((~ok).sum())} columns, first {_first(~ok)}"
    rm_old = before["rm"][G:G + d]
    rv_old = before["rv"][G:G + d]
    want_rm = _running32(rm_old, variants[0][0])
    _assert_within(bn.rm.v.cpu(), want_rm, _ulp(want_rm), "running_mean")
    got_rv = bn.rv.v.cpu().double()
    ok = torch.zeros(d, dtype=torch.bool)
    for v in variants:
        want = _running32(rv_old, v[2]).double()
        ok |= (got_rv - want).abs() <= _ulp(want)
    assert ok.all(), f"running_var off the float32 update at {int((~ok).sum())} columns, first {_first(~ok)}"
    assert int(bn.nbt[1]) == int(before["nbt"][1]) + calls, "num_batches_tracked must go up by 1 per call"


def check_untouched(bn, before, keys):
    for k in keys:
        x, y = getattr(bn, k).buf if k != "nbt" else bn.nbt, before[k]
        same = torch.equal(x.view(torch.int64) if x.dtype == torch.float64 else x.view(torch.int32) if x.dtype == torch.float32 else x,
                           y.view(torch.int64) if y.dtype == torch.float64 else y.view(torch.int32) if y.dtype == torch.float32 else y)
        assert same, f"{k} written"


def eval_stats(bn):
    """Mode 2: mean = running_mean, invstd = rsqrtf(running_var + eps), the sum in float32.  The exact cases' running_var
    makes that sum a power of four, whose reciprocal square root is a power of two."""
    return bn.rm.v, torch.rsqrt((bn.rv.v + float(EPS32)).double()).float()


def apply32(z, mean, invstd, w, b):
    """BnRegs::apply in float32: fmaf((z - mean) * invstd, gamma, beta)."""
    zh = (z - mean) * invstd
    return _fma32(zh, w.expand_as(zh), b.expand_as(zh))


def fwd32(z, mean, invstd, bn, act, p, mask, R):
    """R + drop(act(BN(z))) as OpBnActRes::row computes it, float32."""
    v = apply32(z, mean, invstd, bn.w.v, bn.b.v)
    if act == RELU:
        v = torch.where(v > 0, v, torch.zeros_like(v))
    if p > 0:
        v = v * (mask * _keep_scale(p))
    if R is not None:
        v = v + R
    return v


def exact_sums(gen, rows, d):
    """Producer column sums that finalise to a mean on the 2^-3 grid and a biased variance of 4^j - (double)eps, so the
    float32 invstd is exactly 2^-j.  Exact only for power-of-two rows; other row counts give ordinary sums."""
    n = max(rows, 1)
    mu = _ints(gen, d, lo=-4, hi=4).double()
    j = torch.randint(-1, 2, (d,), generator=gen).double().to(DEV)
    var = 4.0 ** j - EPS64
    return torch.cat([mu * n, (var + mu * mu) * n])


# ---------------------------------------------------------------------------------------------------- forward recipes
def _fwd_single(rows, d, *, act, p, site, train, residual, planes, stats, ldx=None, seed=0, offset_dev=False,
                planes_lo=True):
    """One BN_ACT_RESIDUAL call and its checks.  Returns the outputs for reproducibility comparisons."""
    gen = torch.Generator().manual_seed(seed)
    bn = Bn(d, gen, train)
    bn.sums.v.copy_(exact_sums(gen, rows, d))
    z = Mat(rows, d, ldx, _ints(gen, rows, d))
    R = Mat(rows, d, None, _ints(gen, rows, d)) if residual else None
    out = Mat(rows, d)
    pl = PlanesBuf(rows, d, planes_lo) if planes else None
    st = Guarded(2 * d, torch.float64, torch.zeros(2 * d, dtype=torch.float64)) if stats else None
    od = torch.tensor([OFFSET_DEV], dtype=torch.int64, device=DEV) if offset_dev else None
    before = bn.snapshot()
    _call("bn_act_residual", rows, d, x=z, ldx=z.ld, R=R, out=out, planes=pl, bns=[bn], act=act, p=p, site=site,
          stats=st, offset_dev=od)
    out.check("out")
    bn.check_guards()
    if rows == 0:
        check_untouched(bn, before, ("saved", "rm", "rv", "nbt"))
        assert torch.isnan(out.buf).all()
        return
    if train:
        check_finalised(bn, before, rows)
        mean, invstd = bn.mean_invstd()
    else:
        check_untouched(bn, before, ("saved", "rm", "rv", "nbt"))
        mean, invstd = eval_stats(bn)
    mask = _mask(rows, d, p, site, OFFSET + (OFFSET_DEV if offset_dev else 0)) if p > 0 else None
    want = fwd32(z.v, mean, invstd, bn, act, p, mask, R.v if R else None)
    _assert_equal(out.v, want, "out")
    if pl is not None:
        pl.check(out.v)
    if st is not None:
        check_stats(st, out.v, rows, d)
    return [out.buf.clone(), bn.saved.buf.clone(), bn.rm.buf.clone(), bn.rv.buf.clone()] + (
        [st.buf.clone()] if st is not None else [])


def check_stats(st, v, rows, d, what="stats"):
    st.check(what)
    got = st.v.view(2, d).cpu()
    c = v.double().cpu()
    n = stats_chain(rows, d)
    for i, (want, mag) in enumerate(((c.sum(0), c.abs().sum(0)), ((c * c).sum(0), (c * c).sum(0)))):
        _assert_within(got[i], want, n * U * mag + 2.0 ** -50 * mag, f"{what}[{i}]")


# rows x d covering every row_geom branch: RY from 16 (d <= 256) down to 1 (d = 4096), the 66- and 1056-CTA caps (rows
# 3620 at d = 304, 100003 at d = 64: ~95 rows per thread), one and few CTAs, fewer rows than a CTA's row lanes
FWD_SHAPES = [(1, 4), (2, 84), (5, 256), (64, 304), (3620, 304), (7455, 608), (100003, 64), (3620, 1024), (64, 4096),
              (7455, 84)]


@pytest.mark.parametrize("rows,d", FWD_SHAPES)
@pytest.mark.parametrize("train", [True, False])
def test_genconv_bn_relu(rows, d, train):
    """layer.cu GENConv MLP: r = relu(BN(h1)) at width 2d (so d here is 2 d_layer), planes, no dropout or residual."""
    _fwd_single(rows, d, act=RELU, p=0.0, site=0, train=train, residual=False, planes=True, stats=False)


@pytest.mark.parametrize("rows,d", FWD_SHAPES)
@pytest.mark.parametrize("p", [0.5, 0.75])
def test_bn_act_residual_all_fields(rows, d, p):
    """The single-launch op with every field: x at pitch d + 12, ReLU, dropout with a device offset, residual, planes
    without the lo plane, and the next BatchNorm's column sums (the fused op's node half when E == 0)."""
    _fwd_single(rows, d, act=RELU, p=p, site=SITE_GCN_X, train=True, residual=True, planes=True, stats=True,
                ldx=d + 12, offset_dev=True, planes_lo=False)


def test_bn_act_residual_no_rows():
    _fwd_single(0, 64, act=RELU, p=0.5, site=SITE_GCN_X, train=True, residual=True, planes=True, stats=True)


@pytest.mark.parametrize("rows,d", [(3620, 304), (5, 64)])
def test_gelu_and_layer_dropout(rows, d):
    """GELU (erff) and p = 0.1 (keep scale 1/0.9 rounds): per-element bounds against float64 from the same float32
    BatchNorm output.  GELU: 8u |v| (test_gemm_epilogue_gpu.py); times the inexact scale: one more u, and the residual
    add after it may be contracted into an fma: 1 ulp of the largest magnitude the two roundings see."""
    gen = torch.Generator().manual_seed(3)
    bn = Bn(d, gen, True)
    bn.sums.v.copy_(exact_sums(gen, rows, d))
    z = Mat(rows, d, None, _ints(gen, rows, d))
    R = Mat(rows, d, None, _ints(gen, rows, d))
    out = Mat(rows, d)
    _call("bn_act_residual", rows, d, x=z, R=R, out=out, bns=[bn], act=GELU, p=0.1, site=SITE_LOCAL)
    out.check("out")
    mean, invstd = bn.mean_invstd()
    y = apply32(z.v, mean, invstd, bn.w.v, bn.b.v).double()
    g = 0.5 * y * (1.0 + torch.erf(y / 2.0 ** 0.5))
    s = _mask(rows, d, 0.1, SITE_LOCAL).double() * (1.0 / 0.9)
    x = g * s
    ref = x + R.v.double()
    bound = 8 * U * y.abs() * s + 2 * U * x.abs() + _ulp(torch.maximum(x.abs(), ref.abs()))
    _assert_within(out.v, ref, bound, "out")


# ---------------------------------------------------------------------------------------------------- the fused launch
def _fused(N, E, d, *, train, stats, residual, act=RELU, p=0.5, site=SITE_GCN_X, site2=SITE_GCN_E, seed=0,
           planes=True):
    gen = torch.Generator().manual_seed(seed)
    bx, be = Bn(d, gen, train), Bn(d, gen, train)
    bx.sums.v.copy_(exact_sums(gen, N, d))
    be.sums.v.copy_(exact_sums(gen, E, d))
    zx, ze = Mat(N, d, None, _ints(gen, N, d)), Mat(E, d, None, _ints(gen, E, d))
    Rx = Mat(N, d, None, _ints(gen, N, d)) if residual else None
    Re = Mat(E, d, None, _ints(gen, E, d)) if residual else None
    ox, oe = Mat(N, d), Mat(E, d)
    pl = PlanesBuf(E, d) if planes else None
    st = Guarded(2 * d, torch.float64, torch.zeros(2 * d, dtype=torch.float64)) if stats else None
    snaps = bx.snapshot(), be.snapshot()
    _call("bn_act_residual2", N, d, E=E, x=zx, R=Rx, out=ox, x2=ze, R2=Re, out2=oe, planes=pl, bns=[bx, be], act=act,
          p=p, site=site, site2=site2, stats=st)
    res = []
    for bn, before, z, R, o, rows, s in ((bx, snaps[0], zx, Rx, ox, N, site), (be, snaps[1], ze, Re, oe, E, site2)):
        o.check("out")
        bn.check_guards()
        if rows == 0:
            check_untouched(bn, before, ("saved", "rm", "rv", "nbt"))
            continue
        if train:
            check_finalised(bn, before, rows)
            mean, invstd = bn.mean_invstd()
        else:
            check_untouched(bn, before, ("saved", "rm", "rv", "nbt"))
            mean, invstd = eval_stats(bn)
        mask = _mask(rows, d, p, s) if p > 0 else None
        _assert_equal(o.v, fwd32(z.v, mean, invstd, bn, act, p, mask, R.v if R else None), "out")
        res += [o.buf.clone(), bn.saved.buf.clone(), bn.rm.buf.clone(), bn.rv.buf.clone()]
    if pl is not None and E > 0:
        pl.check(oe.v)
    if st is not None:
        if N > 0:
            check_stats(st, ox.v, N, d, "stats_x")
        res.append(st.buf.clone())
    return res


# (N, E, d): edges on both sides of nodes, the node op's fat block shape (RY 16, 13, 6, 1) walking more edges than it
# has CTAs for, and one side empty (two-launch form)
FUSED_SHAPES = [(3620, 7455, 304), (7455, 3620, 304), (64, 100003, 64), (100003, 64, 64), (5, 2, 608), (1, 64, 4096),
                (3620, 0, 304), (0, 3620, 304)]


@pytest.mark.parametrize("N,E,d", FUSED_SHAPES)
def test_bn_node_x_bn_edge_e(N, E, d):
    """layer.cu GatedGCN outputs: x_loc = x + drop(relu(BN_x(x~))) with norm1_local's sums, e_out = e + drop(relu(
    BN_e(e^))) with e_out's planes, in one launch (blocks [0, ga) the node op, the rest the edge op)."""
    _fused(N, E, d, train=True, stats=True, residual=True)


@pytest.mark.parametrize("N,E,d", FUSED_SHAPES[:4])
def test_bn_node_x_bn_edge_e_eval(N, E, d):
    """Eval mode: no statistics, so the two-launch form, reading the running statistics."""
    _fused(N, E, d, train=False, stats=False, residual=True, p=0.0)


@pytest.mark.parametrize("N,E,d", [(3620, 7455, 304), (7455, 3620, 64), (5, 64, 84)])
@pytest.mark.parametrize("p", [0.0, 0.75])
def test_customgnn_bn(N, E, d, p):
    """custom_gnn.cu GatedGCN: the fused launch with a statistics sink and no residual, its own dropout sites."""
    _fused(N, E, d, train=True, stats=True, residual=False, p=p, site=SITE_CG_X, site2=SITE_CG_E, planes=False)


def test_fused_publishes_once_per_call_at_every_cta_count():
    """num_batches_tracked + 1 per BatchNorm per call, over node and edge grids of 1 to 66 and 1 to 264 CTAs."""
    for N, E in [(1, 1), (64, 4), (832, 900), (3620, 7455), (100003, 100003)]:
        _fused(N, E, 64, train=True, stats=True, residual=True, p=0.0, planes=False)


# ---------------------------------------------------------------------------------------------------- combine
@pytest.mark.parametrize("rows,d", FWD_SHAPES)
@pytest.mark.parametrize("two", [False, True])
def test_norm1_combine(rows, d, two):
    """layer.cu h = norm1_local(x_loc) + norm1_attn(h_attn) (two BatchNorms, each finalising its own statistics), or one
    of them alone (local-only or global-only layers), with planes."""
    gen = torch.Generator().manual_seed(5)
    bns = [Bn(d, gen, True) for _ in range(2 if two else 1)]
    for bn in bns:
        bn.sums.v.copy_(exact_sums(gen, rows, d))
    a, b = Mat(rows, d, None, _ints(gen, rows, d)), Mat(rows, d, None, _ints(gen, rows, d))
    out = Mat(rows, d)
    pl = PlanesBuf(rows, d)
    snaps = [bn.snapshot() for bn in bns]
    _call("bn_combine", rows, d, x=a, x2=b if two else None, out=out, planes=pl, bns=bns)
    out.check("out")
    want = None
    for bn, before, z in zip(bns, snaps, (a, b)):
        bn.check_guards()
        check_finalised(bn, before, rows)
        m, s = bn.mean_invstd()
        y = apply32(z.v, m, s, bn.w.v, bn.b.v)
        want = y if want is None else want + y
    _assert_equal(out.v, want, "out")
    pl.check(out.v)


@pytest.mark.parametrize("rows,d", [(3620, 304), (7455, 64), (1, 4), (100003, 84)])
@pytest.mark.parametrize("train", [True, False])
def test_norm2_san_bn(rows, d, train):
    """layer.cu x_out = norm2(t) and san.cu h1 = bn1(z1), x_out = bn2(z2): one BatchNorm, no planes."""
    gen = torch.Generator().manual_seed(6)
    bn = Bn(d, gen, train)
    bn.sums.v.copy_(exact_sums(gen, rows, d))
    z = Mat(rows, d, None, _ints(gen, rows, d))
    out = Mat(rows, d)
    before = bn.snapshot()
    _call("bn_combine", rows, d, x=z, out=out, bns=[bn])
    out.check("out")
    bn.check_guards()
    if train:
        check_finalised(bn, before, rows)
        m, s = bn.mean_invstd()
    else:
        check_untouched(bn, before, ("saved", "rm", "rv", "nbt"))
        m, s = eval_stats(bn)
    _assert_equal(out.v, apply32(z.v, m, s, bn.w.v, bn.b.v), "out")


# ---------------------------------------------------------------------------------------------------- backward
def _bwd(rows, d, *, act, p, site, train, ldg=None, ldx=None, ldo=None, accumulate=False, planes=False, seed=0,
         offset_dev=False):
    """BN_BWD_REDUCE then BN_BWD_APPLY on exact data (power-of-two rows: S / n and every term of the apply are exact):
    both sums, out, its planes and the parameter gradients against the float32 replay, bit for bit."""
    gen = torch.Generator().manual_seed(seed)
    bn = Bn(d, gen, train)
    mean = _ints(gen, d, lo=-4, hi=4)
    invstd = 2.0 ** torch.randint(-1, 2, (d,), generator=gen).float().to(DEV)
    bn.saved.v.copy_(torch.cat([mean, invstd]))
    bn.sums.v.zero_()
    g = Mat(rows, d, ldg, _ints(gen, rows, d, lo=-4, hi=4))
    z = Mat(rows, d, ldx, _ints(gen, rows, d))
    out = Mat(rows, d, ldo)
    pl = PlanesBuf(rows, d) if planes else None
    if accumulate:
        bn.gw.v.copy_(_ints(gen, d))
        bn.gb.v.copy_(_ints(gen, d))
    gw0, gb0 = bn.gw.v.clone(), bn.gb.v.clone()
    od = torch.tensor([OFFSET_DEV], dtype=torch.int64, device=DEV) if offset_dev else None
    kw = dict(x=z, ldx=z.ld, g=g, ldg=g.ld, bns=[bn], act=act, p=p, site=site, offset_dev=od)
    before = bn.snapshot()
    _call("bn_bwd_reduce", rows, d, **kw)
    _call("bn_bwd_apply", rows, d, out=out, ldo=out.ld, planes=pl, accumulate=accumulate, **kw)
    out.check("out")
    bn.check_guards()
    check_untouched(bn, before, ("saved", "rm", "rv", "nbt", "w", "b"))
    if not train:
        mean, invstd = eval_stats(bn)
    zh = (z.v - mean) * invstd
    gp = g.v.clone()
    if p > 0 and rows > 0:
        gp = gp * (_mask(rows, d, p, site, OFFSET + (OFFSET_DEV if offset_dev else 0)) * _keep_scale(p))
    if act == RELU:
        gp = torch.where(_fma32(zh, bn.w.v.expand_as(zh), bn.b.v.expand_as(zh)) > 0, gp, torch.zeros_like(gp))
    S1, S2 = gp.double().sum(0), (gp.double() * zh.double()).sum(0)
    _assert_equal(bn.sums.v[:d], S1, "S1 (sum g')")
    _assert_equal(bn.sums.v[d:], S2, "S2 (sum g' zhat)")
    if rows == 0:
        assert torch.isnan(out.buf).all()
        for v, v0 in ((bn.gw.v, gw0), (bn.gb.v, gb0)):
            if accumulate:
                assert torch.equal(v, v0), "accumulating gradients changed by a backward over no rows"
            else:
                assert (v == 0).all(), "gradients of a backward over no rows must be zero"
        return
    n = np.float32(rows)
    inv_n = float(np.float32(1.0) / n)
    m1, m2 = S1.float() * inv_n, S2.float() * inv_n
    if not train:
        m1, m2 = torch.zeros_like(m1), torch.zeros_like(m2)
    inner = gp.double() - m1.double() - zh.double() * m2.double()
    for t in (gp.double() - m1.double(), zh.double() * m2.double(), inner):
        assert torch.equal(t.float().double(), t), "test precondition: the apply's inner terms are exact in float32"
    want = (bn.w.v * invstd) * inner.float()
    _assert_equal(out.v, want, "out")
    if pl is not None:
        pl.check(out.v)
    for v, v0, s, name in ((bn.gw.v, gw0, S2, "grad_weight"), (bn.gb.v, gb0, S1, "grad_bias")):
        _assert_equal(v, v0 + s.float() if accumulate else s.float(), name)


# bn_node_x_bwd: layer.cu bn_node_x's backward writes gY1's first block, pitch 7d; custom_gnn.cu's writes gY at 4 dp
@pytest.mark.parametrize("rows,d,ldo", [(64, 304, 7 * 304), (4096, 64, 7 * 64), (2, 84, 4 * 84), (1, 4096, 4096),
                                        (4096, 1024, 4 * 1024), (64, 4, 28)])
@pytest.mark.parametrize("p", [0.0, 0.5])
def test_bn_node_x_bwd(rows, d, ldo, p):
    _bwd(rows, d, act=RELU, p=p, site=SITE_GCN_X, train=True, ldo=ldo, planes=True, offset_dev=True)


@pytest.mark.parametrize("rows,d", [(4096, 304), (64, 608), (1, 84), (0, 64)])
@pytest.mark.parametrize("train", [True, False])
def test_bn_edge_e_bwd(rows, d, train):
    """layer.cu bn_edge_e's backward accumulating into the parameter gradients (GPS_FLAG_GRADS_ACCUMULATE), dropout."""
    _bwd(rows, d, act=RELU, p=0.75, site=SITE_GCN_E, train=train, accumulate=True)


@pytest.mark.parametrize("rows,d", [(4096, 304), (64, 608), (2, 256), (0, 64)])
def test_norm_bwd(rows, d):
    """norm2 / norm1_local / norm1_attn / SAN's bn1, bn2 backward: no act, no dropout, written gradients; and
    GENConv's 2d-wide one with ReLU."""
    _bwd(rows, d, act=-1, p=0.0, site=0, train=True, planes=True)
    _bwd(rows, d, act=RELU, p=0.0, site=0, train=True, seed=1)


@pytest.mark.parametrize("rows,d", [(64, 304), (4096, 84), (2, 4096)])
def test_bwd_pitches(rows, d):
    """g, z and out at three different pitches, dropout indexed over the dense [rows, d] grid whatever the pitches."""
    _bwd(rows, d, act=RELU, p=0.5, site=SITE_LOCAL, train=True, ldg=d + 8, ldx=d + 12, ldo=d + 4)


# ---------------------------------------------------------------------------------------------------- dropmul, colsum
@pytest.mark.parametrize("rows,d", [(3620, 304), (7455, 64), (5, 4), (100003, 84)])
@pytest.mark.parametrize("p,p2,offset_dev", [(0.5, 0.0, False), (0.75, 0.0, True), (0.5, 0.75, True), (0.0, 0.5, False)])
def test_dropmul(rows, d, p, p2, offset_dev):
    """layer.cu dropmul: the gradient in front of one dropout site (FF2, local) or two (attention output then
    Performer's own, site2), with planes."""
    gen = torch.Generator().manual_seed(7)
    src = Mat(rows, d, None, _ints(gen, rows, d))
    out = Mat(rows, d)
    pl = PlanesBuf(rows, d)
    od = torch.tensor([OFFSET_DEV], dtype=torch.int64, device=DEV) if offset_dev else None
    _call("dropmul", rows, d, x=src, out=out, planes=pl, p=p, site=SITE_FF2, p2=p2, site2=7, offset_dev=od)
    out.check("out")
    off = OFFSET + (OFFSET_DEV if offset_dev else 0)
    want = src.v.clone()
    if p > 0:
        want = want * (_mask(rows, d, p, SITE_FF2, off) * _keep_scale(p))
    if p2 > 0:
        want = want * (_mask(rows, d, p2, 7, off) * _keep_scale(p2))
    _assert_equal(out.v, want, "out")
    pl.check(out.v)


# (rows, d, lda): fewer rows than the cluster's 8 x RY row lanes, d = 4 (one column per CTA), one full and a final partial
# column chunk of 128 float4 columns (d = 608 + ... = 2128 -> 532 float4: 4 full chunks + 20), lda > d, the layer's 7d
COLSUM_SHAPES = [(1, 4, 8), (5, 64, 68), (127, 2128, 2136), (3620, 304, 7 * 304), (100003, 64, 64), (7455, 4100, 4104),
                 (64, 1024, 1028)]


@pytest.mark.parametrize("rows,d,lda", COLSUM_SHAPES)
def test_colsum(rows, d, lda):
    """layers_ops.cuh wgrad_add in bf16 mode: the bias gradient as an exact float32 column sum added into a non-zero
    out.  Exact data: every partial is exact, so out must be the float32 sum of the float64 total and the initial out."""
    gen = torch.Generator().manual_seed(8)
    a = Mat(rows, d, lda, _ints(gen, rows, d))
    out = Guarded(d, init=_ints(gen, d))
    o0 = out.v.clone()
    _call("colsum", rows, d, x=a, ldx=lda, out=out)
    out.check("out")
    _assert_equal(out.v, o0 + a.v.double().sum(0).float(), "out")
    again = Guarded(d, init=o0)
    _call("colsum", rows, d, x=a, ldx=lda, out=again)
    assert torch.equal(again.v, out.v)


# ---------------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("d", [6, 4100])
def test_unsupported_width(op, d):
    """d outside the row-wise stages' range is the kernels' GPS_ERR_UNSUPPORTED, with nothing written.  The dropout and
    column-sum passes are flat over float4 groups and take d = 4100."""
    if op in ("dropmul", "colsum") and d == 4100:
        pytest.skip("takes any d % 4 == 0")
    gen = torch.Generator().manual_seed(9)
    rows = 8
    bns = [Bn(d, gen, True), Bn(d, gen, True)]
    for bn in bns:
        bn.sums.v.zero_()
        bn.saved.v.zero_()
    x = Mat(rows, d, None, torch.zeros(rows, d, device=DEV))
    out, out2 = Mat(rows, d), Mat(rows, d)
    snaps = [bn.snapshot() for bn in bns]
    rc = stage(op, rows, d, x=x, g=x, out=out, x2=x, out2=out2, E=rows, bns=bns)
    assert rc == _lib.GPS_ERR_UNSUPPORTED, (rc, _lib.load().gps_last_error())
    assert torch.isnan(out.buf).all() and torch.isnan(out2.buf).all(), "refused, but wrote"
    for bn, before in zip(bns, snaps):
        check_untouched(bn, before, ("saved", "rm", "rv", "nbt", "sums", "gw", "gb"))


# ---------------------------------------------------------------------------------------------------- random cases
def _random_z(gen, rows, d):
    """Columns with means within 4 standard deviations of zero: std in [0.5, 2], mean = t std with |t| <= 4, so
    K = (mean^2 + var) / var <= 17 for the population (K_MAX leaves room for the sample)."""
    std = torch.rand(d, generator=gen) * 1.5 + 0.5
    mean = (torch.rand(d, generator=gen) * 8 - 4) * std
    return (torch.randn(rows, d, generator=gen) * std + mean).to(DEV)


K_MAX = 20.0


def _delta(rows):
    """Relative error of the float64 variance E[z^2] - mean^2 from host-summed float64 sums: (4 + log2 n) 2^-52 K."""
    return (4 + math.log2(max(rows, 2))) * 2.0 ** -52 * K_MAX


def _random_fwd(rows, d, train, act, p, seed):
    gen = torch.Generator().manual_seed(seed)
    bn = Bn(d, gen, train, random=True)
    z = Mat(rows, d, None, _random_z(gen, rows, d))
    zd = z.v.double()
    bn.sums.v.copy_(torch.cat([zd.sum(0), (zd * zd).sum(0)]))
    R = Mat(rows, d, None, (torch.rand(rows, d, generator=gen) + 2).to(DEV))
    out = Mat(rows, d)
    st = Guarded(2 * d, torch.float64, torch.zeros(2 * d, dtype=torch.float64))
    rm0, rv0 = bn.rm.v.double().clone(), bn.rv.v.double().clone()
    _call("bn_act_residual", rows, d, x=z, R=R, out=out, bns=[bn], act=act, p=p, site=SITE_LOCAL, stats=st)
    out.check("out")
    bn.check_guards()
    w, b = bn.w.v.double(), bn.b.v.double()
    mu, var = zd.mean(0), zd.var(0, unbiased=False)
    if train:
        y = F.batch_norm(zd, None, None, w, b, training=True, eps=EPS64)
        invstd = 1.0 / torch.sqrt(var + EPS64)
        zh = (zd - mu) * invstd
        delta = _delta(rows)
        dz = zh.abs() * (3 * U + delta) + invstd * U * mu.abs()
        m, s = bn.mean_invstd()
        _assert_within(m, mu, U * mu.abs() + 2.0 ** -50 * mu.abs(), "save_mean")
        _assert_within(s, invstd, (U + delta) * invstd, "save_invstd")
        # running statistics: torch's update, unbiased variance; two float32 roundings of the update, 0.1 mean's own
        rm_ref = 0.9 * rm0 + 0.1 * mu
        rv_ref = 0.9 * rv0 + 0.1 * var * rows / max(rows - 1, 1)
        _assert_within(bn.rm.v, rm_ref, 3 * U * (0.9 * rm0.abs() + 0.1 * mu.abs()) + 0.1 * U * mu.abs(), "running_mean")
        _assert_within(bn.rv.v, rv_ref, 3 * U * rv_ref.abs() + 0.1 * var * (U + 2 * delta) * 2, "running_var")
        assert int(bn.nbt[1]) == 6
    else:
        rm, rv = bn.rm.v.double(), bn.rv.v.double()
        y = F.batch_norm(zd, rm, rv, w, b, training=False, eps=EPS64)
        zh = (zd - rm) / torch.sqrt(rv + EPS64)
        dz = zh.abs() * 6 * U      # z - m, the product, rv + eps and rsqrtf (2 ulp)
    by = w.abs() * dz + U * y.abs()
    a = torch.relu(y) if act == RELU else y
    sc = _mask(rows, d, p, SITE_LOCAL).double() * _keep_scale(p) if p > 0 else torch.ones_like(y)
    ref = a * sc + R.v.double()
    bound = 2 * (by * sc + 2 * U * (a * sc).abs() + U * ref.abs())
    _assert_within(out.v, ref, bound, "out")
    check_stats(st, out.v, rows, d)
    return [out.buf.clone(), bn.saved.buf.clone(), bn.rm.buf.clone(), bn.rv.buf.clone(), st.buf.clone()]


RANDOM_SHAPES = [(3620, 304), (7455, 608), (100003, 64), (3620, 4096), (64, 84)]


@pytest.mark.parametrize("rows,d", RANDOM_SHAPES)
@pytest.mark.parametrize("train", [True, False])
def test_random_forward_against_torch(rows, d, train):
    first = _random_fwd(rows, d, train, RELU, 0.1, seed=11)
    again = _random_fwd(rows, d, train, RELU, 0.1, seed=11)
    for x, y in zip(first, again):
        assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x.view(torch.int64),
                           y.view(torch.int32) if y.dtype == torch.float32 else y.view(torch.int64)), "not reproducible"


def _random_bwd(rows, d, train, p, seed):
    """Forward stage (training: finalising and saving the statistics), then the backward pair, against the float64
    autograd of R + mask * relu(BN(z)).  The cotangent is zeroed where the float64 pre-activation lies within the
    forward's bound of 0, so both arithmetics take the same ReLU branch."""
    gen = torch.Generator().manual_seed(seed)
    bn = Bn(d, gen, train, random=True)
    z = Mat(rows, d, None, _random_z(gen, rows, d))
    zd = z.v.double()
    bn.sums.v.copy_(torch.cat([zd.sum(0), (zd * zd).sum(0)]))
    out = Mat(rows, d)
    _call("bn_act_residual", rows, d, x=z, out=out, bns=[bn], act=RELU, p=p, site=SITE_LOCAL)
    w = bn.w.v.double().requires_grad_(True)
    b = bn.b.v.double().requires_grad_(True)
    zr = zd.clone().requires_grad_(True)
    mu, var = zd.mean(0), zd.var(0, unbiased=False)
    if train:
        y = F.batch_norm(zr, None, None, w, b, training=True, eps=EPS64)
        invstd = 1.0 / torch.sqrt(var + EPS64)
        m_used = mu
        delta = _delta(rows)
    else:
        rm, rv = bn.rm.v.double(), bn.rv.v.double()
        y = F.batch_norm(zr, rm, rv, w, b, training=False, eps=EPS64)
        invstd = 1.0 / torch.sqrt(rv + EPS64)
        m_used = rm
        delta = 4 * U
    zh = ((zd - m_used) * invstd).detach()
    y_bound = w.detach().abs() * (zh.abs() * (3 * U + delta) + invstd * U * m_used.abs()) + U * y.detach().abs()
    # gradient with a positive column mean (same-signed partials: reproducible sums), correlated with zhat so that
    # sum g' zhat has no cancellation either
    gcot = (0.5 + zh + 0.25 * torch.randn(rows, d, generator=gen, dtype=torch.float64).to(DEV)).float()
    gcot = torch.where(y.detach().abs() <= 4 * y_bound, torch.zeros_like(gcot), gcot)
    sc = _mask(rows, d, p, SITE_LOCAL).double() * _keep_scale(p) if p > 0 else torch.ones_like(zd)
    o = torch.relu(y) * sc
    (o * gcot.double()).sum().backward()
    g = Mat(rows, d, None, gcot)
    dz = Mat(rows, d)
    bn.sums.v.zero_()
    bn.gw.v.zero_()
    bn.gb.v.zero_()
    kw = dict(x=z, g=g, bns=[bn], act=RELU, p=p, site=SITE_LOCAL)
    _call("bn_bwd_reduce", rows, d, **kw)
    _call("bn_bwd_apply", rows, d, out=dz, **kw)
    dz.check("out")
    bn.check_guards()
    gp = gcot.double() * sc * (y.detach() > 0)
    n = rows
    chain = stats_chain(rows, d)
    S1, S2 = gp.sum(0), (gp * zh).sum(0)
    A1, A2 = gp.abs().sum(0), (gp * zh).abs().sum(0)
    gis = (w.detach() * invstd).abs()
    Mterm = invstd * m_used.abs()
    # S1 = grad_beta: the float32 chain of g' (g * s rounds once for an inexact keep scale), then the float32 cast
    _assert_within(bn.gb.v, b.grad, (chain + 1) * U * A1 + U * S1.abs(), "grad_beta (S1)")
    # S2 = grad_gamma: the chain, the fma's rounding, zhat's error ((3u + delta) |zhat| + u invstd |mean|), the cast
    _assert_within(bn.gw.v, w.grad, (chain + 5) * U * A2 + delta * A2 + U * Mterm * A1 + U * S2.abs(),
                   "grad_gamma (S2)")
    if train:
        A = gp.abs() + S1.abs() / n + zh.abs() * S2.abs() / n
        B = (A1 + zh.abs() * A2) / n
        bound = gis * (10 * U * A + (chain + 6) * U * B + 2 * delta * (A + B) + U * Mterm * (S2.abs() + zh.abs() * A1) / n)
    else:
        bound = gis * 6 * U * gp.abs()
    _assert_within(dz.v, zr.grad, 2 * bound + U * zr.grad.abs(), "grad_z")
    return [dz.buf.clone(), bn.sums.buf.clone(), bn.gw.buf.clone(), bn.gb.buf.clone()]


@pytest.mark.parametrize("rows,d", RANDOM_SHAPES)
@pytest.mark.parametrize("train", [True, False])
def test_random_backward_against_autograd(rows, d, train):
    first = _random_bwd(rows, d, train, 0.1, seed=12)
    again = _random_bwd(rows, d, train, 0.1, seed=12)
    for x, y in zip(first, again):
        assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x.view(torch.int64),
                           y.view(torch.int32) if y.dtype == torch.float32 else y.view(torch.int64)), "not reproducible"
