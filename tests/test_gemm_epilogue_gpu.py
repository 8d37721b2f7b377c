"""GPU: the fused epilogue of the dense products (GemmParams, csrc/gemm.cuh) stage by stage, on each of the three kernels
that implement it: the exact CUDA-core kernel (gemm_simt.cu), the register-staged tensor-core kernel (gemm_tc.cu) and
the TMA-fed tensor-core kernel the layers run (gemm_tma.cu), through gps_gemm_epilogue.

Exact operands.  A, B, bias, residuals and act' inputs are small integers times 2^-3: exact in bf16 (zero lo plane),
and every partial sum of the product is a multiple of 2^-6 far below 2^24 ulps, so every kernel, in either precision and
in any summation order, produces the product exactly.  Any mismatch is then the epilogue's.  The dropout probabilities
0.5 and 0.75 keep with scales 2 and 4, so x * s is exact and an FMA contraction of x * s + r cannot change the bits.
Every epilogue step without a transcendental function must then equal, bit for bit, a float32 replay of the documented
order on the host side: bias, relu, the post-activation act' mask, both dropouts, R1, R2, the stored C, C_pre and the
planes.  GELU and its derivative (erff, __expf) are compared with float64 within a per-element bound (see _GELU_ULPS).

Sentinels.  C and C_pre start as NaN and sit inside wider buffers (ld > N), planes start as 0xFFFF, and the float64
statistics sit inside a NaN guard region: an element written that should not be, or left unwritten, shows.

Recipes are named after the layer steps that issue them, so a failure names the step.  Each runs on every kernel, in
fp32-grade and bf16 mode, at shapes covering M in {1, 13, 128, 129, 3620} (last row tiles of 1, 13, 128, 1 and 36
rows: fewer rows than the 16 row classes of the TMA kernel's statistics, and padding rows that must contribute nothing),
N in {64, 304, 608, 912, 1000} and K in {64, 72, 304}.  On the TMA
kernel every tile width the layout takes is forced as well as the policy's choice, and all outputs must be bitwise
equal across widths."""
import ctypes as C

import numpy as np
import pytest
import torch

from graphgps_b200 import _lib
from util import _nan, _stream, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

KERNELS = {"simt": 1, "tc": 2, "tma": 3}
PRECISIONS = {"fp32": 0, "bf16": 1}
RELU, GELU = _lib.ACT["relu"], _lib.ACT["gelu"]
U = 2.0 ** -24               # unit roundoff of float32
SEED, OFFSET, OFFSET_DEV = 0x5EED1234, 4096, 8192
SITE_ATTN_OUT, SITE_FF1, SITE_PERF_OUT = 4, 5, 7     # common.cuh: the layers' dropout sites
SENTINEL16 = -1              # 0xFFFF as int16: the plane sentinel

# (M, N, K): every value of M, N and K named above at least once, without the full product of them
SHAPES = [(1, 64, 64), (13, 304, 72), (129, 608, 304), (128, 912, 64), (3620, 1000, 72), (3620, 304, 304)]

# Longest chain of float32 additions a column statistic goes through inside one CTA before the float64 atomics (the
# float64 part adds ~2^-53 relative, negligible):
#   simt: each thread sums its 4 rows (4 additions), plus the rounding of v * v;
#   tc:   a 5-level butterfly over the warp's 32 rows, plus the rounding of v * v;
#   tma:  8 rows per row class (128 / 16), then the 16 classes in order; v * v is fused (fmaf), so no extra rounding.
# |computed - exact| <= n u sum|x| for a recursive float32 sum of n additions.
_STATS_CHAIN = {"simt": 5, "tc": 6, "tma": 24}

# GELU (0.5 v (1 + erff(v / sqrt 2))): erff is within 2 ulps, the argument's rounding moves erf by < u, and 1 + erf
# rounds once, so 1 + erf is off by at most ~6u absolute; times 0.5 v and one more rounding: <= 4u |v|.  The error is
# bounded relative to v, not to the result, because 1 + erf cancels for negative v.  8u |v| leaves a factor 2.
_GELU_ULPS = 8
# GELU' (cdf + v pdf, pdf with __expf): cdf is off by <= 3u, __expf by 2 + 1.2 |x| ulps (x = -v^2 / 2 >= -8 for
# |v| <= 4, the act' inputs here), so v pdf (|v pdf| <= 0.25) by <= ~6u, the sum rounds once: <= ~10u absolute.
_GELU_D_ULPS = 16


# ---------------------------------------------------------------------------------------------------- operands
def _ints(g, *shape, lo=-8, hi=8):
    """Small integers times 2^-3 (exact in bf16), on the device."""
    return (torch.randint(lo, hi + 1, shape, generator=g).float() * 0.125).to(DEV)


def _planes_of(x, lo):
    """gps_to_planes of an fp32 [rows, cols] view: int16 [2, rows, ld] (plane 1 untouched when lo is False)."""
    r, c = x.shape
    ld = (c + 7) // 8 * 8
    buf = torch.full((2, r, ld), SENTINEL16, dtype=torch.int16, device=DEV)
    _lib.check(_lib.load().gps_to_planes(x.data_ptr(), x.stride(0), r, c, buf[0].data_ptr(), buf[1].data_ptr() if lo else 0,
                                     ld, _stream()), "gps_to_planes")
    return buf, ld


def _dropout_mask(M, N, p, site, offset):
    m = torch.empty(M, N, device=DEV)
    _lib.check(_lib.load().gps_dropout_mask(m.data_ptr(), M, N, p, SEED, offset, site, _stream()), "gps_dropout_mask")
    return m


def _keep_scale(p):
    """1 / (1 - p) exactly as the kernels compute it in float32."""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))


def _gelu64(v):
    return 0.5 * v * (1.0 + torch.erf(v / 2.0 ** 0.5))


def _gelu_d64(v):
    return 0.5 * (1.0 + torch.erf(v / 2.0 ** 0.5)) + v * torch.exp(-0.5 * v * v) / (2.0 * torch.pi) ** 0.5


class Spec:
    """One epilogue: which GemmParams fields are set.  r1 = "alias" makes R1 the output buffer itself (C += product)."""

    def __init__(self, name, tb=0, bias=False, c_pre=False, act=-1, mask=None, p=0.0, site=0, p2=0.0, site2=0,
                 r1=False, r2=False, stats=False, cp=None, splitk=1, offset_dev=False):
        self.__dict__.update(locals())
        del self.__dict__["self"]


# ---------------------------------------------------------------------------------------------------- one run
class Run:
    """Device buffers for one product with its epilogue, the call, and the float32 / float64 replay."""

    def __init__(self, spec, M, N, K, precision, seed=0, random=False):
        self.s, self.M, self.N, self.K, self.prec = spec, M, N, K, precision
        g = torch.Generator().manual_seed(seed)
        if random:
            self.A = torch.randn(M, K, generator=g).to(DEV)
            self.B = (torch.randn(*((K, N) if spec.tb else (N, K)), generator=g) / K ** 0.5).to(DEV)
        else:
            self.A = _ints(g, M, K)
            self.B = _ints(g, *((K, N) if spec.tb else (N, K)))
        lo = precision == 0
        self.Ap, self.lda_p = _planes_of(self.A, lo)
        self.Bp, self.ldb_p = _planes_of(self.B, lo)
        self.bias = _ints(g, N) if spec.bias else None
        # C: columns [4, 4 + N) of a NaN buffer 12 columns wider (ldc != N, guard columns on both sides)
        self.Cbuf = _nan(M, N + 12)
        self.C = self.Cbuf[:, 4:4 + N]
        if spec.splitk > 1:
            self.C.zero_()
        self.R1 = self.R2 = None
        if spec.r1 == "alias":
            self.C.copy_(_ints(g, M, N))
            self.R1_init = self.C.clone()
        elif spec.r1:
            self.R1 = torch.zeros(M, N + 4, device=DEV)[:, :N]
            self.R1.copy_(_ints(g, M, N))
        if spec.r2:
            self.R2 = torch.zeros(M, N + 8, device=DEV)[:, :N]
            self.R2.copy_(_ints(g, M, N))
        self.Cpre_buf = _nan(M, N + 8) if spec.c_pre else None
        self.mask_src = None
        if spec.mask == "relu_post":     # a saved post-activation: >= 0, zero where the pre-activation was <= 0
            self.mask_src = torch.zeros(M, N + 4, device=DEV)[:, :N]
            self.mask_src.copy_(_ints(g, M, N).clamp_min(0.0))
        elif spec.mask == "gelu_pre":    # a saved pre-activation in [-4, 4]
            self.mask_src = torch.zeros(M, N + 4, device=DEV)[:, :N]
            self.mask_src.copy_(_ints(g, M, N, lo=-32, hi=32))
        self.stats_buf = None
        if spec.stats:
            self.stats_buf = torch.full((2 * N + 32,), float("nan"), dtype=torch.float64, device=DEV)
            self.stats_buf[16:16 + 2 * N] = 0.0
        # output planes: identity [M, N] or the per-head padded layout; plane 2 is a guard
        self.cp_hd = self.cp_pad = 0
        self.Cp = None
        if spec.cp is not None:
            width = N
            if spec.cp != "identity":
                self.cp_hd, self.cp_pad = spec.cp, (spec.cp + 15) // 16 * 16
                assert N % self.cp_hd == 0
                width = N // self.cp_hd * self.cp_pad
            self.cp_width = width
            self.Cp = torch.full((3, M, (width + 7) // 8 * 8 + 8), SENTINEL16, dtype=torch.int16, device=DEV)
        self.offset_dev = torch.tensor([OFFSET_DEV], dtype=torch.int64, device=DEV) if spec.offset_dev else None

    def args(self, with_cp=True):
        s, a = self.s, _lib.GpsGemmArgs()
        a.M, a.N, a.K = self.M, self.N, self.K
        a.A, a.lda, a.B, a.ldb, a.ta, a.tb = self.A.data_ptr(), self.A.stride(0), self.B.data_ptr(), self.B.stride(0), 0, s.tb
        lo = self.prec == 0
        a.Ap = _lib.GpsPlanes(self.Ap[0].data_ptr(), self.Ap[1].data_ptr() if lo else 0, self.lda_p)
        a.Bp = _lib.GpsPlanes(self.Bp[0].data_ptr(), self.Bp[1].data_ptr() if lo else 0, self.ldb_p)
        if self.Cp is not None and with_cp:
            a.Cp = _lib.GpsPlanes(self.Cp[0].data_ptr(), self.Cp[1].data_ptr() if lo else 0, self.Cp.shape[2])
            a.cp_hd, a.cp_hd_pad = self.cp_hd, self.cp_pad
        a.C, a.ldc = self.C.data_ptr(), self.C.stride(0)
        a.bias = _lib.ptr(self.bias)
        if self.Cpre_buf is not None:
            a.C_pre, a.ldpre = self.Cpre_buf.data_ptr(), self.Cpre_buf.stride(0)
        a.act = s.act
        a.mask_act = -1
        if self.mask_src is not None:
            a.mask_src, a.ldmask = self.mask_src.data_ptr(), self.mask_src.stride(0)
            a.mask_act, a.mask_is_post = (RELU, 1) if s.mask == "relu_post" else (GELU, 0)
        a.p_drop, a.site, a.p_drop2, a.site2 = s.p, s.site, s.p2, s.site2
        a.seed, a.offset, a.offset_dev = SEED, OFFSET, _lib.ptr(self.offset_dev)
        if s.r1 == "alias":
            a.R1, a.ldr1 = self.C.data_ptr(), self.C.stride(0)
        elif self.R1 is not None:
            a.R1, a.ldr1 = self.R1.data_ptr(), self.R1.stride(0)
        if self.R2 is not None:
            a.R2, a.ldr2 = self.R2.data_ptr(), self.R2.stride(0)
        if self.stats_buf is not None:
            a.stats = self.stats_buf[16:].data_ptr()
        a.splitk, a.precision = s.splitk, self.prec
        return a

    def call(self, impl, with_cp=True):
        a = self.args(with_cp)
        rc = _lib.load().gps_gemm_epilogue(C.byref(a), impl, _stream())
        torch.cuda.synchronize()
        return rc

    def outputs(self, stats=True):
        """Everything the call wrote (or must not have written), for bitwise comparisons between runs."""
        out = [self.Cbuf, self.Cpre_buf, self.stats_buf if stats else None, self.Cp]
        return [t.clone() for t in out if t is not None]

    # ------------------------------------------------------------------------------------------------ replay
    def replay(self):
        """(ref, bound, pre): the documented order replayed.  bound is None when ref is float32 and must match bit for
        bit; else ref is float64 and |C - ref| <= bound elementwise."""
        s, M, N = self.s, self.M, self.N
        acc = self.A.double() @ (self.B.double() if s.tb else self.B.double().t())
        v = acc.float()                                   # exact: multiples of 2^-6 far below 2^24 ulps
        if self.bias is not None:
            v = v + self.bias
        pre = v.clone()
        bound = None
        if s.act == RELU:
            v = torch.where(v > 0, v, torch.zeros_like(v))
        elif s.act == GELU:
            bound = _GELU_ULPS * U * pre.double().abs()
            v = _gelu64(pre.double())
        if s.mask == "relu_post":
            v = torch.where(self.mask_src > 0, v, torch.zeros_like(v))
        elif s.mask == "gelu_pre":
            d = _gelu_d64(self.mask_src.double())
            w = v.double()
            bound = (0.0 if bound is None else bound * d.abs()) + _GELU_D_ULPS * U * w.abs() + U * (w * d).abs()
            v = w * d
        off = OFFSET + (OFFSET_DEV if s.offset_dev else 0)
        inexact = False
        for p, site in ((s.p2, s.site2), (s.p, s.site)):
            if p > 0:
                sc = _keep_scale(p)
                keep = _dropout_mask(M, N, p, site, off)
                inexact |= sc not in (2.0, 4.0)
                v = v * (keep * sc).to(v.dtype)
                if bound is not None:
                    bound = bound * keep * sc
        if inexact and (self.R1 is not None or self.R2 is not None or s.r1 == "alias"):
            # x * s rounds and the residual add after it may be contracted into one FMA: compare the float64 value
            # within 1 ulp of the largest magnitude the two roundings see
            assert bound is None and self.R2 is None
            x = self._drop_scaled64()
            ref = x + self.R1.double()
            bound = _ulp(torch.maximum(x.abs(), ref.abs()))
            return ref, bound, pre
        r1 = self.R1_init if s.r1 == "alias" else self.R1
        for r in (r1, self.R2):
            if r is not None:
                if bound is not None:
                    v = v + r.double()
                    bound = bound + U * v.abs()
                else:
                    v = v + r
        if bound is not None:
            bound = bound + U * v.abs()
        return v, bound, pre

    def _drop_scaled64(self):
        """float64 (acc + bias) * keep * s for the single-dropout epilogues, exact."""
        s = self.s
        acc = self.A.double() @ (self.B.double() if s.tb else self.B.double().t())
        v = acc + (self.bias.double() if self.bias is not None else 0.0)
        off = OFFSET + (OFFSET_DEV if s.offset_dev else 0)
        for p, site in ((s.p2, s.site2), (s.p, s.site)):
            if p > 0:
                v = v * _dropout_mask(self.M, self.N, p, site, off).double() * _keep_scale(p)
        return v


def _ulp(x):
    """Spacing of float32 at |x| (float64 tensor in, float64 out)."""
    x32 = x.float().abs()
    return (torch.nextafter(x32, torch.full_like(x32, float("inf"))) - x32).double()


# ---------------------------------------------------------------------------------------------------- checks
def _check(run, kernel):
    """Every output of one run against the replay and the sentinels.  Returns nothing; asserts."""
    N = run.N
    # guard columns of C (and C_pre) keep the NaN sentinel
    assert torch.isnan(run.Cbuf[:, :4]).all() and torch.isnan(run.Cbuf[:, 4 + N:]).all(), "C written outside [0, N)"
    ref, bound, pre = run.replay()
    got = run.C
    assert not torch.isnan(got).any(), "C left unwritten"
    if bound is None:
        bad = (got != ref)
        assert not bad.any(), f"C differs from the float32 replay at {int(bad.sum())} elements, first {_first(bad)}"
    else:
        err = (got.double() - ref).abs()
        bad = err > bound
        assert not bad.any(), (f"C off its bound at {int(bad.sum())} elements, first {_first(bad)}, "
                               f"worst {float((err / (bound + 1e-300)).max()):.3g} x bound")
    if run.Cpre_buf is not None:
        cp = run.Cpre_buf
        assert torch.isnan(cp[:, N:]).all(), "C_pre written past N"
        assert torch.equal(cp[:, :N], pre), "C_pre differs from acc + bias"
    if run.stats_buf is not None:
        _check_stats(run, kernel)
    if run.Cp is not None and kernel == "tma":
        _check_planes(run)


def _first(mask):
    idx = mask.nonzero()
    return tuple(idx[0].tolist()) if idx.numel() else None


def _check_stats(run, kernel):
    N = run.N
    st = run.stats_buf
    assert torch.isnan(st[:16]).all() and torch.isnan(st[16 + 2 * N:]).all(), "stats written outside [2, N]"
    c = run.C.double()
    got = st[16:16 + 2 * N].view(2, N)
    n = _STATS_CHAIN[kernel]
    for i, (want, mag) in enumerate(((c.sum(0), c.abs().sum(0)), ((c * c).sum(0), (c * c).sum(0)))):
        bound = n * U * mag + 2.0 ** -50 * mag + 1e-300
        err = (got[i] - want).abs()
        bad = err > bound
        assert not bad.any(), (f"stats[{i}] off at {int(bad.sum())} columns, first {_first(bad)}: "
                               f"{float((err / bound).max()):.3g} x bound")


def _check_planes(run):
    """hi / lo equal gps_to_planes of the returned C, remapped for the per-head layout; pads 0; nothing else touched."""
    M, N = run.M, run.N
    lo = run.prec == 0
    want, _ = _planes_of(run.C, lo)
    Cp = run.Cp
    assert (Cp[2] == SENTINEL16).all(), "written past the planes"
    if not lo:
        assert (Cp[1] == SENTINEL16).all(), "lo plane written in bf16 mode with lo = NULL"
    planes = (0, 1) if lo else (0,)
    width = run.cp_width
    assert (Cp[:, :, width:] == SENTINEL16).all(), "planes written past the layout's width"
    if run.cp_hd == 0:
        for pl in planes:
            assert torch.equal(Cp[pl, :, :N], want[pl, :, :N]), f"plane {pl} differs from to_planes(C)"
        return
    hd, hp = run.cp_hd, run.cp_pad
    cols = torch.arange(N, device=DEV)
    pcol = cols // hd * hp + cols % hd
    pads = torch.tensor([h * hp + k for h in range(N // hd) for k in range(hd, hp)], dtype=torch.long, device=DEV)
    for pl in planes:
        assert torch.equal(Cp[pl][:, pcol], want[pl, :, :N]), f"plane {pl} differs from the remapped to_planes(C)"
        if pads.numel():
            assert (Cp[pl][:, pads] == 0).all(), f"plane {pl}: head pad columns are not zero"


def _forced(bn):
    _lib.load().gps_debug_tma(bn, 0)


def _widths(spec):
    """Every tile width the TMA kernel takes for this layout (A is K-major throughout: 256 always; 152 needs a
    K-major B), then the policy's choice again."""
    return (0, 64, 128, 256, 0) if spec.tb else (0, 64, 128, 152, 256, 0)


def _exact_data(spec):
    return spec.act != GELU and spec.mask != "gelu_pre" and all(
        p == 0 or _keep_scale(p) in (2.0, 4.0) for p in (spec.p, spec.p2))


def _run_recipe(spec, kernel, precision, M, N, K, seed=0):
    """Runs spec on one kernel and checks it; on the TMA kernel once per width, all widths bitwise equal."""
    impl = KERNELS[kernel]
    prec = PRECISIONS[precision]
    if kernel != "tma":
        run = Run(spec, M, N, K, prec, seed)
        rc = run.call(impl, with_cp=False)   # the fp32 kernels never write planes (gps_gemm_epilogue refuses Cp)
        if rc == _lib.GPS_ERR_UNSUPPORTED:
            pytest.skip(f"{kernel} does not take this shape: {_lib.load().gps_last_error().decode()}")
        _lib.check(rc, spec.name)
        _check(run, kernel)
        return run
    outs, ran = {}, None
    try:
        for i, bn in enumerate(_widths(spec)):
            _forced(bn)
            run = Run(spec, M, N, K, prec, seed)
            rc = run.call(impl)
            assert rc != _lib.GPS_ERR_UNSUPPORTED or bn != 0, _lib.load().gps_last_error()
            if rc == _lib.GPS_ERR_UNSUPPORTED:
                continue
            _lib.check(rc, f"{spec.name} bn={bn}")
            _check(run, kernel)
            # the float64 atomics of the statistics add the row tiles' partials in any order: bitwise only when every
            # partial sum is exact (exact-operand epilogues without GELU or an inexact keep scale)
            outs[bn if bn not in outs else f"{bn} again"] = run.outputs(stats=_exact_data(spec))
            ran = run
    finally:
        _forced(0)
    first = outs[0]
    for bn, res in outs.items():
        for j, (x, y) in enumerate(zip(res, first)):
            assert _bitwise_equal(x, y), f"width {bn}: output {j} differs from the policy's width"
    return ran


def _bitwise_equal(x, y):
    """Bitwise equality that counts NaN sentinels as equal."""
    if x.dtype in (torch.float32, torch.float64):
        it = torch.int32 if x.dtype == torch.float32 else torch.int64
        return torch.equal(x.contiguous().view(it), y.contiguous().view(it))
    return torch.equal(x, y)


# ---------------------------------------------------------------------------------------------------- recipes
def qkv_planes(hd):
    """layer.cu Q|K|V projection and graphormer.cu in_proj: bias, fp32 C, and the planes in the per-head padded
    layout the wgmma attention reads."""
    return Spec(f"qkv_planes(hd={hd})", bias=True, cp=hd)


def ff1_fwd(act, p):
    """layer.cu / graphormer.cu / custom_gnn.cu first FFN Linear: bias, act, the pre-activation copy, planes, dropout."""
    return Spec(f"ff1_fwd(act={act}, p={p})", bias=True, act=act, c_pre=True, cp="identity", p=p, site=SITE_FF1,
                offset_dev=True)


def out_proj_stats(p, r2):
    """layer.cu / san.cu output projections: bias, dropout, the residual x (and the local branch), BatchNorm sums."""
    return Spec(f"out_proj_stats(p={p}, r2={r2})", bias=True, p=p, site=SITE_ATTN_OUT, r1=True, r2=r2, stats=True,
                offset_dev=True)


def performer_out(p2=0.5, p=0.75, r1=True):
    """layer.cu Performer to_out: SelfAttention's dropout (site2) inside GPSLayer.dropout_attn (site), residual, sums."""
    return Spec(f"performer_out(p2={p2}, p={p}, r1={r1})", bias=True, p2=p2, site2=SITE_PERF_OUT, p=p,
                site=SITE_ATTN_OUT, r1=r1, stats=True)


def dgrad_mask(kind, p=0.5):
    """layer.cu / graphormer.cu FFN data gradient: g W (tb = 1) times act'(saved activation), dropout, planes."""
    return Spec(f"dgrad_mask({kind}, p={p})", tb=1, mask=kind, p=p, site=SITE_FF1, cp="identity", offset_dev=True)


def dgrad_inplace():
    """layer.cu Performer g_q += g_dd Pn: R1 is the output buffer itself."""
    return Spec("dgrad_inplace", tb=1, r1="alias")


def dgrad_splitk():
    """layer.cu grad_x = gY Wcat + g_x_local + g_hA: split-K 4 into a pre-zeroed C with two residuals."""
    return Spec("dgrad_splitk", tb=1, r1=True, r2=True, splitk=4)


kernel_param = pytest.mark.parametrize("kernel", list(KERNELS))
precision_param = pytest.mark.parametrize("precision", list(PRECISIONS))
shape_param = pytest.mark.parametrize("M,N,K", SHAPES)


# hd 16, 24, 64, 76, 128 with 4, 4, 4, 4, 2 heads (N = 3 H hd); 24 and 76 have pad columns
@kernel_param
@precision_param
@pytest.mark.parametrize("hd,M,K,heads", [(16, 13, 64, 4), (24, 129, 72, 4), (64, 1, 304, 4), (76, 3620, 304, 4),
                                          (128, 128, 304, 2)])
def test_qkv_planes(kernel, precision, hd, M, K, heads):
    _run_recipe(qkv_planes(hd), kernel, precision, M, 3 * heads * hd, K)


@kernel_param
@precision_param
@shape_param
@pytest.mark.parametrize("act", ["relu", "gelu"])
@pytest.mark.parametrize("p", [0.0, 0.75])
def test_ff1_fwd(kernel, precision, M, N, K, act, p):
    _run_recipe(ff1_fwd(_lib.ACT[act], p), kernel, precision, M, N, K)


@kernel_param
@precision_param
@shape_param
@pytest.mark.parametrize("p", [0.0, 0.5])
@pytest.mark.parametrize("r2", [False, True])
def test_out_proj_stats(kernel, precision, M, N, K, p, r2):
    _run_recipe(out_proj_stats(p, r2), kernel, precision, M, N, K)


@kernel_param
@pytest.mark.parametrize("M,N,K", [(3620, 304, 304), (129, 1000, 72)])
def test_out_proj_stats_layer_dropout(kernel, M, N, K):
    """p = 0.1, the layers' value: the keep scale 1/0.9 rounds, so C is within 1 ulp of the float64 value."""
    _run_recipe(out_proj_stats(0.1, False), kernel, "fp32", M, N, K)


@kernel_param
@precision_param
@shape_param
def test_performer_out(kernel, precision, M, N, K):
    _run_recipe(performer_out(), kernel, precision, M, N, K)


@kernel_param
@pytest.mark.parametrize("M,N,K", [(3620, 304, 304), (129, 1000, 72)])
def test_performer_out_site2_applies_first(kernel, M, N, K):
    """Both keep scales inexact (p2 = 0.1, p = 0.3) and no residual after them: (x s2) s and (x s) s2 round differently,
    so the bitwise float32 replay in the documented order (site2, then site) tells the two orders apart."""
    spec = performer_out(0.1, 0.3, r1=False)
    run = _run_recipe(spec, kernel, "fp32", M, N, K)
    # the check is only meaningful if the other order gives other bits somewhere
    v = run.replay()[2]
    m2 = _dropout_mask(M, N, 0.1, SITE_PERF_OUT, OFFSET) * _keep_scale(0.1)
    m1 = _dropout_mask(M, N, 0.3, SITE_ATTN_OUT, OFFSET) * _keep_scale(0.3)
    assert not torch.equal((v * m2) * m1, (v * m1) * m2)


@kernel_param
@precision_param
@shape_param
@pytest.mark.parametrize("kind", ["relu_post", "gelu_pre"])
@pytest.mark.parametrize("p", [0.0, 0.5])
def test_dgrad_mask(kernel, precision, M, N, K, kind, p):
    _run_recipe(dgrad_mask(kind, p), kernel, precision, M, N, K)


@kernel_param
@precision_param
@shape_param
def test_dgrad_inplace(kernel, precision, M, N, K):
    _run_recipe(dgrad_inplace(), kernel, precision, M, N, K)


@kernel_param
@precision_param
@shape_param
def test_dgrad_splitk(kernel, precision, M, N, K):
    _run_recipe(dgrad_splitk(), kernel, precision, M, N, K)


# ---------------------------------------------------------------------------------------------------- dropout masks
@kernel_param
def test_forward_and_backward_draw_the_same_mask(kernel):
    """ff1_fwd (forward) and dgrad_mask (backward) at the same (M, N, seed, offset, site) drop the same elements:
    where the value before dropout is non-zero in both runs, an element survives in one iff it survives in the other."""
    M, N, K = 1000, 608, 72
    known, kept = [], []
    for run in (Run(ff1_fwd(RELU, 0.5), M, N, K, 0, seed=1), Run(dgrad_mask("relu_post"), M, N, K, 0, seed=2)):
        _lib.check(run.call(KERNELS[kernel], with_cp=kernel == "tma"), run.s.name)
        run.s.p = 0.0
        known.append(run.replay()[0] != 0)
        kept.append(run.C != 0)
    both = known[0] & known[1]
    assert both.float().mean() > 0.2
    assert torch.equal(kept[0][both], kept[1][both])
    mask = _dropout_mask(M, N, 0.5, SITE_FF1, OFFSET + OFFSET_DEV) != 0
    assert torch.equal(kept[0][both], mask[both])


def test_three_kernels_give_identical_results():
    """The same exact-operand epilogue with both dropout sites on all three kernels: bitwise the same C and planes
    wherever a kernel writes them (hence the same dropout masks)."""
    spec = performer_out()
    res = []
    for kernel in KERNELS:
        run = Run(spec, 3620, 304, 304, 0)
        _lib.check(run.call(KERNELS[kernel], with_cp=False), kernel)
        res.append(run.C.clone())
    assert all(torch.equal(r, res[0]) for r in res[1:])


# ---------------------------------------------------------------------------------------------------- random operands
@kernel_param
@precision_param
@pytest.mark.parametrize("M,N,K", [(3620, 304, 304), (3620, 608, 304)])
def test_random_operands_at_layer_shapes(kernel, precision, M, N, K):
    """Gaussian operands with non-zero lo planes at the d = 304 shapes (out_proj and ff1), against float64 at the
    tolerances of test_gemm_schedule_gpu.py: the exact-operand choice above hides nothing in the lo-plane products."""
    spec = Spec("random", bias=True, r1=True, stats=True, cp="identity")
    run = Run(spec, M, N, K, PRECISIONS[precision], seed=7, random=True)
    rc = run.call(KERNELS[kernel], with_cp=kernel == "tma")
    _lib.check(rc, f"random {kernel}")
    ref = run.A.double() @ run.B.double().t() + run.bias.double() + run.R1.double()
    tol = 2e-5 * max(1.0, K ** 0.5 / 8) if precision == "fp32" else 2e-2
    assert rel_err(run.C, ref) < tol
    _check_stats(run, kernel)
    if kernel == "tma":
        _check_planes(run)


# ---------------------------------------------------------------------------------------------------- refusals
def _small_run(spec, prec=0):
    return Run(spec, 128, 64, 64, prec)


@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("field", ["bias", "act", "mask", "stats", "c_pre", "p", "p2"])
def test_splitk_refuses_a_fused_epilogue(kernel, field):
    kw = {"bias": {"bias": True}, "act": {"act": RELU}, "mask": {"mask": "relu_post"}, "stats": {"stats": True},
          "c_pre": {"c_pre": True}, "p": {"p": 0.5, "site": 5}, "p2": {"p2": 0.5, "site2": 7}}[field]
    run = _small_run(Spec("splitk+" + field, splitk=4, **kw))
    before = run.outputs()
    assert run.call(KERNELS[kernel], with_cp=False) == _lib.GPS_ERR_ARG
    assert all(_bitwise_equal(x, y) for x, y in zip(run.outputs(), before)), "refused, but wrote"


def test_splitk_refuses_planes_on_tma():
    run = _small_run(Spec("splitk+Cp", splitk=4, cp="identity"))
    assert run.call(KERNELS["tma"]) == _lib.GPS_ERR_ARG


@pytest.mark.parametrize("kernel", list(KERNELS))
def test_colsum_needs_transposed_a(kernel):
    run = _small_run(Spec("colsum"))
    a = run.args(with_cp=False)
    colsum = torch.zeros(128, device=DEV)
    a.colsum_a = colsum.data_ptr()
    assert _lib.load().gps_gemm_epilogue(C.byref(a), KERNELS[kernel], _stream()) == _lib.GPS_ERR_ARG


# ---------------------------------------------------------------------------------------------------- dispatcher
def _rejected_by_tma(run):
    """fp32-grade precision with A's lo plane missing: the TMA kernel rejects the product and the dispatcher falls back
    to the fp32 kernels."""
    a = run.args()
    a.Ap = _lib.GpsPlanes(run.Ap[0].data_ptr(), 0, run.lda_p)
    return a


@pytest.mark.parametrize("M,N,K", [(129, 304, 72), (3620, 912, 304)])
def test_dispatcher_fallback_converts_identity_planes(M, N, K):
    run = Run(Spec("fallback", bias=True, cp="identity"), M, N, K, 0)
    rc = _lib.load().gps_gemm_epilogue(C.byref(_rejected_by_tma(run)), 0, _stream())
    torch.cuda.synchronize()
    _lib.check(rc, "dispatcher fallback")
    _check(run, "tc")
    _check_planes(run)


def test_dispatcher_fallback_refuses_per_head_planes():
    """The fallback converts C with to_planes, which writes the identity layout: a per-head padded Cp (the attention's
    Q|K|V) would be read with heads at the wrong columns and unwritten pads, so the dispatcher refuses it."""
    run = Run(qkv_planes(76), 129, 912, 72, 0)
    before = run.outputs()
    rc = _lib.load().gps_gemm_epilogue(C.byref(_rejected_by_tma(run)), 0, _stream())
    torch.cuda.synchronize()
    assert rc == _lib.GPS_ERR_UNSUPPORTED
    assert b"M=129 N=912 K=72" in _lib.load().gps_last_error()
    assert all(_bitwise_equal(x, y) for x, y in zip(run.outputs(), before)), "refused, but wrote"
