"""GPU: the softmax attention stages (csrc/attention.cu, csrc/attention_tc.cu) one by one through gps_attention_stage,
against the float64 restatement of tests/attention_reference.py with the kernels' dropout mask replayed on the host.

  * The host Philox replica equals gps_dropout_mask bit for bit, and the attention kernels' own keep decisions, read
    out through one-hot V (forward) and one-hot dO (the key-major backward pass), equal the replica's.
  * Every (VW, CH, LPR) instantiation of the CUDA-core forward and backward, biased and unbiased, at p = 0 and 0.5;
    float4 rows forced to scalar through odd leading dimensions, and the float4-forward / scalar-backward mix.
  * Batches: the BASELINE shapes, empty and single-node graphs, B = 1, one 3000-node graph, fewer rows than a warp
    holds, N not a multiple of 128, scores up to |s| ~ 60, all-equal scores; the wgmma forward at every head dim that
    is a multiple of 4 up to 128, in fp32-grade and bf16, over CTAs that start mid-graph and span many graphs.
  * Per-element bounds (attention_reference.fwd_bounds / bwd_bounds); the worst error as a fraction of its bound is
    printed per stage.  Outputs start as NaN inside wider buffers and input pitch padding (and padded bias entries)
    hold NaN, so stray writes, missing writes and reads past the declared columns all show.
  * The O planes (both forwards) and the dQ / dK / dV planes equal gps_to_planes of the fp32 outputs bit for bit.
  * The wgmma forward followed by the CUDA-core backward, as the layer runs them at large graphs; two runs bitwise
    equal; refusals before any CUDA call."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import attention_reference as ar
from graphgps_b200 import _lib
from graphgps_b200.batch import batch_from_lists, make_batch
from graphgps_b200.graph import graph_of
from util import _elem_check, _stream

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 0x5EED1234ABCD
OFFSET = 4096 * 5
WORST = {}
BF16_NAN = 0x7FC0
CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "graphgps_b200", "csrc")


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst error / bound per stage:")
    for k in sorted(WORST):
        print(f"  {k:28s} {WORST[k]:.3g}")


def _lib_():
    return _lib.load()


def _ru(x, a):
    return (x + a - 1) // a * a


# ------------------------------------------------------------------------------------------------ harness
class Case:
    """A batch on the device with its graph descriptor, its node offsets on the host and the attention geometry."""

    def __init__(self, b, H, hd, seed=0):
        self.b = b.to(DEV)
        self.gs = graph_of(self.b)
        self.ptr = np.concatenate([[0], np.cumsum(torch.bincount(b.batch.cpu(), minlength=b.num_graphs).numpy())])
        self.N, self.B, self.H, self.hd, self.D = int(self.ptr[-1]), b.num_graphs, H, hd, H * hd
        self.nmax = max(1, int((self.ptr[1:] - self.ptr[:-1]).max()) if self.B else 1)
        self.gen = torch.Generator(device=DEV).manual_seed(seed)

    def randn(self, *shape):
        return torch.randn(*shape, generator=self.gen, device=DEV)


def _sizes(sizes, H, hd, seed=0):
    return Case(batch_from_lists(sizes, [[] for _ in sizes], d=8), H, hd, seed)


def _shape(shape, B, H, hd, seed=0):
    return Case(make_batch(shape, seed=4, dim=8, num_graphs=B), H, hd, seed)


def _nanbuf(rows, cols, dtype=torch.float32):
    if dtype == torch.bfloat16:
        return torch.full((rows, cols), BF16_NAN, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    return torch.full((rows, cols), float("nan"), dtype=dtype, device=DEV)


def _inputs(c, ld, scale=1.0, equal_keys=False):
    """Q | K | V in a [N + 1, ld] buffer whose pad columns and extra row are NaN."""
    buf = _nanbuf(c.N + 1, ld)
    qkv = c.randn(c.N, 3 * c.D)
    qkv[:, :2 * c.D] *= scale
    if equal_keys:   # every key of a head equal: all scores of a row equal
        qkv[:, c.D:2 * c.D] = qkv[:1, c.D:2 * c.D]
    buf[:c.N, :3 * c.D] = qkv
    return buf


def _bias(c):
    """[B*H, nmax, nmax] bias whose entries outside each graph are NaN (never read)."""
    ab = _nanbuf(c.B * c.H * c.nmax, c.nmax).view(c.B * c.H, c.nmax, c.nmax)
    for g in range(c.B):
        n = int(c.ptr[g + 1] - c.ptr[g])
        ab[g * c.H:(g + 1) * c.H, :n, :n] = 2 * c.randn(c.H, n, n)
    return ab


def _planes_buf(rows, cols, lo=True):
    ldp = _ru(cols, 8) + 8
    return _nanbuf(rows, ldp, torch.bfloat16), (_nanbuf(rows, ldp, torch.bfloat16) if lo else None), ldp


def _gp(hi, lo, ld, col=0):
    return _lib.GpsPlanes(hi.data_ptr() + 2 * col, 0 if lo is None else lo.data_ptr() + 2 * col, ld)


def _stage(c, op, **f):
    a = _lib.GpsAttnStageArgs()
    a.graph = c.gs.desc
    a.heads, a.hd, a.seed = c.H, c.hd, SEED
    for k, v in f.items():
        setattr(a, k, v)
    _lib.check(_lib_().gps_attention_stage(C.byref(a), _lib.ATTN[op], _stream()), "gps_attention_stage " + op)


def _bias_arg(c, ab, gb=None):
    if ab is None:
        return None
    return C.pointer(_lib.GpsAttnBias(ab.data_ptr(), c.nmax, 0 if gb is None else gb.data_ptr()))


def _to_planes(x):
    """gps_to_planes of an fp32 [rows, cols] tensor: (hi, lo) as int16 bit patterns [rows, cols]."""
    rows, cols = x.shape
    src = torch.zeros(rows, _ru(cols, 4), device=DEV)
    src[:, :cols] = x
    ldp = _ru(cols, 8)
    hi = torch.empty(rows, ldp, dtype=torch.bfloat16, device=DEV)
    lo = torch.empty(rows, ldp, dtype=torch.bfloat16, device=DEV)
    if rows:
        _lib.check(_lib_().gps_to_planes(src.data_ptr(), src.shape[1], rows, cols, hi.data_ptr(), lo.data_ptr(), ldp,
                                         _stream()), "gps_to_planes")
    return hi[:, :cols].view(torch.int16), lo[:, :cols].view(torch.int16)


def _check_planes(name, hi, lo, x, col0, cols):
    """Planes [N+1, ldp] hold exactly gps_to_planes(x) in columns [col0, col0 + cols); the extra row stays NaN."""
    N = x.shape[0]
    whi, wlo = _to_planes(x)
    assert torch.equal(hi[:N, col0:col0 + cols].view(torch.int16), whi), name + ": hi plane differs"
    assert bool((hi[N].view(torch.int16) == BF16_NAN).all()), name + ": hi plane written past N"
    if lo is not None:
        assert torch.equal(lo[:N, col0:col0 + cols].view(torch.int16), wlo), name + ": lo plane differs"


def _untouched(name, buf, rows, cols):
    """The region outside [:rows, :cols] of a NaN-initialised buffer is still NaN."""
    pad = torch.ones_like(buf, dtype=torch.bool)
    pad[:rows, :cols] = False
    assert bool(torch.isnan(buf[pad].float()).all()), name + ": written outside its rows / columns"


# ------------------------------------------------------------------------------------------------ stage runners
def _fwd(c, qkv, ld, p, ab=None, offset=OFFSET, offset_dev=None, planes_lo=True, ldo=None):
    D, N = c.D, c.N
    ldo = D + 4 if ldo is None else ldo
    O, lse = _nanbuf(N + 1, ldo), _nanbuf(N + 1, c.H)
    hi, lo, ldp = _planes_buf(N + 1, D, planes_lo)
    base = qkv.data_ptr()
    _stage(c, "fwd", Q=base, K=base + 4 * D, V=base + 8 * D, ld=ld, O=O.data_ptr(), ldo=ldo, lse=lse.data_ptr(),
           O_planes=_gp(hi, lo, ldp), p_drop=p, offset=offset, offset_dev=offset_dev, bias=_bias_arg(c, ab))
    return O, lse, hi, lo


def _fwd_tc(c, qkv, p, precision, ab=None, offset=OFFSET, offset_dev=None, extra=8):
    D, N = c.D, c.N
    planes, ld = ar.padded_planes(qkv[:N, :3 * D], c.H, c.hd, extra)
    ldo = D + 5
    O, lse = _nanbuf(N + 1, ldo), _nanbuf(N + 1, c.H)
    hi, lo, ldp = _planes_buf(N + 1, D, precision == 0)
    _stage(c, "fwd_tc", qkv=_lib.GpsPlanes(planes[0].data_ptr(), planes[1].data_ptr() if precision == 0 else 0, ld),
           precision=precision, O=O.data_ptr(), ldo=ldo, lse=lse.data_ptr(), O_planes=_gp(hi, lo, ldp), p_drop=p,
           offset=offset, offset_dev=offset_dev, bias=_bias_arg(c, ab))
    return O, lse, hi, lo


def _bwd(c, qkv, ld, O_in, lse_in, dO, p, ab=None, ldo=None, ldg=None, planes_lo=True):
    """The CUDA-core backward from fp32 O_in [N, D], lse_in [N, H] and dO [N, D]; returns the raw output buffers."""
    D, N = c.D, c.N
    ldo = D + 2 if ldo is None else ldo
    ldg = 3 * D + 4 if ldg is None else ldg
    Ob, dOb = _nanbuf(N + 1, ldo), _nanbuf(N + 1, ldo)
    Ob[:N, :D], dOb[:N, :D] = O_in, dO
    lse = lse_in.contiguous()
    g, delta = _nanbuf(N + 1, ldg), _nanbuf(N + 1, c.H)
    hi, lo, ldp = _planes_buf(N + 1, 3 * D, planes_lo)
    gb = None if ab is None else torch.full_like(ab, float("nan"))
    base, gbase = qkv.data_ptr(), g.data_ptr()
    _stage(c, "bwd", Q=base, K=base + 4 * D, V=base + 8 * D, ld=ld, O=Ob.data_ptr(), dO=dOb.data_ptr(), ldo=ldo,
           lse=lse.data_ptr(), delta=delta.data_ptr(), dQ=gbase, dK=gbase + 4 * D, dV=gbase + 8 * D, ldg=ldg,
           dQ_planes=_gp(hi, lo, ldp, 0), dK_planes=_gp(hi, lo, ldp, D), dV_planes=_gp(hi, lo, ldp, 2 * D), p_drop=p,
           offset=OFFSET, bias=_bias_arg(c, ab, gb))
    return g, delta, hi, lo, gb


def _ref64(c, qkv, p, ab=None, offset=OFFSET):
    D = c.D
    Q, K, V = (qkv[:c.N, i * D:(i + 1) * D].double().requires_grad_(True) for i in range(3))
    b64 = None if ab is None else torch.nan_to_num(ab.double(), nan=0.0).requires_grad_(True)
    keep = ar.keep_masks(c.ptr, c.H, p, SEED, offset, DEV)
    O, lse = ar.attention(Q, K, V, c.ptr, c.H, c.hd, b64, keep, p)
    return Q, K, V, b64, keep, O, lse


def _check_fwd(tag, c, O, lse, ref, p, tc_precision=None):
    Q, K, V, b64, keep, O64, lse64 = ref
    D, N = c.D, c.N
    with torch.no_grad():
        bO, bl = ar.fwd_bounds(Q, K, V, c.ptr, c.H, c.hd, b64, keep, p, tc_precision)
    _elem_check(WORST, tag + " O", O[:N, :D], O64.detach(), bO)
    _elem_check(WORST, tag + " lse", lse[:N], lse64.detach(), bl)
    _untouched(tag + " O", O, N, D)
    _untouched(tag + " lse", lse, N, c.H)


def _run_fwd_bwd(tag, c, ld, p, biased, planes_lo=True, ldo=None, ldg=None, scale=1.0, equal_keys=False):
    """CUDA-core forward and backward of one case against float64; the planes of both; returns the raw outputs."""
    qkv = _inputs(c, ld, scale, equal_keys)
    ab = _bias(c) if biased else None
    ref = _ref64(c, qkv, p, ab)
    O, lse, ohi, olo = _fwd(c, qkv, ld, p, ab, planes_lo=planes_lo, ldo=ldo)
    _check_fwd(tag + " fwd", c, O, lse, ref, p)
    _check_planes(tag + " O planes", ohi, olo, O[:c.N, :c.D], 0, c.D)
    Q, K, V, b64, keep, O64, lse64 = ref
    dO = c.randn(c.N, c.D)
    (O64 * dO.double()).sum().backward()
    O_in, lse_in = O64.detach().float(), lse64.detach().float()
    g, delta, hi, lo, gb = _bwd(c, qkv, ld, O_in, lse_in, dO, p, ab, ldo, ldg, planes_lo)
    D, N = c.D, c.N
    with torch.no_grad():
        bq, bk, bv, bgb = ar.bwd_bounds(Q, K, V, dO.double(), c.ptr, c.H, c.hd, b64, keep, p)
        dl64 = (dO.double() * O_in.double()).reshape(N, c.H, c.hd).sum(-1)
        bdl = 2 * (c.hd + 8) * ar.U * (dO.double().abs() * O_in.double().abs()).reshape(N, c.H, c.hd).sum(-1)
    _elem_check(WORST, tag + " delta", delta[:N], dl64, bdl)
    _elem_check(WORST, tag + " dQ", g[:N, :D], Q.grad, bq)
    _elem_check(WORST, tag + " dK", g[:N, D:2 * D], K.grad, bk)
    _elem_check(WORST, tag + " dV", g[:N, 2 * D:3 * D], V.grad, bv)
    _untouched(tag + " dQKV", g, N, 3 * D)
    _untouched(tag + " delta", delta, N, c.H)
    for i, name in enumerate(("dQ", "dK", "dV")):
        _check_planes(f"{tag} {name} planes", hi, lo, g[:N, i * D:(i + 1) * D], i * D, D)
    if ab is not None:
        _elem_check(WORST, tag + " grad_bias", gb, b64.grad, bgb)   # padded entries: bound 0, so exactly 0
    return O, lse, g, gb


# ------------------------------------------------------------------------------------------------ the dropout stream
@pytest.mark.parametrize("p", [0.1, 0.5, 0.9])
@pytest.mark.parametrize("offset", [0, 4096 * 3 + 1, (1 << 40) + 7])
@pytest.mark.parametrize("site", [3, 16, 19, 4095])
def test_host_philox_replica_equals_gps_dropout_mask(p, offset, site):
    rows, cols = 37, 52
    m = torch.empty(rows, cols, device=DEV)
    _lib.check(_lib_().gps_dropout_mask(m.data_ptr(), rows, cols, p, SEED, offset, site, _stream()), "mask")
    assert torch.equal(m.cpu(), torch.from_numpy(ar.dropout_mask(rows, cols, p, SEED, offset, site)))


def _mask_case(n_graphs=3, n=128, H=4):
    """Graphs of n nodes, hd = n: Q = 0 (uniform probabilities 1/n), V and dO one-hot in the node's local index, so
    O_i = keep_i. / ((1 - p) n) and dV_j = keep_.j / ((1 - p) n) read the kernels' masks out directly."""
    c = _sizes([n] * n_graphs, H, n, seed=5)
    qkv = torch.zeros(c.N + 1, 3 * c.D, device=DEV)
    eye = torch.eye(n, device=DEV).repeat(n_graphs, 1)
    for h in range(H):
        qkv[:c.N, 2 * c.D + h * n:2 * c.D + (h + 1) * n] = eye
    dO = torch.cat([eye] * H, 1)
    return c, qkv, dO


def _masks_from(c, X, p, n):
    """[B, H, n, n] keep decisions from the one-hot read-out X [N, H*n]."""
    k = (X[:c.N, :c.D].double() * (1 - p) * n).reshape(c.B, n, c.H, n).permute(0, 2, 1, 3)
    assert bool(((k - k.round()).abs() < 1e-2).all()) and bool(((k.round() == 0) | (k.round() == 1)).all())
    return k.round().bool()


def _replica(c, p, offset, n):
    keep = ar.keep_masks(c.ptr, c.H, p, SEED, offset, DEV)
    return torch.stack(keep)


@pytest.mark.parametrize("p", [0.1, 0.5, 0.9])
def test_kernel_masks_equal_the_replica_and_keep_rate(p):
    n = 128
    c, qkv, dO = _mask_case(n=n)
    want = _replica(c, p, OFFSET, n)
    O, _, _, _ = _fwd(c, qkv, 3 * c.D, p)
    assert torch.equal(_masks_from(c, O, p, n), want), "CUDA-core forward mask"
    for prec in (0, 1):
        O2, _, _, _ = _fwd_tc(c, qkv, p, prec)
        assert torch.equal(_masks_from(c, O2, p, n), want), f"wgmma forward mask (precision {prec})"
    # key-major backward pass: with dO one-hot, dV_j = sum_i P_ij keep_ij / (1 - p) dO_i = keep_.j / ((1 - p) n)
    lse = torch.full((c.N, c.H), float(np.log(n)), device=DEV)
    g, _, _, _, _ = _bwd(c, qkv, 3 * c.D, torch.zeros(c.N, c.D, device=DEV), lse, dO, p)
    dV = g[:c.N, 2 * c.D:3 * c.D]
    assert torch.equal(_masks_from(c, dV, p, n).transpose(2, 3), want), "key-major backward mask"
    # keep rate per head: binomial, 6 standard deviations
    cnt = c.B * n * n
    rate = want.double().mean((0, 2, 3))
    sd = (p * (1 - p) / cnt) ** 0.5
    assert bool(((rate - (1 - p)).abs() < 6 * sd).all()), rate
    # heads and offsets draw different masks
    for h in range(1, c.H):
        assert not torch.equal(want[:, h], want[:, 0])
    other = _replica(c, p, OFFSET + 4096, n)
    assert not torch.equal(other, want)
    O3, _, _, _ = _fwd(c, qkv, 3 * c.D, p, offset=OFFSET + 4096)
    assert torch.equal(_masks_from(c, O3, p, n), other)


def test_offset_dev_adds_to_the_host_offset():
    n, p = 64, 0.5
    c, qkv, dO = _mask_case(n_graphs=2, n=n, H=2)
    dev_off = torch.tensor([4096 * 7 + 3], dtype=torch.int64, device=DEV)
    want = _replica(c, p, OFFSET + 4096 * 7 + 3, n)
    assert not torch.equal(want, _replica(c, p, OFFSET, n))
    O, _, _, _ = _fwd(c, qkv, 3 * c.D, p, offset_dev=dev_off.data_ptr())
    assert torch.equal(_masks_from(c, O, p, n), want), "CUDA-core forward"
    O2, _, _, _ = _fwd_tc(c, qkv, p, 0, offset_dev=dev_off.data_ptr())
    assert torch.equal(_masks_from(c, O2, p, n), want), "wgmma forward"
    lse = torch.full((c.N, c.H), float(np.log(n)), device=DEV)
    D, N = c.D, c.N
    Ob, dOb = torch.zeros(N, D, device=DEV), dO.contiguous()
    g, delta = _nanbuf(N, 3 * D), _nanbuf(N, c.H)
    base, gbase = qkv.data_ptr(), g.data_ptr()
    _stage(c, "bwd", Q=base, K=base + 4 * D, V=base + 8 * D, ld=3 * D, O=Ob.data_ptr(), dO=dOb.data_ptr(), ldo=D,
           lse=lse.data_ptr(), delta=delta.data_ptr(), dQ=gbase, dK=gbase + 4 * D, dV=gbase + 8 * D, ldg=3 * D,
           p_drop=p, offset=OFFSET, offset_dev=dev_off.data_ptr())
    assert torch.equal(_masks_from(c, g[:, 2 * D:], p, n).transpose(2, 3), want), "key-major backward"


# ------------------------------------------------------------------------------------------------ instantiations
def _kernel_of(hd, vec4):
    vw = 4 if vec4 and hd % 4 == 0 else 1
    nch = hd // vw
    lpr = 1
    while -(-nch // lpr) > 6:
        lpr *= 2
    return vw, -(-nch // lpr), lpr


def _dispatch_table():
    src = open(os.path.join(CSRC, "attention.cu")).read()
    return {tuple(int(x) for x in m) for m in re.findall(r"GPS_ATTN_CASE\((\d+), (\d+), (\d+)\)", src)}


def _one_hd_per_kernel():
    """One head dim per (VW, CH, LPR): the smallest, preferring one where CH * LPR exceeds the chunk count (the lanes'
    last chunks fall past the head) and, for VW = 1, one that is not a multiple of 4.  VW = 1 at a multiple of 4 is
    reached through an odd leading dimension."""
    cands = {}
    for hd in range(1, 193):
        for vec4 in ((True, False) if hd % 4 == 0 else (False,)):
            k = _kernel_of(hd, vec4)
            nch = hd // k[0]
            cands.setdefault(k, []).append(((not vec4 and hd % 4 == 0), nch == k[1] * k[2], hd, vec4))
    return {k: min(v)[2:] for k, v in cands.items()}


PICK = _one_hd_per_kernel()


def test_the_chosen_head_dims_cover_the_dispatch_table():
    table = _dispatch_table()
    assert len(table) == 36
    assert set(PICK) == table
    assert {_kernel_of(hd, v) for hd in range(1, 193) for v in (True, False)} == table


def _inst_params():
    out = []
    for k, (hd, vec4) in sorted(PICK.items()):
        mode = "vec" if vec4 else ("odd_ld" if hd % 4 == 0 else "scalar")
        out.append(pytest.param(hd, mode, id=f"VW{k[0]}_CH{k[1]}_LPR{k[2]}_hd{hd}"))
    # float4 head dims forced to scalar rows: through ld, through ldo, and only through ldg (float4 forward, scalar
    # backward)
    out += [pytest.param(64, "odd_ld", id="hd64_odd_ld"), pytest.param(64, "odd_ldo", id="hd64_odd_ldo"),
            pytest.param(76, "odd_ldg", id="hd76_odd_ldg_fwd_vec_bwd_scalar")]
    return out


@pytest.mark.parametrize("hd,mode", _inst_params())
def test_every_instantiation_forward_backward(hd, mode):
    H = 2
    c = _sizes([3, 0, 17, 1, 40, 9, 0], H, hd, seed=hd)
    D = c.D
    ld = 3 * D + (4 if mode == "vec" else 1 if mode in ("odd_ld", "scalar") else 4)
    ldo = D + (1 if mode == "odd_ldo" else 4)
    ldg = 3 * D + (1 if mode == "odd_ldg" else 4)
    if mode == "scalar":
        ldo, ldg = D + 1, 3 * D + 1
    fwd_vw = 4 if hd % 4 == 0 and ld % 4 == 0 and ldo % 4 == 0 else 1
    bwd_vw = 4 if fwd_vw == 4 and ldg % 4 == 0 else 1
    assert (fwd_vw, bwd_vw) == {"vec": (4, 4), "scalar": (1, 1), "odd_ld": (1, 1), "odd_ldo": (1, 1),
                                "odd_ldg": (4, 1)}[mode]
    for biased in (False, True):
        for p in (0.0, 0.5):
            _run_fwd_bwd(f"inst hd{hd} {mode} b{int(biased)} p{p}", c, ld, p, biased, ldo=ldo, ldg=ldg,
                         planes_lo=not biased)


# ------------------------------------------------------------------------------------------------ batches
def _batch_run(tag, c, p, scale=1.0, equal_keys=False, cuda_core=True, precisions=(0, 1)):
    """The CUDA-core forward and backward, and the wgmma forward (when it takes the head dim) in the given
    precisions, of one batch at attention dropout p; returns the forward outputs by kernel."""
    ld = 3 * c.D + 4
    out = {}
    if cuda_core:
        out["cc"] = _run_fwd_bwd(f"{tag} p{p}", c, ld, p, False, scale=scale, equal_keys=equal_keys)[:2]
    if c.hd % 4 == 0 and c.hd <= 128 and precisions:
        qkv = _inputs(c, ld, scale, equal_keys)
        ref = _ref64(c, qkv, p)
        for prec in precisions:
            O, lse, hi, lo = _fwd_tc(c, qkv, p, prec)
            _check_fwd(f"{tag} tc{prec} p{p}", c, O, lse, ref, p, prec)
            _check_planes(f"{tag} tc{prec} O planes", hi, lo, O[:c.N, :c.D], 0, c.D)
            out[f"tc{prec}"] = (O, lse)
    return out


# (shape, H, hd, B) at the head dims of the BASELINE configs
BASELINE_CUDA_CORE = [("pcqm4m-small", 4, 76, 32), ("zinc-gatedgcn", 4, 16, 8), ("pcqm4m-small", 16, 24, 16),
                      ("code2", 4, 64, 6)]
BASELINE_WGMMA = [("pcqm4m-small", 4, 76, 256), ("zinc-gatedgcn", 4, 16, 32), ("pcqm4m-small", 16, 24, 40),
                  ("code2", 4, 64, 12), ("code2", 2, 128, 5)]


@pytest.mark.parametrize("shape,H,hd,B", BASELINE_CUDA_CORE)
def test_cuda_core_forward_backward_baseline_shapes(shape, H, hd, B):
    c = _shape(shape, B, H, hd, seed=B)
    for p in (0.0, 0.5):
        _batch_run(f"{shape} H{H} hd{hd} B{B}", c, p, precisions=())


@pytest.mark.parametrize("shape,H,hd,B", BASELINE_WGMMA)
@pytest.mark.parametrize("precision", [0, 1])
def test_wgmma_forward_baseline_shapes(shape, H, hd, B, precision):
    """The wgmma forward in one precision; the fp32-grade case also runs the CUDA-core forward and backward."""
    c = _shape(shape, B, H, hd, seed=B)
    for p in (0.0, 0.5):
        _batch_run(f"{shape} H{H} hd{hd} B{B}", c, p, cuda_core=precision == 0, precisions=(precision,))


def test_wgmma_and_cuda_core_forward_edge_cases_and_dropout():
    """Empty graphs, single-node graphs and graphs straddling two 128-row tiles, with and without attention dropout:
    each kernel against float64 under the replayed mask, and the wgmma fp32-grade forward against the CUDA-core one
    within the sum of their bounds (the same Philox stream: the same masks)."""
    c = _sizes([1, 0, 130, 3, 0, 1, 200], 4, 76, seed=11)
    for p in (0.0, 0.5):
        assert set(_batch_run("tile_straddling", c, p)) == {"cc", "tc0", "tc1"}
        qkv = _inputs(c, 3 * c.D + 4)
        ref = _ref64(c, qkv, p)
        O1, l1, _, _ = _fwd(c, qkv, 3 * c.D + 4, p)
        O2, l2, _, _ = _fwd_tc(c, qkv, p, 0)
        Q, K, V, b64, keep = ref[:5]
        with torch.no_grad():
            b1, bl1 = ar.fwd_bounds(Q, K, V, c.ptr, c.H, c.hd, None, keep, p)
            b2, bl2 = ar.fwd_bounds(Q, K, V, c.ptr, c.H, c.hd, None, keep, p, 0)
        _elem_check(WORST, f"tile_straddling tc0 vs cc p{p} O", O2[:c.N, :c.D], O1[:c.N, :c.D].double(), b1 + b2)
        _elem_check(WORST, f"tile_straddling tc0 vs cc p{p} lse", l2[:c.N], l1[:c.N].double(), bl1 + bl2)


EDGE_BATCHES = {
    "empty_and_single_nodes": ([0, 0, 1, 5, 0, 33, 1, 0], 4, 16),
    "one_graph": ([57], 2, 32),
    "one_3000_node_graph": ([3000], 2, 16),
    "below_one_warp": ([3], 2, 16),
    "n_not_multiple_of_128": ([200, 67], 2, 24),
    "scores_to_60": ([40, 90, 7], 2, 32),
    "all_equal_scores": ([40, 90, 7], 2, 32),
}


@pytest.mark.parametrize("name", list(EDGE_BATCHES))
def test_batches(name):
    sizes, H, hd = EDGE_BATCHES[name]
    c = _sizes(sizes, H, hd, seed=len(name))
    scale = 3.9 if name == "scores_to_60" else 1.0   # score std 3.9^2 ~ 15: the largest |s| about 60
    eq = name == "all_equal_scores"
    for p in (0.0, 0.5):
        _batch_run(name, c, p, scale=scale, equal_keys=eq)
    if name == "scores_to_60":
        qkv = _inputs(c, 3 * c.D + 4, scale)
        Q, K = qkv[:c.N, :c.D].double(), qkv[:c.N, c.D:2 * c.D].double()
        s_max = max(float((Q[s:e].reshape(e - s, c.H, c.hd).transpose(0, 1) @ K[s:e].reshape(e - s, c.H, c.hd)
                           .transpose(0, 1).transpose(1, 2)).abs().max()) / c.hd ** 0.5
                    for s, e in zip(c.ptr[:-1], c.ptr[1:]) if e > s)
        assert 40 < s_max < 120, s_max


# ------------------------------------------------------------------------------------------------ wgmma forward
@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("hd", list(range(4, 129, 4)))
def test_wgmma_forward_every_head_dim(hd, precision):
    """CTAs of 128 rows that start mid-graph and span many graphs, a 300-node graph over three key tiles; a qkv plane
    pitch wider than 3 H hd_pad whose extra columns are NaN."""
    H = 2
    c = _sizes([50, 100, 3, 0, 140, 7, 1, 60, 300, 2], H, hd, seed=hd + precision)
    ld = 3 * c.D
    qkv = _inputs(c, ld)
    for biased in (False, True):
        ab = _bias(c) if biased else None
        for p in (0.0, 0.5):
            ref = _ref64(c, qkv, p, ab)
            O, lse, hi, lo = _fwd_tc(c, qkv, p, precision, ab, extra=8 * (1 + hd % 3))
            tag = f"tc{precision} hd{hd} b{int(biased)} p{p}"
            _check_fwd(tag, c, O, lse, ref, p, precision)
            _check_planes(tag + " O planes", hi, lo, O[:c.N, :c.D], 0, c.D)


# ------------------------------------------------------------------------------------------------ composition
@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("biased", [False, True])
@pytest.mark.parametrize("p", [0.0, 0.5])
def test_wgmma_forward_then_cuda_core_backward(precision, biased, p):
    """The layer at mean graph size >= 64: the wgmma forward's O and lse feed the CUDA-core backward.  The bound is
    the backward's with the forward's own bounds as the errors of its O and lse inputs."""
    H, hd = 4, 64
    c = _sizes([120, 64, 300, 1, 0, 90], H, hd, seed=7)
    ld = 3 * c.D + 4
    qkv = _inputs(c, ld)
    ab = _bias(c) if biased else None
    Q, K, V, b64, keep, O64, lse64 = _ref64(c, qkv, p, ab)
    O, lse, _, _ = _fwd_tc(c, qkv, p, precision, ab)
    dO = c.randn(c.N, c.D)
    (O64 * dO.double()).sum().backward()
    g, _, _, _, gb = _bwd(c, qkv, ld, O[:c.N, :c.D], lse[:c.N], dO, p, ab)
    D, N = c.D, c.N
    with torch.no_grad():
        bO, bl = ar.fwd_bounds(Q, K, V, c.ptr, H, hd, b64, keep, p, precision)
        bq, bk, bv, bgb = ar.bwd_bounds(Q, K, V, dO.double(), c.ptr, H, hd, b64, keep, p, O_err=bO, lse_err=bl)
    tag = f"tc{precision}+bwd b{int(biased)} p{p}"
    _elem_check(WORST, tag + " dQ", g[:N, :D], Q.grad, bq)
    _elem_check(WORST, tag + " dK", g[:N, D:2 * D], K.grad, bk)
    _elem_check(WORST, tag + " dV", g[:N, 2 * D:3 * D], V.grad, bv)
    if biased:
        _elem_check(WORST, tag + " grad_bias", gb, b64.grad, bgb)


# ------------------------------------------------------------------------------------------------ determinism, refusals
@pytest.mark.parametrize("biased", [False, True])
def test_two_runs_are_bitwise_equal(biased):
    c = _shape("pcqm4m-small", 64, 4, 76, seed=3)
    ld = 3 * c.D + 4
    qkv = _inputs(c, ld)
    ab = _bias(c) if biased else None
    dO = c.randn(c.N, c.D)
    runs = []
    for _ in range(2):
        O, lse, _, _ = _fwd(c, qkv, ld, 0.5, ab)
        g, delta, hi, lo, gb = _bwd(c, qkv, ld, O[:c.N, :c.D], lse[:c.N], dO, 0.5, ab)
        runs.append([O, lse, g, delta, hi, lo] + ([gb] if biased else []))
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.nan_to_num(7.0),
                           b.view(torch.int16) if b.dtype == torch.bfloat16 else b.nan_to_num(7.0))


def test_refusals_happen_before_any_cuda_call():
    """An unsupported head dim leaves a sentinel grad_bias untouched and launches nothing (the grad_bias clear comes
    after the checks); so do a bad pitch and p = 1."""
    lib = _lib_()
    c = _sizes([5, 3], 2, 193)
    D = c.D
    buf = torch.zeros(c.N, 3 * D, device=DEV)
    gb = torch.full((c.B * c.H, c.nmax, c.nmax), 3.25, device=DEV)
    ab = torch.zeros_like(gb)
    bias = _lib.GpsAttnBias(ab.data_ptr(), c.nmax, gb.data_ptr())
    b = buf.data_ptr()
    torch.cuda.synchronize()
    before = lib.gps_launch_count()
    rc = lib.gps_attention_backward_biased(C.byref(c.gs.desc), 2, 193, b, b, b, 3 * D, b, b, D, b, b, b, b, b, 3 * D,
                                           0.0, 0, 0, C.byref(bias), _stream())
    assert rc == _lib.GPS_ERR_UNSUPPORTED
    a = _lib.GpsAttnStageArgs()
    a.graph, a.heads, a.hd = c.gs.desc, 2, 16
    a.Q = a.K = a.V = a.O = a.lse = a.dO = a.delta = a.dQ = a.dK = a.dV = b
    a.ld, a.ldo, a.ldg = 3 * 32, 32, 3 * 32
    a.bias = C.pointer(bias)
    a.p_drop = 1.0
    assert lib.gps_attention_stage(C.byref(a), _lib.ATTN["bwd"], _stream()) == _lib.GPS_ERR_ARG
    a.p_drop, a.ldg = 0.0, 31
    assert lib.gps_attention_stage(C.byref(a), _lib.ATTN["bwd"], _stream()) == _lib.GPS_ERR_ARG
    torch.cuda.synchronize()
    assert lib.gps_launch_count() == before
    assert bool((gb == 3.25).all())
