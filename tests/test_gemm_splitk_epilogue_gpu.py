"""GPU: K-splits with the fused epilogue on the TMA-fed GEMM (csrc/gemm_tma.cu).  The K-splits of an output tile form a
thread-block cluster; the ranks sum their partial tiles in rank order and each then runs the whole epilogue on its own
rows (bias, act, act' mask, both dropout sites, two residuals, fp32 store, planes in the identity or per-head padded
layout, BatchNorm column sums).  The launch policy picks the split from the shape; gps_debug_tma_splits forces it.

Every epilogue recipe of test_gemm_epilogue_gpu.py (with the layer's g_x product as it now runs: C = sum + R1 + R2
written by the epilogue instead of added into a pre-zeroed C) runs with the split forced to 1, 2 and 4, in fp32-grade and bf16 mode, at
M not a multiple of 128, K of 2 k-blocks and the d = 304 shapes of the layer's node-row products.  With the exact
operands of that file the product is exact in any summation order, so every output must equal the float32 replay bit
for bit (float64 within a bound for GELU) whatever the split: the dropout masks, the planes and the head pads exactly.
Gaussian operands then check the split against the unsplit result within the reordered-sum bound, and two runs of a
split for the same bits."""
import pytest
import torch

from graphgps_b200 import _lib
from test_gemm_epilogue_gpu import (GELU, RELU, U, Run, Spec, _bitwise_equal, _check, _check_planes, _check_stats,
                                    _exact_data, dgrad_inplace, dgrad_mask, ff1_fwd, out_proj_stats, performer_out,
                                    qkv_planes)
from util import _stream, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TMA = 3
SPLITS = (1, 2, 4)


def gx_direct():
    """layer.cu grad_x = gY1 Wcat + g_x_local + g_hA: g W (tb = 1) plus two residuals, written (not added into a zeroed
    C)."""
    return Spec("gx_direct", tb=1, r1=True, r2=True)


RECIPES = {
    "qkv_planes": lambda: qkv_planes(76),
    "ff1_fwd_relu": lambda: ff1_fwd(RELU, 0.75),
    "ff1_fwd_gelu": lambda: ff1_fwd(GELU, 0.0),
    "out_proj_stats": lambda: out_proj_stats(0.5, True),
    "performer_out": lambda: performer_out(),
    "dgrad_mask_relu": lambda: dgrad_mask("relu_post", 0.5),
    "dgrad_mask_gelu": lambda: dgrad_mask("gelu_pre", 0.0),
    "dgrad_inplace": dgrad_inplace,
    "gx_direct": gx_direct,
}

# (M, N, K): 129 rows (a last row tile of 1 row) with K of 2 k-blocks; the d = 304 products: out-proj (K = d), FF2
# forward and FF1 data gradient (K = 2d), g_x (K = 7d); N = 912 for the per-head planes (4 heads of 76 = 3 x 304).
SHAPES = {
    "qkv_planes": [(129, 912, 128), (3620, 912, 304)],
    "gx_direct": [(129, 304, 128), (3620, 304, 2128)],
}
DEFAULT_SHAPES = [(129, 304, 128), (3620, 304, 304), (3620, 304, 608)]
CASES = [(r, shape) for r in RECIPES for shape in SHAPES.get(r, DEFAULT_SHAPES)]


def _lib_():
    return _lib.load()


class forced_splits:
    def __init__(self, s):
        self.s = s

    def __enter__(self):
        _lib_().gps_debug_tma_splits(self.s)

    def __exit__(self, *exc):
        _lib_().gps_debug_tma_splits(0)


def _run(spec, M, N, K, prec, splits, seed=0, random=False):
    run = Run(spec, M, N, K, prec, seed, random=random)
    with forced_splits(splits):
        rc = run.call(TMA)
    _lib.check(rc, f"{spec.name} splits={splits}")
    return run


@pytest.mark.parametrize("precision", [0, 1], ids=["fp32", "bf16"])
@pytest.mark.parametrize("recipe,shape", CASES, ids=[f"{r}-{m}x{n}x{k}" for r, (m, n, k) in CASES])
def test_recipe_with_forced_splits(recipe, shape, precision):
    M, N, K = shape
    spec = RECIPES[recipe]()
    outs = {}
    for s in SPLITS:
        run = _run(spec, M, N, K, precision, s)
        _check(run, "tma")   # the column statistics within the chain bound of one CTA's rows
        outs[s] = run.outputs(stats=False)
    again = _run(spec, M, N, K, precision, 4)
    for j, (x, y) in enumerate(zip(again.outputs(stats=False), outs[4])):
        assert _bitwise_equal(x, y), f"two runs with 4 splits differ in output {j}"
    if _exact_data(spec) and spec.stats:
        # the statistics' float64 atomics add per-CTA partials in any order: bitwise when each partial is exact
        assert _bitwise_equal(again.stats_buf, run.stats_buf), "two runs with 4 splits differ in the statistics"
    # exact operands: every split computes the same exact product, so the outputs (dropout masks, planes, pads) agree;
    # the float32 column statistics group the rows by split and are checked against their bound above
    for s in SPLITS[1:]:
        for j, (x, y) in enumerate(zip(outs[s], outs[1])):
            assert _bitwise_equal(x, y), f"{s} splits: output {j} differs from the unsplit launch"


def _chain_bound(run, splits):
    """|C_split - C_unsplit| elementwise: both sum the same K products, each a float32 chain of at most one addition per
    16-deep MMA step (three MMA passes in fp32-grade mode) plus the splits' partial tiles; each addition is off by at
    most 2u of the running magnitude (the tensor core may truncate), bounded by sum |a_k b_k|."""
    s = run.s
    B = run.B.double() if s.tb else run.B.double().t()
    mag = run.A.double().abs() @ B.abs()
    steps = (3 if run.prec == 0 else 1) * (run.K + 15) // 16 + splits
    return 2 * 2 * steps * U * mag


@pytest.mark.parametrize("precision", [0, 1], ids=["fp32", "bf16"])
@pytest.mark.parametrize("splits", [2, 4])
@pytest.mark.parametrize("M,N,K", [(3620, 304, 304), (3620, 304, 608), (3620, 608, 304), (1000, 304, 2128),
                                   (129, 304, 128)])
def test_random_operands_split_against_unsplit(M, N, K, splits, precision):
    """Gaussian operands with non-zero lo planes, bias, residual, statistics and planes: the split agrees with the
    unsplit launch within the reordered-sum bound and with float64 at the tolerances of test_gemm_epilogue_gpu.py; two
    runs give the same bits; and the split really ran (its bits differ from the unsplit ones somewhere)."""
    spec = Spec("random", bias=True, r1=True, stats=True, cp="identity")
    one = _run(spec, M, N, K, precision, 1, seed=7, random=True)
    runs = [_run(spec, M, N, K, precision, splits, seed=7, random=True) for _ in range(2)]
    for j, (x, y) in enumerate(zip(runs[0].outputs(), runs[1].outputs())):
        assert _bitwise_equal(x, y), f"two runs with {splits} splits differ in output {j}"
    run = runs[0]
    err = (run.C.double() - one.C.double()).abs()
    bound = _chain_bound(run, splits)
    assert (err <= bound).all(), f"split off the unsplit result by {float((err / bound).max()):.3g} x the chain bound"
    if K >= 256:
        assert not torch.equal(run.C, one.C), "no element changed: the split did not run"
    ref = run.A.double() @ run.B.double().t() + run.bias.double() + run.R1.double()
    tol = 2e-5 * max(1.0, K ** 0.5 / 8) if precision == 0 else 2e-2
    assert rel_err(run.C, ref) < tol
    _check_stats(run, "tma")
    _check_planes(run)


def _plain(M, N, K, precision, splitk, C):
    g = torch.Generator().manual_seed(11)
    A = (torch.randint(-8, 9, (M, K), generator=g).float() * 0.125).to(DEV)
    W = (torch.randint(-8, 9, (N, K), generator=g).float() * 0.125).to(DEV)
    lib = _lib_()
    bufs = []
    for x in (A, W):
        r, c = x.shape
        ld = (c + 7) // 8 * 8
        buf = torch.zeros(2, r, ld, dtype=torch.bfloat16, device=DEV)
        _lib.check(lib.gps_to_planes(x.data_ptr(), x.stride(0), r, c, buf[0].data_ptr(),
                                     buf[1].data_ptr() if precision == 0 else 0, ld, _stream()), "gps_to_planes")
        bufs.append((buf, ld))
    (Ap, lda), (Wp, ldw) = bufs
    rc = lib.gps_gemm_planes(Ap[0].data_ptr(), Ap[1].data_ptr() if precision == 0 else 0, lda, 0,
                             Wp[0].data_ptr(), Wp[1].data_ptr() if precision == 0 else 0, ldw, 0,
                             C.data_ptr(), N, 0, 0, 0, M, N, K, splitk, precision, 0, _stream())
    torch.cuda.synchronize()
    _lib.check(rc, "gps_gemm_planes")
    return (A.double() @ W.double().t()).float()


@pytest.mark.parametrize("precision", [0, 1], ids=["fp32", "bf16"])
@pytest.mark.parametrize("M,N,K,tb,splits", [(1000, 304, 2128, 0, 5), (4000, 256, 1792, 1, 2), (3620, 304, 608, 0, 1),
                                              (3620, 304, 2128, 1, 1)])
def test_policy_split_follows_the_shape(M, N, K, tb, splits, precision):
    """Long reductions over few row tiles are split by the launch policy (M = 1000, K = 7d at d = 304: 24 tiles of 128
    columns, 34 k-blocks, 5 splits; g_x at d = 256 over 4000 rows: 64 tiles of 128 columns, 2 splits): the result equals
    the forced split bit for bit and, with Gaussian operands, differs from the unsplit one.  The d = 304 layer products
    (FF2 forward at K = 2d; g_x at K = 7d with its MN-major W, 87 tiles of 128 columns) are not split."""
    spec = Spec("random", tb=tb, bias=True, r1=True, stats=True, cp="identity")
    pol = Run(spec, M, N, K, precision, 7, random=True)
    _lib.check(pol.call(TMA), "policy")
    forced = _run(spec, M, N, K, precision, splits, seed=7, random=True)
    assert torch.equal(pol.C, forced.C) and torch.equal(pol.Cp, forced.Cp)
    if splits > 1:
        one = _run(spec, M, N, K, precision, 1, seed=7, random=True)
        assert not torch.equal(pol.C, one.C)


@pytest.mark.parametrize("splitk", [2, 4])
def test_accumulating_split_still_adds_into_c(splitk):
    """gps_gemm_planes with splitk > 1 and no epilogue keeps its meaning: the product is added into C."""
    M, N, K = 3620, 304, 608
    C = torch.full((M, N), 0.5, device=DEV)
    prod = _plain(M, N, K, 0, splitk, C)
    assert torch.equal(C, prod + 0.5)
