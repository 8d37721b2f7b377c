"""GPU: the tile widths of the TMA-fed GEMM (csrc/gemm_tma.cu).  Every width computes each output element with the same
wgmma sequence, and the BatchNorm column sums of the epilogue are added in the same order for every width, so the
product and the whole layer must come out bitwise equal whichever width the launch policy picks; each result is also
checked against float64 torch at the tolerances of test_gemm_planes_gpu.py."""
import pytest
import torch

import graphgps_b200
from graphgps_b200 import _call, _lib
from graphgps_b200.graph import graph_of
from util import _stream, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _planes(x, lo=True):
    lib = _lib.load()
    r, c = x.shape
    ldp = (c + 7) // 8 * 8
    buf = torch.zeros(2, r, ldp, dtype=torch.bfloat16, device=DEV)
    _lib.check(lib.gps_to_planes(x.data_ptr(), x.stride(0), r, c, buf[0].data_ptr(), buf[1].data_ptr() if lo else 0, ldp,
                                 _stream()), "gps_to_planes")
    return buf, ldp


def _forced(bn):
    lib = _lib.load()
    lib.gps_debug_tma(bn, 0)
    return lib


# K-major B (y = x W^T) with a K-major A (ta = 0) or an MN-major A (ta = 1, A stored [K, M], optionally with the
# bias-gradient row sums colsum_a): every width the layout takes and the policy; M not a multiple of 128,
# N = 304 / 608 / 912 / 1216 and N not a multiple of 152 (296, 1000), more tiles than CTA slots (7455 x 1216: 472
# tiles) with a count that is no multiple of the grid's wave
@pytest.mark.parametrize("M,N,K", [(3620, 304, 304), (3620, 608, 304), (3620, 912, 304), (3620, 1216, 304),
                                   (7455, 1216, 304), (3620, 304, 608), (7455, 304, 304), (333, 296, 200), (1000, 1000, 96)])
@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("ta,colsum", [(0, False), (1, False), (1, True)])
def test_k_major_b_every_width_bitwise(M, N, K, precision, ta, colsum):
    g = torch.Generator().manual_seed(3)
    A = torch.randn(M, K, generator=g).to(DEV)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
    if ta:   # A stored [K, M]; the fp32 source rows are padded to 16 bytes for the plane converter
        At = torch.zeros(K, (M + 3) // 4 * 4, device=DEV)
        At[:, :M] = A.t()
        Ap, lda = _planes(At[:, :M], lo=precision == 0)
    else:
        Ap, lda = _planes(A, lo=precision == 0)
    Wp, ldw = _planes(W, lo=precision == 0)
    ref = A.double() @ W.double().t()
    tol = 2e-5 * max(1.0, K ** 0.5 / 8) if precision == 0 else 2e-2
    widths = (0, 64, 128, 152, 0) if ta else (0, 64, 128, 152, 256, 0)
    outs = {}
    try:
        for bn in widths:
            lib = _forced(bn)
            C = torch.full((M, N), float("nan"), device=DEV)
            Cp = torch.zeros(2, M, (N + 7) // 8 * 8, dtype=torch.bfloat16, device=DEV)
            db = torch.zeros(M, device=DEV)
            rc = lib.gps_gemm_planes(Ap[0].data_ptr(), Ap[1].data_ptr() if precision == 0 else 0, lda, ta,
                                     Wp[0].data_ptr(), Wp[1].data_ptr() if precision == 0 else 0, ldw, 0,
                                     C.data_ptr(), N, Cp[0].data_ptr(), Cp[1].data_ptr() if precision == 0 else 0,
                                     Cp.shape[2], M, N, K, 1, precision, db.data_ptr() if colsum else 0, _stream())
            _lib.check(rc, f"gps_gemm_planes bn={bn}")
            assert rel_err(C.cpu(), ref.cpu()) < tol, bn
            if colsum:
                assert rel_err(db.cpu(), A.double().sum(1).cpu()) < tol, bn
            if bn in outs:
                assert all(torch.equal(x, y) for x, y in zip((C, Cp, db), outs[bn])), "two launches differ"
            outs[bn] = (C, Cp, db)
    finally:
        _forced(0)
    for bn, res in outs.items():
        assert all(torch.equal(x, y) for x, y in zip(res, outs[64])), f"width {bn} differs from width 64"


@pytest.mark.parametrize("bn,ta,tb", [(152, 0, 1), (152, 1, 1), (256, 1, 0), (256, 1, 1), (96, 0, 0)])
def test_widths_a_layout_cannot_take_are_rejected(bn, ta, tb):
    """152 needs a K-major B, 256 a K-major A; a forced width the layout cannot take fails instead of running."""
    lib = _forced(bn)
    try:
        x = torch.randn(304, 304, device=DEV)
        Xp, ldx = _planes(x)
        C = torch.zeros(304, 304, device=DEV)
        rc = lib.gps_gemm_planes(Xp[0].data_ptr(), Xp[1].data_ptr(), ldx, ta, Xp[0].data_ptr(), Xp[1].data_ptr(), ldx,
                                 tb, C.data_ptr(), 304, 0, 0, 0, 304, 304, 304, 1, 0, 0, _stream())
        assert rc == _lib.GPS_ERR_UNSUPPORTED
    finally:
        _forced(0)


def _layer_step(wl, precision, drop, adrop):
    """One GPSLayer fwd + bwd on the workload's batch: every Linear epilogue of the layer runs (bias, ReLU, dropout,
    residuals, plane outputs and BatchNorm statistics)."""
    spec = graphgps_b200.SHAPES[wl]
    _call._drop_counters.clear()   # the same dropout masks in every run
    torch.manual_seed(0)
    layer = graphgps_b200.GPSLayer(spec.dim, spec.local_gnn, spec.global_model, spec.heads, dropout=drop,
                                   attn_dropout=adrop, precision=precision).to(DEV).train()
    b = graphgps_b200.make_batch(wl, seed=0).to(DEV)
    graph_of(b)
    g = torch.Generator().manual_seed(5)
    ct_x = torch.randn(b.x.shape, generator=g).to(DEV)
    ct_e = torch.randn(b.edge_attr.shape, generator=g).to(DEV)
    x = b.x.detach().requires_grad_(True)
    e = b.edge_attr.detach().requires_grad_(True)
    bb = graphgps_b200.GraphBatch(x=x, edge_index=b.edge_index, edge_attr=e, batch=b.batch, num_graphs=b.num_graphs)
    bb.__dict__["_gps_b200_graph"] = b.__dict__["_gps_b200_graph"]
    out = layer(bb)
    torch.autograd.backward([out.x, out.edge_attr], [ct_x, ct_e])
    torch.cuda.synchronize()
    res = [out.x.detach().clone(), out.edge_attr.detach().clone(), x.grad.clone(), e.grad.clone()]
    res += [p.grad.clone() for p in layer.parameters() if p.grad is not None]
    res += [t.clone() for t in layer.buffers() if t.is_floating_point()]
    return res


@pytest.mark.parametrize("precision,drop,adrop", [("fp32", 0.0, 0.5), ("fp32", 0.2, 0.2), ("bf16", 0.0, 0.5)])
def test_layer_step_bitwise_across_tile_widths(precision, drop, adrop):
    """The pcqm4m-small layer (d = 304, ~3600 nodes) with the policy's widths, run twice, and with every GEMM forced to
    64-wide tiles: all outputs, input and parameter gradients and BatchNorm running statistics are bitwise equal."""
    try:
        runs = [_layer_step("pcqm4m-small", precision, drop, adrop) for _ in range(2)]
        _forced(64)
        runs.append(_layer_step("pcqm4m-small", precision, drop, adrop))
    finally:
        _forced(0)
    for other in runs[1:]:
        assert len(other) == len(runs[0])
        for i, (a, b) in enumerate(zip(runs[0], other)):
            assert torch.equal(a, b), f"tensor {i} differs"


def test_layer_with_128_wide_tiles_matches_fp64_oracle():
    """Every GEMM of the pcqm4m-small layer forced to 128-wide tiles (a width every layout takes) against the fp64
    oracle at the tolerances of test_layer_gpu.py: the epilogues (bias, ReLU, residuals, plane outputs, BatchNorm
    statistics, split-K) checked independently of the 64-wide path.  The policy's own
    widths are checked the same way by test_layer_gpu.py::test_layer_matches_oracle_full_size."""
    from test_layer_gpu import _full_size
    _forced(128)
    try:
        _full_size("pcqm4m-small", "CustomGatedGCN", "Transformer", 4, "fp32")
    finally:
        _forced(0)
