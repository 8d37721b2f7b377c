"""GPU: the TMA-fed wgmma GEMM (csrc/gemm_tma.cu) on bf16 hi/lo plane operands, every operand orientation the layer
uses, against float64 torch: y = x W^T (forward Linears, gatedgcn_layer.py:57-61, gps_layer.py:253-257), g_x = g_y W
(data gradients) and dW = G^T X with db = colsum(G) (weight/bias gradients).  fp32-grade mode: <= 2e-5 * max(1, sqrt(K)/8)
scaled max-abs (the tolerance of the register-staged kernel's tests); bf16 mode: 2e-2."""
import pytest
import torch

from graphgps_b200 import _lib
from util import _stream, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _planes(x, lo=True, pad=0):
    """fp32 [r, c] -> (hi, lo) bf16 planes with pitch round_up(c, 8) + pad, via the library's own converter."""
    lib = _lib.load()
    r, c = x.shape
    ldp = (c + 7) // 8 * 8 + pad
    buf = torch.zeros(2, r, ldp, dtype=torch.bfloat16, device=DEV)
    _lib.check(lib.gps_to_planes(x.data_ptr(), x.stride(0), r, c, buf[0].data_ptr(), buf[1].data_ptr() if lo else 0, ldp,
                                 _stream()), "gps_to_planes")
    return buf, ldp


def test_to_planes_hi_plus_lo_is_fp32_grade():
    x = torch.randn(333, 300, device=DEV) * 3
    buf, ldp = _planes(x)
    assert ldp == 304
    rec = buf[0, :, :300].float() + buf[1, :, :300].float()
    assert float((rec - x).abs().max()) <= 2.0 ** -16 * float(x.abs().max())
    assert torch.equal(buf[0, :, :300], x.to(torch.bfloat16))
    assert float(buf[:, :, 300:].float().abs().max()) == 0.0     # the pad columns of the last 8-element chunk are zero


@pytest.mark.parametrize("M,N,K", [(3620, 1216, 304), (3620, 304, 304), (7455, 304, 304), (3620, 608, 304),
                                   (3620, 304, 608), (130, 64, 64), (1, 8, 8), (333, 608, 296), (257, 48, 72)])
@pytest.mark.parametrize("precision", [0, 1])
def test_linear_forward_planes(M, N, K, precision):
    lib = _lib.load()
    g = torch.Generator().manual_seed(0)
    A = torch.randn(M, K, generator=g).to(DEV)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
    Ap, lda = _planes(A, lo=precision == 0)
    Wp, ldw = _planes(W, lo=precision == 0, pad=8)
    Cc = torch.full((M, N), float("nan"), device=DEV)
    Cp = torch.zeros(2, M, (N + 7) // 8 * 8, dtype=torch.bfloat16, device=DEV)
    rc = lib.gps_gemm_planes(Ap[0].data_ptr(), Ap[1].data_ptr() if precision == 0 else 0, lda, 0,
                             Wp[0].data_ptr(), Wp[1].data_ptr() if precision == 0 else 0, ldw, 0,
                             Cc.data_ptr(), N, Cp[0].data_ptr(), Cp[1].data_ptr() if precision == 0 else 0, Cp.shape[2],
                             M, N, K, 1, precision, 0, _stream())
    _lib.check(rc, "gps_gemm_planes")
    ref = A.double() @ W.double().t()
    tol = 2e-5 * max(1.0, K ** 0.5 / 8) if precision == 0 else 2e-2
    assert rel_err(Cc.cpu(), ref.cpu()) < tol
    rec = Cp[0, :, :N].float() + (Cp[1, :, :N].float() if precision == 0 else 0)
    assert rel_err(rec.cpu(), ref.cpu()) < (2 * tol if precision == 0 else 3e-2)


@pytest.mark.parametrize("M,N,K,splitk", [(3620, 304, 2128, 1), (3620, 304, 2128, 4), (3620, 608, 304, 1),
                                          (7455, 304, 304, 1), (100, 72, 40, 1), (3620, 1024, 384, 1)])
def test_data_gradient_planes(M, N, K, splitk):
    """g_x[M,N] = G[M,K] W[K,N]: A K-major, B = W stored [K, N] (MN-major operand)."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(1)
    G = torch.randn(M, K, generator=g).to(DEV)
    W = (torch.randn(K, N, generator=g) / K ** 0.5).to(DEV)
    Gp, ldg = _planes(G)
    Wp, ldw = _planes(W)
    Cc = torch.zeros(M, N, device=DEV)
    rc = lib.gps_gemm_planes(Gp[0].data_ptr(), Gp[1].data_ptr(), ldg, 0, Wp[0].data_ptr(), Wp[1].data_ptr(), ldw, 1,
                             Cc.data_ptr(), N, 0, 0, 0, M, N, K, splitk, 0, 0, _stream())
    _lib.check(rc, "gps_gemm_planes")
    ref = G.double() @ W.double()
    assert rel_err(Cc.cpu(), ref.cpu()) < 2e-5 * max(1.0, K ** 0.5 / 8)


@pytest.mark.parametrize("rows,out,inn,splitk", [(3620, 304, 608, 8), (3620, 2128, 304, 4), (7455, 304, 304, 16),
                                                 (3620, 608, 304, 6), (200, 72, 40, 2), (64, 304, 304, 1)])
def test_weight_gradient_planes(rows, out, inn, splitk):
    """dW[out,in] = G[rows,out]^T X[rows,in], db = colsum(G): both operands MN-major, reduction over rows."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(2)
    G = torch.randn(rows, out, generator=g).to(DEV)
    X = torch.randn(rows, inn, generator=g).to(DEV)
    Gp, ldg = _planes(G)
    Xp, ldx = _planes(X)
    dW = torch.zeros(out, inn, device=DEV)
    db = torch.zeros(out, device=DEV)
    rc = lib.gps_gemm_planes(Gp[0].data_ptr(), Gp[1].data_ptr(), ldg, 1, Xp[0].data_ptr(), Xp[1].data_ptr(), ldx, 1,
                             dW.data_ptr(), inn, 0, 0, 0, out, inn, rows, max(splitk, 2), 0, db.data_ptr(), _stream())
    _lib.check(rc, "gps_gemm_planes")
    ref = G.double().t() @ X.double()
    assert rel_err(dW.cpu(), ref.cpu()) < 2e-5 * max(1.0, rows ** 0.5 / 8)
    assert rel_err(db.cpu(), G.double().sum(0).cpu()) < 2e-5 * max(1.0, rows ** 0.5 / 8)
