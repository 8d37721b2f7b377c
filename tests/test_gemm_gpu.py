"""GPU: the dense-product kernels (wgmma and exact CUDA-core) against a float64 torch product,
all four operand orientations (K-major / MN-major), split-K, ragged sizes."""
import pytest
import torch

from graphgps_b200 import _lib
from util import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

SHAPES = [
    # M, N, K
    (3620, 2128, 304), (7455, 304, 304), (3620, 608, 304), (3620, 304, 608), (128, 128, 64),
    (130, 64, 72), (1, 16, 8), (257, 100, 200), (136, 96, 72), (3624, 2128, 304), (3624, 608, 304), (2128, 304, 3620), (304, 304, 7455), (64, 912, 64),
]


def _run(M, N, K, ta, tb, splitk, precision, impl, seed=0):
    lib = _lib.load()
    g = torch.Generator().manual_seed(seed)
    A = torch.randn((K, M) if ta else (M, K), generator=g).to(DEV)
    B = torch.randn((K, N) if tb else (N, K), generator=g).to(DEV)
    C = torch.zeros(M, N, device=DEV)
    rc = lib.gps_gemm(A.data_ptr(), A.shape[1], ta, B.data_ptr(), B.shape[1], tb, C.data_ptr(), N, M, N, K, splitk,
                      precision, impl, torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "gps_gemm")
    Aop = A.double().t() if ta else A.double()
    Bop = B.double() if tb else B.double().t()
    ref = Aop @ Bop
    torch.cuda.synchronize()
    return rel_err(C.cpu(), ref.cpu()) / max(1.0, K ** 0.5 / 8)


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("ta,tb", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_gemm_simt_exact(M, N, K, ta, tb):
    assert _run(M, N, K, ta, tb, 1, 0, 1) < 1e-5


@pytest.mark.parametrize("M,N,K", [s for s in SHAPES if s[1] % 4 == 0])
@pytest.mark.parametrize("ta,tb", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("precision,tol", [(0, 2e-5), (1, 4e-3)])
def test_gemm_tcgen05(M, N, K, ta, tb, precision, tol):
    lda = M if ta else K
    ldb = N if tb else K
    if lda % 4 or ldb % 4:
        pytest.skip("128-bit operand path needs leading dimensions that are multiples of 4")
    if (not ta and K % 8) or (not tb and K % 8) or (ta and M % 8) or (tb and N % 8):
        pytest.skip("the tensor-core kernel takes whole 8-element operand chunks; the dispatcher uses the CUDA-core kernel here")
    err = _run(M, N, K, ta, tb, 1, precision, 2)
    assert err < tol, err


@pytest.mark.parametrize("M,N,K,splitk", [(2128, 304, 3620, 8), (304, 608, 3620, 14), (304, 304, 7455, 29)])
@pytest.mark.parametrize("impl", [1, 2])
def test_gemm_splitk_weight_gradient_shape(M, N, K, splitk, impl):
    assert _run(M, N, K, 1, 1, splitk, 0, impl) < 5e-5
