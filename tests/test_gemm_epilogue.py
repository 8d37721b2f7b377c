"""CPU: the argument contract of gps_gemm_epilogue, the stage entry point of the dense product and its fused epilogue.
Every call here is rejected before any CUDA call, so it needs no device memory (the addresses are placeholders that
are never dereferenced).  The arithmetic is pinned on the GPU by test_gemm_epilogue_gpu.py."""
import ctypes as C

import pytest

from graphgps_b200 import _lib

P = 1 << 20    # placeholder address: never dereferenced


def _args(**kw):
    """A well-formed 64 x 64 x 64 product with fp32 operands, operand planes and fp32 C; kw overrides fields."""
    a = _lib.GpsGemmArgs()
    a.M = a.N = a.K = 64
    a.A, a.lda, a.B, a.ldb = P, 64, P, 64
    a.Ap = _lib.GpsPlanes(P, P, 64)
    a.Bp = _lib.GpsPlanes(P, P, 64)
    a.C, a.ldc = P, 64
    a.act = a.mask_act = -1
    a.splitk = 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _call(a, impl):
    lib = _lib.load()
    return lib.gps_gemm_epilogue(None if a is None else C.byref(a), impl, None)


@pytest.mark.parametrize("impl", [0, 1, 2, 3])
def test_null_args(impl):
    assert _call(None, impl) == _lib.GPS_ERR_ARG
    assert _lib.load().gps_last_error()


@pytest.mark.parametrize("impl", [0, 1, 2, 3])
@pytest.mark.parametrize("field", ["M", "N", "K"])
@pytest.mark.parametrize("value", [-1, 1 << 31])
def test_sizes_out_of_range(impl, field, value):
    assert _call(_args(**{field: value}), impl) == _lib.GPS_ERR_ARG


@pytest.mark.parametrize("impl", [-1, 4, 99])
def test_bad_impl(impl):
    assert _call(_args(), impl) == _lib.GPS_ERR_ARG
    assert b"impl" in _lib.load().gps_last_error()


@pytest.mark.parametrize("impl", [0, 1, 2, 3])
def test_no_output(impl):
    """Neither C nor Cp: the product would write nothing."""
    assert _call(_args(C=0), impl) == _lib.GPS_ERR_ARG


@pytest.mark.parametrize("impl", [1, 2])
@pytest.mark.parametrize("with_c", [True, False])
def test_planes_output_on_fp32_kernels(impl, with_c):
    """The CUDA-core and register-staged kernels never write planes: Cp there is refused, not ignored."""
    a = _args(Cp=_lib.GpsPlanes(P, P, 64), **({} if with_c else {"C": 0}))
    assert _call(a, impl) == _lib.GPS_ERR_ARG
    assert b"Cp" in _lib.load().gps_last_error()


@pytest.mark.parametrize("impl", [1, 2])
@pytest.mark.parametrize("field", ["A", "B"])
def test_fp32_kernels_need_fp32_operands(impl, field):
    assert _call(_args(**{field: 0}), impl) == _lib.GPS_ERR_ARG
