"""CPU: the argument contract of gps_rowwise_stage, the stage entry point of the row-wise BatchNorm, dropout-gradient and
bias-gradient passes.  Every call here is rejected before any CUDA call, so it needs no device memory (the addresses
are placeholders that are never dereferenced).  The arithmetic is pinned on the GPU by test_bn_stages_gpu.py."""
import ctypes as C

import pytest

from graphgps_b200 import _lib

P = 1 << 20    # placeholder address: never dereferenced
OPS = _lib.ROWWISE
BN_OPS = ["bn_act_residual", "bn_act_residual2", "bn_combine", "bn_bwd_reduce", "bn_bwd_apply"]


def _bn(train=1):
    m = _lib.GpsBatchNorm(P, P, P, P, P, P, P)
    return _lib.GpsRowwiseBn(m, P, P, train, 0)


def _args(**kw):
    """A well-formed 64 x 64 call with every tensor and both BatchNorms (training mode) given; kw overrides fields."""
    a = _lib.GpsRowwiseArgs()
    a.rows, a.E, a.d = 64, 64, 64
    a.x = a.x2 = a.g = a.R = a.R2 = a.out = a.out2 = P
    a.bn[0], a.bn[1] = _bn(), _bn()
    a.act = -1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _call(a, op):
    return _lib.load().gps_rowwise_stage(None if a is None else C.byref(a), OPS[op] if isinstance(op, str) else op, None)


def test_exported():
    lib = _lib.load()
    assert hasattr(lib, "gps_rowwise_stage")
    assert lib.gps_abi_version() == 4
    assert sorted(OPS.values()) == list(range(7))


@pytest.mark.parametrize("op", list(OPS))
def test_null_args(op):
    assert _call(None, op) == _lib.GPS_ERR_ARG
    assert b"null args" in _lib.load().gps_last_error()


@pytest.mark.parametrize("op", [-1, 7, 99])
def test_unknown_op(op):
    assert _call(_args(), op) == _lib.GPS_ERR_ARG
    assert b"unknown op" in _lib.load().gps_last_error()


@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("field", ["rows", "E", "d"])
def test_negative_sizes(op, field):
    assert _call(_args(**{field: -1}), op) == _lib.GPS_ERR_ARG
    assert b"negative size" in _lib.load().gps_last_error()


# (op, ld field) pairs whose kernels take a pitch
FREE_LD = {("bn_act_residual", "ldx"), ("bn_bwd_reduce", "ldx"), ("bn_bwd_reduce", "ldg"), ("bn_bwd_apply", "ldx"),
           ("bn_bwd_apply", "ldg"), ("bn_bwd_apply", "ldo"), ("colsum", "ldx")}


@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("field", ["ldx", "ldg", "ldo"])
@pytest.mark.parametrize("ld", [60, 66, 70])
def test_leading_dimension_below_d_or_unaligned(op, field, ld):
    """Below d (60) or not a multiple of 4 (66, 70): refused whether or not the op reads that pitch."""
    assert _call(_args(**{field: ld}), op) == _lib.GPS_ERR_ARG
    assert field.encode() in _lib.load().gps_last_error()


@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("field", ["ldx", "ldg", "ldo"])
def test_pitch_only_where_the_kernel_takes_one(op, field):
    """ld = 68 > d is refused where the op's kernel has pitch d; elsewhere it passes validation (the call then reaches
    CUDA, so it is not made here)."""
    if (op, field) in FREE_LD:
        pytest.skip("the op takes this pitch")
    assert _call(_args(**{field: 68}), op) == _lib.GPS_ERR_ARG
    assert b"takes " + field.encode() + b" = d only" in _lib.load().gps_last_error()


def _needed(op):
    """The pointers each op needs (with both BatchNorms in training mode)."""
    need = ["x"] + ([] if op == "bn_bwd_reduce" else ["out"])
    if op in ("bn_bwd_reduce", "bn_bwd_apply"):
        need.append("g")
    if op == "bn_act_residual2":
        need += ["x2", "out2"]
    return need


@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("field", ["x", "x2", "g", "out", "out2"])
def test_null_tensor(op, field):
    if field not in _needed(op):
        pytest.skip("the op does not need it")
    assert _call(_args(**{field: 0}), op) == _lib.GPS_ERR_ARG
    assert b"needs" in _lib.load().gps_last_error()


def _bn_ops():
    """(op, BatchNorm index) for every BatchNorm an op reads; bn_combine reads bn[1] only with x2."""
    return [(op, i) for op in BN_OPS for i in ((0, 1) if op in ("bn_act_residual2", "bn_combine") else (0,))]


@pytest.mark.parametrize("op,i", _bn_ops())
@pytest.mark.parametrize("field", ["weight", "bias"])
@pytest.mark.parametrize("train", [0, 1])
def test_null_affine(op, i, field, train):
    a = _args()
    a.bn[0].train = a.bn[1].train = train
    setattr(a.bn[i].bn, field, 0)
    assert _call(a, op) == _lib.GPS_ERR_ARG
    assert b"bn[%d] needs weight and bias" % i in _lib.load().gps_last_error()


@pytest.mark.parametrize("op,i", _bn_ops())
@pytest.mark.parametrize("field", ["running_mean", "running_var"])
def test_eval_needs_running_statistics(op, i, field):
    a = _args()
    a.bn[0].train = a.bn[1].train = 0
    setattr(a.bn[i].bn, field, 0)
    assert _call(a, op) == _lib.GPS_ERR_ARG
    assert b"running statistics" in _lib.load().gps_last_error()


@pytest.mark.parametrize("op,i", _bn_ops())
def test_training_needs_saved(op, i):
    a = _args()
    a.bn[i].saved = 0
    assert _call(a, op) == _lib.GPS_ERR_ARG
    assert b"needs saved" in _lib.load().gps_last_error()


@pytest.mark.parametrize("op,i", _bn_ops())
@pytest.mark.parametrize("train", [0, 1])
def test_sums(op, i, train):
    """Training forward reads the producer's sums; both backward ops read or add their S1 / S2 in either mode.  Only
    the eval forward has no use for them."""
    if not (op in ("bn_bwd_reduce", "bn_bwd_apply") or train):
        pytest.skip("the eval forward does not read sums")
    a = _args()
    a.bn[0].train = a.bn[1].train = train
    a.bn[i].sums = 0
    assert _call(a, op) == _lib.GPS_ERR_ARG
    assert b"needs sums" in _lib.load().gps_last_error()


def test_combine_with_x2_needs_the_second_batchnorm():
    a = _args()
    a.bn[1].bn.weight = 0
    assert _call(a, "bn_combine") == _lib.GPS_ERR_ARG
