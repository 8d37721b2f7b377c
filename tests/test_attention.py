"""CPU: the float64 attention reference and its Philox replica (tests/attention_reference.py), and the argument contract
of gps_attention_stage and the six gps_attention_* entry points that are calls of it.

  * Philox4x32-10: Random123's published known-answer vectors, on the vectorised replica and on a scalar transcription
    of csrc/common.cuh's round function; the keep threshold from the float32 p.
  * The reference against the attention block of the layer's oracle: to_dense_batch, then torch's
    nn.MultiheadAttention with a key padding mask, to 1e-12, undropped and with the keep mask injected where
    nn.MultiheadAttention applies its dropout.
  * Every refusal of the argument contract, before any CUDA call: the addresses are placeholders that are never
    dereferenced.  The arithmetic is pinned on the GPU by test_attention_gpu.py."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import attention_reference as ar
from graphgps_b200 import _lib
from oracle.gps_oracle import to_dense_batch

# ------------------------------------------------------------------------------------------------ Philox
# Random123 kat_vectors, philox4x32 10: counter words, key words, output words
KAT = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
       ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
       ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
        (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]


def _philox_scalar(seed, ctr_hi, ctr_lo):
    """csrc/common.cuh philox4x32, transcribed line for line in Python integers."""
    M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
    m32 = 0xFFFFFFFF
    c0, c1, c2, c3 = ctr_lo & m32, ctr_lo >> 32, ctr_hi & m32, ctr_hi >> 32
    k0, k1 = seed & m32, seed >> 32
    for _ in range(10):
        hi0, lo0 = (M0 * c0) >> 32, (M0 * c0) & m32
        hi1, lo1 = (M1 * c2) >> 32, (M1 * c2) & m32
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + W0) & m32, (k1 + W1) & m32
    return (c0, c1, c2, c3)


def _words(ctr, key):
    return key[0] | key[1] << 32, ctr[2] | ctr[3] << 32, ctr[0] | ctr[1] << 32   # seed, counter hi, counter lo


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_philox_known_answer_vectors(ctr, key, want):
    seed, hi, lo = _words(ctr, key)
    assert _philox_scalar(seed, hi, lo) == want
    assert tuple(int(x) for x in ar.philox4x32_10(seed, hi, lo)) == want


def test_philox_vectorised_matches_scalar():
    rng = np.random.default_rng(0)
    seeds = rng.integers(0, 2 ** 63, 64, dtype=np.uint64)
    his = rng.integers(0, 2 ** 63, 64, dtype=np.uint64)
    los = rng.integers(0, 2 ** 63, 64, dtype=np.uint64)
    got = ar.philox4x32_10(seeds, his, los)
    for s, h, lo, g in zip(seeds, his, los, got):
        assert tuple(int(x) for x in g) == _philox_scalar(int(s), int(h), int(lo))


@pytest.mark.parametrize("p", [0.1, 0.2, 0.5, 0.9, 1e-9, 0.999999])
def test_keep_threshold_is_computed_from_float32_p(p):
    p32 = float(np.float32(p))
    assert ar.keep_threshold(p) == int(p32 * 2 ** 32)
    assert ar.keep_threshold(0.0) == 0


def test_attention_keep_layout():
    """keep(i, jl, h) is component jl & 3 of the draw at counter (offset + 16 + h, (i << 20) | (jl >> 2))."""
    seed, offset, p = 1234, 4096 * 3, 0.5
    rows = np.array([0, 5, 77, 1023])
    keep = ar.attention_keep(seed, offset, p, rows, 11, 2)
    thr = ar.keep_threshold(p)
    for r, i in enumerate(rows):
        for jl in range(11):
            bits = _philox_scalar(seed, offset + 16 + 2, (int(i) << 20) | (jl >> 2))[jl & 3]
            assert keep[r, jl] == (bits >= thr)


# ------------------------------------------------------------------------------------------------ the reference
def _mha_block(Q, K, V, batch, B, H, p=0.0, keep=None):
    """The oracle's attention block with identity projections: to_dense_batch, nn.MultiheadAttention with the key
    padding mask, [mask].  keep (dense [B, H, nmax, nmax]) is injected where nn.MultiheadAttention drops its weights."""
    D = Q.shape[1]
    mha = torch.nn.MultiheadAttention(D, H, dropout=p, batch_first=True).double()
    with torch.no_grad():
        mha.in_proj_weight.copy_(torch.eye(D, dtype=torch.float64).repeat(3, 1))
        mha.in_proj_bias.zero_()
        mha.out_proj.weight.copy_(torch.eye(D, dtype=torch.float64))
        mha.out_proj.bias.zero_()
    mha.train(p > 0)
    qd, mask = to_dense_batch(Q, batch, B)
    kd, _ = to_dense_batch(K, batch, B)
    vd, _ = to_dense_batch(V, batch, B)
    if keep is None:
        return mha(qd, kd, vd, attn_mask=None, key_padding_mask=~mask, need_weights=False)[0][mask]

    def dropout(w, p, training=True, inplace=False):   # w [B*H... or B, H, L, S]
        return w * keep.reshape(w.shape).to(w.dtype) / (1 - p)

    orig = F.dropout
    F.dropout = dropout
    try:
        out = mha(qd, kd, vd, attn_mask=None, key_padding_mask=~mask, need_weights=True, average_attn_weights=False)[0]
    finally:
        F.dropout = orig
    return out[mask]


@pytest.mark.parametrize("p", [0.0, 0.5])
def test_reference_matches_the_oracle_attention_block(p):
    torch.manual_seed(3)
    sizes = [5, 1, 0, 17, 9, 0]
    H, hd = 4, 6
    ptr = np.concatenate([[0], np.cumsum(sizes)])
    N, B, D = int(ptr[-1]), len(sizes), H * hd
    batch = torch.repeat_interleave(torch.arange(B), torch.tensor(sizes))
    Q, K, V = (torch.randn(N, D, dtype=torch.float64) for _ in range(3))
    keep = ar.keep_masks(ptr, H, p, 99, 8192)
    O, lse = ar.attention(Q, K, V, ptr, H, hd, keep=keep, p=p)
    dense = None
    if keep is not None:
        nmax = max(sizes)
        dense = torch.ones(B, H, nmax, nmax, dtype=torch.bool)
        for g in range(B):
            n = sizes[g]
            if n:
                dense[g, :, :n, :n] = keep[g]
        assert 0.3 < float(torch.cat([k.flatten() for k in keep if k.numel()]).double().mean()) < 0.7
    ref = _mha_block(Q, K, V, batch, B, H, p, dense)
    assert float((O - ref).detach().abs().max()) < 1e-12
    want = []
    for g in range(B):
        s, e = int(ptr[g]), int(ptr[g + 1])
        if e > s:
            q, k = Q[s:e].view(e - s, H, hd).transpose(0, 1), K[s:e].view(e - s, H, hd).transpose(0, 1)
            want.append(torch.logsumexp(q @ k.transpose(1, 2) / math.sqrt(hd), -1).t())
    assert float((lse - torch.cat(want)).abs().max()) < 1e-12


# ------------------------------------------------------------------------------------------------ argument contract
P = 1 << 20    # placeholder address: never dereferenced
OPS = _lib.ATTN
H, HD = 4, 16
D = H * HD
HP = 16        # hd_pad of HD


def _args(op, **kw):
    """A well-formed 64-node call of op (every tensor and plane the op takes given); kw overrides fields."""
    a = _lib.GpsAttnStageArgs()
    a.graph.N, a.graph.B, a.graph.graph_ptr = 64, 4, P
    a.heads, a.hd = H, HD
    a.Q = a.K = a.V = a.O = a.lse = a.dO = a.delta = a.dQ = a.dK = a.dV = P
    a.ld, a.ldo, a.ldg = 3 * D, D, 3 * D
    a.qkv = _lib.GpsPlanes(P, P, 3 * H * HP)
    for f in ("O_planes", "dQ_planes", "dK_planes", "dV_planes"):
        setattr(a, f, _lib.GpsPlanes(P, P, D))
    for k, v in kw.items():
        if k == "graph_ptr":
            a.graph.graph_ptr = v
        elif k in ("N", "B"):
            setattr(a.graph, k, v)
        else:
            setattr(a, k, v)
    return a


def _call(a, op):
    return _lib.load().gps_attention_stage(None if a is None else C.byref(a), OPS[op] if isinstance(op, str) else op,
                                           None)


def _refused(a, op, code=_lib.GPS_ERR_ARG, msg=None):
    before = _lib.load().gps_launch_count()
    assert _call(a, op) == code, _lib.load().gps_last_error()
    assert _lib.load().gps_launch_count() == before
    if msg is not None:
        assert msg.encode() in _lib.load().gps_last_error(), _lib.load().gps_last_error()


def test_exported():
    lib = _lib.load()
    assert hasattr(lib, "gps_attention_stage")
    assert lib.gps_abi_version() == 4
    assert sorted(OPS.values()) == [0, 1, 2]


@pytest.mark.parametrize("op", list(OPS))
def test_null_args(op):
    _refused(None, op, msg="null args")


@pytest.mark.parametrize("op", [-1, 3, 99])
def test_unknown_op(op):
    _refused(_args("fwd"), op, msg="unknown op")


@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("kw", [{"N": -1}, {"B": -1}, {"N": 1 << 31}, {"B": 0}, {"graph_ptr": 0}],
                         ids=["N<0", "B<0", "N>=2^31", "B=0", "no_graph_ptr"])
def test_graph(op, kw):
    _refused(_args(op, **kw), op)


@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("heads", [0, -1])
def test_heads_below_one(op, heads):
    _refused(_args(op, heads=heads), op, msg="heads must be >= 1")


@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("p", [-0.1, 1.0, 1.5, float("nan"), float("inf"), -float("inf")])
def test_p_drop_outside_0_1(op, p):
    _refused(_args(op, p_drop=p), op, msg="p_drop")


NEEDED = {"fwd": ["Q", "K", "V", "O", "lse"], "fwd_tc": ["O", "lse"],
          "bwd": ["Q", "K", "V", "O", "lse", "dO", "delta", "dQ", "dK", "dV"]}


@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("field", ["Q", "K", "V", "O", "lse", "dO", "delta", "dQ", "dK", "dV"])
def test_null_tensor(op, field):
    if field not in NEEDED[op]:
        pytest.skip("the op does not read or write it")
    _refused(_args(op, **{field: 0}), op, msg="needs")


def test_fwd_tc_needs_qkv_planes():
    _refused(_args("fwd_tc", qkv=_lib.GpsPlanes(0, 0, 3 * H * HP)), "fwd_tc", msg="qkv planes")


PITCHES = {"fwd": ["ld", "ldo"], "fwd_tc": ["ldo"], "bwd": ["ld", "ldo", "ldg"]}


@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("field", ["ld", "ldo", "ldg"])
@pytest.mark.parametrize("ld", [D - 1, 0, -4])
def test_pitch_below_heads_times_hd(op, field, ld):
    """Rows would overlap: reads of one row see the next, and writes race."""
    if field not in PITCHES[op]:
        pytest.skip("the op does not take this pitch")
    _refused(_args(op, **{field: ld}), op, msg=field + " ")


OUT_PLANES = {"fwd": ["O_planes"], "fwd_tc": ["O_planes"], "bwd": ["dQ_planes", "dK_planes", "dV_planes"]}


@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("field", ["O_planes", "dQ_planes", "dK_planes", "dV_planes"])
def test_output_plane_pitch(op, field):
    if field not in OUT_PLANES[op]:
        pytest.skip("the op does not write these planes")
    _refused(_args(op, **{field: _lib.GpsPlanes(P, P, D - 8)}), op, msg="pitch")
    _refused(_args(op, **{field: _lib.GpsPlanes(0, P, D)}), op, msg="lo without hi")
    _refused(_args(op, **{field: _lib.GpsPlanes(P, 0, D + 4)}), op, _lib.GPS_ERR_UNSUPPORTED, "multiple of 8")


def test_qkv_plane_pitch():
    _refused(_args("fwd_tc", qkv=_lib.GpsPlanes(P, P, 3 * H * HP - 8)), "fwd_tc", msg="qkv pitch")
    _refused(_args("fwd_tc", qkv=_lib.GpsPlanes(P, P, 3 * H * HD - 1 + 3 * H * (HP - HD))), "fwd_tc", msg="qkv pitch")
    _refused(_args("fwd_tc", qkv=_lib.GpsPlanes(P, P, 3 * H * HP + 4)), "fwd_tc", _lib.GPS_ERR_UNSUPPORTED,
             "multiple of 8")
    # the pad columns count: hd 20 pads to 32, so 3 * H * 20 columns are too few
    _refused(_args("fwd_tc", hd=20, ldo=H * 20, O_planes=_lib.GpsPlanes(P, P, H * 24),
                   qkv=_lib.GpsPlanes(P, P, 3 * H * 24)), "fwd_tc", msg="qkv pitch")


@pytest.mark.parametrize("precision", [-1, 2])
def test_fwd_tc_precision(precision):
    _refused(_args("fwd_tc", precision=precision), "fwd_tc", msg="precision")


def test_fwd_tc_fp32_needs_lo_planes():
    _refused(_args("fwd_tc", qkv=_lib.GpsPlanes(P, 0, 3 * H * HP), precision=0), "fwd_tc", _lib.GPS_ERR_UNSUPPORTED,
             "qkv.lo")


@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("hd", [0, -3, 193, 256])
def test_head_dim_outside_1_192(op, hd):
    _refused(_args(op, hd=hd, ld=3 * H * 256, ldo=H * 256, ldg=3 * H * 256), op, _lib.GPS_ERR_UNSUPPORTED, "head dim")


@pytest.mark.parametrize("hd", [6, 130, 132, 192])
def test_fwd_tc_head_dims(hd):
    hp = (hd + 15) // 16 * 16
    _refused(_args("fwd_tc", hd=hd, ldo=H * hd, O_planes=_lib.GpsPlanes(P, P, H * hp),
                   qkv=_lib.GpsPlanes(P, P, 3 * H * hp)), "fwd_tc", _lib.GPS_ERR_UNSUPPORTED, "multiple of 4")


@pytest.mark.parametrize("op", list(OPS))
def test_bias(op):
    b = _lib.GpsAttnBias(0, 8, 0)
    _refused(_args(op, bias=C.pointer(b)), op, msg="null attention bias")
    b = _lib.GpsAttnBias(P, 0, P)
    _refused(_args(op, bias=C.pointer(b)), op, msg="nmax")


# the six fixed-signature entry points share the contract
def _graph(N=64, B=4):
    g = _lib.GpsGraph()
    g.N, g.B, g.graph_ptr = N, B, P
    return g


def _entry(name, g=None, heads=H, hd=HD, ld=3 * D, ldo=D, ldg=3 * D, p=0.0, bias=None, precision=0, lo=P):
    lib = _lib.load()
    g = _graph() if g is None else g
    gp = C.byref(g)
    if name == "forward":
        return lib.gps_attention_forward(gp, heads, hd, P, P, P, ld, P, ldo, P, p, 0, 0, None)
    if name == "forward_tc":
        return lib.gps_attention_forward_tc(gp, heads, hd, P, lo, 3 * heads * HP, P, ldo, P, p, 0, 0, precision, None)
    if name == "backward":
        return lib.gps_attention_backward(gp, heads, hd, P, P, P, ld, P, P, ldo, P, P, P, P, P, ldg, p, 0, 0, None)
    bp = None if bias is None else C.byref(bias)
    if name == "forward_biased":
        return lib.gps_attention_forward_biased(gp, heads, hd, P, P, P, ld, P, ldo, P, p, 0, 0, bp, None)
    if name == "forward_tc_biased":
        return lib.gps_attention_forward_tc_biased(gp, heads, hd, P, lo, 3 * heads * HP, P, ldo, P, p, 0, 0, precision,
                                                   bp, None)
    return lib.gps_attention_backward_biased(gp, heads, hd, P, P, P, ld, P, P, ldo, P, P, P, P, P, ldg, p, 0, 0, bp,
                                             None)


ENTRIES = ["forward", "forward_tc", "backward", "forward_biased", "forward_tc_biased", "backward_biased"]


@pytest.mark.parametrize("name", ENTRIES)
@pytest.mark.parametrize("case", ["heads", "p1", "pnan", "ldo", "hd193", "B0", "nobias", "nmax0"])
def test_entry_points_share_the_contract(name, case):
    lib = _lib.load()
    biased = name.endswith("biased")
    good = _lib.GpsAttnBias(P, 8, 0) if biased else None
    kw = {"bias": good}
    want = _lib.GPS_ERR_ARG
    if case == "heads":
        kw["heads"] = 0
    elif case == "p1":
        kw["p"] = 1.0
    elif case == "pnan":
        kw["p"] = float("nan")
    elif case == "ldo":
        kw["ldo"] = D - 4
    elif case == "hd193":
        kw.update(hd=193, ld=3 * H * 193, ldo=H * 193, ldg=3 * H * 193)
        want = _lib.GPS_ERR_UNSUPPORTED
    elif case == "B0":
        kw["g"] = _graph(B=0)
    elif case == "nobias":
        if not biased:
            pytest.skip("unbiased entry point")
        kw["bias"] = None
    elif case == "nmax0":
        if not biased:
            pytest.skip("unbiased entry point")
        kw["bias"] = _lib.GpsAttnBias(P, 0, 0)
    before = lib.gps_launch_count()
    assert _entry(name, **kw) == want, lib.gps_last_error()
    assert lib.gps_launch_count() == before


@pytest.mark.parametrize("name", ENTRIES)
def test_entry_points_refuse_a_null_graph(name):
    lib = _lib.load()
    fn = getattr(lib, "gps_attention_" + name)
    numeric = (C.c_int64, C.c_int32, C.c_float, C.c_uint64)
    args = [0 if t in numeric else None for t in fn.argtypes]
    assert fn(*args) == _lib.GPS_ERR_ARG
