"""CPU: (1) the fp64 Performer stage references of tests/performer_reference.py, composed with fp64 to_q/k/v,
dd = (x 64^-1/4) P^T and to_out, equal OraclePerformerSelfAttention on the zero-padded dense batch, output and every
gradient (the path through the un-detached amax included) to 1e-12, in both attention forms; (2) the argument contract
of the Performer stage entry points and of gps_layer_plan's int32 index range: every call here is rejected before any
CUDA call, so it needs no device memory (the addresses are placeholders that are never dereferenced)."""
import ctypes as C

import pytest
import torch

from graphgps_b200 import _lib
from oracle.gps_oracle import OraclePerformerSelfAttention
import performer_reference as R

TOL = 1e-12
F64 = torch.float64


def _close(a, b, what):
    a, b = a.detach(), b.detach()
    err = float((a - b).abs().max() / max(1.0, float(b.abs().max())))
    assert err <= TOL, f"{what}: {err}"


# graph sizes: padding of every depth, an empty graph between non-empty ones, single-node graphs
SIZES = [5, 1, 0, 9, 3, 1, 7]


@pytest.mark.parametrize("form", [0, 1])
@pytest.mark.parametrize("heads", [1, 2])
def test_stages_compose_to_the_oracle(form, heads):
    torch.manual_seed(0)
    d = 24
    ora = OraclePerformerSelfAttention(d, heads).double()
    P = ora.fast_attention.projection_matrix
    m = P.shape[0]
    ptr = torch.tensor([0] + SIZES).cumsum(0)
    batch, pos, B, Nmax = R.layout(ptr)
    N = batch.numel()
    x = torch.randn(N, d, dtype=F64, requires_grad=True)
    dense = x.new_zeros(B, Nmax, d).index_put((batch, pos), x)
    mask = torch.zeros(B, Nmax, dtype=torch.bool).index_put((batch, pos), torch.ones(N, dtype=torch.bool))
    out_o = ora(dense, mask)[batch, pos]

    dn = R.DH ** -0.25
    q, k, v = (lin(x).reshape(N * heads, R.DH) for lin in (ora.to_q, ora.to_k, ora.to_v))
    fq, fk, gmax = R.features((q * dn) @ P.t(), (k * dn) @ P.t(), q, k, ptr, heads, m)
    O, _ = R.attention(fq, fk, v, gmax, ptr, heads, Nmax, form)
    out_s = ora.to_out(O.reshape(N, heads * R.DH))
    _close(out_s, out_o, "out")

    ct = torch.randn(out_o.shape, generator=torch.Generator().manual_seed(1), dtype=F64)
    leaves = [x] + list(ora.parameters())
    names = ["x"] + [n for n, _ in ora.named_parameters()]
    go = torch.autograd.grad(out_o, leaves, ct, retain_graph=True)
    gs = torch.autograd.grad(out_s, leaves, ct, retain_graph=True)
    for a, b, n in zip(gs, go, names):
        _close(a, b, "grad " + n)

    # the stage backwards chained by hand: attention, features, then g_q = g_dd (dn P) + the diag path
    gO = torch.autograd.grad(out_s, O, ct, retain_graph=True)[0]
    g_fq, g_fk, gV, g_gmax = R.attention_backward(fq, fk, v, gmax, ptr, heads, Nmax, form, gO)
    dd_q, dd_k = (q * dn) @ P.t(), (k * dn) @ P.t()
    g_ddq, g_ddk, gQ, gK = R.features_backward(dd_q, dd_k, q, k, ptr, heads, m, g_fq, g_fk, g_gmax)
    wq, wk, wv = torch.autograd.grad(out_s, [q, k, v], ct)
    _close(g_ddq @ P * dn + gQ, wq, "g_q through the stages")
    _close(g_ddk @ P * dn + gK, wk, "g_k through the stages")
    _close(gV, wv, "g_v through the stages")
    assert float(g_gmax.abs().max()) > 0, "the padded rows give the key max a gradient"


def test_forms_agree():
    torch.manual_seed(1)
    ptr = torch.tensor([0] + SIZES).cumsum(0)
    _, _, B, Nmax = R.layout(ptr)
    N, H, m = int(ptr[-1]), 2, 266
    qf, kf = (torch.rand(N * H, m, dtype=F64) for _ in range(2))
    V, gmax = torch.randn(N * H, R.DH, dtype=F64), torch.rand(B * H, dtype=F64)
    gO = torch.randn(N * H, R.DH, dtype=F64)
    for a, b in zip(R.attention(qf, kf, V, gmax, ptr, H, Nmax, 0), R.attention(qf, kf, V, gmax, ptr, H, Nmax, 1)):
        _close(a, b, "forward")
    for a, b in zip(R.attention_backward(qf, kf, V, gmax, ptr, H, Nmax, 0, gO),
                    R.attention_backward(qf, kf, V, gmax, ptr, H, Nmax, 1, gO)):
        _close(a, b, "backward")


def test_ties_first_moves_the_split_share_to_the_lowest_index():
    """ties="first" gives a tied maximum's whole gradient to its lowest index; torch.amax splits it.  The totals agree,
    and outside the tied elements both are equal."""
    torch.manual_seed(2)
    ptr = torch.tensor([0, 3, 5])
    H, m = 1, 260
    dd_q, dd_k = torch.randn(5, m, dtype=F64), torch.randn(5, m, dtype=F64)
    dd_q[:, 7] = dd_q[:, 3] = dd_q.amax(1) + 0.5          # every query row: a tie between features 3 and 7
    dd_k[1] = dd_k[0]                                     # graph 0: its max is tied between rows 0 and 1
    Q, K = torch.randn(5, R.DH, dtype=F64), torch.randn(5, R.DH, dtype=F64)
    g = [torch.randn(5, m, dtype=F64), torch.randn(5, m, dtype=F64), torch.randn(2, dtype=F64)]
    split = R.features_backward(dd_q, dd_k, Q, K, ptr, H, m, *g)
    first = R.features_backward(dd_q, dd_k, Q, K, ptr, H, m, *g, ties="first")
    _close(first[0][:, 3] + first[0][:, 7], split[0][:, 3] + split[0][:, 7], "query tie total")
    assert not torch.allclose(first[0][:, 3], split[0][:, 3])
    rest = [j for j in range(m) if j not in (3, 7)]
    _close(first[0][:, rest], split[0][:, rest], "query rows off the tie")
    j = int(dd_k[0].argmax())
    _close(first[1][0, j] + first[1][1, j], split[1][0, j] + split[1][1, j], "key tie total")
    _close(first[1][2:], split[1][2:], "graph 1 has no tie")


# ---------------------------------------------------------------------------------------------------- argument contract
P = 1 << 20    # placeholder address: never dereferenced, every call below fails validation first


def _graph(N=8, B=2):
    return _lib.GpsGraph(N, 0, B, P, P, P, P, P, P, P)


def _calls(lib, g, H, dh, m, form, null):
    """(pointer names, thunk) for every Performer stage entry point; `null` names the one pointer passed as NULL"""
    def a(name):
        return 0 if name == null else P
    return {
        "gps_performer_prep": (
            ["P", "Pn", "nmax", "gmax", "argk"],
            lambda: lib.gps_performer_prep(C.byref(g), H, dh, m, a("P"), a("Pn"), a("nmax"), a("gmax"), a("argk"), 0)),
        "gps_performer_features_forward": (
            ["fq", "fk", "Q", "K", "gmax", "argq", "argk"],
            lambda: lib.gps_performer_features_forward(C.byref(g), H, dh, m, a("fq"), a("fk"), a("Q"), a("K"),
                                                       a("gmax"), a("argq"), a("argk"), 0)),
        "gps_performer_attention_forward": (
            ["nmax", "qf", "kf", "V", "gmax", "O"] + (["den"] if form == 1 else []),
            lambda: lib.gps_performer_attention_forward(C.byref(g), H, dh, m, form, a("nmax"), a("qf"), a("kf"),
                                                        a("V"), a("gmax"), a("O"), a("den"), 0)),
        "gps_performer_attention_backward": (
            ["nmax", "qf", "kf", "V", "gmax", "gO", "g_qf", "g_kf", "gV"] +
            (["ggmax"] if form == 0 else ["O", "den", "gden", "gmrow"]),
            lambda: lib.gps_performer_attention_backward(C.byref(g), H, dh, m, form, a("nmax"), a("qf"), a("kf"),
                                                         a("V"), a("gmax"), a("O"), a("den"), a("gO"), a("gden"),
                                                         a("g_qf"), a("g_kf"), a("gV"), a("ggmax"), a("gmrow"), 0)),
        "gps_performer_features_backward": (
            ["g_fq", "g_fk", "fq", "fk", "Q", "K", "gQ", "gK", "argq", "argk", "gmrow"] +
            (["ggmax"] if form == 0 else []),
            lambda: lib.gps_performer_features_backward(C.byref(g), H, dh, m, form, a("g_fq"), a("g_fk"), a("fq"),
                                                        a("fk"), a("Q"), a("K"), a("gQ"), a("gK"), a("argq"),
                                                        a("argk"), a("ggmax"), a("gmrow"), 0)),
    }


NAMES = list(_calls(None, _graph(), 1, 64, 266, 0, None))


@pytest.mark.parametrize("form", [0, 1])
@pytest.mark.parametrize("name", NAMES)
def test_stage_entry_points_reject_null_pointers(name, form):
    lib = _lib.load()
    g = _graph()
    ptrs, _ = _calls(lib, g, 2, 64, 266, form, None)[name]
    for p in ptrs:
        rc = _calls(lib, g, 2, 64, 266, form, p)[name][1]()
        assert rc == _lib.GPS_ERR_ARG, (name, form, p, rc)
        assert lib.gps_last_error()


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("dh,m,H,N", [(64, 256, 1, 8), (64, 273, 1, 8), (64, 0, 1, 8), (32, 266, 1, 8),
                                      (128, 266, 1, 8), (64, 266, 0, 8), (64, 266, 4, (2 ** 31 - 1) // 272 // 4 + 1),
                                      (64, 266, 1, 2 ** 40)])
def test_stage_entry_points_reject_unsupported_shapes(name, dh, m, H, N):
    lib = _lib.load()
    for form in (0, 1):
        rc = _calls(lib, _graph(N=N), H, dh, m, form, None)[name][1]()
        assert rc == _lib.GPS_ERR_UNSUPPORTED, (name, dh, m, H, N, form, rc)


@pytest.mark.parametrize("name", ["gps_performer_attention_forward", "gps_performer_attention_backward",
                                  "gps_performer_features_backward"])
@pytest.mark.parametrize("form", [-1, 2])
def test_stage_entry_points_reject_unknown_forms(name, form):
    lib = _lib.load()
    assert _calls(lib, _graph(), 1, 64, 266, form, None)[name][1]() == _lib.GPS_ERR_ARG


def _plan(N, heads):
    a = _lib.GpsLayerArgs()
    a.d, a.heads, a.global_type, a.act, a.training = 64, heads, _lib.GLOBAL["Performer"], 0, 1
    a.perf_features, a.perf_dim_head = 266, 64
    a.graph.N, a.graph.E, a.graph.B = N, 0, 1
    plan = _lib.GpsLayerPlan()
    return _lib.load().gps_layer_plan(C.byref(a), C.byref(plan)), plan


@pytest.mark.parametrize("heads", [1, 4, 16])
def test_plan_rejects_feature_maps_beyond_int32_indexing(heads):
    """argk holds the flat index (n H + h) 272 + j of the key feature map in an int: N H 272 must stay below 2^31"""
    limit = (2 ** 31 - 1) // 272 // heads
    rc, plan = _plan(limit, heads)
    assert rc == _lib.GPS_OK, _lib.load().gps_last_error()
    assert limit * heads * 272 < 2 ** 31
    rc, _ = _plan(limit + 1, heads)
    assert rc == _lib.GPS_ERR_UNSUPPORTED
    assert b"int32" in _lib.load().gps_last_error()
