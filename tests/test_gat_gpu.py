"""GPU: the GAT local model (PyG GATConv, gps_layer.py:70-74,183-189) stage by stage and in the layer.

Stages against the float64 restatement of tests/gat_reference.py: the fold, the forward (the saved scores and
log-sum-exp included) and the backward (gY, grad_edge_attr, g_v, g_att_src, g_att_dst, g_bias), on the BASELINE shapes,
MalNet-like hubs, degenerate graphs and an in-degree sweep, with C = d / H in {1, 9, 16, 24, 64, 76}.  Every output
starts as NaN.  Every element is held to a bound of the gamma_n kind: K n 2^-24 sum|terms| with n the length of the sums
that produce it (a head's C channels, an edge's d, a node's in- or out-degree + 1, a column sum's chunk), with the
score errors carried through exp into the attention weights (tests/gat_reference.py::error_bounds); the worst error as
a fraction of its bound is printed.  Structural cases are exact.  The layer
against the reference's own fp64 fixtures (tests/golden/gat/), a finite-difference check with dropout, a 2-layer stack
against two oracle layers, a captured step against eager execution, and the graphgym-built layer, through the checks
tests/local_model_harness.py shares with GENConv and PNA."""
import ctypes as C
import math

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import batch_from_lists, make_batch
from graphgps_b200.graph import graph_of
import gat_reference as R
from gat_oracle import gat_batch
from local_model_harness import (SPECS, check_dropout_forward_backward_consistent, check_golden,
                                 check_graphgym_built_layer, check_two_layer_stack_and_capture, golden_names)
from util import DEV, _elem_check, _nan, _stream

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
WORST = {}


def _bound_check(name, got, ref, absref, n, K=4.0):
    """|got - ref| <= K n u absref + tiny, elementwise; absref = the same computation on absolute values."""
    got, ref, absref = got.double().cpu(), ref.double().cpu(), absref.double().cpu()
    assert not torch.isnan(got).any(), f"{name}: NaN left in the output"
    bound = K * max(n, 1) * U * absref + 1e-30
    frac = float(((got - ref).abs() / bound).max()) if got.numel() else 0.0
    WORST[name] = max(WORST.get(name, 0.0), frac)
    assert frac <= 1.0, f"{name}: error {frac:.3g} x its bound"
    return frac


# ------------------------------------------------------------------------------------------------- stage inputs
def _stage_batch(kind, d):
    if kind == "degenerate":   # empty graph, single nodes, a node with only self loops, an isolated node, duplicates
        return batch_from_lists([1, 0, 3, 2, 4], [[], [], [(0, 0), (0, 0), (1, 2)], [(0, 0)],
                                                  [(0, 1), (0, 1), (2, 1), (1, 1), (3, 1)]], d=d, seed=3)
    if kind == "sweep":        # in-degree 0..5, 64, 65
        sizes, lists = [], []
        for k in (0, 1, 2, 3, 4, 5, 64, 65):
            sizes.append(k + 1)
            lists.append([(j + 1, 0) for j in range(k)])
        return batch_from_lists(sizes, lists, d=d, seed=4)
    if kind == "malnet":       # hubs with thousands of in-edges
        n = 3000
        lists = [[(j, 0) for j in range(1, n)] + [(0, j) for j in range(1, n, 7)] + [(j, j + 1) for j in range(1, n - 1)]]
        return batch_from_lists([n], lists, d=d, seed=5)
    return gat_batch(kind, 9, d, 12 if kind == "zinc-gine" else 6)


def _params(d, H, seed):
    g = torch.Generator().manual_seed(seed)
    C_ = d // H
    a = 3.0 * math.sqrt(6.0 / (H + C_))
    att = [(torch.rand(H * C_, generator=g) * 2 - 1) * a for _ in range(3)]
    W = torch.randn(d, d, generator=g) / math.sqrt(d)
    bias = torch.randn(d, generator=g) * 0.3
    return att, W, bias


STAGE_CASES = [("zinc-gine", 64, 4), ("pcqm4m-small", 64, 4), ("zinc-gine", 36, 4), ("zinc-gine", 64, 1),
               ("zinc-gine", 96, 4), ("pcqm4m-small", 304, 4), ("zinc-gine", 64, 64), ("malnet", 64, 4),
               ("degenerate", 36, 4), ("sweep", 48, 2)]


def _run_stages(b, d, H, seed=1):
    lib = _lib.load()
    bd = b.clone().to(DEV)   # GraphBatch.to moves in place
    gs = graph_of(bd)
    N, E = b.num_nodes, b.num_edges
    (att_src, att_dst, att_edge), W, bias = _params(d, H, seed)
    g = torch.Generator().manual_seed(seed + 1)
    Y = torch.randn(N, d, generator=g)
    x = torch.randn(N, d, generator=g)
    dv = lambda t: t.to(DEV).contiguous()
    v = _nan(H, d)
    Wd, aed = dv(W), dv(att_edge)
    _lib.check(lib.gps_gat_fold_forward(Wd.data_ptr(), aed.data_ptr(), d, H, v.data_ptr(), _stream()), "fold")
    scores = _nan((4 * N + E) * H)
    xloc = _nan(N, d)
    Yd, xd, ead, asd, add_, bd_ = dv(Y), dv(x), dv(b.edge_attr), dv(att_src), dv(att_dst), dv(bias)
    _lib.check(lib.gps_gat_forward(C.byref(gs.desc), d, H, Yd.data_ptr(), d, _lib.ptr(ead) if E else 0, v.data_ptr(),
                                   asd.data_ptr(), add_.data_ptr(), bd_.data_ptr(), xd.data_ptr(), scores.data_ptr(),
                                   xloc.data_ptr(), 0.0, 0, 0, None, _stream()), "gat_forward")
    g_h = torch.randn(N, d, generator=g)
    ghd = dv(g_h)
    ws = torch.empty(max(int(lib.gps_gat_workspace_bytes(N, E, H, d)), 4), dtype=torch.uint8, device=DEV)

    def bwd():
        out = dict(gY=_nan(N, d), gea=_nan(max(E, 1), d), gv=_nan(H, d), gas=_nan(d), gad=_nan(d), gb=_nan(d),
                   gW=_nan(d, d), gae=_nan(d))
        _lib.check(lib.gps_gat_backward(C.byref(gs.desc), d, H, Yd.data_ptr(), d, _lib.ptr(ead) if E else 0,
                                        v.data_ptr(), asd.data_ptr(), add_.data_ptr(), scores.data_ptr(), ghd.data_ptr(),
                                        ws.data_ptr(), ws.numel(), out["gY"].data_ptr(), d, None,
                                        out["gea"].data_ptr() if E else 0, out["gv"].data_ptr(), out["gas"].data_ptr(),
                                        out["gad"].data_ptr(), out["gb"].data_ptr(), 0, _stream()), "gat_backward")
        _lib.check(lib.gps_gat_fold_backward(Wd.data_ptr(), aed.data_ptr(), out["gv"].data_ptr(), d, H,
                                             out["gW"].data_ptr(), out["gae"].data_ptr(), 0, _stream()), "fold_backward")
        torch.cuda.synchronize()
        return {k: t.cpu() for k, t in out.items()}

    res = bwd()
    res2 = bwd()
    for k in res:
        assert torch.equal(res[k].nan_to_num(7.0), res2[k].nan_to_num(7.0)), f"{k}: two runs differ"
    torch.cuda.synchronize()
    return dict(N=N, E=E, Y=Y, x=x, W=W, att=(att_src, att_dst, att_edge), bias=bias, g_h=g_h, v=v.cpu(),
                scores=scores.cpu(), xloc=xloc.cpu(), bwd=res)


@pytest.mark.parametrize("kind,d,H", STAGE_CASES)
def test_gat_stages_match_fp64(kind, d, H):
    b = _stage_batch(kind, d)
    r = _run_stages(b, d, H)
    N, E = r["N"], r["E"]
    ei = b.edge_index
    dd = lambda t: t.double().requires_grad_(True)
    W, bias, Y, ea = dd(r["W"]), dd(r["bias"]), dd(r["Y"]), dd(b.edge_attr)
    a_s, a_d, a_e = dd(r["att"][0]), dd(r["att"][1]), dd(r["att"][2])
    C_ = d // H
    # fold
    v64 = R.fold(W, a_e, H)
    _bound_check("fold", r["v"], v64.detach(), R.fold(W.detach().abs(), a_e.detach().abs(), H), C_)
    vleaf = r["v"].double().requires_grad_(True)   # the stages below read the library's v
    # scores and forward
    s = R.scores(Y, ei, ea, vleaf, a_s, a_d, H)
    sc = r["scores"]
    NH = N * H
    absY, absv = Y.detach().abs(), vleaf.detach().abs()
    sa = R.scores(absY, ei, ea.detach().abs(), absv, a_s.detach().abs(), a_d.detach().abs(), H)
    _bound_check("a_src", sc[:NH].view(N, H), s["a_src"].detach(), sa["a_src"], C_)
    _bound_check("a_dst", sc[NH:2 * NH].view(N, H), s["a_dst"].detach(), sa["a_dst"], C_)
    _bound_check("a_edge", sc[4 * NH:].view(E, H), s["a_edge"].detach(), sa["a_edge"], d)
    out = R.aggregate(Y, ei, ea, vleaf, a_s, a_d, bias, H)
    g_h = r["g_h"].double()
    B = R.error_bounds(Y.detach(), ei, ea.detach(), vleaf.detach(), a_s.detach(), a_d.detach(), bias.detach(),
                       r["x"].double(), g_h, H)
    _elem_check(WORST, "a_self", sc[2 * NH:3 * NH].view(N, H), s["a_self"].detach(), B["a_self"])
    _elem_check(WORST, "lse", sc[3 * NH:4 * NH].view(N, H), s["lse"].detach(), B["lse"])
    _elem_check(WORST, "xloc", r["xloc"], r["x"].double() + out.detach(), B["xloc"])
    # backward
    grads = torch.autograd.grad((out * g_h).sum(), [Y, ea, vleaf, a_s, a_d, bias])
    gres = r["bwd"]
    for name, got, ref in (("gY", gres["gY"], grads[0]), ("grad_edge_attr", gres["gea"][:E], grads[1]),
                           ("g_v", gres["gv"], grads[2]), ("g_att_src", gres["gas"], grads[3]),
                           ("g_att_dst", gres["gad"], grads[4]), ("g_bias", gres["gb"], grads[5])):
        _elem_check(WORST, name, got, ref.reshape(got.shape), B[name])
    # fold backward from the library's g_v: g_W_edge[hC+c, :] = att_edge[hC+c] g_v[h], g_att_edge = W_edge . g_v
    gv = gres["gv"].double()
    ae64 = a_e.detach()
    gv_rows = gv.repeat_interleave(C_, 0)                                   # [d, d]: row hC+c holds g_v[h]
    _elem_check(WORST, "g_W_edge", gres["gW"], ae64[:, None] * gv_rows, 2 * U * (ae64[:, None] * gv_rows).abs())
    _elem_check(WORST, "g_att_edge", gres["gae"], (W.detach() * gv_rows).sum(1),
                4 * d * U * (W.detach().abs() * gv_rows.abs()).sum(1))
    # removed self loops: grad_edge_attr exactly 0
    if E:
        selfe = ei[0] == ei[1]
        assert bool((gres["gea"][:E][selfe] == 0).all())
    print(kind, d, H, {k: round(v, 3) for k, v in sorted(WORST.items())})


def test_gat_structural_cases_are_exact():
    """An isolated node has alpha = 1 (x_loc = x + (Y + bias) bit for bit); an all-self-loop batch and E = 0 give
    out = Y + bias everywhere."""
    lib = _lib.load()
    d, H = 36, 4
    for b in (batch_from_lists([3, 1, 2], [[(0, 0), (1, 1), (2, 2)], [(0, 0), (0, 0)], [(1, 1)]], d=d, seed=6),
              batch_from_lists([4, 2], [[], []], d=d, seed=7),
              gat_batch("zinc-gine", 9, d, 4)):
        r = _run_stages(b, d, H, seed=2)
        expect = r["x"] + (r["Y"] + r["bias"])
        deg = torch.bincount(b.edge_index[1][b.edge_index[0] != b.edge_index[1]], minlength=r["N"])
        iso = deg == 0
        assert bool(iso.any())
        assert torch.equal(r["xloc"][iso], expect[iso])
        if not bool((b.edge_index[0] != b.edge_index[1]).any()):
            assert torch.equal(r["xloc"], expect)
            assert bool((r["bwd"]["gea"][:r["E"]] == 0).all())


# ------------------------------------------------------------------------------------------------- layer
# the checks every local model shares, from tests/local_model_harness.py
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", golden_names(SPECS["GAT"]))
def test_layer_matches_gat_golden(name, precision):
    check_golden(SPECS["GAT"], name, precision)


def test_gat_dropout_forward_backward_consistent():
    check_dropout_forward_backward_consistent(SPECS["GAT"])


def test_two_layer_stack_matches_two_oracle_layers_and_capture_matches_eager():
    check_two_layer_stack_and_capture(SPECS["GAT"])


def test_graphgym_built_gat_transformer_layer_runs(monkeypatch):
    check_graphgym_built_layer(SPECS["GAT"], monkeypatch)


def test_gat_layer_validation():
    layer = graphgps_b200.GPSLayer(32, "GAT", "Transformer", 4).to(DEV)
    b = make_batch("zinc-gine", seed=1, dim=32, num_graphs=3).to(DEV)
    b.edge_attr = b.edge_attr[:, :16].contiguous()
    with pytest.raises(ValueError):
        layer(b)
