"""GPU: the PNA local model (PyG PNAConv, gps_layer.py:75-90,183-189) stage by stage and in the layer.

Stages against the float64 restatement of tests/pna_reference.py: the edge fold and its backward, the aggregation
(Z = [x | mean | max | sum] and the saved argmax) and its backward (g_q, g_P_dst | g_P_src, g_x), on the BASELINE shapes,
a hub with thousands of in-edges, E = 0, isolated nodes and exact ties.  Every output starts as NaN and every element is
held to its bound; the argmax may pick any edge of a near-tied set.  Then the layer against the reference's own fp64
fixtures (tests/golden/pna/), a finite-difference check with dropout, a 2-layer stack against two oracle layers, a
captured step against eager execution, the graphgym-built layer, and no dense product leaving the TMA GEMM under
GPS_B200_STRICT=1, through the checks tests/local_model_harness.py shares with GAT and GENConv."""
import ctypes as C

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import batch_from_lists, make_batch
from graphgps_b200.graph import graph_of
import pna_reference as R
from local_model_harness import (DEG, SPECS, check_dropout_forward_backward_consistent, check_golden,
                                 check_graphgym_built_layer, check_no_gemm_fallback_under_strict_mode,
                                 check_two_layer_stack_and_capture, golden_names)
from pna_oracle import pna_batch, tie_edge
from util import DEV, _elem_check, _nan, _stream

pytestmark = pytest.mark.gpu
WORST = {}


# ------------------------------------------------------------------------------------------------- stages
def _stage_batch(kind, d):
    if kind == "degenerate":   # an empty graph, single nodes, self loops only, an isolated node, duplicates
        return batch_from_lists([1, 0, 3, 2, 4], [[], [], [(0, 0), (0, 0), (1, 2)], [(0, 0)],
                                                  [(0, 1), (0, 1), (2, 1), (1, 1), (3, 1)]], d=d, seed=3)
    if kind == "no-edges":
        return batch_from_lists([4, 2, 1], [[], [], []], d=d, seed=7)
    if kind == "hub":          # a 3000-node graph whose node 0 has 2999 in-edges
        n = 3000
        lists = [[(j, 0) for j in range(1, n)] + [(0, j) for j in range(1, n, 7)] + [(j, j + 1) for j in range(1, n - 1)]]
        return batch_from_lists([n], lists, d=d, seed=5)
    if kind == "zinc-gine":
        return pna_batch(kind, 9, d, 12)
    return make_batch(kind, seed=9, dim=d, num_graphs=64 if kind == "pcqm4m-small" else 8)


STAGE_CASES = [("zinc-gine", 64), ("zinc-gine", 4), ("pcqm4m-small", 304), ("pcqm4m-small", 36), ("code2", 64),
               ("hub", 36), ("hub", 304), ("degenerate", 4), ("degenerate", 36), ("no-edges", 64)]


def _run_aggregate(b, d, Y, q, x, gZ, add):
    lib = _lib.load()
    bd = b.clone().to(DEV)
    gs = graph_of(bd)
    N, E = b.num_nodes, b.num_edges
    dv = lambda t: t.float().to(DEV).contiguous()
    Yd, qd, xd, gZd, addd = dv(Y), dv(q), dv(x), dv(gZ), dv(add)
    Z, arg = _nan(N, 4 * d), torch.full((N, d), -7, dtype=torch.int32, device=DEV)
    _lib.check(lib.gps_pna_aggregate_forward(C.byref(gs.desc), d, xd.data_ptr(), Yd.data_ptr(), 2 * d,
                                             qd.data_ptr() if E else 0, Z.data_ptr(), arg.data_ptr(), _stream()),
               "pna_aggregate_forward")

    def bwd():
        gq, gY, gx = _nan(max(E, 1), d), _nan(N, 2 * d), _nan(N, d)
        _lib.check(lib.gps_pna_aggregate_backward(C.byref(gs.desc), d, gZd.data_ptr(), arg.data_ptr(), addd.data_ptr(),
                                                  gq.data_ptr() if E else 0, gY.data_ptr(), 2 * d, gx.data_ptr(),
                                                  _stream()), "pna_aggregate_backward")
        torch.cuda.synchronize()
        return gq[:E].cpu(), gY.cpu(), gx.cpu()

    r1, r2 = bwd(), bwd()
    for a, c in zip(r1, r2):
        assert torch.equal(a.nan_to_num(7.0), c.nan_to_num(7.0)), "two runs differ"
    return Z.cpu(), arg.cpu(), r1


@pytest.mark.parametrize("kind,d", STAGE_CASES)
def test_pna_aggregate_stages_match_fp64(kind, d):
    b = _stage_batch(kind, d)
    N, E, ei = b.num_nodes, b.num_edges, b.edge_index
    g = torch.Generator().manual_seed(1)
    Y = torch.randn(N, 2 * d, generator=g)
    q = torch.randn(E, d, generator=g)
    gZ = torch.randn(N, 4 * d, generator=g)
    add = torch.randn(N, d, generator=g)
    Z, arg, (gq, gY, gx) = _run_aggregate(b, d, Y, q, b.x, gZ, add)
    Zr, B, m, bm, bmax = R.aggregate(b.x.double(), Y.double(), q.double(), ei)
    _elem_check(WORST, "Z", Z, Zr, B)
    assert R.argmax_ok(arg, m, ei, Zr[:, 2 * d:3 * d], bmax), "argmax outside the near-tied set"
    gqr, bq, gYr, bY, gxr, bx = R.backward(gZ.double(), arg, ei, N, d, add.double())
    if E:
        _elem_check(WORST, "g_q", gq, gqr, bq)
    _elem_check(WORST, "gY", gY, gYr, bY)
    _elem_check(WORST, "g_x", gx, gxr, bx)
    iso = torch.bincount(ei[1], minlength=N) == 0
    assert bool((Z[iso, d:] == 0).all()) and bool((arg[iso] == -1).all())
    assert torch.equal(Z[:, :d], b.x)
    print(kind, d, {k: round(v, 3) for k, v in sorted(WORST.items())})


def test_exact_tie_sends_the_max_gradient_to_the_first_copy():
    """The exact duplicate of pna_batch has the same message bits as its original in every channel.  Where the pair
    holds the segment max, the argmax is the original (the lower edge id), the copy's g_q has no max share, and the
    original's has all of it."""
    d = 64
    b = pna_batch("zinc-gine", 9, d, 12)
    N, E, ei = b.num_nodes, b.num_edges, b.edge_index
    k, last = tie_edge(b), E - 1
    g = torch.Generator().manual_seed(4)
    Y = torch.randn(N, 2 * d, generator=g)
    q = torch.randn(E, d, generator=g)
    q[last] = q[k]
    gZ = torch.randn(N, 4 * d, generator=g)
    Z, arg, (gq, _, _) = _run_aggregate(b, d, Y, q, b.x, gZ, torch.zeros(N, d))
    t = int(ei[1, k])
    m, _ = R.messages(Y.double(), q.double(), ei, d)
    held = m[k] == m[ei[1] == t].max(0).values
    assert bool(held.any()) and bool((~held).any())
    assert bool((arg[t][held] == k).all()) and not bool((arg[t] == last).any())
    n = float((ei[1] == t).sum())
    base = gZ[t, d:2 * d] / n + gZ[t, 3 * d:]
    assert torch.allclose(gq[last], base, rtol=1e-6, atol=1e-6)
    assert torch.allclose(gq[k][held], (base + gZ[t, 2 * d:3 * d])[held], rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("d", [8, 64, 160, 304])
def test_fold_stages_match_fp64(d):
    lib = _lib.load()
    de = min(128, d)
    g = torch.Generator().manual_seed(d)
    Wpre, bpre = torch.randn(d, 3 * d, generator=g), torch.randn(d, generator=g)
    Wenc, benc = torch.randn(d, de, generator=g), torch.randn(d, generator=g)
    gF, gc = torch.randn(d, de, generator=g), torch.randn(d, generator=g)
    dv = lambda t: t.to(DEV).contiguous()
    W, bp, We, be, gFd, gcd = map(dv, (Wpre, bpre, Wenc, benc, gF, gc))
    F, c = _nan(d, de), _nan(d)
    _lib.check(lib.gps_pna_fold_forward(W.data_ptr(), bp.data_ptr(), We.data_ptr(), be.data_ptr(), d, de, F.data_ptr(),
                                        c.data_ptr(), _stream()), "pna_fold_forward")
    Fr, bF, cr, bc = R.fold(Wpre.double(), bpre.double(), Wenc.double(), benc.double())
    _elem_check(WORST, "F", F.cpu(), Fr, bF)
    _elem_check(WORST, "c", c.cpu(), cr, bc)
    gW = torch.full((d, 3 * d), 5.0, device=DEV)   # blocks 0..2d untouched
    gbp, gWe, gbe = _nan(d), _nan(d, de), _nan(d)
    for acc in (0, 1):
        _lib.check(lib.gps_pna_fold_backward(W.data_ptr(), We.data_ptr(), be.data_ptr(), gFd.data_ptr(), gcd.data_ptr(),
                                             d, de, gW.data_ptr(), gbp.data_ptr(), gWe.data_ptr(), gbe.data_ptr(), acc,
                                             _stream()), "pna_fold_backward")
        torch.cuda.synchronize()
        if acc == 0:
            first = [t.cpu().clone() for t in (gW, gbp, gWe, gbe)]
    gWeR, bWe, gWencR, bWenc, gbencR, bbenc = R.unfold(Wpre.double(), Wenc.double(), benc.double(), gF.double(),
                                                      gc.double())
    _elem_check(WORST, "g_W_e", first[0][:, 2 * d:], gWeR, bWe)
    _elem_check(WORST, "g_W_enc", first[2], gWencR, bWenc)
    _elem_check(WORST, "g_b_enc", first[3], gbencR, bbenc)
    assert torch.equal(first[1], gc)
    assert bool((first[0][:, :2 * d] == 5.0).all())
    assert torch.equal(gW.cpu()[:, 2 * d:], 2 * first[0][:, 2 * d:])   # accumulate adds the same bits again
    assert torch.equal(gbe.cpu(), 2 * first[3])


# ------------------------------------------------------------------------------------------------- layer
# the checks every local model shares, from tests/local_model_harness.py
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", golden_names(SPECS["PNA"]))
def test_layer_matches_pna_golden(name, precision):
    check_golden(SPECS["PNA"], name, precision)


def test_edge_width_is_checked():
    layer = graphgps_b200.GPSLayer(160, "PNA", "None", 4, pna_degrees=DEG).to(DEV)
    b = pna_batch("zinc-gine", 1, 160, 2).to(DEV)
    b.edge_attr = torch.zeros(b.edge_attr.shape[0], 160, device=DEV)
    with pytest.raises(ValueError, match="min\\(128, dim_h\\) = 128"):
        layer(b)


def test_pna_dropout_forward_backward_consistent():
    check_dropout_forward_backward_consistent(SPECS["PNA"])


def test_two_layer_stack_matches_two_oracle_layers_and_capture_matches_eager():
    check_two_layer_stack_and_capture(SPECS["PNA"])


def test_graphgym_built_pna_transformer_layer_runs(monkeypatch):
    check_graphgym_built_layer(SPECS["PNA"], monkeypatch)


def test_no_gemm_fallback_under_strict_mode():
    check_no_gemm_fallback_under_strict_mode(SPECS["PNA"])
