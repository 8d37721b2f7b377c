"""GPU: the GENConv local model (PyG GENConv, gps_layer.py:60-61,183-189) stage by stage and in the layer.

Stages against the float64 restatement of tests/genconv_reference.py: the softmax aggregation (agg, the saved log-sum-exp
and u = agg + x) and its backward (grad_edge_attr and g_x), on the BASELINE shapes (zinc-gine, pcqm4m-small, code2), a
hub with thousands of in-edges, E = 0 and isolated nodes, with d in {4, 36, 64, 304, 2048}.  Every output starts as NaN.
Every element is held to a bound of the K n 2^-24 sum|terms| kind with the message errors carried through exp
(tests/genconv_reference.py::error_bounds); the worst error as a fraction of its bound is printed.  The layer against
the reference's own fp64 fixtures (tests/golden/genconv/), a finite-difference check with dropout, a 2-layer stack
against two oracle layers, a captured step against eager execution, the graphgym-built layer, and no dense product
leaving the TMA GEMM under GPS_B200_STRICT=1, through the checks tests/local_model_harness.py shares with GAT and PNA."""
import ctypes as C

import pytest
import torch

from graphgps_b200 import _lib
from graphgps_b200.batch import batch_from_lists, make_batch
from graphgps_b200.graph import graph_of
import genconv_reference as R
from genconv_oracle import dead_node, genconv_batch
from local_model_harness import (SPECS, check_dropout_forward_backward_consistent, check_golden,
                                 check_graphgym_built_layer, check_no_gemm_fallback_under_strict_mode,
                                 check_two_layer_stack_and_capture, golden_names)
from util import DEV, _elem_check, _nan, _stream

pytestmark = pytest.mark.gpu
WORST = {}


# ------------------------------------------------------------------------------------------------- stages
def _stage_batch(kind, d):
    if kind == "degenerate":   # an empty graph, single nodes, self loops only, an isolated node, duplicates
        b = batch_from_lists([1, 0, 3, 2, 4], [[], [], [(0, 0), (0, 0), (1, 2)], [(0, 0)],
                                                [(0, 1), (0, 1), (2, 1), (1, 1), (3, 1)]], d=d, seed=3)
    elif kind == "no-edges":
        b = batch_from_lists([4, 2, 1], [[], [], []], d=d, seed=7)
    elif kind == "hub":        # a 3000-node graph whose node 0 has 2999 in-edges
        n = 3000
        lists = [[(j, 0) for j in range(1, n)] + [(0, j) for j in range(1, n, 7)] + [(j, j + 1) for j in range(1, n - 1)]]
        b = batch_from_lists([n], lists, d=d, seed=5)
    elif kind == "zinc-gine":
        return genconv_batch(kind, 9, d, 8 if d > 1000 else 12)
    else:
        b = make_batch(kind, seed=9, dim=d, num_graphs=64 if kind == "pcqm4m-small" else 8)
    b.x, b.edge_attr = b.x * 3.0, b.edge_attr * 3.0
    return b


STAGE_CASES = [("zinc-gine", 64), ("zinc-gine", 4), ("zinc-gine", 2048), ("pcqm4m-small", 304), ("pcqm4m-small", 36),
               ("code2", 64), ("hub", 36), ("hub", 304), ("degenerate", 4), ("degenerate", 36), ("no-edges", 64)]


def _run_stages(b, d, seed=1):
    lib = _lib.load()
    bd = b.clone().to(DEV)
    gs = graph_of(bd)
    N, E = b.num_nodes, b.num_edges
    g = torch.Generator().manual_seed(seed)
    g_u = torch.randn(N, d, generator=g)
    add = torch.randn(N, d, generator=g)
    dv = lambda t: t.to(DEV).contiguous()
    xd, ed, gud, addd = dv(b.x), dv(b.edge_attr), dv(g_u), dv(add)
    agg, lse, u = _nan(N, d), _nan(N, d), _nan(N, d)
    _lib.check(lib.gps_genconv_aggregate_forward(C.byref(gs.desc), d, xd.data_ptr(), _lib.ptr(ed) if E else 0,
                                                 agg.data_ptr(), lse.data_ptr(), u.data_ptr(), _stream()),
               "genconv_aggregate_forward")

    def bwd():
        ge, gx = _nan(max(E, 1), d), _nan(N, d)
        _lib.check(lib.gps_genconv_aggregate_backward(C.byref(gs.desc), d, xd.data_ptr(), _lib.ptr(ed) if E else 0,
                                                      agg.data_ptr(), lse.data_ptr(), gud.data_ptr(), addd.data_ptr(),
                                                      ge.data_ptr() if E else 0, gx.data_ptr(), _stream()),
                   "genconv_aggregate_backward")
        torch.cuda.synchronize()
        return ge[:E].cpu(), gx.cpu()

    r1, r2 = bwd(), bwd()
    for a, c in zip(r1, r2):
        assert torch.equal(a.nan_to_num(7.0), c.nan_to_num(7.0)), "two runs differ"
    return dict(N=N, E=E, agg=agg.cpu(), lse=lse.cpu(), u=u.cpu(), g_u=g_u, add=add, g_e=r1[0], g_x=r1[1])


@pytest.mark.parametrize("kind,d", STAGE_CASES)
def test_genconv_stages_match_fp64(kind, d):
    b = _stage_batch(kind, d)
    r = _run_stages(b, d)
    ei = b.edge_index
    x = b.x.double().requires_grad_(True)
    e = b.edge_attr.double().requires_grad_(True)
    agg, lse, u = R.aggregate(x, ei, e)
    g_u, add = r["g_u"].double(), r["add"].double()
    B = R.error_bounds(x.detach(), ei, e.detach(), g_u, add)
    _elem_check(WORST, "agg", r["agg"], agg.detach(), B["agg"])
    _elem_check(WORST, "lse", r["lse"], lse.detach(), B["lse"])
    _elem_check(WORST, "u", r["u"], u.detach(), B["u"])
    gx, ge = torch.autograd.grad((u * g_u).sum(), [x, e])
    _elem_check(WORST, "g_e", r["g_e"], ge, B["g_e"])
    _elem_check(WORST, "g_x", r["g_x"], gx + add, B["g_x"])
    # structural cases are exact: a node without in-edges has agg = 0, lse = 0, u = x; an edge whose x_src + e <= 0
    # in a channel gets exactly 0 there
    iso = torch.bincount(ei[1], minlength=r["N"]) == 0
    assert bool((r["agg"][iso] == 0).all()) and bool((r["lse"][iso] == 0).all())
    assert torch.equal(r["u"][iso], b.x[iso])
    if r["E"]:
        dead = (b.x[ei[0]] + b.edge_attr) <= 0
        assert bool((r["g_e"][dead] == 0).all())
    print(kind, d, {k: round(v, 3) for k, v in sorted(WORST.items())})


def test_all_1e7_messages_give_uniform_weights():
    """The node of genconv_batch whose messages are all 1e-7: agg = 1e-7 and its in-edges get no gradient."""
    b = genconv_batch("zinc-gine", 9, 64, 4)
    r = _run_stages(b, 64)
    t = dead_node(b)
    assert torch.allclose(r["agg"][t], torch.full((64,), 1e-7), rtol=1e-5, atol=0)
    k = b.edge_index[1] == t
    assert bool((r["g_e"][k] == 0).all())


# ------------------------------------------------------------------------------------------------- layer
# the checks every local model shares, from tests/local_model_harness.py
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", golden_names(SPECS["GENConv"]))
def test_layer_matches_genconv_golden(name, precision):
    check_golden(SPECS["GENConv"], name, precision)


def test_genconv_dropout_forward_backward_consistent():
    check_dropout_forward_backward_consistent(SPECS["GENConv"])


def test_two_layer_stack_matches_two_oracle_layers_and_capture_matches_eager():
    check_two_layer_stack_and_capture(SPECS["GENConv"])


def test_graphgym_built_genconv_transformer_layer_runs(monkeypatch):
    check_graphgym_built_layer(SPECS["GENConv"], monkeypatch)


def test_no_gemm_fallback_under_strict_mode():
    check_no_gemm_fallback_under_strict_mode(SPECS["GENConv"])
