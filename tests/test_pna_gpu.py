"""GPU: the PNA local model (PyG PNAConv, gps_layer.py:75-90,183-189) stage by stage and in the layer.

Stages against the float64 restatement of tests/pna_reference.py: the edge fold and its backward, the aggregation
(Z = [x | mean | max | sum] and the saved argmax) and its backward (g_q, g_P_dst | g_P_src, g_x), on the BASELINE shapes,
a hub with thousands of in-edges, E = 0, isolated nodes and exact ties.  Every output starts as NaN and every element is
held to its bound; the argmax may pick any edge of a near-tied set.  Then the layer against the reference's own fp64
fixtures (tests/golden/pna/), a finite-difference check with dropout, a 2-layer stack against two oracle layers, a
captured step against eager execution, the graphgym-built layer, and no dense product leaving the TMA GEMM under
GPS_B200_STRICT=1."""
import ctypes as C
import glob as _glob
import os
import subprocess
import sys

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import GraphBatch, batch_from_lists, make_batch
from graphgps_b200.graph import graph_of
import pna_reference as R
from biased_util import compare_biased
from pna_oracle import pna_batch, pna_oracle_layer, seeded_state, tie_edge
from util import GOLDEN_DIR, golden_batch, pin_dropout_counter, rel_err, rel_l2, run_layer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = {"fp32": 1e-3, "bf16": 1e-2}
GRAD_L2 = {"fp32": 5e-3, "bf16": 1e-1}
DEG = [0, 3, 11, 9, 4, 1]
WORST = {}


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _elem_check(name, got, ref, bound):
    got, ref, bound = got.double().cpu(), ref.double().cpu(), bound.double().cpu()
    assert got.shape == ref.shape == bound.shape, (name, got.shape, ref.shape, bound.shape)
    assert not torch.isnan(got).any(), f"{name}: NaN left in the output"
    err = (got - ref).abs()
    frac = float((err / (bound + 1e-300)).max()) if got.numel() else 0.0
    WORST[name] = max(WORST.get(name, 0.0), frac)
    assert bool((err <= bound).all()), f"{name}: error {frac:.3g} x its bound"
    return frac


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
    _elem_check("Z", Z, Zr, B)
    assert R.argmax_ok(arg, m, ei, Zr[:, 2 * d:3 * d], bmax), "argmax outside the near-tied set"
    gqr, bq, gYr, bY, gxr, bx = R.backward(gZ.double(), arg, ei, N, d, add.double())
    if E:
        _elem_check("g_q", gq, gqr, bq)
    _elem_check("gY", gY, gYr, bY)
    _elem_check("g_x", gx, gxr, bx)
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
    _elem_check("F", F.cpu(), Fr, bF)
    _elem_check("c", c.cpu(), cr, bc)
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
    _elem_check("g_W_e", first[0][:, 2 * d:], gWeR, bWe)
    _elem_check("g_W_enc", first[2], gWencR, bWenc)
    _elem_check("g_b_enc", first[3], gbencR, bbenc)
    assert torch.equal(first[1], gc)
    assert bool((first[0][:, :2 * d] == 5.0).all())
    assert torch.equal(gW.cpu()[:, 2 * d:], 2 * first[0][:, 2 * d:])   # accumulate adds the same bits again
    assert torch.equal(gbe.cpu(), 2 * first[3])


# ------------------------------------------------------------------------------------------------- layer
def _pna_names():
    names = sorted(os.path.basename(p)[:-3] for p in _glob.glob(os.path.join(GOLDEN_DIR, "pna", "*.pt")))
    return [n for n in names if not n.startswith("reference_live")]


def _load(name):
    return torch.load(os.path.join(GOLDEN_DIR, "pna", name + ".pt"), weights_only=False)


def _state(fix, layer):
    return fix["state"] if "state" in fix else seeded_state(layer, fix["state_seed"])


def _layer(fix, precision):
    cfg = fix["config"]
    layer = graphgps_b200.GPSLayer(cfg["d"], "PNA", cfg["glob"], cfg["heads"], act=cfg["act"],
                                   pna_degrees=cfg["pna_degrees"], batch_norm=cfg["batch_norm"], precision=precision)
    layer.load_state_dict(_state(fix, layer), strict=True)
    return layer.to(DEV).train(cfg["training"])


def _bf16_l2_bounds(fix):
    """{result key: relative L2 bound} for the bf16 comparison of a training fixture: max(0.1, 4 x the relative L2 error
    that rounding the fixture's inputs and parameters to bf16 alone causes in the fp64 oracle)."""
    cfg = fix["config"]
    bf = lambda t: t.to(torch.bfloat16).double()
    o = pna_oracle_layer(cfg["d"], cfg["glob"], cfg["heads"], cfg["pna_degrees"], act=cfg["act"],
                         batch_norm=cfg["batch_norm"])
    o.load_state_dict({k: (bf(v) if v.is_floating_point() and "running" not in k else v)
                       for k, v in _state(fix, o).items()})
    o = o.double().train()
    b = golden_batch(fix, dtype=torch.float64)
    b.x, b.edge_attr = bf(b.x).requires_grad_(True), bf(b.edge_attr).requires_grad_(True)
    x, e = b.x, b.edge_attr
    if "attn_bias" in fix:
        b.attn_bias = fix["attn_bias"].double()
    (o(b).x * fix["ct_x"].double()).sum().backward()
    emu = {"grad_x": rel_l2(x.grad, fix["grad_x"]), "grad_e": rel_l2(e.grad, fix["grad_e"])}
    for n, q in o.named_parameters():
        if n in fix["grad_params"]:
            emu["grad:" + n] = rel_l2(q.grad, fix["grad_params"][n])
    return {k: max(GRAD_L2["bf16"], 4 * v) for k, v in emu.items()}


def _compare_per_key(res, fix, tol, l2, what):
    bad, worst = {}, 0.0
    e = rel_err(res["out_x"], fix["out_x"])
    worst = max(worst, e)
    if not e <= tol:
        bad["out_x"] = e
    for n, v in fix.get("state_after", {}).items():
        if v.is_floating_point() and not rel_err(res["state_after"][n], v) <= tol:
            bad["state:" + n] = rel_err(res["state_after"][n], v)
        if not v.is_floating_point() and not torch.equal(res["state_after"][n], v):
            bad["state:" + n] = "differs"
    pairs = [(k, res.get(k), fix[k]) for k in ("grad_x", "grad_e", "grad_attn_bias") if k in fix]
    pairs += [("grad:" + n, res["grad_params"].get(n), g) for n, g in fix.get("grad_params", {}).items()]
    for k, a, g in pairs:
        assert a is not None, f"{what}: {k} missing"
        e = rel_err(a, g)
        worst = max(worst, e)
        if e <= tol:
            continue
        if float(g.abs().max()) < 1e-9 and float(a.abs().max()) <= GRAD_L2["bf16"]:
            # zero in exact arithmetic (post's bias: its gradient is a column sum of what a training-mode BatchNorm
            # passes back, which sums to zero); the bf16 products leave an absolute residue, and no relative measure
            continue
        bound = l2.get(k, GRAD_L2["bf16"])
        if not rel_l2(a, g) <= bound:
            bad[k] = (e, rel_l2(a, g), bound)
    assert not bad, f"{what}: {bad}"
    return worst


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", _pna_names())
def test_layer_matches_pna_golden(name, precision):
    fix = _load(name)
    cfg = fix["config"]
    fb0 = _lib.load().gps_fallback_count()
    b = golden_batch(fix, DEV)
    layer = _layer(fix, precision)
    if "attn_bias" in fix:
        b.attn_bias = fix["attn_bias"].to(DEV).requires_grad_(cfg["training"])
    res = run_layer(layer, b, fix, backward=cfg["training"])
    if "attn_bias" in fix and cfg["training"]:
        res["grad_attn_bias"] = b.attn_bias.grad.detach().cpu()
    what = f"CUDA {precision} vs PNA golden {name}"
    if precision == "fp32":
        # an argmax that flips between two messages closer than fp32 noise moves a whole max gradient: relative L2
        errs = compare_biased(res, fix, TOL[precision], what, grad_l2_tol=GRAD_L2[precision])
        worst = max(v for k, v in errs.items() if not k.startswith("raw:"))
    else:
        worst = _compare_per_key(res, fix, TOL[precision], _bf16_l2_bounds(fix) if cfg["training"] else {}, what)
    if cfg["training"]:
        for n in ("local_model.edge_encoder.weight", "local_model.pre_nns.0.0.weight", "local_model.lin.weight"):
            assert n in res["grad_params"] and n in fix["grad_params"], n
        assert "grad_e" in res
    print(name, precision, "max err", worst)
    assert _lib.load().gps_fallback_count() == fb0


def test_edge_width_is_checked():
    layer = graphgps_b200.GPSLayer(160, "PNA", "None", 4, pna_degrees=DEG).to(DEV)
    b = pna_batch("zinc-gine", 1, 160, 2).to(DEV)
    b.edge_attr = torch.zeros(b.edge_attr.shape[0], 160, device=DEV)
    with pytest.raises(ValueError, match="min\\(128, dim_h\\) = 128"):
        layer(b)


def test_pna_dropout_forward_backward_consistent():
    """With the Philox offset pinned, the PNA+Transformer layer with dropout 0.2 is a deterministic function of x and
    edge_attr: its backward equals a central finite difference of its forward along a direction in each."""
    torch.manual_seed(5)
    d, H = 64, 4
    layer = graphgps_b200.GPSLayer(d, "PNA", "Transformer", H, act="gelu", dropout=0.2, pna_degrees=DEG).to(DEV).train()
    b = pna_batch("zinc-gine", 3, d, 8).to(DEV)
    g = torch.Generator().manual_seed(2)
    ct_x = torch.randn(b.x.shape, generator=g).to(DEV)
    vx = torch.randn(b.x.shape, generator=g).to(DEV)
    ve = torch.randn(b.edge_attr.shape, generator=g).to(DEV)

    def f(x, e):
        pin_dropout_counter(DEV, 7 * 4096)
        bb = GraphBatch(x=x, edge_index=b.edge_index, edge_attr=e, batch=b.batch, num_graphs=b.num_graphs)
        out = layer(bb)
        return (out.x * ct_x).sum(), out

    x0, e0 = b.x.clone().requires_grad_(True), b.edge_attr.clone().requires_grad_(True)
    loss, out0 = f(x0, e0)
    loss.backward()
    eps = 1e-2
    for which, analytic, dx, de in (("x", float((x0.grad * vx).sum()), eps * vx, 0.0),
                                    ("edge_attr", float((e0.grad * ve).sum()), 0.0, eps * ve)):
        with torch.no_grad():
            lp, _ = f(b.x + dx, b.edge_attr + de)
            lm, _ = f(b.x - dx, b.edge_attr - de)
        numeric = float((lp - lm) / (2 * eps))
        # an argmax switch or a GELU / BatchNorm curvature inside +-eps moves the central difference by O(eps)
        print("finite difference", which, numeric, analytic)
        assert abs(numeric - analytic) <= 1e-1 * max(1.0, abs(analytic)), (which, numeric, analytic)
    with torch.no_grad():
        _, again = f(b.x.clone(), b.edge_attr.clone())
    assert torch.equal(again.x, out0.x.detach())


def test_two_layer_stack_matches_two_oracle_layers_and_capture_matches_eager():
    torch.manual_seed(6)
    L, d, H = 2, 64, 4
    stack = graphgps_b200.GPSStack(L, d, "PNA", "Transformer", H, pna_degrees=DEG).to(DEV).train()
    oras = [pna_oracle_layer(d, "Transformer", H, DEG) for _ in range(L)]
    for o, l in zip(oras, stack.layers):
        o.load_state_dict({k: v.cpu() for k, v in l.state_dict().items()}, strict=True)
    b = pna_batch("zinc-gine", 7, d, 24)
    ct_x = torch.randn(b.x.shape, generator=torch.Generator().manual_seed(3))
    fb0 = _lib.load().gps_fallback_count()
    ob = b.clone()
    ob.x, ob.edge_attr = ob.x.double().requires_grad_(True), ob.edge_attr.double().requires_grad_(True)
    ox, oe = ob.x, ob.edge_attr
    for o in oras:
        ob = o.double().train()(ob)
    (ob.x * ct_x.double()).sum().backward()

    gb = b.clone().to(DEV)
    graph_of(gb)
    ct = ct_x.to(DEV)
    runs = []
    for _ in range(2):   # two eager steps from the same parameters and running statistics: identical bits
        state = {k: v.clone() for k, v in stack.state_dict().items()}
        eb = gb.clone()
        eb.__dict__["_gps_b200_graph"] = graph_of(gb)
        eb.x.requires_grad_(True)
        eb.edge_attr.requires_grad_(True)
        ex, ee = eb.x, eb.edge_attr
        out = stack(eb)
        out.x.backward(ct)
        runs.append((out.x.detach().clone(), ex.grad.clone(), ee.grad.clone(),
                     [p.grad.clone() for p in stack.parameters()]))
        for p in stack.parameters():
            p.grad = None
        stack.load_state_dict(state)
        del out, eb
    eager = runs[0]
    for a, c in zip(runs[0][:3], runs[1][:3]):
        assert torch.equal(a, c)
    for a, c in zip(runs[0][3], runs[1][3]):
        assert torch.equal(a, c)
    assert rel_err(eager[0].cpu(), ob.x.detach()) < 1e-3
    for a, r in ((eager[1], ox.grad), (eager[2], oe.grad)):
        assert rel_err(a.cpu(), r) < 1e-3 or rel_l2(a.cpu(), r) < 5e-3, (rel_err(a.cpu(), r), rel_l2(a.cpu(), r))
    step = stack.capture(gb, ct)
    step.replay()
    step.replay()
    torch.cuda.synchronize()
    assert torch.equal(step.x_out, eager[0]) and torch.equal(step.grad_x, eager[1])
    assert torch.equal(step.grad_e, eager[2])
    for (n, p), g in zip(stack.named_parameters(), eager[3]):
        assert torch.equal(p.grad, g), n
    assert _lib.load().gps_fallback_count() == fb0


def test_graphgym_built_pna_transformer_layer_runs(monkeypatch):
    import types
    from graphgps_b200 import graphgym
    registry = {}

    def register_layer(key, module=None):
        registry[key] = module
        return module

    ns = types.SimpleNamespace
    cfg = ns(gt=ns(layer_type="PNA+Transformer", n_heads=4, dropout=0.0, attn_dropout=0.0, layer_norm=False,
                   batch_norm=True, pna_degrees=DEG), gnn=ns(act="relu"))
    for name, attrs in (("torch_geometric", {}), ("torch_geometric.graphgym", {}),
                        ("torch_geometric.graphgym.register", {"register_layer": register_layer}),
                        ("torch_geometric.graphgym.config", {"cfg": cfg})):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        monkeypatch.setitem(sys.modules, name, m)
    cls = graphgym.register("gpslayer_b200_pna")
    layer = cls(ns(dim_out=64)).to(DEV)
    assert layer.local_gnn_type == "PNA" and layer.local_model.deg == DEG
    ora = pna_oracle_layer(64, "Transformer", 4, DEG)
    ora.load_state_dict({k: v.cpu() for k, v in layer.state_dict().items()}, strict=True)
    b = pna_batch("zinc-gine", 2, 64, 6)
    out = layer(b.clone().to(DEV)).x.detach().cpu()
    ref = ora.double()(GraphBatch(x=b.x.double(), edge_index=b.edge_index, edge_attr=b.edge_attr.double(),
                                  batch=b.batch, num_graphs=b.num_graphs)).x.detach()
    assert rel_err(out, ref) < 1e-3
    cfg.gt.pna_degrees = None
    with pytest.raises(NotImplementedError):
        cls(ns(dim_out=64))


_STRICT_SCRIPT = r"""
import sys, torch
sys.path[:0] = [{root!r}, {tests!r}]
import graphgps_b200
from graphgps_b200 import _lib
from pna_oracle import pna_batch
for d, shape, B in ((64, "zinc-gine", 24), (304, "pcqm4m-small", 64)):
    for norm in (True, False):
        layer = graphgps_b200.GPSLayer(d, "PNA", "Transformer", 4, batch_norm=norm, dropout=0.1,
                                       pna_degrees=[0, 3, 11, 9, 4, 1]).cuda().train()
        b = pna_batch(shape, 1, d, B).to("cuda")
        b.x.requires_grad_(True)
        b.edge_attr.requires_grad_(True)
        layer(b).x.sum().backward()
torch.cuda.synchronize()
print("fallbacks", _lib.load().gps_fallback_count())
"""


def test_no_gemm_fallback_under_strict_mode():
    """GPS_B200_STRICT=1 turns a dense product that would leave the TMA GEMM into an error; the PNA layer's products at
    d = 64 and 304 (edge products with K = de = 128 there; both normalisation modes, dropout on) all stay on it.  The
    switch is read once per process, so the layer runs in a child process."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = _STRICT_SCRIPT.format(root=root, tests=os.path.join(root, "tests"))
    env = dict(os.environ, GPS_B200_STRICT="1")
    r = subprocess.run([sys.executable, "-s", "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "fallbacks 0" in r.stdout, r.stdout
