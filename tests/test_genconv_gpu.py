"""GPU: the GENConv local model (PyG GENConv, gps_layer.py:60-61,183-189) stage by stage and in the layer.

Stages against the float64 restatement of tests/genconv_reference.py: the softmax aggregation (agg, the saved log-sum-exp
and u = agg + x) and its backward (grad_edge_attr and g_x), on the BASELINE shapes (zinc-gine, pcqm4m-small, code2), a
hub with thousands of in-edges, E = 0 and isolated nodes, with d in {4, 36, 64, 304, 2048}.  Every output starts as NaN.
Every element is held to a bound of the K n 2^-24 sum|terms| kind with the message errors carried through exp
(tests/genconv_reference.py::error_bounds); the worst error as a fraction of its bound is printed.  The layer against
the reference's own fp64 fixtures (tests/golden/genconv/), a finite-difference check with dropout, a 2-layer stack
against two oracle layers, a captured step against eager execution, the graphgym-built layer, and no dense product
leaving the TMA GEMM under GPS_B200_STRICT=1."""
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
import genconv_reference as R
from biased_util import compare_biased
from genconv_oracle import dead_node, genconv_batch, genconv_oracle_layer
from util import GOLDEN_DIR, golden_batch, pin_dropout_counter, rel_err, rel_l2, run_layer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = {"fp32": 1e-3, "bf16": 1e-2}
GRAD_L2 = {"fp32": 5e-3, "bf16": 1e-1}
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
    _elem_check("agg", r["agg"], agg.detach(), B["agg"])
    _elem_check("lse", r["lse"], lse.detach(), B["lse"])
    _elem_check("u", r["u"], u.detach(), B["u"])
    gx, ge = torch.autograd.grad((u * g_u).sum(), [x, e])
    _elem_check("g_e", r["g_e"], ge, B["g_e"])
    _elem_check("g_x", r["g_x"], gx + add, B["g_x"])
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
def _gen_names():
    names = sorted(os.path.basename(p)[:-3] for p in _glob.glob(os.path.join(GOLDEN_DIR, "genconv", "*.pt")))
    return [n for n in names if not n.startswith("reference_live")]


def _load(name):
    return torch.load(os.path.join(GOLDEN_DIR, "genconv", name + ".pt"), weights_only=False)


def _layer(fix, precision):
    cfg = fix["config"]
    layer = graphgps_b200.GPSLayer(cfg["d"], "GENConv", cfg["glob"], cfg["heads"], act=cfg["act"],
                                   batch_norm=cfg["batch_norm"], precision=precision)
    layer.load_state_dict(fix["state"], strict=True)
    return layer.to(DEV).train(cfg["training"])


def _bf16_l2_bounds(fix):
    """{result key: relative L2 bound} for the bf16 comparison of a training fixture: max(0.1, 4 x the relative L2 error
    that rounding the fixture's inputs and parameters to bf16 alone causes in the fp64 oracle)."""
    cfg = fix["config"]
    bf = lambda t: t.to(torch.bfloat16).double()
    o = genconv_oracle_layer(cfg["d"], cfg["glob"], cfg["heads"], act=cfg["act"], batch_norm=cfg["batch_norm"])
    o.load_state_dict({k: (bf(v) if v.is_floating_point() and "running" not in k else v)
                       for k, v in fix["state"].items()})
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
        bound = l2.get(k, GRAD_L2["bf16"])
        if not rel_l2(a, g) <= bound:
            bad[k] = (e, rel_l2(a, g), bound)
    assert not bad, f"{what}: {bad}"
    return worst


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", _gen_names())
def test_layer_matches_genconv_golden(name, precision):
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
    what = f"CUDA {precision} vs GENConv golden {name}"
    assert any("mlp.1.running_var" in k for k in fix["state_after"])
    if precision == "fp32":
        errs = compare_biased(res, fix, TOL[precision], what, grad_l2_tol=GRAD_L2[precision])
        worst = max(v for k, v in errs.items() if not k.startswith("raw:"))
    else:
        worst = _compare_per_key(res, fix, TOL[precision], _bf16_l2_bounds(fix) if cfg["training"] else {}, what)
    if cfg["training"]:
        got = res["grad_params"]
        for n in ("local_model.mlp.0.weight", "local_model.mlp.1.weight", "local_model.mlp.1.bias",
                  "local_model.mlp.4.weight"):
            assert n in got and n in fix["grad_params"], n
        assert "grad_e" in res
    print(name, precision, "max err", worst)
    assert _lib.load().gps_fallback_count() == fb0


def test_genconv_dropout_forward_backward_consistent():
    """With the Philox offset pinned, the GENConv+Transformer layer with dropout 0.2 is a deterministic function of x and
    edge_attr: its backward equals a central finite difference of its forward along a direction in each."""
    torch.manual_seed(5)
    d, H = 64, 4
    layer = graphgps_b200.GPSLayer(d, "GENConv", "Transformer", H, act="gelu", dropout=0.2).to(DEV).train()
    b = genconv_batch("zinc-gine", 3, d, 8).to(DEV)
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
        # every message or MLP ReLU whose pre-activation crosses 0 inside +-eps moves the central difference by O(eps)
        print("finite difference", which, numeric, analytic)
        assert abs(numeric - analytic) <= 1e-1 * max(1.0, abs(analytic)), (which, numeric, analytic)
    with torch.no_grad():
        _, again = f(b.x.clone(), b.edge_attr.clone())
    assert torch.equal(again.x, out0.x.detach())


def test_two_layer_stack_matches_two_oracle_layers_and_capture_matches_eager():
    torch.manual_seed(6)
    L, d, H = 2, 64, 4
    stack = graphgps_b200.GPSStack(L, d, "GENConv", "Transformer", H).to(DEV).train()
    oras = [genconv_oracle_layer(d, "Transformer", H) for _ in range(L)]
    for o, l in zip(oras, stack.layers):
        with torch.no_grad():
            bn = l.local_model.mlp[1]
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.uniform_(-0.3, 0.3)
        o.load_state_dict({k: v.cpu() for k, v in l.state_dict().items()}, strict=True)
    b = genconv_batch("zinc-gine", 7, d, 24)
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
                     [p.grad.clone() for p in stack.parameters()],
                     {k: v.clone() for k, v in stack.state_dict().items()}))
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


def test_graphgym_built_genconv_transformer_layer_runs(monkeypatch):
    import types
    from graphgps_b200 import graphgym
    registry = {}

    def register_layer(key, module=None):
        registry[key] = module
        return module

    ns = types.SimpleNamespace
    cfg = ns(gt=ns(layer_type="GENConv+Transformer", n_heads=4, dropout=0.0, attn_dropout=0.0, layer_norm=False,
                   batch_norm=True), gnn=ns(act="relu"))
    for name, attrs in (("torch_geometric", {}), ("torch_geometric.graphgym", {}),
                        ("torch_geometric.graphgym.register", {"register_layer": register_layer}),
                        ("torch_geometric.graphgym.config", {"cfg": cfg})):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        monkeypatch.setitem(sys.modules, name, m)
    cls = graphgym.register("gpslayer_b200_genconv")
    layer = cls(ns(dim_out=64)).to(DEV)
    assert layer.local_gnn_type == "GENConv"
    ora = genconv_oracle_layer(64, "Transformer", 4)
    ora.load_state_dict({k: v.cpu() for k, v in layer.state_dict().items()}, strict=True)
    b = genconv_batch("zinc-gine", 2, 64, 6)
    out = layer(b.clone().to(DEV)).x.detach().cpu()
    ref = ora.double()(GraphBatch(x=b.x.double(), edge_index=b.edge_index, edge_attr=b.edge_attr.double(),
                                  batch=b.batch, num_graphs=b.num_graphs)).x.detach()
    assert rel_err(out, ref) < 1e-3


_STRICT_SCRIPT = r"""
import sys, torch
sys.path[:0] = [{root!r}, {tests!r}]
import graphgps_b200
from graphgps_b200 import _lib
from genconv_oracle import genconv_batch
for d, shape, B in ((64, "zinc-gine", 24), (304, "pcqm4m-small", 64)):
    for norm in (True, False):
        layer = graphgps_b200.GPSLayer(d, "GENConv", "Transformer", 4, batch_norm=norm, dropout=0.1).cuda().train()
        b = genconv_batch(shape, 1, d, B).to("cuda")
        b.x.requires_grad_(True)
        b.edge_attr.requires_grad_(True)
        layer(b).x.sum().backward()
torch.cuda.synchronize()
print("fallbacks", _lib.load().gps_fallback_count())
"""


def test_no_gemm_fallback_under_strict_mode():
    """GPS_B200_STRICT=1 turns a dense product that would leave the TMA GEMM into an error; the GENConv layer's products
    at d = 64 and 304 (both normalisation modes, dropout on) all stay on it.  The switch is read once per process, so the
    layer runs in a child process."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = _STRICT_SCRIPT.format(root=root, tests=os.path.join(root, "tests"))
    env = dict(os.environ, GPS_B200_STRICT="1")
    r = subprocess.run([sys.executable, "-s", "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "fallbacks 0" in r.stdout, r.stdout
