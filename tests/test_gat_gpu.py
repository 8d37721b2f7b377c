"""GPU: the GAT local model (PyG GATConv, gps_layer.py:70-74,183-189) stage by stage and in the layer.

Stages against the float64 restatement of tests/gat_reference.py: the fold, the forward (the saved scores and
log-sum-exp included) and the backward (gY, grad_edge_attr, g_v, g_att_src, g_att_dst, g_bias), on the BASELINE shapes,
MalNet-like hubs, degenerate graphs and an in-degree sweep, with C = d / H in {1, 9, 16, 24, 64, 76}.  Every output
starts as NaN.  Every element is held to a bound of the gamma_n kind: K n 2^-24 sum|terms| with n the length of the sums
that produce it (a head's C channels, an edge's d, a node's in- or out-degree + 1, a column sum's chunk), with the
score errors carried through exp into the attention weights (tests/gat_reference.py::error_bounds); the worst error as
a fraction of its bound is printed.  Structural cases are exact.  The layer
against the reference's own fp64 fixtures (tests/golden/gat/), a finite-difference check with dropout, a 2-layer stack
against two oracle layers, a captured step against eager execution, and the graphgym-built layer."""
import ctypes as C
import math

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import GraphBatch, batch_from_lists, make_batch
from graphgps_b200.graph import graph_of
import gat_reference as R
from biased_util import compare_biased
from gat_oracle import gat_batch, gat_oracle_layer
from util import GOLDEN_DIR, golden_batch, pin_dropout_counter, rel_err, rel_l2, run_layer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = {"fp32": 1e-3, "bf16": 1e-2}
GRAD_L2 = {"fp32": 5e-3, "bf16": 1e-1}
# bf16 gradient bounds are derived per fixture and per gradient: max(0.1, 4 x the relative L2 error that rounding the
# fixture's inputs and parameters to bf16 alone causes in the fp64 oracle).  GAT's score-path gradients are sums that
# cancel (sum_e alpha (g_alpha - Delta) = 0 per node and head), so bf16 rounding anywhere upstream moves them by far more
# than 2^-9: at H = 1 (one head of 64 channels, scores of ~10 units) att_*, lin_src, lin_edge and grad_e reach a
# relative L2 error of ~0.7, and they alone get 0.75 there.
SCORE_PATH = ("grad_e", "grad:local_model.att_src", "grad:local_model.att_dst", "grad:local_model.att_edge",
              "grad:local_model.lin_src.weight", "grad:local_model.lin_edge.weight")


def _bf16_l2_bounds(fix):
    """{result key: relative L2 bound} for the bf16 comparison of a training fixture."""
    cfg = fix["config"]
    bf = lambda t: t.to(torch.bfloat16).double()
    o = gat_oracle_layer(cfg["d"], cfg["glob"], cfg["heads"], act=cfg["act"], batch_norm=cfg["batch_norm"])
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
    out = {k: max(GRAD_L2["bf16"], 4 * v) for k, v in emu.items()}
    if cfg["heads"] == 1:
        for k in SCORE_PATH:
            out[k] = max(out[k], 0.75)
    return out


def _compare_per_key(res, fix, tol, l2, what):
    """util.compare with a relative-L2 bound per gradient (l2[key]) instead of one for all."""
    bad, worst = {}, 0.0
    for k in ("out_x",):
        e = rel_err(res[k], fix[k])
        worst = max(worst, e)
        if not e <= tol:
            bad[k] = e
    for n, v in fix.get("state_after", {}).items():
        if v.is_floating_point() and not rel_err(res["state_after"][n], v) <= tol:
            bad["state:" + n] = rel_err(res["state_after"][n], v)
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


U = 2.0 ** -24
WORST = {}


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _bound_check(name, got, ref, absref, n, K=4.0):
    """|got - ref| <= K n u absref + tiny, elementwise; absref = the same computation on absolute values."""
    got, ref, absref = got.double().cpu(), ref.double().cpu(), absref.double().cpu()
    assert not torch.isnan(got).any(), f"{name}: NaN left in the output"
    bound = K * max(n, 1) * U * absref + 1e-30
    frac = float(((got - ref).abs() / bound).max()) if got.numel() else 0.0
    WORST[name] = max(WORST.get(name, 0.0), frac)
    assert frac <= 1.0, f"{name}: error {frac:.3g} x its bound"
    return frac


def _elem_check(name, got, ref, bound):
    """|got - ref| <= bound elementwise (bounds from gat_reference.error_bounds: actual reduction lengths, per element)."""
    got, ref, bound = got.double().cpu(), ref.double().cpu(), bound.double().cpu()
    assert got.shape == ref.shape == bound.shape, (name, got.shape, ref.shape, bound.shape)
    assert not torch.isnan(got).any(), f"{name}: NaN left in the output"
    err = (got - ref).abs()
    frac = float((err / (bound + 1e-300)).max()) if got.numel() else 0.0
    WORST[name] = max(WORST.get(name, 0.0), frac)
    assert bool((err <= bound).all()), f"{name}: error {frac:.3g} x its bound"
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
    _elem_check("a_self", sc[2 * NH:3 * NH].view(N, H), s["a_self"].detach(), B["a_self"])
    _elem_check("lse", sc[3 * NH:4 * NH].view(N, H), s["lse"].detach(), B["lse"])
    _elem_check("xloc", r["xloc"], r["x"].double() + out.detach(), B["xloc"])
    # backward
    grads = torch.autograd.grad((out * g_h).sum(), [Y, ea, vleaf, a_s, a_d, bias])
    gres = r["bwd"]
    for name, got, ref in (("gY", gres["gY"], grads[0]), ("grad_edge_attr", gres["gea"][:E], grads[1]),
                           ("g_v", gres["gv"], grads[2]), ("g_att_src", gres["gas"], grads[3]),
                           ("g_att_dst", gres["gad"], grads[4]), ("g_bias", gres["gb"], grads[5])):
        _elem_check(name, got, ref.reshape(got.shape), B[name])
    # fold backward from the library's g_v: g_W_edge[hC+c, :] = att_edge[hC+c] g_v[h], g_att_edge = W_edge . g_v
    gv = gres["gv"].double()
    ae64 = a_e.detach()
    gv_rows = gv.repeat_interleave(C_, 0)                                   # [d, d]: row hC+c holds g_v[h]
    _elem_check("g_W_edge", gres["gW"], ae64[:, None] * gv_rows, 2 * U * (ae64[:, None] * gv_rows).abs())
    _elem_check("g_att_edge", gres["gae"], (W.detach() * gv_rows).sum(1),
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
def _gat_names():
    import glob
    import os
    names = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(GOLDEN_DIR, "gat", "*.pt")))
    return [n for n in names if not n.startswith("reference_live")]


def _load(name):
    import os
    return torch.load(os.path.join(GOLDEN_DIR, "gat", name + ".pt"), weights_only=False)


def _layer(fix, precision):
    cfg = fix["config"]
    layer = graphgps_b200.GPSLayer(cfg["d"], "GAT", cfg["glob"], cfg["heads"], act=cfg["act"],
                                   batch_norm=cfg["batch_norm"], precision=precision)
    layer.load_state_dict(fix["state"], strict=True)
    return layer.to(DEV).train(cfg["training"])


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", _gat_names())
def test_layer_matches_gat_golden(name, precision):
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
    what = f"CUDA {precision} vs GAT golden {name}"
    if precision == "fp32":
        errs = compare_biased(res, fix, TOL[precision], what, grad_l2_tol=GRAD_L2[precision])
        worst = max(v for k, v in errs.items() if not k.startswith("raw:"))
    else:
        worst = _compare_per_key(res, fix, TOL[precision], _bf16_l2_bounds(fix) if cfg["training"] else {}, what)
        errs = {"grad:" + n: 0 for n in res.get("grad_params", {})}
    if cfg["training"]:
        assert "grad_e" in res and "grad:local_model.att_edge" in errs and "grad:local_model.lin_src.weight" in errs
    print(name, precision, "max err", worst)
    assert _lib.load().gps_fallback_count() == fb0


def test_gat_dropout_forward_backward_consistent():
    """With the Philox offset pinned, the GAT+Transformer layer with dropout 0.2 is a deterministic function of x and
    edge_attr: its backward equals a central finite difference of its forward along a direction in each."""
    torch.manual_seed(5)
    d, H = 64, 4
    layer = graphgps_b200.GPSLayer(d, "GAT", "Transformer", H, act="gelu", dropout=0.2).to(DEV).train()
    b = gat_batch("zinc-gine", 3, d, 8).to(DEV)
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
        # every edge whose score crosses LeakyReLU's kink inside +-eps moves the central difference by O(eps)
        print("finite difference", which, numeric, analytic)
        assert abs(numeric - analytic) <= 1e-1 * max(1.0, abs(analytic)), (which, numeric, analytic)
    with torch.no_grad():
        _, again = f(b.x.clone(), b.edge_attr.clone())
    assert torch.equal(again.x, out0.x.detach())


def test_two_layer_stack_matches_two_oracle_layers_and_capture_matches_eager():
    torch.manual_seed(6)
    L, d, H = 2, 64, 4
    stack = graphgps_b200.GPSStack(L, d, "GAT", "Transformer", H).to(DEV).train()
    oras = [gat_oracle_layer(d, "Transformer", H) for _ in range(L)]
    for o, l in zip(oras, stack.layers):
        with torch.no_grad():
            for p in (l.local_model.att_src, l.local_model.att_dst, l.local_model.att_edge):
                p.mul_(3.0)
        o.load_state_dict({k: v.cpu() for k, v in l.state_dict().items()}, strict=True)
    b = gat_batch("zinc-gine", 7, d, 24)
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
    eb = gb.clone()
    eb.__dict__["_gps_b200_graph"] = graph_of(gb)
    eb.x.requires_grad_(True)
    eb.edge_attr.requires_grad_(True)
    ex, ee = eb.x, eb.edge_attr
    out = stack(eb)
    out.x.backward(ct)
    eager = (out.x.detach().clone(), ex.grad.clone(), ee.grad.clone(), [p.grad.clone() for p in stack.parameters()])
    del out, eb
    assert rel_err(eager[0].cpu(), ob.x.detach()) < 1e-3
    for a, r in ((eager[1], ox.grad), (eager[2], oe.grad)):
        assert rel_err(a.cpu(), r) < 1e-3 or rel_l2(a.cpu(), r) < 5e-3, (rel_err(a.cpu(), r), rel_l2(a.cpu(), r))
    for p in stack.parameters():
        p.grad = None
    step = stack.capture(gb, ct)
    step.replay()
    step.replay()
    torch.cuda.synchronize()
    assert torch.equal(step.x_out, eager[0]) and torch.equal(step.grad_x, eager[1])
    assert torch.equal(step.grad_e, eager[2])
    for (n, p), g in zip(stack.named_parameters(), eager[3]):
        assert torch.equal(p.grad, g), n
    assert _lib.load().gps_fallback_count() == fb0


def test_graphgym_built_gat_transformer_layer_runs(monkeypatch):
    import sys
    import types
    from graphgps_b200 import graphgym
    registry = {}

    def register_layer(key, module=None):
        registry[key] = module
        return module

    ns = types.SimpleNamespace
    cfg = ns(gt=ns(layer_type="GAT+Transformer", n_heads=4, dropout=0.0, attn_dropout=0.0, layer_norm=False,
                   batch_norm=True), gnn=ns(act="relu"))
    for name, attrs in (("torch_geometric", {}), ("torch_geometric.graphgym", {}),
                        ("torch_geometric.graphgym.register", {"register_layer": register_layer}),
                        ("torch_geometric.graphgym.config", {"cfg": cfg})):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        monkeypatch.setitem(sys.modules, name, m)
    cls = graphgym.register("gpslayer_b200_gat")
    layer = cls(ns(dim_out=64)).to(DEV)
    ora = gat_oracle_layer(64, "Transformer", 4)
    ora.load_state_dict({k: v.cpu() for k, v in layer.state_dict().items()}, strict=True)
    b = gat_batch("zinc-gine", 2, 64, 6)
    out = layer(b.clone().to(DEV)).x.detach().cpu()
    ref = ora.double()(GraphBatch(x=b.x.double(), edge_index=b.edge_index, edge_attr=b.edge_attr.double(),
                                  batch=b.batch, num_graphs=b.num_graphs)).x.detach()
    assert rel_err(out, ref) < 1e-3


def test_gat_layer_validation():
    layer = graphgps_b200.GPSLayer(32, "GAT", "Transformer", 4).to(DEV)
    b = make_batch("zinc-gine", seed=1, dim=32, num_graphs=3).to(DEV)
    b.edge_attr = b.edge_attr[:, :16].contiguous()
    with pytest.raises(ValueError):
        layer(b)
