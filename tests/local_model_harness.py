"""The GPSLayer local models GAT, GENConv and PNA (gps_layer.py:60-90,183-189), one spec each, and the pieces of their
tests that do not depend on the model: the layer checks each model's GPU test file runs (fixtures in fp32 and bf16,
dropout, stack and capture, graphgym, strict mode) and the C ABI builders of the CPU tests."""
import ctypes as C
import os
import subprocess
import sys
import types

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import GraphBatch
from graphgps_b200.graph import graph_of
from gat_oracle import gat_batch, gat_oracle_layer
from genconv_oracle import genconv_batch, genconv_oracle_layer
from pna_oracle import pna_batch, pna_oracle_layer, seeded_state
from util import DEV, GOLDEN_DIR, compare, golden_batch, pin_dropout_counter, rel_err, rel_l2, run_layer

TOL = {"fp32": 1e-3, "bf16": 1e-2}
GRAD_L2 = {"fp32": 5e-3, "bf16": 1e-1}
DEG = [0, 3, 11, 9, 4, 1]   # the PNA in-degree histogram of the tests that build their own layer

# GAT's score-path gradients are sums that cancel (sum_e alpha (g_alpha - Delta) = 0 per node and head), so bf16 rounding
# anywhere upstream moves them by far more than 2^-9: at H = 1 (one head of 64 channels, scores of ~10 units) att_*,
# lin_src, lin_edge and grad_e reach a relative L2 error of ~0.7, and they alone get 0.75 there.
SCORE_PATH = ("grad_e", "grad:local_model.att_src", "grad:local_model.att_dst", "grad:local_model.att_edge",
              "grad:local_model.lin_src.weight", "grad:local_model.lin_edge.weight")


def _gat_score_path(bounds, cfg):
    if cfg["heads"] == 1:
        for k in SCORE_PATH:
            bounds[k] = max(bounds[k], 0.75)


def _pna_zero(key, expected):
    # zero in exact arithmetic (post's bias: its gradient is a column sum of what a training-mode BatchNorm passes back,
    # which sums to zero); the bf16 products leave an absolute residue, and no relative measure bounds it
    return float(expected.abs().max()) < 1e-9


def _perturb_gat(layer):
    with torch.no_grad():
        for p in (layer.local_model.att_src, layer.local_model.att_dst, layer.local_model.att_edge):
            p.mul_(3.0)


def _perturb_genconv(layer):
    with torch.no_grad():
        bn = layer.local_model.mlp[1]
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.3, 0.3)


# name: the GPSLayer local_gnn_type.  extra(cfg): the GPSLayer / oracle keyword arguments a config adds.  oracle: the
# fp64 oracle layer's builder.  state(fix, module): the fixture's state dict (PNA's large fixtures store a seed).
# grads: parameters whose gradients a training fixture must hold and the layer must produce; state_keys: entries every
# fixture's state_after must hold.  bf16_widen(bounds, cfg) and bf16_zero(key, expected): the model's own bf16 rules.
# perturb(layer): moves the stack test's layers off their initial values where those hide a term.  graphgym_gt: the
# cfg.gt options the GraphGym-built layer needs.
SPECS = {
    "GAT": types.SimpleNamespace(
        name="GAT", batch=gat_batch, extra=lambda cfg: {}, oracle=gat_oracle_layer,
        state=lambda fix, module: fix["state"],
        grads=("local_model.att_edge", "local_model.lin_src.weight"), state_keys=(),
        bf16_widen=_gat_score_path, bf16_zero=None, perturb=_perturb_gat, graphgym_gt={}),
    "GENConv": types.SimpleNamespace(
        name="GENConv", batch=genconv_batch, extra=lambda cfg: {}, oracle=genconv_oracle_layer,
        state=lambda fix, module: fix["state"],
        grads=("local_model.mlp.0.weight", "local_model.mlp.1.weight", "local_model.mlp.1.bias",
               "local_model.mlp.4.weight"), state_keys=("local_model.mlp.1.running_var",),
        bf16_widen=None, bf16_zero=None, perturb=_perturb_genconv, graphgym_gt={}),
    "PNA": types.SimpleNamespace(
        name="PNA", batch=pna_batch, extra=lambda cfg: {"pna_degrees": cfg["pna_degrees"]},
        oracle=lambda d, glob, heads, pna_degrees, **kw: pna_oracle_layer(d, glob, heads, pna_degrees, **kw),
        state=lambda fix, module: fix["state"] if "state" in fix else seeded_state(module, fix["state_seed"]),
        grads=("local_model.edge_encoder.weight", "local_model.pre_nns.0.0.weight", "local_model.lin.weight"),
        state_keys=(), bf16_widen=None, bf16_zero=_pna_zero, perturb=None, graphgym_gt={"pna_degrees": DEG}),
}


def default_cfg(**kw):
    """The configuration of the tests that build their own layer."""
    return dict(dict(d=64, glob="Transformer", heads=4, act="relu", batch_norm=True, pna_degrees=DEG), **kw)


def golden_dir(spec):
    return os.path.join(GOLDEN_DIR, spec.name.lower())


def golden_names(spec):
    names = sorted(p[:-3] for p in os.listdir(golden_dir(spec)) if p.endswith(".pt"))
    return [n for n in names if not n.startswith("reference_live")]


def load(spec, name):
    return torch.load(os.path.join(golden_dir(spec), name + ".pt"), weights_only=False)


def gps_layer(spec, cfg, **kw):
    return graphgps_b200.GPSLayer(cfg["d"], spec.name, cfg["glob"], cfg["heads"], act=cfg["act"],
                                  batch_norm=cfg["batch_norm"], **spec.extra(cfg), **kw)


def oracle_layer(spec, cfg):
    return spec.oracle(cfg["d"], cfg["glob"], cfg["heads"], act=cfg["act"], batch_norm=cfg["batch_norm"],
                       **spec.extra(cfg))


def _bf16_l2_bounds(spec, fix):
    """{result key: relative L2 bound} for the bf16 comparison of a training fixture: max(0.1, 4 x the relative L2 error
    that rounding the fixture's inputs and parameters to bf16 alone causes in the fp64 oracle), then the model's own
    rule."""
    cfg = fix["config"]
    bf = lambda t: t.to(torch.bfloat16).double()
    o = oracle_layer(spec, cfg)
    o.load_state_dict({k: (bf(v) if v.is_floating_point() and "running" not in k else v)
                       for k, v in spec.state(fix, o).items()})
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
    bounds = {k: max(GRAD_L2["bf16"], 4 * v) for k, v in emu.items()}
    if spec.bf16_widen is not None:
        spec.bf16_widen(bounds, cfg)
    return bounds


# ------------------------------------------------------------------------------------------------- layer checks (GPU)
def check_golden(spec, name, precision):
    """The layer against one of the reference's own fp64 fixtures (tests/golden/<model>/)."""
    fix = load(spec, name)
    cfg = fix["config"]
    fb0 = _lib.load().gps_fallback_count()
    b = golden_batch(fix, DEV)
    layer = gps_layer(spec, cfg, precision=precision)
    layer.load_state_dict(spec.state(fix, layer), strict=True)
    layer = layer.to(DEV).train(cfg["training"])
    if "attn_bias" in fix:
        b.attn_bias = fix["attn_bias"].to(DEV).requires_grad_(cfg["training"])
    res = run_layer(layer, b, fix, backward=cfg["training"])
    if "attn_bias" in fix and cfg["training"]:
        res["grad_attn_bias"] = b.attn_bias.grad.detach().cpu()
    what = f"CUDA {precision} vs {spec.name} golden {name}"
    for k in spec.state_keys:
        assert k in fix["state_after"], k
    if precision == "fp32":
        # relative L2 as well: a ReLU or LeakyReLU kink, or a PNA argmax between two messages closer than fp32 noise,
        # moves single gradient entries by O(|g|)
        errs = compare(res, fix, TOL[precision], what, grad_l2_tol=GRAD_L2[precision])
    else:
        bounds = dict(_bf16_l2_bounds(spec, fix) if cfg["training"] else {}, default=GRAD_L2["bf16"])
        errs = compare(res, fix, TOL[precision], what, grad_l2_tol=bounds, zero=spec.bf16_zero,
                       zero_tol=GRAD_L2["bf16"])
    if cfg["training"]:
        for n in spec.grads:
            assert n in res["grad_params"] and n in fix["grad_params"], n
        assert "grad_e" in res
    print(name, precision, "max err", max(v for k, v in errs.items() if not k.startswith("raw:")))
    assert _lib.load().gps_fallback_count() == fb0


def check_dropout_forward_backward_consistent(spec):
    """With the Philox offset pinned, the <model>+Transformer layer with dropout 0.2 is a deterministic function of x and
    edge_attr: its backward equals a central finite difference of its forward along a direction in each."""
    torch.manual_seed(5)
    layer = gps_layer(spec, default_cfg(act="gelu"), dropout=0.2).to(DEV).train()
    b = spec.batch("zinc-gine", 3, 64, 8).to(DEV)
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
        # every kink crossed inside +-eps moves the central difference by O(eps): a GAT score at LeakyReLU's kink, a
        # GENConv message or MLP ReLU pre-activation at 0, a PNA argmax switch; and GELU / BatchNorm curvature
        print("finite difference", which, numeric, analytic)
        assert abs(numeric - analytic) <= 1e-1 * max(1.0, abs(analytic)), (which, numeric, analytic)
    with torch.no_grad():
        _, again = f(b.x.clone(), b.edge_attr.clone())
    assert torch.equal(again.x, out0.x.detach())


def check_two_layer_stack_and_capture(spec):
    """A 2-layer stack against two oracle layers, two eager steps against each other, and a captured step against
    eager execution."""
    torch.manual_seed(6)
    L, d, H = 2, 64, 4
    cfg = default_cfg()
    stack = graphgps_b200.GPSStack(L, d, spec.name, "Transformer", H, **spec.extra(cfg)).to(DEV).train()
    oras = [oracle_layer(spec, cfg) for _ in range(L)]
    for o, l in zip(oras, stack.layers):
        if spec.perturb is not None:
            spec.perturb(l)
        o.load_state_dict({k: v.cpu() for k, v in l.state_dict().items()}, strict=True)
    b = spec.batch("zinc-gine", 7, d, 24)
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


def check_graphgym_built_layer(spec, monkeypatch):
    """The <model>+Transformer layer GraphGym builds runs and matches the oracle."""
    from graphgps_b200 import graphgym
    registry = {}

    def register_layer(key, module=None):
        registry[key] = module
        return module

    ns = types.SimpleNamespace
    cfg = ns(gt=ns(layer_type=f"{spec.name}+Transformer", n_heads=4, dropout=0.0, attn_dropout=0.0, layer_norm=False,
                   batch_norm=True, **spec.graphgym_gt), gnn=ns(act="relu"))
    for name, attrs in (("torch_geometric", {}), ("torch_geometric.graphgym", {}),
                        ("torch_geometric.graphgym.register", {"register_layer": register_layer}),
                        ("torch_geometric.graphgym.config", {"cfg": cfg})):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        monkeypatch.setitem(sys.modules, name, m)
    cls = graphgym.register(f"gpslayer_b200_{spec.name.lower()}")
    layer = cls(ns(dim_out=64)).to(DEV)
    assert layer.local_gnn_type == spec.name
    if spec.name == "PNA":
        assert layer.local_model.deg == spec.graphgym_gt["pna_degrees"]
    ora = oracle_layer(spec, default_cfg())
    ora.load_state_dict({k: v.cpu() for k, v in layer.state_dict().items()}, strict=True)
    b = spec.batch("zinc-gine", 2, 64, 6)
    out = layer(b.clone().to(DEV)).x.detach().cpu()
    ref = ora.double()(GraphBatch(x=b.x.double(), edge_index=b.edge_index, edge_attr=b.edge_attr.double(),
                                  batch=b.batch, num_graphs=b.num_graphs)).x.detach()
    assert rel_err(out, ref) < 1e-3
    for k in spec.graphgym_gt:   # an option the model needs, left unset, is refused
        setattr(cfg.gt, k, None)
        with pytest.raises(NotImplementedError):
            cls(ns(dim_out=64))


_STRICT_SCRIPT = r"""
import sys, torch
sys.path[:0] = [{root!r}, {tests!r}]
import graphgps_b200
from graphgps_b200 import _lib
from local_model_harness import SPECS, default_cfg
spec = SPECS[{model!r}]
for d, shape, B in ((64, "zinc-gine", 24), (304, "pcqm4m-small", 64)):
    for norm in (True, False):
        layer = graphgps_b200.GPSLayer(d, spec.name, "Transformer", 4, batch_norm=norm, dropout=0.1,
                                       **spec.extra(default_cfg())).cuda().train()
        b = spec.batch(shape, 1, d, B).to("cuda")
        b.x.requires_grad_(True)
        b.edge_attr.requires_grad_(True)
        layer(b).x.sum().backward()
torch.cuda.synchronize()
print("fallbacks", _lib.load().gps_fallback_count())
"""


def check_no_gemm_fallback_under_strict_mode(spec):
    """GPS_B200_STRICT=1 turns a dense product that would leave the TMA GEMM into an error; the layer's products at d =
    64 and 304 (both normalisation modes, dropout on; PNA's edge products with K = de = 128 at 304) all stay on it.
    The switch is read once per process, so the layer runs in a child process."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = _STRICT_SCRIPT.format(root=root, tests=os.path.join(root, "tests"), model=spec.name)
    env = dict(os.environ, GPS_B200_STRICT="1")
    r = subprocess.run([sys.executable, "-s", "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "fallbacks 0" in r.stdout, r.stdout


# ------------------------------------------------------------------------------------------------- C ABI (CPU tests)
def _args(local, N=10, E=20, d=64, H=4, glob="Transformer", norm="batch"):
    a = _lib.GpsLayerArgs()
    a.d, a.heads = d, H
    a.local_type = _lib.LOCAL[local]
    a.global_type = _lib.GLOBAL[glob]
    a.norm_type = _lib.NORM[norm]
    a.graph.N, a.graph.E, a.graph.B = N, E, 2
    return a


def _plan(a):
    p = _lib.GpsLayerPlan()
    rc = _lib.load().gps_layer_plan(C.byref(a), C.byref(p))
    return rc, p


def _r(n):
    return (n + 255) // 256 * 256


def _planes(rows, cols, lo=True):
    """bytes of one bf16 hi (+ lo) plane pair as the library allocates it"""
    one = _r(2 * (rows * ((cols + 7) // 8 * 8) + 8))
    return one * (2 if lo else 1)
