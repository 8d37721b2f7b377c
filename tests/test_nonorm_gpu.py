"""GPU: GPSLayer(..., batch_norm=False) on the H100 against the reference-verbatim fixtures (tests/golden/nonorm/) and the
fp64 oracle at full size on single-graph node-level batches (the shapes of the six GCN+Transformer configs), dropout
consistency, eval mode, a 2-layer stack with CUDA-graph capture, the graphgym-built layer and the launch count.
Tolerances as in test_layer_gpu.py."""
import copy
import types

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.graph import graph_of
from oracle.gps_oracle import OracleGPSLayer
from nonorm_util import NODE_SHAPES, load_nonorm, node_graph, node_shape_batch, nonorm_names, with_edge_cases
from util import compare, golden_batch, pin_dropout_counter, rel_err, rel_l2, run_layer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = {"fp32": 1e-3, "bf16": 1e-2}
GRAD_L2 = {"fp32": 5e-3, "bf16": 1e-1}
STRICT_GRAD = {"fp32": 1e-3, "bf16": 3e-2}   # GELU: no kink flips, no L2 fallback (test_layer_gelu_strict_gradients_full_size)


def _pair(d, local="GCN", glob="Transformer", heads=4, act="gelu", precision="fp32", seed=0, **kw):
    """fp32 oracle and CUDA layer with the same weights (GCN bias drawn non-zero: PyG initialises it to zero)."""
    torch.manual_seed(seed)
    ora = OracleGPSLayer(d, local, glob, heads, act=act, batch_norm=False, **kw)
    if local == "GCN":
        with torch.no_grad():
            ora.local_model.bias.uniform_(-0.3, 0.3)
    ours = graphgps_b200.GPSLayer(d, local, glob, heads, act=act, precision=precision, batch_norm=False, **kw)
    ours.load_state_dict(ora.state_dict(), strict=True)
    return ora, ours.to(DEV)


def _cts(b, local="GCN", seed=9):
    g = torch.Generator().manual_seed(seed)
    fix = {"config": dict(local=local), "ct_x": torch.randn(b.x.shape, generator=g)}
    if local == "CustomGatedGCN":
        fix["ct_e"] = torch.randn(b.edge_attr.shape, generator=g)
    return fix


def _to64(b, dev="cpu"):
    b = b.clone()
    b.x, b.edge_attr = b.x.to(dev, torch.float64), b.edge_attr.to(dev, torch.float64)
    for k in ("edge_index", "batch"):
        setattr(b, k, getattr(b, k).to(dev))
    return b


def _oracle64(ora, b, fix, dev=DEV):
    """The fp64 oracle, on the GPU (factory calls inside it default to that device): [4, 7600, 7600] fp64 is 1.85 GB."""
    with torch.device(dev):
        res = run_layer(copy.deepcopy(ora).to(dev).double(), _to64(b, dev), fix)
    torch.cuda.empty_cache()
    return res


def _target(ref):
    t = {k: ref[k] for k in ("out_x", "out_e", "grad_x", "grad_e") if k in ref}
    t["grad_params"], t["state_after"] = ref["grad_params"], ref["state_after"]
    return t


# ------------------------------------------------------------------------------------------ fixtures
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", nonorm_names())
def test_layer_matches_nonorm_golden(name, precision):
    fix = load_nonorm(name)
    cfg = fix["config"]
    layer = graphgps_b200.GPSLayer(cfg["d"], cfg["local"], cfg["glob"], cfg["heads"], act=cfg["act"],
                                   precision=precision, batch_norm=False)
    layer.load_state_dict(fix["state"], strict=True)
    layer = layer.to(DEV).train(cfg["training"])
    res = run_layer(layer, golden_batch(fix, DEV), fix, backward=cfg["training"])
    errs = compare(res, fix, TOL[precision], f"CUDA {precision} vs nonorm golden {name}", grad_l2_tol=GRAD_L2[precision])
    print(name, precision, "max err", max(v for k, v in errs.items() if not k.startswith("raw:")))


# ------------------------------------------------------------------------------------------ full size, one graph
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("shape", sorted(NODE_SHAPES))
def test_node_level_full_size_matches_oracle_fp64(shape, precision):
    """GCN+Transformer, GELU, one whole graph per batch (WebKB 183, chameleon 2277 at d = 96 / head dim 24, squirrel
    5201 with in-degrees in the thousands, actor 7600 nodes): outputs and EVERY gradient at the strict max-abs bound."""
    s = NODE_SHAPES[shape]
    b = node_shape_batch(shape, seed=3)
    ora, ours = _pair(s.d, heads=s.heads, precision=precision)
    fix = _cts(b)
    ref = _oracle64(ora, b, fix)
    res = run_layer(ours, b.clone().to(DEV), fix)
    for k in ("out_x",):
        assert rel_err(res[k], ref[k]) < TOL[precision], (k, rel_err(res[k], ref[k]))
    t = _target(ref)
    t.pop("out_x")
    errs = compare(res, t, STRICT_GRAD[precision], f"CUDA {precision} vs oracle fp64 @ {shape}")
    indeg = int(torch.bincount(b.edge_index[1], minlength=s.N).max())
    print(shape, precision, f"N={s.N} E={s.E} d={s.d} max in-degree {indeg}", f"out_x {rel_err(res['out_x'], ref['out_x']):.2e}",
          f"worst grad {max(v for k, v in errs.items() if not k.startswith('raw:')):.2e}")


# ------------------------------------------------------------------------------------------ dropout
@pytest.mark.parametrize("local,glob", [("GCN", "Transformer"), ("GCN", "None"), ("GINE", "Transformer"),
                                        ("CustomGatedGCN", "Performer")])
def test_dropout_forward_backward_consistent(local, glob):
    """Dropout 0.2 on every node-side site and attention dropout 0.5 (wn-chameleon-GPS: d = 96, head dim 24; the
    Performer takes head dim 64): with the Philox offset pinned the layer is a smooth (GELU) function whose backward equals
    a central finite difference of its forward, i.e. forward and backward draw the same masks.  A different offset
    draws different masks."""
    d = 96 if glob == "Transformer" else 64
    _, layer = _pair(d, local, glob, heads=4 if glob != "Performer" else 2, dropout=0.2, attn_dropout=0.5, seed=5)
    layer.train()
    b = node_graph(700, 4000, d, seed=3).to(DEV)
    if local == "GINE":   # its message relu(x_j + e_ij) has a kink whatever the activation: keep the sums away from it
        b.edge_attr += 4.0
    g = torch.Generator().manual_seed(2)
    ct_x = torch.randn(b.x.shape, generator=g).to(DEV)
    ct_e = torch.randn(b.edge_attr.shape, generator=g).to(DEV)
    vx = torch.randn(b.x.shape, generator=g).to(DEV)

    def f(x, counter=7 * 4096):
        pin_dropout_counter(DEV, counter)
        out = layer(graphgps_b200.GraphBatch(x=x, edge_index=b.edge_index, edge_attr=b.edge_attr.clone(), batch=b.batch,
                                             num_graphs=1))
        loss = (out.x * ct_x).sum()
        if local == "CustomGatedGCN":
            loss = loss + (out.edge_attr * ct_e).sum()
        return loss, out

    x0 = b.x.clone().requires_grad_(True)
    loss, out0 = f(x0)
    loss.backward()
    analytic = float((x0.grad * vx).sum())
    eps = 1e-2
    with torch.no_grad():
        lp, _ = f(b.x + eps * vx)
        lm, _ = f(b.x - eps * vx)
        _, again = f(b.x.clone())
        _, other = f(b.x.clone(), counter=9 * 4096)
    numeric = float((lp - lm) / (2 * eps))
    assert torch.equal(again.x, out0.x.detach())                # pinned offset => identical masks
    assert not torch.equal(other.x, out0.x.detach())            # another offset => other masks
    assert abs(numeric - analytic) <= 3e-2 * max(1.0, abs(analytic)), (numeric, analytic)
    print(local, glob, "fd", numeric, "analytic", analytic)


# ------------------------------------------------------------------------------------------ eval mode
@pytest.mark.parametrize("local,glob,shape", [("GCN", "Transformer", "webkb"), ("CustomGatedGCN", "Transformer", None),
                                              ("GINE", "None", None)])
def test_eval_mode_forward_backward_matches_oracle(local, glob, shape):
    """Eval mode: no dropout (the layer is built with 0.2 / 0.5), GatedGCN's BatchNorms on their running statistics."""
    if shape is not None:
        b = with_edge_cases(node_shape_batch(shape, seed=4), 4)
        d = NODE_SHAPES[shape].d
    else:
        b, d = graphgps_b200.make_batch("zinc-gatedgcn", seed=4, dim=48, num_graphs=8), 48
    ora, ours = _pair(d, local, glob, dropout=0.2, attn_dropout=0.5, seed=6)
    with torch.no_grad():
        for m in list(ora.modules()):
            if isinstance(m, torch.nn.BatchNorm1d):
                m.running_mean.uniform_(-0.2, 0.2)
                m.running_var.uniform_(0.6, 1.4)
    ours.load_state_dict(ora.state_dict(), strict=True)
    ora.eval()
    ours.eval()
    fix = _cts(b, local)
    ref = _oracle64(ora, b, fix)
    res = run_layer(ours, b.clone().to(DEV), fix)
    errs = compare(res, _target(ref), TOL["fp32"], f"eval {local}+{glob}", grad_l2_tol=GRAD_L2["fp32"])
    print(local, glob, "eval max err", max(v for k, v in errs.items() if not k.startswith("raw:")))


# ------------------------------------------------------------------------------------------ stack, capture
def test_two_layer_stack_matches_oracle_and_capture_replays_eager():
    """gt.layers = 2 (every GCN+Transformer config): the second layer reads the planes the first layer's FF2 epilogue
    wrote.  The stack equals two fp64 oracle layers; its captured step equals the eager step bitwise."""
    s = NODE_SHAPES["chameleon"]
    b = node_shape_batch("chameleon", seed=5)
    torch.manual_seed(5)
    oras = [OracleGPSLayer(s.d, "GCN", "Transformer", s.heads, act="gelu", batch_norm=False) for _ in range(2)]
    stack = graphgps_b200.GPSStack(2, s.d, "GCN", "Transformer", s.heads, act="gelu", batch_norm=False)
    for lay, o in zip(stack.layers, oras):
        with torch.no_grad():
            o.local_model.bias.uniform_(-0.3, 0.3)
        lay.load_state_dict(o.state_dict(), strict=True)
    stack = stack.to(DEV).train()
    fix = _cts(b)
    with torch.device(DEV):
        ref = run_layer(torch.nn.Sequential(*[copy.deepcopy(o).to(DEV).double() for o in oras]), _to64(b, DEV), fix)
    res = run_layer(stack, b.clone().to(DEV), fix)
    bad = {}
    if not rel_err(res["out_x"], ref["out_x"]) < TOL["fp32"]:
        bad["out_x"] = rel_err(res["out_x"], ref["out_x"])
    got = {"layers." + n: g for n, g in ref["grad_params"].items()}
    pairs = [("grad_x", res["grad_x"], ref["grad_x"])]
    pairs += [(n, p.grad.detach().cpu(), got[n]) for n, p in stack.named_parameters()]
    worst = 0.0
    for k, a, g in pairs:   # GELU: the strict max-abs bound through both layers
        worst = max(worst, rel_err(a, g))
        if not rel_err(a, g) < STRICT_GRAD["fp32"]:
            bad[k] = (rel_err(a, g), rel_l2(a, g))
    assert not bad, bad
    print("2-layer stack: out_x", f"{rel_err(res['out_x'], ref['out_x']):.2e}", f"worst grad max-abs {worst:.2e}")
    # captured step == eager step
    bd = b.clone().to(DEV)
    graph_of(bd)
    ct_x = fix["ct_x"].to(DEV)
    step = stack.capture(bd, ct_x)
    step.replay()
    torch.cuda.synchronize()
    x_out, gx = step.x_out.clone(), step.grad_x.clone()
    grads = [p.grad.clone() for p in stack.parameters()]
    xe = bd.x.detach().clone().requires_grad_(True)
    for p in stack.parameters():
        p.grad = None
    out = stack(graphgps_b200.GraphBatch(x=xe, edge_index=bd.edge_index, edge_attr=bd.edge_attr, batch=bd.batch,
                                         num_graphs=1))
    torch.autograd.backward([out.x], [ct_x])
    assert torch.equal(out.x.detach(), x_out) and torch.equal(xe.grad, gx)
    for (n, p), g in zip(stack.named_parameters(), grads):
        assert torch.equal(p.grad, g), n


def test_bucket_gradients_equal_plain_gradients():
    """dp.GradBucket's in-place accumulation path (GpsLayerArgs.flags, GPS_FLAG_GRADS_ACCUMULATE) on layers without norms."""
    b = node_shape_batch("webkb", seed=6).to(DEV)
    torch.manual_seed(7)
    stack = graphgps_b200.GPSStack(2, 64, "GCN", "Transformer", 4, act="gelu", batch_norm=False).to(DEV).train()
    ct = torch.randn_like(b.x)

    def step():
        x = b.x.clone().requires_grad_(True)
        out = stack(graphgps_b200.GraphBatch(x=x, edge_index=b.edge_index, edge_attr=b.edge_attr, batch=b.batch,
                                             num_graphs=1))
        torch.autograd.backward([out.x], [ct])
        return x.grad

    for p in stack.parameters():
        p.grad = None
    gx = step()
    plain = [p.grad.clone() for p in stack.parameters()]
    bucket = stack.make_grad_bucket()
    bucket.zero_()
    assert torch.equal(step(), gx)
    for (n, p), g in zip(stack.named_parameters(), plain):
        assert torch.equal(p.grad, g), n


def test_graphgym_webkb_tex_layer_trains_and_matches_the_oracle(monkeypatch):
    """A GCN+Transformer layer built by graphgym.register() from a webkb-tex-GPS-style cfg (batch_norm: False, gelu,
    dropout 0.2) runs forward and backward; with dropout off it equals the oracle."""
    import sys
    from graphgps_b200 import graphgym
    ns = types.SimpleNamespace
    cfg = ns(gt=ns(layer_type="GCN+Transformer", n_heads=4, dropout=0.2, attn_dropout=0.0, layer_norm=False,
                   batch_norm=False), gnn=ns(act="gelu"), posenc_EquivStableLapPE=ns(enable=False))
    for mod, attrs in (("torch_geometric", {}), ("torch_geometric.graphgym", {}),
                       ("torch_geometric.graphgym.register", {"register_layer": lambda key, module=None: module}),
                       ("torch_geometric.graphgym.config", {"cfg": cfg})):
        m = types.ModuleType(mod)
        m.__dict__.update(attrs)
        monkeypatch.setitem(sys.modules, mod, m)
    torch.manual_seed(8)
    layer = graphgym.register("gpslayer_b200_webkb")(ns(dim_out=64)).to(DEV).train()
    b = with_edge_cases(node_shape_batch("webkb", seed=8), 8)
    bb = b.clone().to(DEV)
    bb.x.requires_grad_(True)
    x_in = bb.x
    out = layer(bb)
    out.x.square().sum().backward()
    assert torch.isfinite(x_in.grad).all() and all(torch.isfinite(p.grad).all() for p in layer.parameters())
    assert not torch.equal(layer(b.clone().to(DEV)).x, out.x)   # dropout 0.2 draws new masks per call
    layer.dropout = 0.0
    layer.__dict__.pop("_args_cache", None)
    ora = OracleGPSLayer(64, "GCN", "Transformer", 4, act="gelu", batch_norm=False)
    ora.load_state_dict(layer.state_dict(), strict=True)
    fix = _cts(b)
    for p in layer.parameters():
        p.grad = None
    res = run_layer(layer, b.clone().to(DEV), fix)
    compare(res, _target(_oracle64(ora, b, fix)), TOL["fp32"], "graphgym webkb-tex", grad_l2_tol=GRAD_L2["fp32"])


# ------------------------------------------------------------------------------------------ launches
@pytest.mark.parametrize("local,glob,dropout", [("GCN", "Transformer", 0.2), ("GCN", "Transformer", 0.0),
                                                ("CustomGatedGCN", "Transformer", 0.0), ("GINE", "None", 0.2),
                                                ("None", "Performer", 0.0)])
def test_fewer_launches_than_batchnorm_mode(local, glob, dropout):
    lib = _lib.load()
    b = graphgps_b200.make_batch("zinc-gine", seed=2, dim=64, num_graphs=8).to(DEV)
    graph_of(b)
    counts = {}
    for bn in (True, False):
        torch.manual_seed(1)
        layer = graphgps_b200.GPSLayer(64, local, glob, 4, act="gelu", dropout=dropout, batch_norm=bn).to(DEV).train()

        def step():
            bb = graphgps_b200.GraphBatch(x=b.x.clone().requires_grad_(True), edge_index=b.edge_index,
                                          edge_attr=b.edge_attr.clone().requires_grad_(local in ("GINE",)),
                                          batch=b.batch, num_graphs=b.num_graphs)
            bb.__dict__["_gps_b200_graph"] = b.__dict__["_gps_b200_graph"]
            out = layer(bb)
            out.x.sum().backward()

        step()
        torch.cuda.synchronize()
        c0 = lib.gps_launch_count()
        step()
        torch.cuda.synchronize()
        counts[bn] = lib.gps_launch_count() - c0
    print(local, glob, f"dropout={dropout}", "launches fwd+bwd: batch_norm=True", counts[True], "batch_norm=False",
          counts[False])
    assert counts[False] < counts[True]
