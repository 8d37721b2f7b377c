"""CPU: GPSLayer(..., batch_norm=False), the normalisation-free mode of every GCN+Transformer config
(gps_layer.py:125-151, 191-229 with layer_norm = batch_norm = False).  The oracle is pinned to the reference's own fp64
outputs (tests/golden/nonorm/, made by tests/golden/make_nonorm_golden.py); the module keeps the reference's parameters
and constructor behaviour; the library plans the mode without a GPU."""
import ctypes as C
import sys
import types

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import GraphBatch
from oracle.gps_oracle import OracleGPSLayer
from nonorm_util import LIVE_NAME, NODE_SHAPES, load_nonorm, node_graph, nonorm_names
from util import compare, golden_batch, run_layer

NORMS = ("norm1_local", "norm1_attn", "norm2")
COMBOS = [(lo, gl) for lo in ("None", "CustomGatedGCN", "GINE", "GCN") for gl in ("None", "Transformer", "Performer")
          if (lo, gl) != ("None", "None")]


def _oracle(fix, dtype):
    cfg = fix["config"]
    layer = OracleGPSLayer(cfg["d"], cfg["local"], cfg["glob"], cfg["heads"], act=cfg["act"], batch_norm=False)
    layer.load_state_dict(fix["state"], strict=True)
    return layer.to(dtype).train(cfg["training"])


def test_nonorm_fixtures_exist():
    names = nonorm_names()
    assert len(names) == 9
    cfgs = [load_nonorm(n)["config"] for n in names]
    assert all(c["batch_norm"] is False for c in cfgs)
    assert {(c["local"], c["glob"]) for c in cfgs} >= {("GCN", "Transformer"), ("GCN", "None"), ("GINE", "Transformer"),
                                                       ("CustomGatedGCN", "Transformer"), ("None", "Transformer"),
                                                       ("CustomGatedGCN", "Performer")}
    assert any(not c["training"] for c in cfgs)
    assert {c["d"] // c["heads"] for c in cfgs if c["glob"] == "Transformer"} >= {16, 24}


def test_oracle_equals_reference_live_nonorm():
    """The reference GCN+Transformer layer's own fp64 outputs and gradients, batch_norm=False, GELU, one graph."""
    ref = load_nonorm(LIVE_NAME)
    O = OracleGPSLayer(32, "GCN", "Transformer", 4, act="gelu", batch_norm=False)
    O.load_state_dict(ref["state"], strict=True)
    O = O.double()
    b = GraphBatch(x=ref["x"].clone().requires_grad_(True), edge_index=ref["edge_index"], edge_attr=ref["edge_attr"],
                   batch=ref["batch"], num_graphs=ref["num_graphs"])
    x_in = b.x
    o = O(b)
    (o.x ** 2).sum().backward()
    assert (ref["out_x"] - o.x).abs().max() < 1e-10
    assert (ref["grad_x"] - x_in.grad).abs().max() < 1e-9
    po = dict(O.named_parameters())
    assert set(ref["grad_params"]) == {n for n, p in po.items() if p.grad is not None}
    for n, g in ref["grad_params"].items():
        assert (g - po[n].grad).abs().max() < 1e-9, n


@pytest.mark.parametrize("name", nonorm_names())
def test_oracle_matches_nonorm_golden_fp64(name):
    fix = load_nonorm(name)
    res = run_layer(_oracle(fix, torch.float64), golden_batch(fix, dtype=torch.float64), fix,
                    backward=fix["config"]["training"])
    compare(res, fix, 2e-6, f"oracle fp64 vs nonorm golden {name}")


@pytest.mark.parametrize("name", nonorm_names())
def test_oracle_fp32_close_to_nonorm_golden(name):
    fix = load_nonorm(name)
    res = run_layer(_oracle(fix, torch.float32), golden_batch(fix), fix, backward=fix["config"]["training"])
    compare(res, fix, 5e-4, f"oracle fp32 vs nonorm golden {name}")


@pytest.mark.parametrize("name", nonorm_names() + [LIVE_NAME])
def test_state_dict_matches_reference(name):
    """The fixtures hold the reference module's own state_dict: same keys and shapes, strict load both ways."""
    fix = load_nonorm(name)
    cfg = fix.get("config", {"d": 32, "local": "GCN", "glob": "Transformer", "heads": 4, "act": "gelu"})
    ours = graphgps_b200.GPSLayer(cfg["d"], cfg["local"], cfg["glob"], cfg["heads"], act=cfg["act"], batch_norm=False)
    so, sr = ours.state_dict(), fix["state"]
    assert set(so) == set(sr)
    for k in so:
        assert tuple(so[k].shape) == tuple(sr[k].shape), k
    ours.load_state_dict(sr, strict=True)
    ora = OracleGPSLayer(cfg["d"], cfg["local"], cfg["glob"], cfg["heads"], act=cfg["act"], batch_norm=False)
    ora.load_state_dict(ours.state_dict(), strict=True)


@pytest.mark.parametrize("local,glob", COMBOS)
def test_every_built_model_constructs_without_norms(local, glob):
    ours = graphgps_b200.GPSLayer(64, local, glob, 4, batch_norm=False)
    for n in NORMS:
        assert not hasattr(ours, n), n
    assert not any(k.startswith(tuple(n + "." for n in NORMS)) for k in ours.state_dict())
    ora = OracleGPSLayer(64, local, glob, 4, batch_norm=False)
    assert {k: tuple(v.shape) for k, v in ours.state_dict().items()} == \
        {k: tuple(v.shape) for k, v in ora.state_dict().items()}
    # the BatchNorm layer has exactly the three norms more: 2 affine vectors + 3 buffers each
    bn = graphgps_b200.GPSLayer(64, local, glob, 4)
    assert set(bn.state_dict()) - set(ours.state_dict()) == {f"{n}.{p}" for n in NORMS for p in
                                                               ("weight", "bias", "running_mean", "running_var",
                                                                "num_batches_tracked")}
    assert ours._param_names == [n for n in bn._param_names if not n.startswith(NORMS)]


def test_state_dict_loads_into_the_reference_layer():
    """Both directions against the reference module itself (needs the reference layer files)."""
    from oracle.ref_shim import find_reference_layer_dir, load_reference
    if find_reference_layer_dir() is None:
        pytest.skip("reference layer files not present")
    ref = load_reference()
    for local, glob in (("GCN", "Transformer"), ("CustomGatedGCN", "Transformer"), ("GINE", "None"),
                        ("None", "Performer")):
        R = ref.GPSLayer(64, local, glob, 4, act="gelu", batch_norm=False)
        ours = graphgps_b200.GPSLayer(64, local, glob, 4, act="gelu", batch_norm=False)
        if glob == "Performer":   # a buffer drawn at construction: take the reference's
            ours.load_state_dict(R.state_dict(), strict=True)
        R.load_state_dict(ours.state_dict(), strict=True)
        ours.load_state_dict(R.state_dict(), strict=True)
        for n in NORMS:
            assert hasattr(R, n) == hasattr(ours, n) == False  # noqa: E712


def test_error_contract():
    G = graphgps_b200.GPSLayer
    with pytest.raises(ValueError, match="two types of normalization"):
        G(64, "GCN", "Transformer", 4, layer_norm=True, batch_norm=True)
    for bn in (False,):
        with pytest.raises(NotImplementedError, match="LayerNorm") as e:
            G(64, "GCN", "Transformer", 4, layer_norm=True, batch_norm=bn)
        assert "BatchNorm" not in str(e.value) and "every shipped config" not in str(e.value)
    with pytest.raises(ValueError, match="local model or a global model"):
        G(64, "None", "None", 4, batch_norm=False)


def _cfg(layer_type, batch_norm, act="gelu", dropout=0.2, attn_dropout=0.0, heads=4):
    ns = types.SimpleNamespace
    return ns(gt=ns(layer_type=layer_type, n_heads=heads, dropout=dropout, attn_dropout=attn_dropout, layer_norm=False,
                    batch_norm=batch_norm), gnn=ns(act=act), posenc_EquivStableLapPE=ns(enable=False))


def _register(monkeypatch, cfg, name):
    from graphgps_b200 import graphgym
    for mod, attrs in (("torch_geometric", {}), ("torch_geometric.graphgym", {}),
                       ("torch_geometric.graphgym.register", {"register_layer": lambda key, module=None: module}),
                       ("torch_geometric.graphgym.config", {"cfg": cfg})):
        m = types.ModuleType(mod)
        m.__dict__.update(attrs)
        monkeypatch.setitem(sys.modules, mod, m)
    return graphgym.register(name)


def test_graphgym_register_builds_a_webkb_tex_style_layer(monkeypatch):
    """webkb-tex-GPS: gt.layer_type GCN+Transformer, 4 heads, dropout 0.2, batch_norm / layer_norm False, gnn.act gelu."""
    cls = _register(monkeypatch, _cfg("GCN+Transformer", False), "gpslayer_b200_nonorm")
    layer = cls(types.SimpleNamespace(dim_out=64))
    assert (layer.local_gnn_type, layer.global_model_type, layer.batch_norm, layer.act) == ("GCN", "Transformer",
                                                                                          False, "gelu")
    assert layer.dropout == 0.2 and not any(hasattr(layer, n) for n in NORMS)
    ora = OracleGPSLayer(64, "GCN", "Transformer", 4, act="gelu", batch_norm=False)
    ora.load_state_dict(layer.state_dict(), strict=True)
    layer.load_state_dict(ora.state_dict(), strict=True)


def test_build_args_sets_norm_type_and_leaves_the_norm_structs_zero():
    for bn in (True, False):
        layer = graphgps_b200.GPSLayer(32, "GCN", "Transformer", 4, act="gelu", batch_norm=bn)
        named = dict(layer.named_parameters())
        grads = {n: torch.empty_like(p) for n, p in named.items()}
        a = layer._build_args(named, grads)
        assert a.norm_type == (_lib.NORM["batch"] if bn else _lib.NORM["none"])
        for n in NORMS:
            s = getattr(a, n)
            fields = [getattr(s, f) for f, _ in _lib.GpsBatchNorm._fields_]
            assert all(v is None or v == 0 for v in fields) != bn, n
        assert a.ff1.weight and a.attn_out.weight and a.gcn_conv.weight


def _plan(local="GCN", glob="Transformer", norm=1, N=7600, E=30019, B=1, d=64, heads=4, dropout=0.2, training=1):
    a = _lib.GpsLayerArgs()
    a.d, a.heads, a.local_type, a.global_type, a.act, a.training = d, heads, _lib.LOCAL[local], _lib.GLOBAL[glob], 1, training
    a.dropout = dropout
    a.norm_type = norm
    if glob == "Performer":
        a.perf_features, a.perf_dim_head = 266, 64
    a.graph.N, a.graph.E, a.graph.B = N, E, B
    plan = _lib.GpsLayerPlan()
    return _lib.load().gps_layer_plan(C.byref(a), C.byref(plan)), plan, a


@pytest.mark.parametrize("local,glob", COMBOS)
def test_plan_is_smaller_without_norms(local, glob):
    for shape in ("actor", "webkb"):
        s = NODE_SHAPES[shape]
        for dropout in (0.0, 0.2):
            rb, pb, _ = _plan(local, glob, 0, s.N, s.E, 1, s.d, s.heads, dropout)
            rn, pn, _ = _plan(local, glob, 1, s.N, s.E, 1, s.d, s.heads, dropout)
            assert rb == rn == _lib.GPS_OK
            assert pn.saved_bytes < pb.saved_bytes, (shape, dropout)
            assert pn.bwd_workspace_bytes < pb.bwd_workspace_bytes, (shape, dropout)
            assert pn.wplanes_bytes == pb.wplanes_bytes   # the same weights minus three BatchNorms (no planes)


def test_unknown_norm_type_is_unsupported_everywhere():
    lib = _lib.load()
    for norm in (2, -1, 7):
        rc, _, a = _plan(norm=norm)
        assert rc == _lib.GPS_ERR_UNSUPPORTED
        assert b"norm_type" in lib.gps_last_error()
        # forward / backward refuse it while planning, before any device work
        assert lib.gps_layer_forward(C.byref(a), None) == _lib.GPS_ERR_UNSUPPORTED
        assert lib.gps_layer_backward(C.byref(a), None) == _lib.GPS_ERR_UNSUPPORTED


def test_grad_bucket_groups_and_stack_without_norms():
    """GPSStack (2 layers, as the configs) and dp.GradBucket: prefix groups early / mid / late still cover every
    parameter of a layer that has no norms, in the order the backward pass finishes them."""
    from graphgps_b200.dp import EARLY, LATE, MID, GradBucket, _group
    st = graphgps_b200.GPSStack(2, 16, "GCN", "Transformer", 2, act="gelu", dropout=0.2, batch_norm=False)
    keys = list(st.state_dict().keys())
    assert not any(".norm" in k for k in keys)
    ora = [OracleGPSLayer(16, "GCN", "Transformer", 2, act="gelu", batch_norm=False) for _ in range(2)]
    for lay, o in zip(st.layers, ora):
        o.load_state_dict(lay.state_dict(), strict=True)
    groups = {n: _group(n) for n, _ in st.layers[0].named_parameters()}
    assert groups == {"local_model.bias": MID, "local_model.lin.weight": LATE, "self_attn.in_proj_weight": LATE,
                      "self_attn.in_proj_bias": LATE, "self_attn.out_proj.weight": EARLY,
                      "self_attn.out_proj.bias": EARLY, "ff_linear1.weight": EARLY, "ff_linear1.bias": EARLY,
                      "ff_linear2.weight": EARLY, "ff_linear2.bias": EARLY}
    bucket = GradBucket(list(st.layers))
    lo, n = bucket.flat.data_ptr(), bucket.flat.numel()
    for p in st.parameters():
        assert lo <= p.grad.data_ptr() < lo + 4 * n and p.grad.shape == p.shape
    assert [(li, g) for li, g, _, _ in bucket.segments] == [(0, EARLY), (0, MID), (0, LATE), (1, EARLY), (1, MID),
                                                            (1, LATE)]
    for lay in st.layers:
        assert lay._bucket_grads(dict(lay.named_parameters())) is not None
    st2 = graphgps_b200.GPSStack(2, 16, "CustomGatedGCN", "Performer", 2, batch_norm=False)
    early = {n for n, _ in st2.layers[0].named_parameters() if _group(n) == EARLY}
    assert early == {f"{m}.{p}" for m in ("ff_linear1", "ff_linear2", "self_attn.to_out") for p in ("weight", "bias")}
    GradBucket(list(st2.layers)).check_attached()


def test_node_graph_generator():
    """Seeded, vectorised, directed, heavy-tailed in-degrees (thousands at the squirrel shape)."""
    s = NODE_SHAPES["squirrel"]
    b = node_graph(s.N, s.E, 8, seed=1)
    assert b.edge_index.shape == (2, s.E) and b.x.shape == (s.N, 8) and b.num_graphs == 1
    indeg = torch.bincount(b.edge_index[1], minlength=s.N)
    assert int(indeg.max()) >= 1000 and float(indeg.float().median()) < 0.2 * s.E / s.N * 10
    assert torch.equal(node_graph(s.N, s.E, 8, seed=1).edge_index, b.edge_index)
    assert not torch.equal(node_graph(s.N, s.E, 8, seed=2).edge_index, b.edge_index)
