"""CPU: GPSLayer(..., 'BiasedTransformer', ...), Graphormer's additive attention bias (gps_layer.py:104-106, 202-204,
234-241).  The oracle (tests/biased_oracle.py) is pinned to the reference's own fp64 outputs and gradients
(tests/golden/biased/, made by tests/golden/make_biased_golden.py); the module keeps the reference's parameters and
constructor behaviour; the C entry points reject malformed biases before any CUDA call; GpsLayerArgs is unchanged."""
import ctypes as C
import sys
import types

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import GraphBatch, make_batch
from oracle.gps_oracle import OracleGPSLayer, param_count
from biased_oracle import OracleGPSLayerBiased
from biased_util import LIVE_NAME, PAD_VALUE, biased_batch, biased_names, compare_biased, load_biased, make_bias, \
    run_biased


def _oracle(fix, dtype):
    cfg = fix["config"]
    layer = OracleGPSLayerBiased(cfg["d"], cfg["local"], "BiasedTransformer", cfg["heads"], act=cfg["act"],
                                 batch_norm=cfg["batch_norm"])
    layer.load_state_dict(fix["state"], strict=True)
    return layer.to(dtype).train(cfg["training"])


def test_biased_fixtures_exist():
    names = biased_names()
    assert len(names) == 8
    cfgs = [load_biased(n)["config"] for n in names]
    assert {c["local"] for c in cfgs} == {"GINE", "CustomGatedGCN", "None"}
    assert {c["bias_kind"] for c in cfgs} == {"random", "graph_token", "spd"}
    assert {c["act"] for c in cfgs} == {"relu", "gelu"}
    assert {c["batch_norm"] for c in cfgs} == {True, False} and {c["training"] for c in cfgs} == {True, False}


def test_oracle_equals_reference_live_biased():
    """The reference layer's own fp64 outputs and gradients, the attn_bias gradient included."""
    ref = load_biased(LIVE_NAME)
    O = OracleGPSLayerBiased(32, "GINE", "BiasedTransformer", 4)
    O.load_state_dict(ref["state"], strict=True)
    O = O.double()
    b = GraphBatch(x=ref["x"].clone().requires_grad_(True), edge_index=ref["edge_index"],
                   edge_attr=ref["edge_attr"].clone().requires_grad_(True), batch=ref["batch"],
                   num_graphs=ref["num_graphs"], attn_bias=ref["attn_bias"].clone().requires_grad_(True))
    x_in, ab_in = b.x, b.attn_bias
    o = O(b)
    (o.x * ref["ct_x"]).sum().backward()
    assert (ref["out_x"] - o.x).abs().max() < 1e-10
    assert (ref["grad_x"] - x_in.grad).abs().max() < 1e-9
    assert (ref["grad_attn_bias"] - ab_in.grad).abs().max() < 1e-9
    assert float(ref["grad_attn_bias"].norm()) > 1.0
    po = dict(O.named_parameters())
    assert set(ref["grad_params"]) == {n for n, p in po.items() if p.grad is not None}
    for n, g in ref["grad_params"].items():
        assert (g - po[n].grad).abs().max() < 1e-9, n


@pytest.mark.parametrize("name", biased_names())
def test_oracle_matches_biased_golden_fp64(name):
    fix = load_biased(name)
    res = run_biased(_oracle(fix, torch.float64), biased_batch(fix, dtype=torch.float64), fix,
                     backward=fix["config"]["training"])
    compare_biased(res, fix, 2e-6, f"oracle fp64 vs biased golden {name}")


@pytest.mark.parametrize("name", biased_names())
def test_biased_fixture_bias_matters(name):
    """Each fixture's bias reshapes the softmax: the same layer without it (zero bias) moves the output by O(1), and the
    attn_bias gradient is far from 0, zero exactly at the padded entries."""
    fix = load_biased(name)
    b = biased_batch(fix, dtype=torch.float64)
    nob = biased_batch(fix, dtype=torch.float64)
    nob.attn_bias = torch.zeros_like(nob.attn_bias)
    with torch.no_grad():
        d = (_oracle(fix, torch.float64)(b).x - _oracle(fix, torch.float64)(nob).x).abs().max()
    assert float(d) > 0.1, name
    ab = fix["attn_bias"]
    pad = ab == PAD_VALUE
    assert pad.any() and not pad.all()
    if "grad_attn_bias" in fix:
        g = fix["grad_attn_bias"]
        assert float(g.norm()) > 1.0
        assert bool((g[pad] == 0).all())


def test_state_dict_matches_reference_and_transformer():
    """self_attn is the Transformer's nn.MultiheadAttention (gps_layer.py:104-106): key for key the reference's."""
    for name in biased_names() + [LIVE_NAME]:
        fix = load_biased(name)
        cfg = fix.get("config", {"d": 32, "local": "GINE", "heads": 4, "act": "relu", "batch_norm": True})
        ours = graphgps_b200.GPSLayer(cfg["d"], cfg["local"], "BiasedTransformer", cfg["heads"], act=cfg["act"],
                                      batch_norm=cfg["batch_norm"])
        so, sr = ours.state_dict(), fix["state"]
        assert list(so) == list(sr)
        for k in so:
            assert tuple(so[k].shape) == tuple(sr[k].shape), k
        ours.load_state_dict(sr, strict=True)
    for local in ("GINE", "CustomGatedGCN", "GCN", "None"):
        b, t = graphgps_b200.GPSLayer(64, local, "BiasedTransformer", 4), graphgps_b200.GPSLayer(64, local, "Transformer", 4)
        assert [(n, p.shape) for n, p in b.named_parameters()] == [(n, p.shape) for n, p in t.named_parameters()]
        assert isinstance(b.self_attn, torch.nn.MultiheadAttention)
        assert param_count(b) == param_count(OracleGPSLayerBiased(64, local, "BiasedTransformer", 4))


def test_constructor_accepts_the_type_and_keeps_the_reference_errors():
    G = graphgps_b200.GPSLayer
    layer = G(64, "GINE", "BiasedTransformer", 4, dropout=0.0, attn_dropout=0.5)
    assert layer.global_model_type == "BiasedTransformer" and layer.self_attn.dropout == 0.5
    with pytest.raises(ValueError):
        G(66, "GINE", "BiasedTransformer", 4)                # embed_dim % num_heads
    with pytest.raises(NotImplementedError):
        G(64, "GINE", "BiasedTransformer", 4, log_attn_weights=True)
    with pytest.raises(NotImplementedError):
        G(64, "GINE", "BigBird", 4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        layer(make_batch("zinc-gine", dim=64, num_graphs=2))


def test_oracle_reads_attn_bias_and_raises_without_it():
    torch.manual_seed(0)
    O = OracleGPSLayerBiased(32, "GINE", "BiasedTransformer", 4)
    b = make_batch("zinc-gine", seed=1, dim=32, num_graphs=3)
    with pytest.raises(AttributeError):
        O(b.clone())
    T = OracleGPSLayer(32, "GINE", "Transformer", 4)
    T.load_state_dict(O.state_dict(), strict=True)
    zb = b.clone()
    zb.attn_bias = torch.zeros_like(make_bias(b.batch, 3, 4, 0))
    assert torch.allclose(O(zb).x, T(b.clone()).x, atol=1e-6)


def test_graphgym_register_builds_gine_biased_transformer(monkeypatch):
    """graphgym.register splits cfg.gt.layer_type (gps_model.py:80): zinc-GPSwGraphormer's GINE+BiasedTransformer."""
    from graphgps_b200 import graphgym
    ns = types.SimpleNamespace
    cfg = ns(gt=ns(layer_type="GINE+BiasedTransformer", n_heads=4, dropout=0.0, attn_dropout=0.5, layer_norm=False,
                   batch_norm=True), gnn=ns(act="relu"), posenc_EquivStableLapPE=ns(enable=False))
    registry = {}
    for name, attrs in (("torch_geometric", {}), ("torch_geometric.graphgym", {}),
                        ("torch_geometric.graphgym.register",
                         {"register_layer": lambda key, module=None: registry.setdefault(key, module)}),
                        ("torch_geometric.graphgym.config", {"cfg": cfg})):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        monkeypatch.setitem(sys.modules, name, m)
    cls = graphgym.register("gpslayer_b200_biased")
    layer = cls(ns(dim_out=64))
    assert registry["gpslayer_b200_biased"] is cls
    assert layer.local_gnn_type == "GINE" and layer.global_model_type == "BiasedTransformer"
    assert layer.attn_dropout == 0.5 and layer.num_heads == 4


def test_attn_bias_fields_and_abi_version():
    """The bias travels in GpsLayerArgs.attn_bias; the BiasedTransformer is the Transformer global type."""
    assert [f[0] for f in _lib.GpsAttnBias._fields_] == ["bias", "nmax", "grad_bias"]
    assert dict(_lib.GpsLayerArgs._fields_)["attn_bias"] is _lib.GpsAttnBias
    assert _lib.load().gps_abi_version() == 4
    assert _lib.GLOBAL == {"None": 0, "Transformer": 1, "Performer": 2, "BigBird": 3}


def _args(glob="Transformer", N=50, E=120, B=4):
    a = _lib.GpsLayerArgs()
    a.d, a.heads, a.local_type, a.global_type, a.act, a.training = 64, 4, _lib.LOCAL["GINE"], _lib.GLOBAL[glob], 0, 1
    a.graph.N, a.graph.E, a.graph.B = N, E, B
    return a


@pytest.mark.parametrize("fn", ["gps_layer_forward", "gps_layer_backward"])
def test_layer_entry_points_reject_bad_biases(fn):
    """GPS_ERR_ARG before any CUDA call: a bias with another global type, nmax < 1, a NULL bias pointer with nmax or
    grad_bias set, NULL args."""
    lib = _lib.load()
    f = getattr(lib, fn)

    def call(bias, glob="Transformer"):
        a = _args(glob)
        a.attn_bias = bias
        return f(C.byref(a), None)

    good = _lib.GpsAttnBias(0x1000, 37, 0)
    for glob in ("Performer", "None"):
        assert call(good, glob) == _lib.GPS_ERR_ARG
    for nmax in (0, -1):
        assert call(_lib.GpsAttnBias(0x1000, nmax, 0)) == _lib.GPS_ERR_ARG
    assert call(_lib.GpsAttnBias(0, 37, 0x2000)) == _lib.GPS_ERR_ARG
    assert call(_lib.GpsAttnBias(0, 37, 0)) == _lib.GPS_ERR_ARG
    assert call(_lib.GpsAttnBias(0, 0, 0x2000)) == _lib.GPS_ERR_ARG
    assert f(None, None) == _lib.GPS_ERR_ARG
    assert b"nmax" in lib.gps_last_error() or b"null" in lib.gps_last_error() or b"args" in lib.gps_last_error()


def test_stage_entry_points_reject_bad_biases():
    lib = _lib.load()
    g = _lib.GpsGraph()
    g.N, g.E, g.B = 50, 0, 4
    p = 0x1000
    calls = {
        "fwd": lambda ab: lib.gps_attention_forward_biased(C.byref(g), 4, 16, p, p, p, 192, p, 64, p, 0.0, 0, 0, ab,
                                                           None),
        "tc": lambda ab: lib.gps_attention_forward_tc_biased(C.byref(g), 4, 16, p, p, 192, p, 64, p, 0.0, 0, 0, 0, ab,
                                                             None),
        "bwd": lambda ab: lib.gps_attention_backward_biased(C.byref(g), 4, 16, p, p, p, 192, p, p, 64, p, p, p, p, p,
                                                            192, 0.0, 0, 0, ab, None),
    }
    for name, call in calls.items():
        assert call(None) == _lib.GPS_ERR_ARG, name
        assert call(C.byref(_lib.GpsAttnBias(0, 37, 0))) == _lib.GPS_ERR_ARG, name
        assert call(C.byref(_lib.GpsAttnBias(p, 0, 0))) == _lib.GPS_ERR_ARG, name
    assert lib.gps_attention_forward_biased(None, 4, 16, p, p, p, 192, p, 64, p, 0.0, 0, 0,
                                            C.byref(_lib.GpsAttnBias(p, 37, 0)), None) == _lib.GPS_ERR_ARG


def test_make_bias_kinds():
    b = make_batch("zinc-gine", seed=2, dim=8, num_graphs=3)
    n = torch.bincount(b.batch, minlength=3)
    for kind in ("random", "graph_token", "spd"):
        ab = make_bias(b.batch, 3, 4, 1, kind, b.edge_index)
        assert ab.shape == (12, int(n.max()), int(n.max()))
        g0 = ab[0, :n[0], :n[0]]
        assert bool((ab[0, n[0]:, :] == PAD_VALUE).all()) and bool((ab[0, :, n[0]:] == PAD_VALUE).all())
        assert not torch.equal(ab[0, :n[0], :n[0]], ab[1, :n[0], :n[0]])           # per head
        if kind == "spd":
            assert g0.unique().numel() <= 8 and torch.equal(g0.diagonal(), g0[0, 0].expand(int(n[0])))
        else:
            assert not torch.equal(g0, g0.t())                                       # asymmetric
        if kind == "graph_token":
            assert bool((g0[0, :] == g0[0, 0]).all()) and bool((g0[:, 0] == g0[0, 0]).all())


def test_oracle_initial_state_equals_reference():
    """Under one torch seed the oracle draws the reference layer's initial parameters; needs the reference layer files."""
    from oracle.ref_shim import find_reference_layer_dir, load_reference
    if find_reference_layer_dir() is None:
        pytest.skip("reference layer files not present")
    for local in ("GINE", "None"):
        torch.manual_seed(7)
        ref = load_reference().GPSLayer(32, local, "BiasedTransformer", 2).state_dict()
        torch.manual_seed(7)
        ora = OracleGPSLayerBiased(32, local, "BiasedTransformer", 2).state_dict()
        assert set(ref) == set(ora)
        for k in ref:
            assert torch.equal(ref[k], ora[k]), k
