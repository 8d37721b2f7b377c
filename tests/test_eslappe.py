"""CPU: GPSLayer(..., equivstable_pe=True), the EquivStableLapPE edge gate of GatedGCN (gatedgcn_layer.py:29-35,
65-70, 101-104).  The oracle is pinned to the reference's own fp64 outputs (tests/golden/eslappe/, made by
tests/golden/make_eslappe_golden.py) through tests/eslappe_oracle.py; the module keeps the reference's parameters and constructor behaviour."""
import ctypes as C
import sys
import types

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import GraphBatch
from oracle.gps_oracle import OracleGPSLayer, param_count
from eslappe_oracle import OracleGPSLayerESLapPE
from eslappe_util import LIVE_NAME, compare_eslap, eslap_batch, eslap_names, load_eslap, run_eslap


def _oracle(fix, dtype):
    cfg = fix["config"]
    layer = OracleGPSLayerESLapPE(cfg["d"], cfg["local"], cfg["glob"], cfg["heads"], act=cfg["act"])
    layer.load_state_dict(fix["state"], strict=True)
    return layer.to(dtype).train(cfg["training"])


def test_eslappe_fixtures_exist():
    assert len(eslap_names()) == 5
    assert {load_eslap(n)["config"]["pe_dim"] for n in eslap_names()} >= {7, 48, 64}


def test_oracle_equals_reference_live_eslappe():
    """The reference layer's own fp64 outputs and gradients, grad_pe included."""
    ref = load_eslap(LIVE_NAME)
    O = OracleGPSLayerESLapPE(32, "CustomGatedGCN", "Transformer", 4)
    O.load_state_dict(ref["state"], strict=True)
    O = O.double()
    b = GraphBatch(x=ref["x"].clone().requires_grad_(True), edge_index=ref["edge_index"],
                   edge_attr=ref["edge_attr"].clone().requires_grad_(True), batch=ref["batch"],
                   num_graphs=ref["num_graphs"], pe_EquivStableLapPE=ref["pe"].clone().requires_grad_(True))
    x_in, pe_in = b.x, b.pe_EquivStableLapPE
    o = O(b)
    (o.x ** 2).sum().backward()
    assert (ref["out_x"] - o.x).abs().max() < 1e-10
    assert (ref["grad_x"] - x_in.grad).abs().max() < 1e-9
    assert (ref["grad_pe"] - pe_in.grad).abs().max() < 1e-9
    po = dict(O.named_parameters())
    assert set(ref["grad_params"]) == {n for n, p in po.items() if p.grad is not None}
    assert any(n.startswith("local_model.mlp_r_ij.") for n in ref["grad_params"])
    for n, g in ref["grad_params"].items():
        assert (g - po[n].grad).abs().max() < 1e-9, n


@pytest.mark.parametrize("name", eslap_names())
def test_oracle_matches_eslappe_golden_fp64(name):
    fix = load_eslap(name)
    res = run_eslap(_oracle(fix, torch.float64), eslap_batch(fix, dtype=torch.float64), fix,
                    backward=fix["config"]["training"])
    compare_eslap(res, fix, 2e-6, f"oracle fp64 vs eslappe golden {name}")


@pytest.mark.parametrize("name", eslap_names())
def test_oracle_fp32_close_to_eslappe_golden(name):
    fix = load_eslap(name)
    res = run_eslap(_oracle(fix, torch.float32), eslap_batch(fix), fix, backward=fix["config"]["training"])
    compare_eslap(res, fix, 5e-4, f"oracle fp32 vs eslappe golden {name}")


@pytest.mark.parametrize("name", eslap_names() + [LIVE_NAME])
def test_state_dict_matches_reference(name):
    """The fixtures hold the reference module's own state_dict: same keys and shapes, strict load."""
    fix = load_eslap(name)
    cfg = fix.get("config", {"d": 32, "local": "CustomGatedGCN", "glob": "Transformer", "heads": 4, "act": "relu"})
    ours = graphgps_b200.GPSLayer(cfg["d"], cfg["local"], cfg["glob"], cfg["heads"], act=cfg["act"],
                                  equivstable_pe=True)
    so, sr = ours.state_dict(), fix["state"]
    assert set(so) == set(sr)
    for k in so:
        assert tuple(so[k].shape) == tuple(sr[k].shape), k
    ours.load_state_dict(sr, strict=True)
    # the reference registers mlp_r_ij after E and before bn_node_x (gatedgcn_layer.py:21-38)
    keys = [k for k in so if k.startswith("local_model.")]
    assert keys.index("local_model.E.bias") < keys.index("local_model.mlp_r_ij.0.weight") < \
        keys.index("local_model.bn_node_x.weight")


@pytest.mark.parametrize("glob,heads", [("Transformer", 4), ("None", 4)])
def test_parameter_count(glob, heads):
    """mlp_r_ij adds d (Linear(1, d).weight) + d + d (Linear(d, 1).weight) + 1 to the GatedGCN layer."""
    for d in (64, 304):
        ours = graphgps_b200.GPSLayer(d, "CustomGatedGCN", glob, heads, equivstable_pe=True)
        ora = OracleGPSLayerESLapPE(d, "CustomGatedGCN", glob, heads)
        base = param_count(graphgps_b200.GPSLayer(d, "CustomGatedGCN", glob, heads))
        assert param_count(ours) == param_count(ora) == base + 3 * d + 1
        if glob == "Transformer":
            assert param_count(ours) == 13 * d * d + 25 * d + 1


def test_constructor_gine_raises_and_gcn_none_ignore_the_flag():
    G = graphgps_b200.GPSLayer
    for glob in ("Transformer", "None"):
        with pytest.raises(NotImplementedError, match="reference itself fails to construct"):
            G(64, "GINE", glob, 4, equivstable_pe=True)
    with pytest.raises(NotImplementedError):
        OracleGPSLayerESLapPE(64, "GINE", "Transformer", 4)
    for local, glob in (("GCN", "Transformer"), ("None", "Transformer"), ("GCN", "None")):
        on, off = G(64, local, glob, 4, equivstable_pe=True), G(64, local, glob, 4)
        assert [(n, p.shape) for n, p in on.named_parameters()] == [(n, p.shape) for n, p in off.named_parameters()]
        assert not on._eslap
        ora_on, ora_off = OracleGPSLayerESLapPE(64, local, glob, 4), OracleGPSLayer(64, local, glob, 4)
        assert set(ora_on.state_dict()) == set(ora_off.state_dict()) == set(on.state_dict())


def test_oracle_gcn_and_none_ignore_the_pe():
    """GCN / None never read batch.pe_EquivStableLapPE (gps_layer.py:176-187): no PE on the batch is fine."""
    from graphgps_b200.batch import make_batch
    for local, glob in (("GCN", "Transformer"), ("None", "Transformer")):
        torch.manual_seed(0)
        on = OracleGPSLayerESLapPE(32, local, glob, 4)
        off = OracleGPSLayer(32, local, glob, 4)
        off.load_state_dict(on.state_dict(), strict=True)
        b = make_batch("zinc-gatedgcn", seed=1, dim=32, num_graphs=3)
        assert torch.equal(on(b.clone()).x, off(b.clone()).x)


def _plan(local, pe, pe_dim, N=50, E=120, B=4):
    a = _lib.GpsLayerArgs()
    a.d, a.heads, a.local_type, a.global_type, a.act, a.training = 64, 4, _lib.LOCAL[local], _lib.GLOBAL["Transformer"], 0, 1
    a.graph.N, a.graph.E, a.graph.B = N, E, B
    a.pe, a.pe_dim = pe, pe_dim
    plan = _lib.GpsLayerPlan()
    return _lib.load().gps_layer_plan(C.byref(a), C.byref(plan)), plan


def test_abi_pe_fields_and_plan():
    """gps_layer_plan (host-only) sizes r / rho and the backward scratch of the PE fields, and refuses a PE for local
    models that do not read one."""
    rc0, p0 = _plan("CustomGatedGCN", None, 0)
    rc1, p1 = _plan("CustomGatedGCN", 0x1000, 7)
    assert rc0 == rc1 == _lib.GPS_OK
    assert p1.saved_bytes == p0.saved_bytes + 2 * 512          # r_e and rho_e, 120 floats each (256-byte granules)
    assert p1.bwd_workspace_bytes > p0.bwd_workspace_bytes
    for local in ("GINE", "GCN", "None"):
        assert _plan(local, 0x1000, 7)[0] == _lib.GPS_ERR_ARG
    assert _plan("CustomGatedGCN", 0x1000, 0)[0] == _lib.GPS_ERR_ARG


def test_graphgym_register_forwards_the_flag(monkeypatch):
    """GPSModel passes cfg.posenc_EquivStableLapPE.enable as equivstable_pe (gps_model.py:92)."""
    from graphgps_b200 import graphgym
    ns = types.SimpleNamespace
    for enable in (True, False):
        cfg = ns(gt=ns(layer_type="CustomGatedGCN+Transformer", n_heads=4, dropout=0.0, attn_dropout=0.0,
                       layer_norm=False, batch_norm=True), gnn=ns(act="relu"),
                 posenc_EquivStableLapPE=ns(enable=enable))
        registry = {}
        for name, attrs in (("torch_geometric", {}), ("torch_geometric.graphgym", {}),
                            ("torch_geometric.graphgym.register",
                             {"register_layer": lambda key, module=None: registry.setdefault(key, module)}),
                            ("torch_geometric.graphgym.config", {"cfg": cfg})):
            m = types.ModuleType(name)
            m.__dict__.update(attrs)
            monkeypatch.setitem(sys.modules, name, m)
        cls = graphgym.register("gpslayer_b200_pe")
        layer = cls(ns(dim_out=32))
        assert layer.equivstable_pe == enable and layer._eslap == enable
        assert hasattr(layer.local_model, "mlp_r_ij") == enable


@pytest.mark.parametrize("glob", ["Transformer", "Performer", "None"])
def test_oracle_initial_state_equals_reference(glob):
    """Under one torch seed the oracle draws the same initial parameters as the reference layer (mlp_r_ij between E and
    the global model, gatedgcn_layer.py:21-38 / gps_layer.py:44-153); needs the reference layer files."""
    from oracle.ref_shim import find_reference_layer_dir, load_reference
    if find_reference_layer_dir() is None:
        pytest.skip("reference layer files not present")
    torch.manual_seed(7)
    ref = load_reference().GPSLayer(32, "CustomGatedGCN", glob, 2, equivstable_pe=True).state_dict()
    torch.manual_seed(7)
    ora = OracleGPSLayerESLapPE(32, "CustomGatedGCN", glob, 2).state_dict()
    assert set(ref) == set(ora)
    for k in ref:
        assert torch.equal(ref[k], ora[k]), k
