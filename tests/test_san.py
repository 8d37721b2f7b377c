"""SAN layer, CPU side: the float64 restatement against the reference run verbatim, the fake-pair complement, the
parameter container against the reference's, the constructor contract, the C ABI's plan and argument checks, and
install_san.  The checks SAN2Layer runs as well are in tests/san_harness.py."""
import ctypes as C
import os
import types

import pytest
import torch
import torch.nn as nn

import graphgps_b200
from graphgps_b200 import _lib, graphgym
from san_harness import (NOT_BUILT, VARIANTS, _args, _check_oracle, _load, check_constructor_not_built,
                         check_shared_embedding)
from san_oracle import fake_pairs, san_batch

SAN_DIR = VARIANTS["SAN"].dir
HAVE_REFERENCE = os.path.isfile("/root/reference/graphgps/layer/san_layer.py")


def test_oracle_equals_reference_live():
    _check_oracle("SAN", _load("SAN", "reference_live"), 1e-10, 1e-9)


@pytest.mark.skipif(not HAVE_REFERENCE, reason="the reference tree is not present; reference_live pins the oracle")
def test_oracle_equals_reference_run_now():
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    from make_san_golden import CASES, load_san, run_case
    san, _ = load_san()
    for case in CASES:
        if case[0] in ("edge_cases_hd6", "two_layer_shared_hd6", "molhiv_hd16_eval", "saturate_hd8"):
            _check_oracle("SAN", run_case(san, *case, dtype=torch.float64), 1e-10, 1e-9)


def _complement(edge_index, batch, num_graphs):
    """Every ordered pair (j, i), j != i, of one graph without a real edge j -> i, by plain enumeration."""
    real = {(int(s), int(d)) for s, d in edge_index.t().tolist()}
    nodes = {}
    for i, g in enumerate(batch.tolist()):
        nodes.setdefault(g, []).append(i)
    return {(j, i) for g in range(num_graphs) for i in nodes.get(g, []) for j in nodes.get(g, [])
            if j != i and (j, i) not in real}


def test_fake_set_is_the_complement():
    # self loops, a duplicate, a one-way edge, an isolated node, a one-node graph
    fix = _load("SAN", "reference_live")
    want = _complement(fix["edge_index"], fix["batch"], fix["num_graphs"])
    ref = {tuple(p) for p in fix["fake_pairs"].t().tolist()}   # negate_edge_index under torch_scatter's scatter_mul
    assert ref == want
    ours = {tuple(p) for p in fake_pairs(fix["edge_index"], fix["batch"], fix["num_graphs"]).t().tolist()}
    assert ours == want
    assert (5, 0) in want and (0, 5) in want       # the isolated node pairs with every other node of its graph
    assert (0, 1) not in want and (1, 0) not in want and (3, 0) not in want and (0, 3) in want   # the one-way edge
    assert not any(p[0] == p[1] for p in want)
    b = san_batch("sbm", [30, 1, 25], 8, 3)
    assert {tuple(p) for p in fake_pairs(b.edge_index, b.batch, 3).t().tolist()} == _complement(b.edge_index, b.batch, 3)


def test_state_dict_matches_reference():
    fix = _load("SAN", "reference_live")
    torch.manual_seed(fix["init_seed"])
    emb = nn.Embedding(1, 56)
    layer = graphgps_b200.SANLayer(0.1, 56, 56, 8, True, emb, 0.2)
    ours = layer.state_dict()
    ref = fix["init_state"]
    assert list(ours.keys()) == list(ref.keys())
    for k, v in ref.items():
        assert tuple(ours[k].shape) == tuple(v.shape), k
        assert torch.equal(ours[k], v), k      # same modules, same draws from the same seed
    layer.load_state_dict(ref, strict=True)


def test_fixture_states_load_strictly():
    for p in sorted(os.listdir(SAN_DIR)):
        fix = _load("SAN", p[:-3])
        cfg = fix["config"]
        emb = nn.Embedding(1, cfg["d"])
        layers = [graphgps_b200.SANLayer(cfg["gamma"], cfg["d"], cfg["d"], cfg["heads"], True, emb)
                  for _ in range(cfg["layers"])]
        mod = layers[0] if cfg["layers"] == 1 else nn.Sequential(*layers)
        mod.load_state_dict(fix["state"], strict=True)


def test_shared_embedding():
    check_shared_embedding("SAN")


@pytest.mark.parametrize("kw", NOT_BUILT)
def test_constructor_not_built(kw):
    check_constructor_not_built("SAN", kw)


def test_constructor_contract():
    emb = nn.Embedding(1, 48)
    with pytest.raises(NotImplementedError):
        graphgps_b200.SANLayer(0.1, 40, 48, 8, True, emb)          # in_dim != out_dim
    with pytest.raises(ValueError):
        graphgps_b200.SANLayer(0.1, 48, 48, 5, True, emb)          # the reference fails at its view
    with pytest.raises(ValueError):
        graphgps_b200.SANLayer(0.1, 48, 48, 8, True, emb, precision="fp16")
    with pytest.raises(NotImplementedError):
        graphgps_b200.SANLayer(0.1, 400, 400, 2, True, nn.Embedding(1, 400))   # head dim 200 > 192
    layer = graphgps_b200.SANLayer(1e-5, 84, 84, 4, True, nn.Embedding(1, 84), 0.2, precision="bf16")
    assert (layer.gamma, layer.p_dropout, layer.num_heads, layer.precision) == (1e-5, 0.2, 4, "bf16")


def test_forward_refuses_cpu_tensors_and_missing_edge_attr():
    layer = graphgps_b200.SANLayer(0.1, 16, 16, 4, True, nn.Embedding(1, 16))
    b = types.SimpleNamespace(x=torch.zeros(3, 16), batch=torch.zeros(3, dtype=torch.int64),
                              edge_index=torch.zeros(2, 0, dtype=torch.int64), edge_attr=torch.zeros(0, 16))
    with pytest.raises(RuntimeError, match="CUDA"):
        layer(b)


def test_abi_plan():
    lib = _lib.load()
    plan = _lib.GpsSanPlan()
    assert lib.gps_san_plan(C.byref(_args("SAN")), C.byref(plan)) == _lib.GPS_OK
    N, E, d = 133, 300, 56
    # saved holds at least Y (5d), E, attn, z1, h1, hid (2d), z2 in fp32
    assert plan.saved_bytes >= 4 * (N * d * 11 + E * d)
    assert plan.bwd_workspace_bytes >= 4 * (N * d * 12 + E * d)
    big = _lib.GpsSanPlan()
    assert lib.gps_san_plan(C.byref(_args("SAN", nmax=133)), C.byref(big)) == _lib.GPS_OK
    assert big.saved_bytes >= plan.saved_bytes       # the bitmap grows with nmax
    drop = _args("SAN")
    drop.dropout = 0.2
    dp = _lib.GpsSanPlan()
    assert lib.gps_san_plan(C.byref(drop), C.byref(dp)) == _lib.GPS_OK
    assert dp.saved_bytes > plan.saved_bytes         # the dropped attention output is kept beside the plain one


@pytest.mark.parametrize("d,heads,rc", [(56, 5, _lib.GPS_ERR_ARG), (0, 1, _lib.GPS_ERR_ARG),
                                        (54, 6, _lib.GPS_ERR_UNSUPPORTED), (400, 2, _lib.GPS_ERR_UNSUPPORTED)])
def test_abi_plan_rejects(d, heads, rc):
    lib = _lib.load()
    plan = _lib.GpsSanPlan()
    assert lib.gps_san_plan(C.byref(_args("SAN", d, heads)), C.byref(plan)) == rc
    assert lib.gps_san_plan(None, C.byref(plan)) == _lib.GPS_ERR_ARG
    bad = _args("SAN")
    bad.nmax = 0
    assert lib.gps_san_plan(C.byref(bad), C.byref(plan)) == _lib.GPS_ERR_ARG


def test_abi_rejects_before_any_cuda_call():
    """Bad or NULL arguments return GPS_ERR_ARG without touching the device (these pointers are never dereferenced)."""
    lib = _lib.load()
    assert lib.gps_san_forward(None, None) == _lib.GPS_ERR_ARG
    assert lib.gps_san_backward(None, None) == _lib.GPS_ERR_ARG
    a = _args("SAN")
    fake = 1 << 40
    a.x, a.edge_attr, a.x_out, a.saved, a.workspace = fake, fake, fake, fake, fake
    a.saved_bytes = a.workspace_bytes = 1 << 40
    assert lib.gps_san_forward(C.byref(a), None) == _lib.GPS_ERR_ARG          # missing parameters
    for f in ("Q", "K", "V", "Q2", "K2", "E", "E2", "O_h", "ffn1", "ffn2"):
        setattr(a, f, _lib.GpsLinear(fake, fake, 0, 0))
    for f in ("bn1", "bn2"):
        setattr(a, f, _lib.GpsBatchNorm(fake, fake, fake, fake, 0, 0, 0))
    assert lib.gps_san_forward(C.byref(a), None) == _lib.GPS_ERR_ARG          # missing fake_edge_emb
    assert "fake_edge_emb" in lib.gps_last_error().decode()
    a.fake_edge_emb = fake
    a.dropout = 1.0
    assert lib.gps_san_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    a.dropout = 0.0
    assert lib.gps_san_backward(C.byref(a), None) == _lib.GPS_ERR_ARG         # no grad_x_out / grad_x
    a.edge_attr = 0
    assert lib.gps_san_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    a.edge_attr, a.x_out = fake, 0
    assert lib.gps_san_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    a.x_out, a.saved_bytes = fake, 16
    assert lib.gps_san_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "saved buffer too small" in lib.gps_last_error().decode()
    # the attention stage
    g = _lib.GpsGraph()
    g.N, g.E, g.B = 10, 0, 1
    ws = lib.gps_san_attention_workspace_bytes(10, 16, 2, 10)
    assert ws > 0
    assert lib.gps_san_attention_forward(None, 2, 8, fake, 80, 0, fake, 0.1, 10, fake, ws, fake, 16, fake,
                                         None) == _lib.GPS_ERR_ARG
    assert lib.gps_san_attention_forward(C.byref(g), 2, 8, fake, 40, 0, fake, 0.1, 10, fake, ws, fake, 16, fake,
                                         None) == _lib.GPS_ERR_ARG   # ld < 5 d
    assert lib.gps_san_attention_forward(C.byref(g), 2, 8, fake, 80, 0, fake, 0.1, 10, fake, ws - 1, fake, 16, fake,
                                         None) == _lib.GPS_ERR_ARG   # workspace too small


def test_install_san_rebinds_stub_module():
    stub = types.ModuleType("graphgps.network.san_transformer")

    class Original:
        pass

    class San2:
        pass

    stub.SANLayer, stub.SAN2Layer = Original, San2
    prev = graphgym.install_san(stub)
    assert prev is Original
    assert stub.SANLayer is graphgps_b200.SANLayer
    assert stub.SAN2Layer is San2
    assert graphgym.install_san(stub) is graphgps_b200.SANLayer
