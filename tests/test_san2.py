"""SAN2 layer, CPU side: the float64 restatement against the reference run verbatim, the parameter container against
the reference's, the constructor contract, the C ABI's plan and argument checks for variant 1, and install_san2.  The
checks SANLayer runs as well are in tests/san_harness.py."""
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
from san_oracle import fake_pairs

SAN2_DIR = VARIANTS["SAN2"].dir
HAVE_REFERENCE = os.path.isfile("/root/reference/graphgps/layer/san2_layer.py")


def test_oracle_equals_reference_live():
    _check_oracle("SAN2", _load("SAN2", "reference_live"), 1e-10, 1e-9)


@pytest.mark.skipif(not HAVE_REFERENCE, reason="the reference tree is not present; reference_live pins the oracle")
def test_oracle_equals_reference_run_now():
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    from make_san2_golden import CASES, load_san2, run_case
    san2, _ = load_san2()
    for case in CASES:
        if case[0] in ("edge_cases_hd6", "two_layer_shared_hd6", "molhiv_hd16_eval", "no_clamp_hd8", "gamma_zero_hd7"):
            _check_oracle("SAN2", run_case(san2, *case, dtype=torch.float64), 1e-10, 1e-9)


def test_fixtures_cover_the_cases():
    live = _load("SAN2", "reference_live")
    assert live["state"]["0.attention.gamma"].dtype == torch.float64
    assert live["grad_params"]["0.attention.gamma"].dtype == torch.float64
    clamp = _load("SAN2", "no_clamp_hd8")
    assert clamp["max_score"] > 88          # exp would overflow in fp32 without the running max
    zero = _load("SAN2", "gamma_zero_hd7")
    assert float(zero["state"]["attention.gamma"]) == 0.0
    assert abs(float(zero["grad_params"]["attention.gamma"])) > 1e-6   # the fake part has weight 0, its gradient not
    edge = _load("SAN2", "edge_cases_hd6")
    fake = fake_pairs(edge["edge_index"], edge["batch"], edge["num_graphs"])
    ei = edge["edge_index"]
    assert not bool((fake[1] >= 11).any() & (fake[1] <= 13).any())   # the complete graph has no fake pair
    assert not bool((ei[1] == 4).any()) and not bool((ei[1] == 14).any())   # nodes without in-edges
    assert bool((ei[0] == ei[1]).any())                                     # self loops are real edges


def test_state_dict_matches_reference():
    fix = _load("SAN2", "reference_live")
    torch.manual_seed(fix["init_seed"])
    emb = nn.Embedding(1, 56)
    layer = graphgps_b200.SAN2Layer(0.1, 56, 56, 8, True, emb, 0.2)
    ours = layer.state_dict()
    ref = fix["init_state"]
    assert list(ours.keys()) == list(ref.keys())
    assert next(k for k in ours if k.startswith("attention.")) == "attention.gamma"
    for k, v in ref.items():
        assert ours[k].dtype == v.dtype, k
        assert tuple(ours[k].shape) == tuple(v.shape), k
        assert torch.equal(ours[k], v), k      # same modules, same draws from the same seed
    assert ours["attention.gamma"].dtype == torch.float64 and float(ours["attention.gamma"]) == 0.5
    layer.load_state_dict(ref, strict=True)


def test_fixture_states_load_strictly():
    for p in sorted(os.listdir(SAN2_DIR)):
        fix = _load("SAN2", p[:-3])
        cfg = fix["config"]
        emb = nn.Embedding(1, cfg["d"])
        layers = [graphgps_b200.SAN2Layer(0.1, cfg["d"], cfg["d"], cfg["heads"], True, emb)
                  for _ in range(cfg["layers"])]
        mod = layers[0] if cfg["layers"] == 1 else nn.Sequential(*layers)
        mod.load_state_dict(fix["state"], strict=True)
        g = layers[0].attention.gamma
        assert g.dtype == torch.float64 and float(g.detach()) == cfg["gamma"]


def test_gamma_argument_is_ignored():
    torch.manual_seed(3)
    a = graphgps_b200.SAN2Layer(0.1, 24, 24, 4, True, nn.Embedding(1, 24))
    torch.manual_seed(3)
    b = graphgps_b200.SAN2Layer(7.0, 24, 24, 4, True, nn.Embedding(1, 24))
    for (ka, va), (kb, vb) in zip(a.state_dict().items(), b.state_dict().items()):
        assert ka == kb and torch.equal(va, vb), ka
    assert float(a.attention.gamma) == 0.5 and a.attention.gamma.requires_grad
    assert not hasattr(a, "gamma")


def test_shared_embedding():
    check_shared_embedding("SAN2")
    a = graphgps_b200.SAN2Layer(0.1, 24, 24, 4, True, nn.Embedding(1, 24))
    b = graphgps_b200.SAN2Layer(0.1, 24, 24, 4, True, a.attention.fake_edge_emb)
    assert a.attention.gamma is not b.attention.gamma


@pytest.mark.parametrize("kw", NOT_BUILT)
def test_constructor_not_built(kw):
    check_constructor_not_built("SAN2", kw, match="SAN2Layer")


def test_constructor_contract():
    emb = nn.Embedding(1, 48)
    with pytest.raises(NotImplementedError):
        graphgps_b200.SAN2Layer(0.1, 40, 48, 8, True, emb)          # in_dim != out_dim
    with pytest.raises(ValueError):
        graphgps_b200.SAN2Layer(0.1, 48, 48, 5, True, emb)          # the reference fails at its view
    with pytest.raises(ValueError):
        graphgps_b200.SAN2Layer(0.1, 48, 48, 8, True, emb, precision="fp16")
    with pytest.raises(NotImplementedError):
        graphgps_b200.SAN2Layer(0.1, 400, 400, 2, True, nn.Embedding(1, 400))   # head dim 200 > 192
    layer = graphgps_b200.SAN2Layer(0.1, 84, 84, 4, True, nn.Embedding(1, 84), 0.2, precision="bf16")
    assert (layer.p_dropout, layer.num_heads, layer.precision) == (0.2, 4, "bf16")
    assert repr(layer).startswith("SAN2Layer(")


def test_non_float64_gamma_is_refused():
    layer = graphgps_b200.SAN2Layer(0.1, 16, 16, 4, True, nn.Embedding(1, 16))
    b = types.SimpleNamespace(x=torch.zeros(3, 16), batch=torch.zeros(3, dtype=torch.int64),
                              edge_index=torch.zeros(2, 0, dtype=torch.int64), edge_attr=torch.zeros(0, 16))
    with pytest.raises(RuntimeError, match="CUDA"):
        layer(b)                       # float64 gamma: on to the CUDA check of batch.x
    layer.attention.gamma.data = layer.attention.gamma.data.float()
    with pytest.raises(TypeError, match="attention.gamma"):
        layer(b)
    layer.float()                      # as a model-wide .float() would leave it
    with pytest.raises(TypeError, match="float64"):
        layer(b)


def _round(n):
    return (n + 255) // 256 * 256


def test_abi_plan_variant1():
    lib = _lib.load()
    N, E, d, H = 133, 300, 56, 8
    p0, p1 = _lib.GpsSanPlan(), _lib.GpsSanPlan()
    assert lib.gps_san_plan(C.byref(_args("SAN")), C.byref(p0)) == _lib.GPS_OK
    assert lib.gps_san_plan(C.byref(_args("SAN2")), C.byref(p1)) == _lib.GPS_OK
    # R and F [N, d] and the two log-sum-exps [2, N, H] in place of rz [N, H]
    assert p1.saved_bytes - p0.saved_bytes == 2 * _round(4 * N * d) + _round(8 * N * H) - _round(4 * N * H)
    assert p1.bwd_workspace_bytes - p0.bwd_workspace_bytes == _round(8 * N * H) - _round(4 * N * H)   # Dr and Df
    assert p1.fwd_workspace_bytes == p0.fwd_workspace_bytes
    assert p1.saved_bytes >= 4 * (N * d * 13 + E * d)
    z = _lib.GpsSanPlan()                  # a zero-filled args struct is variant 0, as before
    a = _args("SAN")
    a.gamma = -1.0
    assert lib.gps_san_plan(C.byref(a), C.byref(z)) == _lib.GPS_ERR_ARG
    a.variant = 1                          # the gamma field is not read by SAN2
    assert lib.gps_san_plan(C.byref(a), C.byref(z)) == _lib.GPS_OK
    assert z.saved_bytes == p1.saved_bytes


@pytest.mark.parametrize("variant", [2, -1, 7])
def test_abi_unknown_variant(variant):
    lib = _lib.load()
    plan = _lib.GpsSanPlan()
    assert lib.gps_san_plan(C.byref(_args(variant)), C.byref(plan)) == _lib.GPS_ERR_UNSUPPORTED
    assert "variant" in lib.gps_last_error().decode()


def test_abi_rejects_before_any_cuda_call():
    """Bad or NULL arguments of variant 1 return before touching the device (these pointers are never dereferenced)."""
    lib = _lib.load()
    a = _args("SAN2")
    fake = 1 << 40
    a.x, a.edge_attr, a.x_out, a.saved, a.workspace = fake, fake, fake, fake, fake
    a.grad_x_out, a.grad_x = fake, fake
    a.saved_bytes = a.workspace_bytes = 1 << 40
    for f in ("Q", "K", "V", "Q2", "K2", "E", "E2", "O_h", "ffn1", "ffn2"):
        setattr(a, f, _lib.GpsLinear(fake, fake, 0, 0))
    for f in ("bn1", "bn2"):
        setattr(a, f, _lib.GpsBatchNorm(fake, fake, fake, fake, 0, 0, 0))
    a.fake_edge_emb = fake
    for fn in (lib.gps_san_forward, lib.gps_san_backward):
        assert fn(C.byref(a), None) == _lib.GPS_ERR_ARG                # NULL gamma_param
        assert "attention.gamma" in lib.gps_last_error().decode()
    a.gamma_param = fake
    a.variant = 3
    for fn in (lib.gps_san_forward, lib.gps_san_backward):
        assert fn(C.byref(a), None) == _lib.GPS_ERR_UNSUPPORTED
    a.variant = 1
    a.saved_bytes = 16
    assert lib.gps_san_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "saved buffer too small" in lib.gps_last_error().decode()
    # the attention stage
    g = _lib.GpsGraph()
    g.N, g.E, g.B = 10, 0, 1
    ws = lib.gps_san2_attention_workspace_bytes(10, 16, 2, 10)
    assert (lib.gps_san2_attention_workspace_bytes(1000, 16, 2, 100) - lib.gps_san_attention_workspace_bytes(1000, 16, 2, 100)
            == _round(2 * 1000 * 2 * 4) - _round(1000 * 2 * 4))   # Dr and Df in place of D
    args = [C.byref(g), 2, 8, fake, 80, 0, fake, fake, 10, fake, ws, fake, 16, fake, fake, fake, None]
    for i, bad in ((0, None), (4, 40), (7, None), (10, ws - 1), (13, None)):   # graph, ld < 5 d, gamma, ws, R
        b = list(args)
        b[i] = bad
        assert lib.gps_san2_attention_forward(*b) == _lib.GPS_ERR_ARG, i
    bwd = [C.byref(g), 2, 8, fake, 80, 0, fake, fake, 10, fake, ws, fake, fake, fake, fake, 16, fake, 80, 0, fake,
           None, None]
    assert lib.gps_san2_attention_backward(*bwd) == _lib.GPS_ERR_ARG       # NULL dgamma
    bwd[7] = None
    assert lib.gps_san2_attention_backward(*bwd) == _lib.GPS_ERR_ARG       # NULL gamma


def test_install_san2_rebinds_stub_module():
    stub = types.ModuleType("graphgps.network.san_transformer")

    class San1:
        pass

    class Original:
        pass

    stub.SANLayer, stub.SAN2Layer = San1, Original
    prev = graphgym.install_san2(stub)
    assert prev is Original
    assert stub.SAN2Layer is graphgps_b200.SAN2Layer
    assert stub.SANLayer is San1
    assert graphgym.install_san2(stub) is graphgps_b200.SAN2Layer
    stub2 = types.ModuleType("graphgps.network.san_transformer")
    stub2.SANLayer, stub2.SAN2Layer = San1, Original
    graphgym.install_san(stub2)
    assert stub2.SAN2Layer is Original and stub2.SANLayer is graphgps_b200.SANLayer
