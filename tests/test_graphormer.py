"""Graphormer layer, CPU side: the float64 restatement against the reference run verbatim, the parameter container
against the reference's, the constructor contract, the C ABI's plan and argument checks, and install_graphormer."""
import ctypes as C
import os
import types

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib, graphgym
from graphormer_oracle import graphormer_forward
from util import GOLDEN_DIR

GR_DIR = os.path.join(GOLDEN_DIR, "graphormer")


def _load(name):
    return torch.load(os.path.join(GR_DIR, name + ".pt"), weights_only=False)


def test_oracle_equals_reference_live():
    fix = _load("reference_live")
    cfg = fix["config"]
    state = {k: v.double().requires_grad_(True) for k, v in fix["state"].items()}
    x = fix["x"].clone().requires_grad_(True)
    ab = fix["attn_bias"].clone().requires_grad_(True)
    out = graphormer_forward(state, x, fix["batch"], fix["num_graphs"], cfg["heads"], ab)
    assert float((out.detach() - fix["out"]).abs().max()) < 1e-10
    (out * fix["ct"]).sum().backward()
    assert float((x.grad - fix["grad_x"]).abs().max()) < 1e-9
    assert float((ab.grad - fix["grad_attn_bias"]).abs().max()) < 1e-9
    for n, g in fix["grad_params"].items():
        assert float((state[n].grad - g).abs().max()) < 1e-9, n


def test_state_dict_matches_reference():
    fix = _load("reference_live")
    torch.manual_seed(fix["init_seed"])
    layer = graphgps_b200.GraphormerLayer(80, 8, 0.1, 0.1, 0.1)
    ours = layer.state_dict()
    ref = fix["init_state"]
    assert list(ours.keys()) == list(ref.keys())
    for k, v in ref.items():
        assert tuple(ours[k].shape) == tuple(v.shape), k
        assert torch.equal(ours[k], v), k      # same modules, same draws from the same seed
    layer.load_state_dict(fix["init_state"], strict=True)


def test_fixture_states_load_strictly():
    for p in sorted(os.listdir(GR_DIR)):
        fix = _load(p[:-3])
        cfg = fix["config"]
        layer = graphgps_b200.GraphormerLayer(cfg["d"], cfg["heads"], 0.0, 0.0, 0.0)
        layer.load_state_dict(fix["state"], strict=True)


def test_constructor_contract():
    with pytest.raises(ValueError):
        graphgps_b200.GraphormerLayer(80, 7, 0.0, 0.0, 0.0)
    with pytest.raises(ValueError):
        graphgps_b200.GraphormerLayer(80, 8, 0.0, 0.0, 0.0, precision="fp16")
    layer = graphgps_b200.GraphormerLayer(56, 8, 0.2, 0.1, 0.3, precision="bf16")
    assert (layer.p_dropout, layer.p_attn, layer.p_mlp) == (0.2, 0.1, 0.3)
    assert layer.dropout.p == 0.2 and layer.mlp[3].p == 0.3 and layer.mlp[5].p == 0.2
    assert layer.attention.dropout == 0.1


def test_forward_refuses_cpu_tensors():
    layer = graphgps_b200.GraphormerLayer(16, 4, 0.0, 0.0, 0.0)
    b = types.SimpleNamespace(x=torch.zeros(3, 16), batch=torch.zeros(3, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="CUDA"):
        layer(b)


def _args(d=80, heads=8, N=133, B=6):
    a = _lib.GpsGraphormerArgs()
    a.d, a.heads = d, heads
    a.graph.N, a.graph.B = N, B
    return a


def test_abi_plan():
    lib = _lib.load()
    plan = _lib.GpsGraphormerPlan()
    assert lib.gps_graphormer_plan(C.byref(_args()), C.byref(plan)) == _lib.GPS_OK
    N, d = 133, 80
    # saved holds at least h, Y, O, x1, h2, hid, hid_pre (fp32) and the row statistics
    assert plan.saved_bytes >= 4 * (N * d * 9 + 4 * N + N * 8)
    assert plan.bwd_workspace_bytes >= 4 * N * d * 9
    assert plan.fwd_workspace_bytes == 0          # hd 10: the CUDA-core forward, no padded planes
    big = _lib.GpsGraphormerPlan()
    assert lib.gps_graphormer_plan(C.byref(_args(64, 4, 7600, 1)), C.byref(big)) == _lib.GPS_OK
    assert big.fwd_workspace_bytes > 0            # hd 16, one large graph: the wgmma forward's padded planes
    assert big.saved_bytes > plan.saved_bytes
    wg = _lib.GpsGraphormerPlan()   # the hd16_bias_wgmma fixture's batch: two graphs, N >= 64 B
    assert lib.gps_graphormer_plan(C.byref(_args(64, 4, 136, 2)), C.byref(wg)) == _lib.GPS_OK
    assert wg.fwd_workspace_bytes > 0


@pytest.mark.parametrize("d,heads,rc", [(80, 7, _lib.GPS_ERR_ARG), (0, 1, _lib.GPS_ERR_ARG), (78, 6, _lib.GPS_ERR_UNSUPPORTED),
                                        (400, 2, _lib.GPS_ERR_UNSUPPORTED)])
def test_abi_plan_rejects(d, heads, rc):
    lib = _lib.load()
    plan = _lib.GpsGraphormerPlan()
    assert lib.gps_graphormer_plan(C.byref(_args(d, heads)), C.byref(plan)) == rc
    assert lib.gps_graphormer_plan(None, C.byref(plan)) == _lib.GPS_ERR_ARG


def test_abi_rejects_before_any_cuda_call():
    """Bad or NULL arguments return GPS_ERR_ARG without touching the device (these pointers are never dereferenced)."""
    lib = _lib.load()
    assert lib.gps_graphormer_forward(None, None, None) == _lib.GPS_ERR_ARG
    assert lib.gps_graphormer_backward(None, None, None) == _lib.GPS_ERR_ARG
    a = _args()
    fake = 1 << 40
    a.x, a.x_out, a.saved, a.workspace = fake, fake, fake, fake
    a.saved_bytes = a.workspace_bytes = 1 << 40
    # missing parameters
    assert lib.gps_graphormer_forward(C.byref(a), None, None) == _lib.GPS_ERR_ARG
    for f in ("input_norm", "attn_in", "attn_out", "mlp_norm", "mlp_lin1", "mlp_lin2"):
        setattr(a, f, _lib.GpsLinear(fake, fake, 0, 0))
    a.dropout = 1.0
    assert lib.gps_graphormer_forward(C.byref(a), None, None) == _lib.GPS_ERR_ARG
    a.dropout = 0.0
    bad = _lib.GpsAttnBias(fake, 0, 0)
    assert lib.gps_graphormer_forward(C.byref(a), C.byref(bad), None) == _lib.GPS_ERR_ARG
    bad = _lib.GpsAttnBias(0, 30, 0)
    assert lib.gps_graphormer_backward(C.byref(a), C.byref(bad), None) == _lib.GPS_ERR_ARG
    # backward without grad_x_out / grad_x
    assert lib.gps_graphormer_backward(C.byref(a), None, None) == _lib.GPS_ERR_ARG
    a.x_out = 0
    assert lib.gps_graphormer_forward(C.byref(a), None, None) == _lib.GPS_ERR_ARG
    a.x_out, a.saved_bytes = fake, 16
    assert lib.gps_graphormer_forward(C.byref(a), None, None) == _lib.GPS_ERR_ARG
    assert "saved buffer too small" in lib.gps_last_error().decode()


def test_install_graphormer_rebinds_stub_module():
    stub = types.ModuleType("graphgps.network.graphormer")

    class Original:
        pass

    stub.GraphormerLayer = Original
    prev = graphgym.install_graphormer(stub)
    assert prev is Original
    assert stub.GraphormerLayer is graphgps_b200.GraphormerLayer
    assert graphgym.install_graphormer(stub) is graphgps_b200.GraphormerLayer
