"""CPU tests of CustomGNN's GatedGCNLayer / GINEConvLayer drop-ins: the float64 restatement against the reference, the
fixtures, state_dict and seeded initial values, the constructor contract, the C ABI's plan and argument checks, and
graphgym.install_custom_gnn."""
import ctypes as C
import glob
import os
import types

import pytest
import torch
import torch.nn as nn

import graphgps_b200
from graphgps_b200 import _lib, graphgym
from custom_gnn_oracle import SanBatch, oracle_layer, run_stack
from util import GOLDEN_DIR

CG_DIR = os.path.join(GOLDEN_DIR, "custom_gnn")
FIXTURES = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(CG_DIR, "*.pt"))
                  if not os.path.basename(p).startswith("reference_live"))


def load(name):
    return torch.load(os.path.join(CG_DIR, name + ".pt"), weights_only=False)


def oracle_stack(cfg):
    return nn.Sequential(*[oracle_layer(cfg["kind"], cfg["d"], cfg["act"] or "relu", cfg["residual"])
                           for _ in range(cfg["layers"])])


def check_oracle(fix, rtol, atol):
    """Runs the float64 restatement on a fixture and compares outputs, every gradient and the buffers after the call."""
    cfg = fix["config"]
    stack = oracle_stack(cfg).double()
    stack.load_state_dict({k: v.double() if v.is_floating_point() else v for k, v in fix["state"].items()}, strict=True)
    stack.train(cfg["training"])
    x = fix["x"].double().clone().requires_grad_(True)
    e = fix["edge_attr"].double().clone().requires_grad_(True)
    ox, oe = run_stack(list(stack), x, e, fix["edge_index"])
    loss = (ox * fix["ct_x"].double()).sum()
    if fix["ct_e"] is not None:
        loss = loss + (oe * fix["ct_e"].double()).sum()
    loss.backward()
    close = lambda a, b: torch.testing.assert_close(a.double(), b.double(), rtol=rtol, atol=atol)  # noqa: E731
    close(ox, fix["out_x"])
    if fix["out_e"] is not None:
        close(oe, fix["out_e"])
    close(x.grad, fix["grad_x"])
    close(e.grad if e.grad is not None else torch.zeros_like(e), fix["grad_edge_attr"])
    for n, p in stack.named_parameters():
        close(p.grad, fix["grad_params"][n])
    state = stack.state_dict()
    for k, v in fix["state_after"].items():
        if v.is_floating_point():
            close(state[k], v)
        else:
            assert int(state[k]) == int(v), k


def test_oracle_equals_reference_live():
    fix = load("reference_live")
    check_oracle(fix, 1e-10, 1e-9)
    check_oracle(fix["gine"], 1e-10, 1e-9)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_equals_fixture(name):
    check_oracle(load(name), 1e-5, 1e-5)   # the fixtures are the reference's fp64 results stored as fp32


def test_fixtures_cover_the_issue_cases():
    cfgs = [load(n)["config"] for n in FIXTURES]
    ds = {c["d"] for c in cfgs}
    assert {108, 138, 166, 208} <= ds and any(d % 2 for d in ds)
    gated = [c for c in cfgs if c["kind"] == "gatedgcn"]
    assert {c["act"] for c in gated} == {"relu", "gelu"}
    assert any(not c["residual"] for c in cfgs) and any(not c["training"] for c in cfgs)
    assert any(c["layers"] >= 3 for c in gated)
    for n in FIXTURES + ["reference_live"]:
        assert os.path.getsize(os.path.join(CG_DIR, n + ".pt")) < 1_000_000, n


def test_edge_case_fixture_shapes():
    f = load("gatedgcn_edge_cases_d20")
    ei, b = f["edge_index"], f["batch"]
    assert (ei[0] == ei[1]).any()                                    # self loop
    pairs = [tuple(p) for p in ei.t().tolist()]
    assert len(pairs) != len(set(pairs))                             # duplicate edge
    assert (torch.bincount(b) == 1).any()                            # one-node graph
    assert set(range(b.numel())) - set(ei.flatten().tolist())        # isolated node
    assert load("gatedgcn_no_edges_d20")["edge_index"].shape[1] == 0


def ours(cfg):
    d = cfg["d"]
    if cfg["kind"] == "gatedgcn":
        return graphgps_b200.GatedGCNLayer(d, d, dropout=0.0, residual=cfg["residual"], act=cfg["act"])
    return graphgps_b200.GINEConvLayer(d, d, dropout=0.0, residual=cfg["residual"])


def test_state_dict_and_init_match_reference():
    fix = load("reference_live")
    d = fix["init_d"]
    for cls, ref in ((lambda: graphgps_b200.GatedGCNLayer(d, d, 0.1, True), fix["init_state"]),
                     (lambda: graphgps_b200.GINEConvLayer(d, d, 0.1, True), fix["init_state_gine"])):
        torch.manual_seed(fix["init_seed"])
        sd = cls().state_dict()
        assert list(sd) == list(ref)
        for k in ref:
            assert torch.equal(sd[k].to(ref[k].dtype), ref[k]), k


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_states_load_strictly(name):
    fix = load(name)
    stack = nn.Sequential(*[ours(fix["config"]) for _ in range(fix["config"]["layers"])])
    stack.load_state_dict(fix["state"], strict=True)


@pytest.mark.parametrize("kw", [dict(in_dim=64, out_dim=32), dict(equivstable_pe=True), dict(act="swish"),
                                dict(in_dim=5000, out_dim=5000)])
def test_gatedgcn_not_built(kw):
    args = dict(in_dim=64, out_dim=64, dropout=0.0, residual=True)
    args.update(kw)
    with pytest.raises(NotImplementedError):
        graphgps_b200.GatedGCNLayer(**args)


def test_constructor_contract():
    with pytest.raises(NotImplementedError):
        graphgps_b200.GINEConvLayer(64, 32, 0.0, True)
    for cls in (graphgps_b200.GatedGCNLayer, graphgps_b200.GINEConvLayer):
        with pytest.raises(ValueError):
            cls(64, 64, 0.0, True, precision="fp16")
        with pytest.raises(ValueError):
            cls(64, 64, 1.0, True)
    layer = graphgps_b200.GatedGCNLayer(138, 138, 0.2, False, act="gelu", precision="bf16")
    assert (layer.act, layer.residual, layer.dropout, layer.precision) == ("gelu", False, 0.2, "bf16")
    with pytest.raises(RuntimeError):   # CPU tensors: no fallback
        layer(SanBatch(torch.zeros(3, 138), torch.zeros(0, 138), torch.zeros(2, 0, dtype=torch.int64),
                       torch.zeros(3, dtype=torch.int64), 1))


def _args(kind=_lib.CUSTOM_GATEDGCN, d=138, N=100, E=300, **kw):
    a = _lib.GpsCustomGnnArgs()
    a.d, a.kind, a.act, a.precision, a.training, a.residual = d, kind, _lib.ACT["relu"], 0, 1, 1
    a.graph.N, a.graph.E, a.graph.B = N, E, 2
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _plan(a):
    p = _lib.GpsCustomGnnPlan()
    assert _lib.load().gps_custom_gnn_plan(C.byref(a), C.byref(p)) == _lib.GPS_OK
    return p


def test_abi_plan_sizes():
    # d = 138 runs at the pitch 144: its weight planes are those of d = 144; its saved state adds the padded inputs
    p138, p144 = _plan(_args(d=138)), _plan(_args(d=144))
    assert p138.wplanes_bytes == p144.wplanes_bytes > 2 * 5 * 144 * 144
    assert p138.saved_bytes > p144.saved_bytes >= 4 * (100 * 4 * 144 + 300 * 144 + 100 * 144)
    assert p138.bwd_workspace_bytes > p144.bwd_workspace_bytes
    # bf16 keeps no lo planes
    assert _plan(_args(d=144, precision=1)).wplanes_bytes < p144.wplanes_bytes
    g = _plan(_args(kind=_lib.CUSTOM_GINE, d=208))
    assert g.wplanes_bytes < p144.wplanes_bytes and g.saved_bytes >= 4 * 3 * 100 * 208
    # more rows, more memory
    assert _plan(_args(N=200, E=600)).saved_bytes > p138.saved_bytes
    for d in (1, 7, 37, 4096):
        _plan(_args(d=d))


@pytest.mark.parametrize("field,value,rc", [("kind", 2, _lib.GPS_ERR_ARG), ("d", 0, _lib.GPS_ERR_ARG),
                                            ("d", 4097, _lib.GPS_ERR_UNSUPPORTED), ("precision", 3, _lib.GPS_ERR_ARG),
                                            ("act", 5, _lib.GPS_ERR_ARG), ("dropout", 1.0, _lib.GPS_ERR_ARG),
                                            ("flags", 1, _lib.GPS_ERR_ARG)])
def test_abi_plan_rejects(field, value, rc):
    lib = _lib.load()
    plan = _lib.GpsCustomGnnPlan()
    assert lib.gps_custom_gnn_plan(None, C.byref(plan)) == _lib.GPS_ERR_ARG
    assert lib.gps_custom_gnn_plan(C.byref(_args(**{field: value})), C.byref(plan)) == rc
    bad = _args()
    bad.graph.N = -1
    assert lib.gps_custom_gnn_plan(C.byref(bad), C.byref(plan)) == _lib.GPS_ERR_ARG


def test_abi_rejects_before_any_cuda_call():
    """Every refusal below happens before the library touches the device (this machine may have none)."""
    lib = _lib.load()
    assert lib.gps_custom_gnn_forward(None, None) == _lib.GPS_ERR_ARG
    assert lib.gps_custom_gnn_backward(None, None) == _lib.GPS_ERR_ARG
    fake = 256   # never dereferenced: each call fails its checks first
    a = _args()
    assert lib.gps_custom_gnn_forward(C.byref(a), None) == _lib.GPS_ERR_ARG          # no x / saved / workspace
    p = _plan(a)
    a.x, a.edge_attr, a.x_out, a.edge_out = fake, fake, fake, fake
    a.saved, a.saved_bytes = fake, p.saved_bytes
    a.workspace, a.workspace_bytes = fake, max(p.fwd_workspace_bytes, p.bwd_workspace_bytes)
    a.wplanes, a.wplanes_bytes = fake, p.wplanes_bytes
    assert lib.gps_custom_gnn_forward(C.byref(a), None) == _lib.GPS_ERR_ARG          # missing parameters
    for f in ("A", "B", "C", "D"):
        setattr(a, f, _lib.GpsLinear(fake, fake, 0, 0))
    a.bn_node_x = a.bn_edge_e = _lib.GpsBatchNorm(fake, fake, fake, fake, 0, 0, 0)
    assert lib.gps_custom_gnn_forward(C.byref(a), None) == _lib.GPS_ERR_ARG          # E is missing
    a.E = _lib.GpsLinear(fake, 0, 0, 0)
    assert lib.gps_custom_gnn_forward(C.byref(a), None) == _lib.GPS_ERR_ARG          # E.bias is missing
    a.E = _lib.GpsLinear(fake, fake, 0, 0)
    a.bn_edge_e = _lib.GpsBatchNorm(fake, fake, 0, fake, 0, 0, 0)
    assert lib.gps_custom_gnn_forward(C.byref(a), None) == _lib.GPS_ERR_ARG          # no running_mean
    a.bn_edge_e = _lib.GpsBatchNorm(fake, fake, fake, fake, 0, 0, 0)
    a.edge_out = 0
    assert lib.gps_custom_gnn_forward(C.byref(a), None) == _lib.GPS_ERR_ARG          # no edge_out
    assert lib.gps_custom_gnn_backward(C.byref(a), None) == _lib.GPS_ERR_ARG         # no grad_x_out / grad_x
    a.saved_bytes -= 256
    a.edge_out = fake
    assert lib.gps_custom_gnn_forward(C.byref(a), None) == _lib.GPS_ERR_ARG          # saved too small
    a.saved_bytes += 256
    a.wplanes_bytes -= 256
    assert lib.gps_custom_gnn_forward(C.byref(a), None) == _lib.GPS_ERR_ARG          # wplanes too small
    g = _args(kind=_lib.CUSTOM_GINE, d=208)
    pg = _plan(g)
    g.x, g.edge_attr, g.x_out = fake, fake, fake
    g.saved, g.saved_bytes, g.workspace, g.workspace_bytes = fake, pg.saved_bytes, fake, pg.fwd_workspace_bytes
    g.wplanes, g.wplanes_bytes = fake, pg.wplanes_bytes
    g.nn0 = _lib.GpsLinear(fake, fake, 0, 0)
    assert lib.gps_custom_gnn_forward(C.byref(g), None) == _lib.GPS_ERR_ARG          # nn.2 is missing
    g.nn2 = _lib.GpsLinear(fake, fake, 0, 0)
    g.edge_attr = 0
    assert lib.gps_custom_gnn_forward(C.byref(g), None) == _lib.GPS_ERR_ARG          # edge_attr with E > 0


def test_install_custom_gnn_on_a_stub():
    stub = types.ModuleType("graphgps.network.custom_gnn")
    stub.GatedGCNLayer, stub.GINEConvLayer = "ref_gated", "ref_gine"
    prev = graphgym.install_custom_gnn(stub)
    assert prev == {"GatedGCNLayer": "ref_gated", "GINEConvLayer": "ref_gine"}
    assert stub.GatedGCNLayer is graphgps_b200.GatedGCNLayer
    assert stub.GINEConvLayer is graphgps_b200.GINEConvLayer
    # CustomGNN's own call: conv_model(dim_in, dim_in, dropout=..., residual=...)
    layer = stub.GINEConvLayer(166, 166, dropout=0.1, residual=True)
    assert isinstance(layer, graphgps_b200.GINEConvLayer) and layer.dim_out == 166
    layer = stub.GatedGCNLayer(138, 138, dropout=0.1, residual=True)
    assert isinstance(layer, graphgps_b200.GatedGCNLayer) and layer.act == "relu"
