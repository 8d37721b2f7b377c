"""The graph-prediction heads, CPU side: the float64 restatement against the reference run verbatim, the state dicts
against the reference's, the constructor contract, CPU refusal, the C ABI's struct layout, plan sizes and argument
checks, and install_graph_heads."""
import ctypes as C
import os
import shutil
import subprocess
import sys
import types

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib, graphgym
from graph_head_oracle import fixture_batch, fixture_ct, oracle
from util import GOLDEN_DIR

GH_DIR = os.path.join(GOLDEN_DIR, "graph_head")
INCLUDE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include")
REF = "/root/reference/graphgps"
FIXTURES = sorted(p[:-3] for p in os.listdir(GH_DIR) if p.endswith(".pt") and p != "reference_live.pt")


def _load(name):
    return torch.load(os.path.join(GH_DIR, name + ".pt"), weights_only=False)


def _head(fix, **kw):
    c = fix["config"]
    if c["kind"] == "san_graph":
        return graphgps_b200.SANGraphHead(c["d"], c["dout"], L=c["L"], graph_pooling=c["pooling"], act=c["act"], **kw)
    return graphgps_b200.GraphormerHead(c["d"], c["dout"], graph_pooling=c["pooling"], **kw)


def test_oracle_equals_reference_live():
    fix = _load("reference_live")
    pred, gx, grads = oracle(fix)
    assert float((pred - fix["pred"]).abs().max()) < 1e-10
    assert float((gx - fix["grad_x"]).abs().max()) < 1e-10
    for k, g in fix["grads"].items():
        assert float((grads[k] - g).abs().max()) < 1e-10, k


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_equals_reference_fixtures(name):
    """Every fp32 fixture (PCQM4Mv2, ZINC, molhiv and molpcba shapes, graph_token under both heads, one-node and empty
    graphs, L = 0 and 3, one graph of 20 000 nodes) against the oracle in float64."""
    fix = _load(name)
    pred, gx, grads = oracle(fix)
    refs = [("pred", pred, fix["pred"])] + [(k, grads[k], g) for k, g in fix["grads"].items()]
    if "grad_x" in fix:
        refs.append(("grad_x", gx, fix["grad_x"]))
    for what, a, r in refs:
        assert float((a - r.double()).abs().max()) <= 1e-5 * max(1.0, float(r.abs().max())), what


def test_fixture_batches_are_what_they_claim():
    c = {n: _load(n) for n in ("edge_cases_L0_add", "one_large_graph", "zinc_graphormer_d80_token")}
    sizes = torch.diff(c["edge_cases_L0_add"]["ptr"])
    assert (sizes == 0).any() and (sizes == 1).any() and int(sizes.max()) > 2 * 64 and int(sizes[-1]) > 0
    assert c["one_large_graph"]["num_graphs"] == 1 and c["one_large_graph"]["x_shape"][0] == 20000
    assert fixture_batch(c["zinc_graphormer_d80_token"]).shape[0] == c["zinc_graphormer_d80_token"]["x_shape"][0]
    assert fixture_ct(c["one_large_graph"]).shape == (1, 1)


def test_graphormer_empty_graph_predicts_the_bias():
    """The reference pools after the LayerNorm, so an empty graph's pooled row is zero and its pred is layers.0.bias;
    ln gets no gradient from it."""
    fix = _load("graphormer_edge_d76_token")
    empty = torch.diff(fix["ptr"]) == 0
    assert fix["config"]["d"] % 8 == 4 and int(empty.sum()) == 2 and not bool(empty[-1])
    bias = fix["state"]["layers.0.bias"]
    assert torch.allclose(fix["pred"][empty], bias.expand(2, -1), rtol=0, atol=1e-7)


def test_state_dict_matches_reference():
    fix = _load("reference_live")
    torch.manual_seed(fix["init_seed"])
    ours = graphgps_b200.SANGraphHead(304, 1).state_dict()
    assert list(ours) == list(fix["init_state"]) == [f"FC_layers.{l}.{p}" for l in range(3) for p in ("weight", "bias")]
    for k, v in fix["init_state"].items():
        assert torch.equal(ours[k], v), k   # nn.Linear's draws from the same seed, in the same order
    torch.manual_seed(fix["init_seed"])
    ours = graphgps_b200.GraphormerHead(80, 1).state_dict()
    assert list(ours) == list(fix["init_state_graphormer"]) == ["ln.weight", "ln.bias", "layers.0.weight",
                                                                 "layers.0.bias"]
    for k, v in fix["init_state_graphormer"].items():
        assert torch.equal(ours[k], v), k


def test_fixture_states_load_strictly():
    for name in FIXTURES + ["reference_live"]:
        fix = _load(name)
        _head(fix).load_state_dict(fix["state"], strict=True)


def test_loads_reference_head_weights_strictly():
    if not os.path.isdir(REF):
        pytest.skip("reference checkout not available")
    sys.path.insert(0, GOLDEN_DIR)
    try:
        from make_graph_head_golden import build_head, load_heads
    finally:
        sys.path.pop(0)
    saved = {k: v for k, v in sys.modules.items() if k.startswith("torch_geometric")}
    try:
        classes = load_heads(REF)
        for ours, args in ((graphgps_b200.SANGraphHead(72, 1), ("san_graph", 72, 1, 2, "mean", "relu")),
                           (graphgps_b200.SANGraphHead(304, 128, L=3), ("san_graph", 304, 128, 3, "add", "gelu")),
                           (graphgps_b200.GraphormerHead(80, 1), ("graphormer_graph", 80, 1, 0, "graph_token", "relu"))):
            ref = build_head(classes, *args)
            ours.load_state_dict(ref.state_dict(), strict=True)
            assert list(ours.state_dict()) == list(ref.state_dict())
    finally:   # the generator's PyG stubs must not leak into the other tests of the session
        for k in [k for k in sys.modules if k.startswith("torch_geometric")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_constructor_contract():
    h = graphgps_b200.SANGraphHead(56, 1)
    assert [tuple(m.weight.shape) for m in h.FC_layers] == [(28, 56), (14, 28), (1, 14)]
    assert [tuple(m.weight.shape) for m in graphgps_b200.SANGraphHead(24, 5, L=0).FC_layers] == [(5, 24)]
    assert graphgps_b200.SANGraphHead(8, 1, L=3).FC_layers[3].weight.shape == (1, 1)
    for kw in (dict(graph_pooling="max"), dict(graph_pooling="sum"), dict(act="elu"), dict(L=4)):
        with pytest.raises(NotImplementedError):
            graphgps_b200.SANGraphHead(8, 1, **kw)   # L = 4 leaves 8 // 16 = 0 columns
    for dims in ((4097, 1), (64, 4097), (0, 1)):
        with pytest.raises(NotImplementedError):
            graphgps_b200.SANGraphHead(*dims)
    with pytest.raises(ValueError):
        graphgps_b200.SANGraphHead(64, 1, precision="fp16")
    for pool in ("mean", "add", "max"):
        with pytest.raises(NotImplementedError):
            graphgps_b200.GraphormerHead(80, 1, graph_pooling=pool)
    with pytest.raises(NotImplementedError):
        graphgps_b200.GraphormerHead(78, 1)   # the Graphormer layer's dim_in % 4 == 0
    assert graphgps_b200.GraphormerHead(76, 3).layers[0].weight.shape == (3, 76)


def test_forward_refuses_cpu_tensors():
    b = types.SimpleNamespace(x=torch.randn(4, 8), edge_index=torch.zeros(2, 0, dtype=torch.int64),
                              batch=torch.zeros(4, dtype=torch.int64), num_graphs=1, y=torch.zeros(1))
    for h in (graphgps_b200.SANGraphHead(8, 1), graphgps_b200.GraphormerHead(8, 1)):
        with pytest.raises(RuntimeError, match="CUDA"):
            h(b)


def test_struct_layout_matches_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    structs = (_lib.GpsGraphHeadArgs, _lib.GpsGraphHeadPlan)
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "gps_b200.h"', "int main(void) {",
             '  printf("MAX_L %d\\n", GPS_GRAPH_HEAD_MAX_L);',
             '  printf("POOL %d %d %d\\n", GPS_POOL_MEAN, GPS_POOL_ADD, GPS_POOL_GRAPH_TOKEN);',
             '  printf("KIND %d %d\\n", GPS_GRAPH_HEAD_SAN, GPS_GRAPH_HEAD_GRAPHORMER);']
    for s in structs:
        t = s.__name__
        lines.append(f'  printf("{t} %zu\\n", sizeof({t}));')
        lines += [f'  printf("{t}.{f} %zu\\n", offsetof({t}, {f}));' for f, _ in s._fields_]
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines) + "\n")
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe)], check=True)
    out = {}
    for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines():
        k, *v = line.split()
        out[k] = [int(u) for u in v]
    assert out["MAX_L"] == [_lib.GRAPH_HEAD_MAX_L]
    assert out["POOL"] == [_lib.POOLING[p] for p in ("mean", "add", "graph_token")]
    assert out["KIND"] == [_lib.GRAPH_HEAD[k] for k in ("san_graph", "graphormer_graph")]
    for s in structs:
        t = s.__name__
        assert C.sizeof(s) == out[t][0]
        for f, _ in s._fields_:
            assert getattr(s, f).offset == out[f"{t}.{f}"][0], f


def _args(kind=0, pooling=0, act=0, L=2, d=304, dout=1, N=6581, B=256, precision=0):
    a = _lib.GpsGraphHeadArgs()
    a.kind, a.pooling, a.act, a.L, a.dim_in, a.dim_out, a.precision = kind, pooling, act, L, d, dout, precision
    a.graph.N, a.graph.B = N, B
    return a


def _plan(**kw):
    plan = _lib.GpsGraphHeadPlan()
    rc = _lib.load().gps_graph_head_plan(C.byref(_args(**kw)), C.byref(plan))
    return rc, plan


def test_abi_plan():
    rc, p = _plan()
    assert rc == _lib.GPS_OK
    # padded weights 304x152, 152x80, 80x8 (+ planes) and the pooled / hidden rows of 256 graphs
    assert p.saved_bytes >= 4 * (304 * 152 + 152 * 80 + 80 * 8 + 256 * (304 + 152 + 80))
    assert p.fwd_workspace_bytes >= 4 * 2 * 103 * 304    # the pooling partials of 103 chunks of 64 rows
    assert p.bwd_workspace_bytes >= 4 * (304 * 152 + 152 * 80 + 80 * 8)
    rc, tok = _plan(pooling=2)
    assert rc == _lib.GPS_OK and tok.fwd_workspace_bytes < p.fwd_workspace_bytes   # graph_token: no partials
    rc, bf = _plan(precision=1)
    assert rc == _lib.GPS_OK and bf.saved_bytes < p.saved_bytes                    # no lo planes
    rc, gl = _plan(act=1)
    assert rc == _lib.GPS_OK and gl.saved_bytes > p.saved_bytes                    # GELU keeps pre-activations
    rc, gr = _plan(kind=1, pooling=2, L=0, d=80)
    assert rc == _lib.GPS_OK and gr.bwd_workspace_bytes >= 4 * 2 * 132 * 80        # LayerNorm partials


@pytest.mark.parametrize("kw,rc", [
    (dict(d=0), _lib.GPS_ERR_ARG), (dict(dout=0), _lib.GPS_ERR_ARG), (dict(d=4097), _lib.GPS_ERR_UNSUPPORTED),
    (dict(dout=4097), _lib.GPS_ERR_UNSUPPORTED), (dict(precision=2), _lib.GPS_ERR_ARG), (dict(kind=2), _lib.GPS_ERR_ARG),
    (dict(L=-1), _lib.GPS_ERR_ARG), (dict(L=9), _lib.GPS_ERR_UNSUPPORTED), (dict(L=13, d=4096), _lib.GPS_ERR_UNSUPPORTED),
    (dict(pooling=3), _lib.GPS_ERR_UNSUPPORTED), (dict(act=2), _lib.GPS_ERR_UNSUPPORTED),
    (dict(kind=1, pooling=0, L=0, d=80), _lib.GPS_ERR_UNSUPPORTED), (dict(kind=1, pooling=2, L=1, d=80), _lib.GPS_ERR_ARG),
    (dict(kind=1, pooling=2, L=0, d=78), _lib.GPS_ERR_UNSUPPORTED), (dict(N=-1), _lib.GPS_ERR_ARG)])
def test_abi_plan_rejects(kw, rc):
    assert _plan(**kw)[0] == rc
    assert _lib.load().gps_graph_head_plan(None, C.byref(_lib.GpsGraphHeadPlan())) == _lib.GPS_ERR_ARG


def test_abi_rejects_before_any_cuda_call():
    """Bad or NULL arguments return GPS_ERR_ARG without touching the device (these pointers are never dereferenced)."""
    lib = _lib.load()
    fake = 1 << 40
    assert lib.gps_graph_head_forward(None, None) == _lib.GPS_ERR_ARG
    assert lib.gps_graph_head_backward(None, None) == _lib.GPS_ERR_ARG
    a = _args()
    assert lib.gps_graph_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # no saved / workspace
    a.saved, a.saved_bytes, a.workspace, a.workspace_bytes = fake, 16, fake, 1 << 30
    assert lib.gps_graph_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "saved buffer too small" in lib.gps_last_error().decode()
    a.saved_bytes = 1 << 30
    assert lib.gps_graph_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # no graph_ptr
    assert "graph_ptr" in lib.gps_last_error().decode()
    a.graph.graph_ptr = fake
    assert lib.gps_graph_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # no weights
    assert "fc[0]" in lib.gps_last_error().decode()
    for l in range(3):
        a.fc[l].weight = a.fc[l].bias = fake
    assert lib.gps_graph_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # no x
    assert "x is required" in lib.gps_last_error().decode()
    a.x = fake
    assert lib.gps_graph_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # no pred
    assert lib.gps_graph_head_backward(C.byref(a), None) == _lib.GPS_ERR_ARG   # no grad_pred
    a.grad_pred = fake
    assert lib.gps_graph_head_backward(C.byref(a), None) == _lib.GPS_ERR_ARG   # no grad_x
    assert "grad_x" in lib.gps_last_error().decode()
    a.flags = 1
    assert lib.gps_graph_head_backward(C.byref(a), None) == _lib.GPS_ERR_ARG
    a.flags, a.workspace_bytes = 0, 64
    assert lib.gps_graph_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "workspace too small" in lib.gps_last_error().decode()
    g = _args(kind=1, pooling=2, L=0, d=80)
    g.saved, g.saved_bytes, g.workspace, g.workspace_bytes = fake, 1 << 30, fake, 1 << 30
    g.graph.graph_ptr = g.fc[0].weight = g.fc[0].bias = g.x = g.pred = fake
    assert lib.gps_graph_head_forward(C.byref(g), None) == _lib.GPS_ERR_ARG    # no LayerNorm parameters
    assert "ln" in lib.gps_last_error().decode()


def test_pool_stages_reject_before_any_cuda_call():
    lib = _lib.load()
    fake = 1 << 40
    g = _lib.GpsGraph(N=300, E=0, B=4)
    assert lib.gps_graph_pool_forward(None, 0, fake, 8, fake, 8, fake, 1 << 20, None) == _lib.GPS_ERR_ARG
    assert lib.gps_graph_pool_forward(C.byref(g), 0, fake, 8, fake, 8, fake, 1 << 20, None) == _lib.GPS_ERR_ARG
    g.graph_ptr = fake
    assert lib.gps_graph_pool_forward(C.byref(g), 3, fake, 8, fake, 8, fake, 1 << 20, None) == _lib.GPS_ERR_UNSUPPORTED
    assert lib.gps_graph_pool_forward(C.byref(g), 0, fake, 8, fake, 7, fake, 1 << 20, None) == _lib.GPS_ERR_ARG
    # mean / add: 2 x 5 chunks x 8 columns of float partials
    assert lib.gps_graph_pool_forward(C.byref(g), 1, fake, 8, fake, 8, fake, 319, None) == _lib.GPS_ERR_ARG
    assert "workspace too small" in lib.gps_last_error().decode()
    assert lib.gps_graph_pool_forward(C.byref(g), 0, 0, 8, fake, 8, fake, 320, None) == _lib.GPS_ERR_ARG
    assert lib.gps_graph_pool_backward(C.byref(g), 0, fake, 7, 8, fake, None) == _lib.GPS_ERR_ARG
    assert lib.gps_graph_pool_backward(C.byref(g), 0, fake, 8, 8, 0, None) == _lib.GPS_ERR_ARG
    assert lib.gps_graph_pool_backward(C.byref(g), 5, fake, 8, 8, fake, None) == _lib.GPS_ERR_UNSUPPORTED
    assert lib.gps_graph_pool_forward(C.byref(g), 0, fake, 8, fake, 8, fake + 8, 1 << 20, None) == _lib.GPS_ERR_ARG
    assert "16-byte aligned" in lib.gps_last_error().decode()
    g.B = 0
    assert lib.gps_graph_pool_backward(C.byref(g), 0, fake, 8, 8, fake, None) == _lib.GPS_ERR_ARG   # rows in no graph


def test_install_graph_heads_sets_registry():
    reg = types.SimpleNamespace(head_dict={"san_graph": "original", "default": "gnn"})
    cfg = types.SimpleNamespace(model=types.SimpleNamespace(graph_pooling="add"), gnn=types.SimpleNamespace(act="gelu"))
    stub = types.ModuleType("torch_geometric.graphgym.config")
    stub.cfg = cfg
    saved = sys.modules.get("torch_geometric.graphgym.config")
    sys.modules["torch_geometric.graphgym.config"] = stub
    try:
        assert graphgym.install_graph_heads(reg) == {"san_graph": "original", "graphormer_graph": None}
        san, gr = reg.head_dict["san_graph"], reg.head_dict["graphormer_graph"]
        assert reg.head_dict["default"] == "gnn"
        h = san(304, 1)   # the reference's (dim_in, dim_out) constructor
        assert isinstance(h, graphgps_b200.SANGraphHead) and (h.graph_pooling, h.act, h.L) == ("add", "gelu", 2)
        cfg.model.graph_pooling = "max"
        with pytest.raises(NotImplementedError):
            san(304, 1)
        with pytest.raises(NotImplementedError):
            gr(80, 1)
        cfg.model.graph_pooling = "graph_token"
        assert isinstance(gr(80, 1), graphgps_b200.GraphormerHead)
        assert graphgym.install_graph_heads(reg) == {"san_graph": san, "graphormer_graph": gr}
    finally:
        if saved is None:
            del sys.modules["torch_geometric.graphgym.config"]
        else:
            sys.modules["torch_geometric.graphgym.config"] = saved
