"""Graphormer's attention-bias encoder, CPU side: the float64 restatement against the reference run verbatim, the
parameter container against the reference's, the constructor contract, CPU refusal, the C ABI's struct layout, plan and
argument checks, and install_graphormer_bias."""
import ctypes as C
import os
import shutil
import subprocess
import types

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib, graphgym
from graphormer_bias_oracle import bias_forward, bias_inputs
from util import GOLDEN_DIR

GB_DIR = os.path.join(GOLDEN_DIR, "graphormer_bias")
INCLUDE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include")


def _load(name):
    return torch.load(os.path.join(GB_DIR, name + ".pt"), weights_only=False)


def test_oracle_equals_reference_live():
    fix = _load("reference_live")
    cfg = fix["config"]
    state = {k: v.double().requires_grad_(True) for k, v in fix["state"].items()}
    st, gi, batch, spt = bias_inputs(fix)
    assert spt is not None and cfg["use_graph_token"]
    out = bias_forward(state, st, gi, batch, cfg["heads"], spt, cfg["use_graph_token"])
    assert out.shape == fix["out"].shape
    assert float((out.detach() - fix["out"]).abs().max()) < 1e-10
    (out * fix["ct"]).sum().backward()
    for n, g in fix["grad_params"].items():
        assert float((state[n].grad - g).abs().max()) < 1e-10, n


def test_oracle_equals_reference_fixtures():
    """Every fp32 fixture (no token, no shortest_path_types, unreachable pairs, truncated paths, one-node graphs, the
    largest graph not first) against the oracle in float64."""
    for p in sorted(os.listdir(GB_DIR)):
        fix = _load(p[:-3])
        cfg = fix["config"]
        state = {k: v.double().requires_grad_(True) for k, v in fix["state"].items()}
        st, gi, batch, spt = bias_inputs(fix)
        out = bias_forward(state, st, gi, batch, cfg["heads"], spt, cfg["use_graph_token"])
        assert out.shape == fix["out"].shape, p
        assert float((out.detach() - fix["out"].double()).abs().max()) < 1e-5, p
        (out * fix["ct"].double()).sum().backward()
        for n, g in fix["grad_params"].items():
            if g is None:   # a parameter the output does not read (the edge tables without shortest_path_types)
                assert spt is None and state[n].grad is None, (p, n)
            else:
                assert float((state[n].grad - g.double()).abs().max()) <= 1e-5 * max(1.0, float(g.abs().max())), (p, n)


def test_state_dict_matches_reference():
    fix = _load("reference_live")
    torch.manual_seed(fix["init_seed"])
    for ref in (fix["init_state"], fix["init_state_no_token"]):
        ours = (graphgps_b200.BiasEncoder(8, 20, 4, True) if "graph_token" in ref else
                graphgps_b200.BiasEncoder(4, 20, 0, False)).state_dict()
        assert list(ours.keys()) == list(ref.keys())
        for k, v in ref.items():
            assert tuple(ours[k].shape) == tuple(v.shape), k
            assert torch.equal(ours[k], v), k      # same modules, same draws from the same seed


def test_fixture_states_load_strictly():
    for p in sorted(os.listdir(GB_DIR)):
        cfg = _load(p[:-3])["config"]
        enc = graphgps_b200.BiasEncoder(cfg["heads"], cfg["num_spatial_types"], cfg["num_edge_types"],
                                        cfg["use_graph_token"])
        enc.load_state_dict(_load(p[:-3])["state"], strict=True)


def test_constructor_contract():
    enc = graphgps_b200.BiasEncoder(8, 20, 4)
    assert enc.use_graph_token and enc.num_heads == 8
    assert tuple(enc.spatial_encoder.weight.shape) == (21, 8)
    assert tuple(enc.edge_dis_encoder.weight.shape) == (20 * 8 * 8, 1)
    assert tuple(enc.edge_encoder.weight.shape) == (4, 8)
    assert tuple(enc.graph_token.shape) == (1, 8, 1)
    enc = graphgps_b200.BiasEncoder(4, 20, 0, use_graph_token=False)   # the actor / webkb / wn configs
    assert not hasattr(enc, "graph_token")
    assert tuple(enc.edge_encoder.weight.shape) == (0, 4)
    assert sorted(n for n, _ in enc.named_parameters()) == ["edge_dis_encoder.weight", "edge_encoder.weight",
                                                             "spatial_encoder.weight"]


def _cpu_batch():
    n = 3
    i = torch.arange(n).repeat_interleave(n)
    j = torch.arange(n).repeat(n)
    return types.SimpleNamespace(spatial_types=(i - j).abs(), graph_index=torch.stack([i, j]),
                                 batch=torch.zeros(n, dtype=torch.int64))


def test_forward_refuses_cpu_tensors():
    enc = graphgps_b200.BiasEncoder(4, 20, 0, False)
    with pytest.raises(RuntimeError, match="CUDA"):
        enc(_cpu_batch())


def test_missing_spatial_types_raises_attribute_error():
    enc = graphgps_b200.BiasEncoder(4, 20, 0, False)
    b = _cpu_batch()
    del b.spatial_types
    with pytest.raises(AttributeError):
        enc(b)


def test_struct_layout_matches_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "gps_b200.h"', "int main(void) {"]
    for s in (_lib.GpsGraphormerBiasArgs, _lib.GpsGraphormerBiasPlan):
        t = s.__name__
        lines.append(f'  printf("{t} %zu\\n", sizeof({t}));')
        lines += [f'  printf("{t}.{f} %zu\\n", offsetof({t}, {f}));' for f, _ in s._fields_]
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines) + "\n")
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe)], check=True)
    out = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True,
                                                        text=True).stdout.splitlines())
    for s in (_lib.GpsGraphormerBiasArgs, _lib.GpsGraphormerBiasPlan):
        t = s.__name__
        assert C.sizeof(s) == int(out[t])
        for f, _ in s._fields_:
            assert getattr(s, f).offset == int(out[f"{t}.{f}"]), f


def _args(P=3151, B=6, nmax=30, H=8, S=20, T=4, token=1, edges=True):
    a = _lib.GpsGraphormerBiasArgs()
    a.num_pairs, a.num_graphs, a.nmax, a.heads = P, B, nmax, H
    a.num_spatial_types, a.num_edge_types, a.use_graph_token = S, T, token
    if edges:
        a.shortest_path_types = 1 << 40   # only its NULL-ness is read by the plan
    return a


def test_abi_plan():
    lib = _lib.load()
    plan = _lib.GpsGraphormerBiasPlan()
    assert lib.gps_graphormer_bias_plan(C.byref(_args()), C.byref(plan)) == _lib.GPS_OK
    assert plan.fwd_workspace_bytes == 0
    # per-CTA partials: at least one CTA's H * (S*T + S + 1) floats and its token share
    assert plan.bwd_workspace_bytes >= 4 * (8 * (20 * 4 + 21) + 8)
    small = _lib.GpsGraphormerBiasPlan()
    assert lib.gps_graphormer_bias_plan(C.byref(_args(edges=False)), C.byref(small)) == _lib.GPS_OK
    assert small.bwd_workspace_bytes < plan.bwd_workspace_bytes
    actor = _lib.GpsGraphormerBiasPlan()   # one graph of 7 600 nodes, 4 heads, no edge types
    assert lib.gps_graphormer_bias_plan(C.byref(_args(7600 ** 2, 1, 7600, 4, 20, 0, 0, False)),
                                        C.byref(actor)) == _lib.GPS_OK


@pytest.mark.parametrize("kw,rc", [
    (dict(H=0), _lib.GPS_ERR_ARG), (dict(S=0), _lib.GPS_ERR_ARG), (dict(P=-1), _lib.GPS_ERR_ARG),
    (dict(token=2), _lib.GPS_ERR_ARG), (dict(nmax=0), _lib.GPS_ERR_ARG), (dict(T=0), _lib.GPS_ERR_ARG),
    (dict(H=33), _lib.GPS_ERR_UNSUPPORTED), (dict(S=20, T=60, H=8), _lib.GPS_ERR_UNSUPPORTED),
    (dict(S=400, H=8, edges=False), _lib.GPS_ERR_UNSUPPORTED), (dict(S=40, T=10, H=2), _lib.GPS_ERR_UNSUPPORTED)])
def test_abi_plan_rejects(kw, rc):
    lib = _lib.load()
    plan = _lib.GpsGraphormerBiasPlan()
    assert lib.gps_graphormer_bias_plan(C.byref(_args(**kw)), C.byref(plan)) == rc
    assert lib.gps_graphormer_bias_plan(None, C.byref(plan)) == _lib.GPS_ERR_ARG


def test_abi_rejects_before_any_cuda_call():
    """Bad or NULL arguments return GPS_ERR_ARG without touching the device (these pointers are never dereferenced)."""
    lib = _lib.load()
    assert lib.gps_graphormer_bias_forward(None, None) == _lib.GPS_ERR_ARG
    assert lib.gps_graphormer_bias_backward(None, None) == _lib.GPS_ERR_ARG
    fake = 1 << 40
    a = _args()
    assert lib.gps_graphormer_bias_forward(C.byref(a), None) == _lib.GPS_ERR_ARG   # no index tensors
    a.spatial_types = a.graph_index = a.node_ptr = fake
    a.spatial_weight = a.edge_dis_weight = a.edge_weight = fake
    assert lib.gps_graphormer_bias_forward(C.byref(a), None) == _lib.GPS_ERR_ARG   # no graph_token
    assert "graph_token" in lib.gps_last_error().decode()
    a.graph_token = fake
    assert lib.gps_graphormer_bias_forward(C.byref(a), None) == _lib.GPS_ERR_ARG   # no output
    a.attn_bias = fake
    a.edge_weight = 0
    assert lib.gps_graphormer_bias_forward(C.byref(a), None) == _lib.GPS_ERR_ARG   # edge term without its table
    a.edge_weight = fake
    assert lib.gps_graphormer_bias_backward(C.byref(a), None) == _lib.GPS_ERR_ARG  # no grad_attn_bias
    a.grad_attn_bias, a.workspace, a.workspace_bytes = fake, fake, 16
    assert lib.gps_graphormer_bias_backward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "workspace too small" in lib.gps_last_error().decode()


def test_install_graphormer_bias_rebinds_stub_module():
    stub = types.ModuleType("graphgps.encoder.graphormer_encoder")

    class Original:
        pass

    stub.BiasEncoder = Original
    prev = graphgym.install_graphormer_bias(stub)
    assert prev is Original
    assert stub.BiasEncoder is graphgps_b200.BiasEncoder
    assert graphgym.install_graphormer_bias(stub) is graphgps_b200.BiasEncoder


def test_install_graphormer_bias_reaches_graphormer_encoder():
    """The reference's GraphormerEncoder (loaded verbatim with the fixture generator's stubs) builds this package's
    BiasEncoder after install_graphormer_bias, keeps its own NodeEncoder, and loads a reference encoder's weights
    strictly."""
    ref = "/root/reference/graphgps/encoder/graphormer_encoder.py"
    if not os.path.isfile(ref):
        pytest.skip("reference checkout not available")
    import sys
    sys.path.insert(0, os.path.join(GOLDEN_DIR))
    try:
        from make_graphormer_bias_golden import load_encoder
    finally:
        sys.path.pop(0)
    saved = {k: v for k, v in sys.modules.items() if k.startswith("torch_geometric")}
    try:
        _check_graphormer_encoder(load_encoder(ref))
    finally:   # the generator's PyG stubs must not leak into the other tests of the session
        for k in [k for k in sys.modules if k.startswith("torch_geometric")]:
            del sys.modules[k]
        sys.modules.update(saved)


def _check_graphormer_encoder(m):
    import torch_geometric.graphgym.config as gcfg
    gcfg.cfg.graphormer = types.SimpleNamespace(num_heads=8, use_graph_token=True, input_dropout=0.0)
    gcfg.cfg.dataset = types.SimpleNamespace(edge_encoder_num_types=4)
    gcfg.cfg.posenc_GraphormerBias.num_spatial_types = 20
    m.cfg = gcfg.cfg
    reference = m.GraphormerEncoder(80)
    prev = graphgym.install_graphormer_bias(m)
    try:
        ours = m.GraphormerEncoder(80)
    finally:
        m.BiasEncoder = prev
    assert isinstance(ours[0], graphgps_b200.BiasEncoder) and type(ours[1]) is m.NodeEncoder
    ours.load_state_dict(reference.state_dict(), strict=True)
