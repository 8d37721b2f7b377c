"""The inductive link-prediction head, CPU side: the float64 restatement against the reference run verbatim, the state
dict against the reference's, the constructor contract, CPU refusal, the C ABI's struct layout and argument checks, and
install_inductive_edge_head."""
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
from inductive_edge_oracle import STATS, fixture_x, head_forward, rank_stats
from util import GOLDEN_DIR

IE_DIR = os.path.join(GOLDEN_DIR, "inductive_edge")
INCLUDE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include")
REF = "/root/reference/graphgps/head/inductive_edge.py"
W, B = "layer_post_mp.model.0.model.weight", "layer_post_mp.model.0.model.bias"


def _load(name):
    fix = torch.load(os.path.join(IE_DIR, name + ".pt"), weights_only=False)
    fix["x"] = fixture_x(fix)
    return fix


def _oracle(fix):
    x = fix["x"].double().requires_grad_(True)
    w = fix["state"][W].double().requires_grad_(True)
    b = fix["state"][B].double().requires_grad_(True)
    y, pred = head_forward(x, w, b, fix["edge_index_labeled"])
    (pred * fix["ct"].double()).sum().backward()
    return y, pred, x.grad, w.grad, b.grad


def test_oracle_equals_reference_live():
    fix = _load("reference_live")
    y, pred, gx, gw, gb = _oracle(fix)
    assert float((pred.detach() - fix["pred"]).abs().max()) < 1e-10
    for a, r in ((gx, fix["grad_x"]), (gw, fix["grad_weight"]), (gb, fix["grad_bias"])):
        assert float((a - r).abs().max()) < 1e-10
    stats = rank_stats(y, fix["edge_index_labeled"], fix["edge_label"], fix["ptr"])
    for k in STATS:   # the reference averages each graph's ranks in float32
        assert abs(stats[k] - fix["stats"][k]) < 1e-6, k


@pytest.mark.parametrize("name", sorted(p[:-3] for p in os.listdir(IE_DIR) if p != "reference_live.pt"))
def test_oracle_equals_reference_fixtures(name):
    """Every fp32 fixture (256-graph contact batches at d 138 and 208, graphs without positives, one- and two-node
    graphs, a graph of 3 000 nodes) against the oracle in float64: the reference's ranks exactly."""
    fix = _load(name)
    y, pred, gx, gw, gb = _oracle(fix)
    scale = max(1.0, float(fix["pred"].abs().max()))
    assert float((pred.detach() - fix["pred"].double()).abs().max()) <= 1e-5 * scale
    refs = [(gw, fix["grad_weight"]), (gb, fix["grad_bias"])]
    if "grad_x" in fix:
        refs.append((gx, fix["grad_x"]))
    for a, r in refs:
        assert float((a - r.double()).abs().max()) <= 1e-5 * max(1.0, float(r.abs().max()))
    stats = rank_stats(y, fix["edge_index_labeled"], fix["edge_label"], fix["ptr"])
    for k in STATS:
        assert abs(stats[k] - fix["stats"][k]) < 1e-6, (k, stats[k], fix["stats"][k])


def test_oracle_tie_rule():
    """Equal scores count in the positive's favour; the target itself is not a candidate, the source is."""
    y = torch.tensor([[1.0, 0.0], [1.0, 0.0], [1.0, 0.0], [2.0, 0.0], [0.5, 0.0]], dtype=torch.float64)
    eli = torch.tensor([[0, 0], [1, 4]])
    stats = rank_stats(y, eli, torch.tensor([1, 1]), torch.tensor([0, 5]))
    # (0, 1): above it only node 3 -> rank 2; (0, 4): nodes 0, 1, 2, 3 -> rank 5
    assert stats == {"hits@1": 0.0, "hits@3": 0.5, "hits@10": 1.0, "mrr": (1 / 2 + 1 / 5) / 2}


def test_state_dict_matches_reference():
    fix = _load("reference_live")
    torch.manual_seed(fix["init_seed"])
    ours = graphgps_b200.InductiveEdgeHead(138, 1).state_dict()
    assert list(ours.keys()) == list(fix["init_state"].keys()) == [W, B]
    for k, v in fix["init_state"].items():
        assert torch.equal(ours[k], v), k   # nn.Linear's draws from the same seed


def test_fixture_states_load_strictly():
    for p in sorted(os.listdir(IE_DIR)):
        fix = _load(p[:-3])
        graphgps_b200.InductiveEdgeHead(fix["config"]["d"], 1).load_state_dict(fix["state"], strict=True)


def _with_reference_head(check):
    if not os.path.isfile(REF):
        pytest.skip("reference checkout not available")
    sys.path.insert(0, GOLDEN_DIR)
    try:
        from make_inductive_edge_golden import load_head
    finally:
        sys.path.pop(0)
    saved = {k: v for k, v in sys.modules.items() if k.startswith("torch_geometric")}
    try:
        check(load_head(REF))
    finally:   # the generator's PyG stubs must not leak into the other tests of the session
        for k in [k for k in sys.modules if k.startswith("torch_geometric")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_loads_reference_head_weights_strictly():
    def check(m):
        ref = m.GNNInductiveEdgeHead(96, 1)
        ours = graphgps_b200.InductiveEdgeHead(96, 1)
        ours.load_state_dict(ref.state_dict(), strict=True)
        assert list(ours.state_dict()) == list(ref.state_dict())
    _with_reference_head(check)


def test_constructor_contract():
    h = graphgps_b200.InductiveEdgeHead(208, 1)
    assert tuple(h.layer_post_mp.model[0].model.weight.shape) == (208, 208)
    with pytest.raises(ValueError):
        graphgps_b200.InductiveEdgeHead(138, 2)   # dot decoding is binary
    with pytest.raises(NotImplementedError):
        graphgps_b200.InductiveEdgeHead(138, 1, edge_decoding="concat")
    with pytest.raises(NotImplementedError):
        graphgps_b200.InductiveEdgeHead(138, 1, edge_decoding="cosine_similarity")
    with pytest.raises(ValueError):
        graphgps_b200.InductiveEdgeHead(138, 1, edge_decoding="bilinear")
    with pytest.raises(NotImplementedError):
        graphgps_b200.InductiveEdgeHead(138, 1, layers_post_mp=2)
    with pytest.raises(ValueError):
        graphgps_b200.InductiveEdgeHead(138, 1, precision="fp16")


def test_forward_refuses_cpu_tensors():
    h = graphgps_b200.InductiveEdgeHead(8, 1)
    b = types.SimpleNamespace(x=torch.randn(4, 8), edge_index_labeled=torch.tensor([[0, 1], [1, 2]]),
                              edge_label=torch.tensor([1, 0]), batch=torch.zeros(4, dtype=torch.int64), num_graphs=1)
    with pytest.raises(RuntimeError, match="CUDA"):
        h(b)


def test_struct_layout_matches_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    structs = (_lib.GpsLinkHeadArgs, _lib.GpsLinkHeadPlan)
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "gps_b200.h"', "int main(void) {"]
    for s in structs:
        t = s.__name__
        lines.append(f'  printf("{t} %zu\\n", sizeof({t}));')
        lines += [f'  printf("{t}.{f} %zu\\n", offsetof({t}, {f}));' for f, _ in s._fields_]
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines) + "\n")
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe)], check=True)
    out = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True,
                                                        text=True).stdout.splitlines())
    for s in structs:
        t = s.__name__
        assert C.sizeof(s) == int(out[t])
        for f, _ in s._fields_:
            assert getattr(s, f).offset == int(out[f"{t}.{f}"]), f


def _args(N=8209, K=4530, B=256, d=138, training=1, precision=0):
    a = _lib.GpsLinkHeadArgs()
    a.d, a.training, a.precision = d, training, precision
    a.pairs.N, a.pairs.E, a.pairs.B = N, K, B
    return a


def test_abi_plan():
    lib = _lib.load()
    plan = _lib.GpsLinkHeadPlan()
    assert lib.gps_link_head_plan(C.byref(_args()), C.byref(plan)) == _lib.GPS_OK
    dp = 144
    assert plan.saved_bytes >= 4 * (2 * 8209 * dp + dp * dp + dp)    # x, y, W, b at pitch dp (+ planes)
    assert plan.fwd_workspace_bytes == 0                              # training: no ranking
    assert plan.bwd_workspace_bytes >= 4 * (2 * 8209 * dp + dp * dp)
    ev = _lib.GpsLinkHeadPlan()
    assert lib.gps_link_head_plan(C.byref(_args(training=0)), C.byref(ev)) == _lib.GPS_OK
    assert ev.fwd_workspace_bytes >= 8 * 4 * 256                       # per-graph values
    bf = _lib.GpsLinkHeadPlan()
    assert lib.gps_link_head_plan(C.byref(_args(precision=1)), C.byref(bf)) == _lib.GPS_OK
    assert bf.saved_bytes < plan.saved_bytes                           # no lo planes


@pytest.mark.parametrize("kw,rc", [
    (dict(d=0), _lib.GPS_ERR_ARG), (dict(d=4097), _lib.GPS_ERR_UNSUPPORTED), (dict(precision=3), _lib.GPS_ERR_ARG),
    (dict(N=-1), _lib.GPS_ERR_ARG), (dict(K=-1), _lib.GPS_ERR_ARG), (dict(B=-1), _lib.GPS_ERR_ARG)])
def test_abi_plan_rejects(kw, rc):
    lib = _lib.load()
    plan = _lib.GpsLinkHeadPlan()
    assert lib.gps_link_head_plan(C.byref(_args(**kw)), C.byref(plan)) == rc
    assert lib.gps_link_head_plan(None, C.byref(plan)) == _lib.GPS_ERR_ARG


def test_abi_rejects_before_any_cuda_call():
    """Bad or NULL arguments return GPS_ERR_ARG without touching the device (these pointers are never dereferenced)."""
    lib = _lib.load()
    fake = 1 << 40
    assert lib.gps_link_head_forward(None, None) == _lib.GPS_ERR_ARG
    assert lib.gps_link_head_backward(None, None) == _lib.GPS_ERR_ARG
    a = _args()
    assert lib.gps_link_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # no saved / workspace
    a.saved, a.saved_bytes, a.workspace, a.workspace_bytes = fake, 16, fake, 1 << 30
    assert lib.gps_link_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "saved buffer too small" in lib.gps_last_error().decode()
    a.saved_bytes = 1 << 30
    assert lib.gps_link_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # no pair graph arrays
    assert "pair graph" in lib.gps_last_error().decode()
    for f in ("dst_ptr", "dst_src", "dst_eid", "src_ptr", "src_dst", "src_eid", "graph_ptr"):
        setattr(a.pairs, f, fake)
    assert lib.gps_link_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # no weights
    assert "weight" in lib.gps_last_error().decode()
    a.lin.weight = a.lin.bias = fake
    assert lib.gps_link_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # no edge_index_labeled
    a.edge_index_labeled = fake
    assert lib.gps_link_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # no x / y
    a.x = a.y = a.pred = fake
    a.training = 0
    assert lib.gps_link_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # eval without stats
    a.stats, a.label_bytes = fake, 2
    assert lib.gps_link_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "label_bytes" in lib.gps_last_error().decode()
    a.label_bytes, a.edge_label = 8, 0
    assert lib.gps_link_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # eval without edge_label
    a.flags = 1
    assert lib.gps_link_head_backward(C.byref(a), None) == _lib.GPS_ERR_ARG
    a.flags = 0
    assert lib.gps_link_head_backward(C.byref(a), None) == _lib.GPS_ERR_ARG   # no grad_x
    assert "grad_x" in lib.gps_last_error().decode()


def test_rank_metrics_rejects_before_any_cuda_call():
    lib = _lib.load()
    fake = 1 << 40
    g = _lib.GpsGraph(N=30, E=12, B=4)
    args = lambda **kw: dict(dict(y=fake, ld=20, d=20, lab=fake, lb=8, stats=fake, ws=fake, wsb=128), **kw)

    def call(g, **kw):
        a = args(**kw)
        return lib.gps_link_rank_metrics(C.byref(g) if g is not None else None, a["y"], a["ld"], a["d"], a["lab"],
                                         a["lb"], a["stats"], a["ws"], a["wsb"], None)

    assert call(None) == _lib.GPS_ERR_ARG
    assert call(g) == _lib.GPS_ERR_ARG   # no CSR arrays
    for f in ("dst_ptr", "dst_src", "dst_eid", "src_ptr", "src_dst", "src_eid", "graph_ptr"):
        setattr(g, f, fake)
    assert call(g, ld=19) == _lib.GPS_ERR_ARG
    assert call(g, lb=3) == _lib.GPS_ERR_ARG
    assert call(g, wsb=127) == _lib.GPS_ERR_ARG
    assert "workspace too small" in lib.gps_last_error().decode()
    assert call(g, lab=0) == _lib.GPS_ERR_ARG
    assert call(g, stats=0) == _lib.GPS_ERR_ARG


def test_install_inductive_edge_head_sets_registry():
    reg = types.SimpleNamespace(head_dict={"inductive_edge": "original"})
    cfg = types.SimpleNamespace(model=types.SimpleNamespace(edge_decoding="dot"),
                                gnn=types.SimpleNamespace(layers_post_mp=1))
    stub = types.ModuleType("torch_geometric.graphgym.config")
    stub.cfg = cfg
    saved = sys.modules.get("torch_geometric.graphgym.config")
    sys.modules["torch_geometric.graphgym.config"] = stub
    try:
        assert graphgym.install_inductive_edge_head(reg) == "original"
        cls = reg.head_dict["inductive_edge"]
        head = cls(138, 1)   # the reference's (dim_in, dim_out) constructor
        assert isinstance(head, graphgps_b200.InductiveEdgeHead) and head.dim_in == 138
        cfg.gnn.layers_post_mp = 2
        with pytest.raises(NotImplementedError):
            cls(138, 1)
        cfg.gnn.layers_post_mp, cfg.model.edge_decoding = 1, "concat"
        with pytest.raises(NotImplementedError):
            cls(138, 1)
        assert graphgym.install_inductive_edge_head(reg) is cls
    finally:
        if saved is None:
            del sys.modules["torch_geometric.graphgym.config"]
        else:
            sys.modules["torch_geometric.graphgym.config"] = saved
