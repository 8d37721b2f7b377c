"""The node-prediction heads and losses, CPU side: the float64 restatement against the reference run verbatim, the state
dicts against the reference's, the constructor contract, CPU refusal, the C ABI's struct layout, plan sizes and argument
checks, and install_node_heads / install_node_losses."""
import ctypes as C
import math
import os
import shutil
import subprocess
import sys
import types

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib, graphgym
from node_head_oracle import fixture_ct, fixture_rows, oracle
from util import GOLDEN_DIR

NH_DIR = os.path.join(GOLDEN_DIR, "node_head")
INCLUDE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include")
REF = "/root/reference/graphgps"
FIXTURES = sorted(p[:-3] for p in os.listdir(NH_DIR) if p.endswith(".pt") and p != "reference_live.pt")


def _load(name):
    return torch.load(os.path.join(NH_DIR, name + ".pt"), weights_only=False)


def _head(c, **kw):
    cls = graphgps_b200.NodeHead if c["head"] == "node" else graphgps_b200.InductiveNodeHead
    return cls(c["d"], c["dout"], layers_post_mp=c["L"], dim_inner=c["dim_inner"], **kw)


def _close(a, r, tol):
    if math.isnan(float(r.double().abs().max())) if r.numel() else False:
        return torch.equal(torch.isnan(a), torch.isnan(r)) and \
            bool(((a - r.to(a.dtype)).abs()[~torch.isnan(r)] <= tol * max(1.0, float(r.nan_to_num().abs().max()))).all())
    return r.numel() == 0 or float((a - r.double()).abs().max()) <= tol * max(1.0, float(r.abs().max()))


@pytest.mark.parametrize("name", ["live_inductive", "live_node", "live_binary"])
def test_oracle_equals_reference_live(name):
    fix = _load("reference_live")["cases"][name]
    for mode, sfx in (("loss", ""), ("ct", "_ct")):
        loss, score, gx, grads = oracle(fix, mode)
        if mode == "loss":
            assert abs(float(loss) - fix["loss"]) < 1e-10
            assert float((score - fix["pred_score"]).abs().max()) < 1e-10
        assert float((gx - fix["grad_x" + sfx]).abs().max()) < 1e-10
        for k, g in fix["grads" + sfx].items():
            assert float((grads[k] - g).abs().max()) < 1e-10, (mode, k)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_equals_reference_fixtures(name):
    """Every fixture (PATTERN, CLUSTER, VOC, COCO, an odd width, an absent class, a one-class batch, ReLU-zeroed rows,
    binary, actor / webkb masks, an empty mask) against the oracle in float64, under both upstream gradients."""
    fix = _load(name)
    for mode, sfx in (("loss", ""), ("ct", "_ct")):
        loss, score, gx, grads = oracle(fix, mode)
        if mode == "loss":
            assert (math.isnan(fix["loss"]) and math.isnan(float(loss))) or abs(float(loss) - fix["loss"]) <= 1e-6
            assert abs(float(score.sum()) - fix["pred_score_sum"]) <= 1e-6 * max(1.0, abs(fix["pred_score_sum"]))
            if "pred_score" in fix:
                assert _close(score, fix["pred_score"], 1e-5)
        refs = [(k, grads[k], g) for k, g in fix["grads" + sfx].items()]
        if "grad_x" + sfx in fix:
            refs.append(("grad_x", gx, fix["grad_x" + sfx]))
        for what, a, r in refs:
            assert _close(a, r, 1e-5), (mode, what)


def test_fixtures_are_what_they_claim():
    one = _load("one_class_C4")
    assert math.isnan(one["loss"]) and one["labels"].unique().tolist() == [2]
    assert set(_load("absent_class_C5")["labels"].unique().tolist()) == {0, 1, 3}
    empty = _load("empty_mask_test")
    assert empty["num_pred"] == 0 and not empty["masks"]["test"].any() and math.isnan(empty["loss"])
    actor = _load("actor_d64_C5_train")
    assert actor["x_shape"][0] == 7600 and fixture_rows(actor).shape[0] == actor["num_pred"]
    assert _load("binary_d64_L3")["config"]["dout"] == 1 and fixture_ct(_load("binary_d64_L3")).dim() == 1
    z = _load("relu_zero_rows")
    b0 = z["state"]["layer_post_mp.model.0.Layer_0.layer.model.bias"]
    assert (b0 < 0).all() and z["config"]["zero_rows"]   # zero rows: every unit of the first hidden layer is 0


def test_state_dict_matches_reference():
    live = _load("reference_live")
    for key, args in (("init_state_L3", (graphgps_b200.InductiveNodeHead, 64, 2, 3, None)),
                      ("init_state_L1", (graphgps_b200.NodeHead, 64, 5, 1, None)),
                      ("init_state_L2_inner", (graphgps_b200.InductiveNodeHead, 37, 3, 2, 40))):
        cls, d, dout, L, di = args
        torch.manual_seed(live["init_seed"])
        ours = cls(d, dout, layers_post_mp=L, dim_inner=di).state_dict()
        assert list(ours) == list(live[key])
        for k, v in live[key].items():
            assert torch.equal(ours[k], v), (key, k)   # nn.Linear's draws from the same seed, in the same order
    names = list(graphgps_b200.InductiveNodeHead(8, 2, layers_post_mp=3).state_dict())
    assert names == [f"layer_post_mp.model.0.Layer_{i}.layer.model.{p}" for i in range(2) for p in ("weight", "bias")] + \
        ["layer_post_mp.model.1.model.weight", "layer_post_mp.model.1.model.bias"]


def test_fixture_states_load_strictly():
    for name in FIXTURES:
        fix = _load(name)
        _head(fix["config"]).load_state_dict(fix["state"], strict=True)
    for fix in _load("reference_live")["cases"].values():
        _head(fix["config"]).load_state_dict(fix["state"], strict=True)


def test_loads_reference_head_weights_strictly():
    if not os.path.isdir(REF):
        pytest.skip("reference checkout not available")
    sys.path.insert(0, GOLDEN_DIR)
    try:
        from make_node_head_golden import build_head, load_reference
    finally:
        sys.path.pop(0)
    saved = {k: v for k, v in sys.modules.items() if k.startswith("torch_geometric")}
    try:
        classes = load_reference(REF)
        for head, d, dout, L, di in (("inductive_node", 64, 2, 3, None), ("node", 64, 5, 1, None),
                                     ("inductive_node", 37, 3, 2, 40)):
            ref = build_head(classes, head, d, dout, L, di)
            ours = _head(dict(head=head, d=d, dout=dout, L=L, dim_inner=di))
            ours.load_state_dict(ref.state_dict(), strict=True)
            assert list(ours.state_dict()) == list(ref.state_dict())
    finally:   # the generator's PyG stubs must not leak into the other tests of the session
        for k in [k for k in sys.modules if k.startswith("torch_geometric")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_constructor_contract():
    h = graphgps_b200.InductiveNodeHead(37, 3, layers_post_mp=2, dim_inner=40)
    assert h.layer_post_mp.model[0].Layer_0.layer.model.weight.shape == (40, 37)
    assert h.layer_post_mp.model[1].model.weight.shape == (3, 40)
    assert graphgps_b200.NodeHead(64, 5).layer_post_mp.model[0].model.weight.shape == (5, 64)
    assert graphgps_b200.InductiveNodeHead(24, 2, layers_post_mp=3).dim_inner == 24   # dim_in when dim_inner is None
    for kw in (dict(layers_post_mp=0), dict(layers_post_mp=9), dict(dim_inner=4097)):
        with pytest.raises(NotImplementedError):
            graphgps_b200.InductiveNodeHead(8, 2, **kw)
    for dims in ((4097, 1), (64, 4097), (0, 1)):
        with pytest.raises(NotImplementedError):
            graphgps_b200.NodeHead(*dims)
    with pytest.raises(ValueError):
        graphgps_b200.NodeHead(64, 1, precision="fp16")


def test_refuses_cpu_tensors():
    b = types.SimpleNamespace(x=torch.randn(4, 8), y=torch.zeros(4, dtype=torch.int64), split="train",
                              train_mask=torch.ones(4, dtype=torch.bool))
    for h in (graphgps_b200.InductiveNodeHead(8, 2), graphgps_b200.NodeHead(8, 2)):
        with pytest.raises(RuntimeError, match="CUDA"):
            h(b)
    for fn in (graphgps_b200.weighted_cross_entropy, graphgps_b200.cross_entropy):
        with pytest.raises(RuntimeError, match="CUDA"):
            fn(torch.randn(4, 3), torch.zeros(4, dtype=torch.int64))


def test_struct_layout_matches_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    structs = (_lib.GpsNodeHeadArgs, _lib.GpsNodeHeadPlan, _lib.GpsNodeLossArgs, _lib.GpsNodeLossPlan)
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "gps_b200.h"', "int main(void) {",
             '  printf("MAX %d %d\\n", GPS_NODE_HEAD_MAX_L, GPS_NODE_LOSS_MAX_C);']
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
    assert out["MAX"] == [_lib.NODE_HEAD_MAX_L, _lib.NODE_LOSS_MAX_C]
    for s in structs:
        t = s.__name__
        assert C.sizeof(s) == out[t][0]
        for f, _ in s._fields_:
            assert getattr(s, f).offset == out[f"{t}.{f}"][0], f


def _args(L=3, d=96, di=96, dout=21, N=15000, M=0, precision=0):
    a = _lib.GpsNodeHeadArgs()
    a.L, a.dim_in, a.dim_inner, a.dim_out, a.N, a.M, a.precision = L, d, di, dout, N, M, precision
    return a


def _plan(**kw):
    plan = _lib.GpsNodeHeadPlan()
    return _lib.load().gps_node_head_plan(C.byref(_args(**kw)), C.byref(plan)), plan


def test_abi_plan():
    rc, p = _plan()
    assert rc == _lib.GPS_OK
    # the padded x and the two normalised hidden rows (+ hi / lo planes), and the padded weights
    assert p.saved_bytes >= 15000 * 96 * 3 * (4 + 4) + 4 * (96 * 96 * 2 + 24 * 96)
    assert p.fwd_workspace_bytes >= 4 * 15000 * 24                      # the padded y
    assert p.bwd_workspace_bytes >= 4 * 15000 * (96 + 96 + 24 + 96)     # g_l and the product output
    rc, bf = _plan(precision=1)
    assert rc == _lib.GPS_OK and bf.saved_bytes < p.saved_bytes         # no lo planes
    rc, one = _plan(L=1, d=64, dout=5, N=7600)
    assert rc == _lib.GPS_OK and one.saved_bytes < p.saved_bytes
    lp = _lib.GpsNodeLossPlan()
    assert _lib.load().gps_node_loss_plan(C.byref(_lib.GpsNodeLossArgs(M=15000, C=21, weighted=1)),
                                          C.byref(lp)) == _lib.GPS_OK
    assert lp.saved_bytes >= 4 * 21 + 4 and lp.fwd_workspace_bytes >= 4 * 15000


@pytest.mark.parametrize("kw,rc", [
    (dict(L=0), _lib.GPS_ERR_ARG), (dict(L=9), _lib.GPS_ERR_UNSUPPORTED), (dict(d=0), _lib.GPS_ERR_ARG),
    (dict(dout=0), _lib.GPS_ERR_ARG), (dict(di=0), _lib.GPS_ERR_ARG), (dict(d=4097), _lib.GPS_ERR_UNSUPPORTED),
    (dict(di=4097), _lib.GPS_ERR_UNSUPPORTED), (dict(dout=4097), _lib.GPS_ERR_UNSUPPORTED),
    (dict(precision=2), _lib.GPS_ERR_ARG), (dict(N=-1), _lib.GPS_ERR_ARG), (dict(M=-1), _lib.GPS_ERR_ARG)])
def test_abi_plan_rejects(kw, rc):
    assert _plan(**kw)[0] == rc
    assert _lib.load().gps_node_head_plan(None, C.byref(_lib.GpsNodeHeadPlan())) == _lib.GPS_ERR_ARG


def test_abi_rejects_before_any_cuda_call():
    """Bad or NULL arguments return GPS_ERR_ARG without touching the device (these pointers are never dereferenced)."""
    lib = _lib.load()
    fake = 1 << 40
    assert lib.gps_node_head_forward(None, None) == _lib.GPS_ERR_ARG
    assert lib.gps_node_head_backward(None, None) == _lib.GPS_ERR_ARG
    a = _args(M=10)
    assert lib.gps_node_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # no saved / workspace
    a.saved, a.saved_bytes, a.workspace, a.workspace_bytes = fake, 16, fake, 1 << 34
    assert lib.gps_node_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "saved buffer too small" in lib.gps_last_error().decode()
    a.saved_bytes = 1 << 34
    assert lib.gps_node_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # no weights
    assert "fc[0]" in lib.gps_last_error().decode()
    for l in range(3):
        a.fc[l].weight = a.fc[l].bias = fake
    assert lib.gps_node_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # M > 0 without rows
    assert "rows" in lib.gps_last_error().decode()
    a.rows = fake
    assert lib.gps_node_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # no x / y
    assert "x and y" in lib.gps_last_error().decode()
    a.x = a.y = fake
    assert lib.gps_node_head_forward(C.byref(a), None) == _lib.GPS_ERR_ARG    # no pred
    assert "pred" in lib.gps_last_error().decode()
    assert lib.gps_node_head_backward(C.byref(a), None) == _lib.GPS_ERR_ARG   # no grad_x
    assert "grad_x" in lib.gps_last_error().decode()
    a.grad_x, a.flags = fake, 1
    assert lib.gps_node_head_backward(C.byref(a), None) == _lib.GPS_ERR_ARG
    a.flags, a.workspace_bytes = 0, 64
    assert lib.gps_node_head_backward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "workspace too small" in lib.gps_last_error().decode()
    # the normalisation stage
    assert lib.gps_row_l2norm_forward(fake, 10, 6, 8, fake, fake, None) == _lib.GPS_ERR_UNSUPPORTED
    assert lib.gps_row_l2norm_forward(fake, 10, 8, 6, fake, fake, None) == _lib.GPS_ERR_ARG
    assert lib.gps_row_l2norm_forward(fake, 10, 8, 8, fake, 0, None) == _lib.GPS_ERR_ARG
    assert lib.gps_row_l2norm_backward(fake, fake, fake, 10, 8, 8, 0, None) == _lib.GPS_ERR_ARG
    assert lib.gps_row_l2norm_backward(fake, fake, fake, 10, 4100, 4100, fake, None) == _lib.GPS_ERR_UNSUPPORTED


@pytest.mark.parametrize("kw,rc", [
    (dict(C=0), _lib.GPS_ERR_ARG), (dict(C=4097), _lib.GPS_ERR_UNSUPPORTED), (dict(M=-1), _lib.GPS_ERR_ARG),
    (dict(weighted=2), _lib.GPS_ERR_ARG), (dict(C=1, weighted=0), _lib.GPS_ERR_UNSUPPORTED),
    (dict(flags=1), _lib.GPS_ERR_ARG)])
def test_loss_rejects_before_any_cuda_call(kw, rc):
    lib = _lib.load()
    fake = 1 << 40
    a = _lib.GpsNodeLossArgs(**{**dict(M=100, C=5, weighted=1), **kw})
    assert lib.gps_node_loss_plan(C.byref(a), C.byref(_lib.GpsNodeLossPlan())) == rc
    a.saved = a.workspace = a.pred = a.label = a.loss = a.pred_score = a.grad_pred = fake
    a.saved_bytes = a.workspace_bytes = 1 << 30
    assert lib.gps_node_loss_forward(C.byref(a), None) == rc
    assert lib.gps_node_loss_backward(C.byref(a), None) == rc


def test_loss_rejects_missing_pointers():
    lib = _lib.load()
    fake = 1 << 40
    assert lib.gps_node_loss_forward(None, None) == _lib.GPS_ERR_ARG
    a = _lib.GpsNodeLossArgs(M=100, C=5, weighted=1)
    assert lib.gps_node_loss_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    a.saved, a.saved_bytes, a.workspace, a.workspace_bytes = fake, 8, fake, 1 << 30
    assert lib.gps_node_loss_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "saved buffer too small" in lib.gps_last_error().decode()
    a.saved_bytes = 1 << 20
    assert lib.gps_node_loss_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "loss is required" in lib.gps_last_error().decode()
    a.loss = fake
    assert lib.gps_node_loss_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "pred, label" in lib.gps_last_error().decode()
    a.workspace_bytes = 16
    a.pred = a.label = a.pred_score = fake
    assert lib.gps_node_loss_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "workspace too small" in lib.gps_last_error().decode()
    assert lib.gps_node_loss_backward(C.byref(a), None) == _lib.GPS_ERR_ARG   # no grad_pred


def _stub_cfg(monkeypatch, **kw):
    ns = types.SimpleNamespace
    cfg = ns(gnn=ns(layers_post_mp=3, dim_inner=40), model=ns(loss_fun="weighted_cross_entropy"),
             dataset=ns(task_type="classification"))
    stub = types.ModuleType("torch_geometric.graphgym.config")
    stub.cfg = cfg
    monkeypatch.setitem(sys.modules, "torch_geometric.graphgym.config", stub)
    return cfg


def test_install_node_heads_sets_registry(monkeypatch):
    cfg = _stub_cfg(monkeypatch)
    reg = types.SimpleNamespace(head_dict={"node": "original", "default": "gnn"})
    assert graphgym.install_node_heads(reg) == {"inductive_node": None, "node": "original"}
    ind, node = reg.head_dict["inductive_node"], reg.head_dict["node"]
    assert reg.head_dict["default"] == "gnn"
    h = ind(37, 3)   # the reference's (dim_in, dim_out) constructor
    assert isinstance(h, graphgps_b200.InductiveNodeHead) and (h.L, h.dim_inner) == (3, 40)
    cfg.gnn.layers_post_mp, cfg.gnn.dim_inner = 1, None
    n = node(64, 5)
    assert isinstance(n, graphgps_b200.NodeHead) and (n.L, n.dim_inner) == (1, 64)
    assert graphgym.install_node_heads(reg) == {"inductive_node": ind, "node": node}


def test_install_node_losses_sets_registry_and_wrapper(monkeypatch):
    cfg = _stub_cfg(monkeypatch)
    calls = []

    def previous(pred, true):
        calls.append((pred, true))
        return "previous"

    reg = types.SimpleNamespace(loss_dict={"weighted_cross_entropy": "ref", "l1": "l1"})
    train = types.SimpleNamespace(compute_loss=previous)
    assert graphgym.install_node_losses(reg, train) == {"weighted_cross_entropy": "ref", "compute_loss": previous}
    wce = reg.loss_dict["weighted_cross_entropy"]
    assert reg.loss_dict["l1"] == "l1" and train.compute_loss is not previous
    cfg.model.loss_fun = "cross_entropy"
    assert wce(torch.randn(4, 3), torch.zeros(4, dtype=torch.int64)) is None   # checks loss_fun itself
    cfg.model.loss_fun = "weighted_cross_entropy"
    with pytest.raises(RuntimeError, match="CUDA"):   # ours, which refuses CPU tensors
        wce(torch.randn(4, 3), torch.zeros(4, dtype=torch.int64))
    # everything the device path does not take goes to the previous compute_loss, unchanged
    cases = [("l1", "classification", torch.randn(4, 3), torch.zeros(4, dtype=torch.int64)),
             ("cross_entropy", "classification_multilabel", torch.randn(4, 3), torch.zeros(4, 3)),
             ("cross_entropy", "classification", torch.randn(4, 3), torch.zeros(4, dtype=torch.int64)),   # CPU
             ("cross_entropy", "classification", torch.randn(4, 1), torch.zeros(4, 1, dtype=torch.int64)),  # binary
             ("cross_entropy", "classification", torch.randn(4, 3).double(), torch.zeros(4, dtype=torch.int64))]
    for loss_fun, task, pred, true in cases:
        cfg.model.loss_fun, cfg.dataset.task_type = loss_fun, task
        calls.clear()
        assert train.compute_loss(pred, true) == "previous"
        assert len(calls) == 1 and calls[0][0] is pred and calls[0][1] is true
