"""RWSE, CPU side: the float64 oracle against the reference run verbatim, the block-diagonal batch against graph by
graph, the encoder's state dict, initial draws and constructor contract, CPU refusal, the C ABI's struct layout, plan
sizes and argument checks, and install_rwse."""
import ctypes as C
import os
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib, graphgym
from rwse_oracle import encoder as oracle_encoder, fixture_names, hashed, landing, landing_batched, load

INCLUDE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include")
FIXTURES = fixture_names()


def test_oracle_equals_reference_live():
    fix = load("reference_live")
    c = fix["config"]
    rw = torch.from_numpy(landing(fix["edge_index"].long().numpy(), fix["ptr"].numpy(), c["ksteps"]))
    assert float((rw - fix["rw64"]).abs().max()) < 1e-10
    N = int(fix["ptr"][-1])
    x, g = hashed(fix["x_seed"], (N, c["dim_in"])), hashed(fix["x_seed"] + 1, (N, c["dim_emb"]))
    out, gx, grads, run = oracle_encoder(fix["state"], c, x, fix["rw64"].float(), g, True)
    assert float((out - fix["out"]).abs().max()) < 1e-10
    assert float((gx - fix["grad_x"]).abs().max()) < 1e-10
    for k, v in fix["grads"].items():
        assert float((grads[k] - v).abs().max()) < 1e-10, k
    for a, r in zip(run, fix["running"]):
        assert float((a - r).abs().max()) < 1e-10


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_equals_reference_fixtures(name):
    fix = load(name)
    c = fix["config"]
    rw = torch.from_numpy(landing(fix["edge_index"].long().numpy(), fix["ptr"].numpy(), c["ksteps"]))
    rows = fix["rw64"].shape[0]
    assert float((rw[:rows] - fix["rw64"]).abs().max()) < 1e-12
    N = int(fix["ptr"][-1])
    x, g = hashed(fix["x_seed"], (N, c["dim_in"])), hashed(fix["x_seed"] + 1, (N, c["dim_emb"]))
    _, _, grads, run = oracle_encoder(fix["state"], c, x, rw.float(), g, c["training"])
    for k, v in fix["grads"].items():
        assert float((grads[k] - v).abs().max()) <= 1e-10 * max(1.0, float(v.abs().max())), k
    if c["batch_norm"]:
        for a, r in zip(run, fix["running"]):
            assert float((a - r).abs().max()) < 1e-10


def test_fixtures_are_what_they_claim():
    ec = load("edge_cases_range5")
    assert ec["config"]["ksteps"] == [0, 1, 2, 3, 4] and len(ec["config"]["ksteps"]) % 4   # the padded BatchNorm
    assert bool((ec["rw64"][:, 0] == 1).all())                   # k = 0: a zero-variance column
    assert load("edge_cases_k3183")["config"]["ksteps"] == [3, 1, 8, 3]
    bip = slice(13, 19)                                          # the bipartite graph of edge_case_graphs()
    assert int(ec["ptr"][4]) == 13 and int(ec["ptr"][5]) == 19
    assert bool((ec["rw64"][bip, 1] == 0).all()) and bool((ec["rw64"][bip, 3] == 0).all())
    assert bool((ec["rw64"][bip, 2] > 0).any())
    pc = load("pcqm4m_k16_pe20_d304")
    assert pc["ptr"].numel() - 1 == 256 and int(torch.diff(pc["ptr"]).min()) == 1   # single atoms without edges
    mal = load("malnet_hubs_5000")
    assert int(mal["ptr"][-1]) == 5000 and int(torch.bincount(mal["edge_index"][1].long()).max()) > 500
    assert load("molpcba_k16_pe20_d384")["ptr"].numel() - 1 == 512
    assert load("zinc_eval")["config"]["training"] is False
    for name in FIXTURES + ["reference_live"]:
        path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rwse", name + ".pt")
        assert os.path.getsize(path) < 1 << 20, name


def test_block_diagonal_batch_equals_graph_by_graph():
    for name in ("edge_cases_k3183", "zinc_k20_pe28"):
        fix = load(name)
        ei, ptr, ks = fix["edge_index"].long().numpy(), fix["ptr"].numpy(), fix["config"]["ksteps"]
        a = landing(ei, ptr, ks)
        b = landing_batched(ei, int(ptr[-1]), ks)
        assert np.array_equal(a, b), name


def test_state_dict_matches_reference_and_loads_strictly():
    fix = load("reference_live")
    c = fix["init_config"]
    torch.manual_seed(1357)
    enc = graphgps_b200.KernelPENodeEncoder(c["dim_in"], c["dim_emb"], c["K"], c["dim_pe"])
    ref = fix["init_state"]
    assert list(enc.state_dict()) == list(ref)
    for k, v in ref.items():
        assert torch.equal(enc.state_dict()[k], v), k   # same seed, same draws
    for name in FIXTURES:
        f = load(name)
        cf = f["config"]
        e = graphgps_b200.KernelPENodeEncoder(cf["dim_in"], cf["dim_emb"], len(cf["ksteps"]), cf["dim_pe"],
                                              raw_norm_type="batchnorm" if cf["batch_norm"] else "none",
                                              expand_x=cf["expand_x"])
        e.load_state_dict(f["state"], strict=True)
    names = list(graphgps_b200.KernelPENodeEncoder(36, 64, 20, 28, expand_x=False).state_dict())
    assert names == ["raw_norm.weight", "raw_norm.bias", "raw_norm.running_mean", "raw_norm.running_var",
                     "raw_norm.num_batches_tracked", "pe_encoder.weight", "pe_encoder.bias"]


def test_constructor_contract():
    E = graphgps_b200.KernelPENodeEncoder
    with pytest.raises(ValueError, match="too large"):
        E(5, 16, 8, 20)
    with pytest.raises(NotImplementedError):
        E(5, 64, 16, 20, model="mlp")
    with pytest.raises(ValueError):
        E(5, 64, 16, 20, model="transformer")
    with pytest.raises(NotImplementedError):
        E(5, 64, 16, 20, pass_as_var=True)
    with pytest.raises(NotImplementedError):
        E(5, 4097, 16, 20)
    with pytest.raises(NotImplementedError):
        E(5, 64, 65, 20)
    with pytest.raises(ValueError):
        E(5, 64, 16, 20, kernel_type="LapPE")
    with pytest.raises(ValueError):
        E(5, 64, 16, 20, kernel_type="HKdiagSE", ksteps=range(1, 17))
    with pytest.raises(ValueError):
        E(5, 64, 16, 20, ksteps=range(1, 9))
    with pytest.raises(NotImplementedError):
        E(5, 64, 1, 20, ksteps=[257])
    with pytest.raises(ValueError, match="dim_in must be"):
        E(5, 64, 16, 20, expand_x=False)
    assert E(5, 64, 16, 20, raw_norm_type="none").raw_norm is None
    assert not hasattr(E(44, 64, 16, 20, expand_x=False), "linear_x")
    assert E(5, 64, 16, 20, ksteps=range(1, 17)).ksteps == tuple(range(1, 17))


def test_forward_refuses_cpu_tensors_and_missing_statistics():
    enc = graphgps_b200.KernelPENodeEncoder(5, 16, 4, 8)
    b = types.SimpleNamespace(x=torch.randn(4, 5), pestat_RWSE=torch.rand(4, 4))
    with pytest.raises(RuntimeError, match="CUDA"):
        enc(b)
    b = types.SimpleNamespace(edge_index=torch.zeros(2, 0, dtype=torch.int64), batch=torch.zeros(4, dtype=torch.int64),
                              num_graphs=1)
    with pytest.raises(RuntimeError, match="CUDA"):
        graphgps_b200.rw_landing_probs(b, [1, 2])


def test_struct_layout_matches_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    structs = (_lib.GpsKernelPeArgs, _lib.GpsKernelPePlan)
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "gps_b200.h"', "int main(void) {",
             '  printf("LIMITS %d %d\\n", GPS_RWSE_MAX_COLS, GPS_RWSE_MAX_STEPS);']
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
    assert out["LIMITS"] == [_lib.RWSE_MAX_COLS, _lib.RWSE_MAX_STEPS]
    for s in structs:
        t = s.__name__
        assert C.sizeof(s) == out[t][0]
        for f, _ in s._fields_:
            assert getattr(s, f).offset == out[f"{t}.{f}"][0], f


def _args(N=4106, K=16, dim_in=284, dim_emb=304, dim_pe=20, expand_x=0, batch_norm=1, training=1):
    a = _lib.GpsKernelPeArgs()
    a.N, a.K, a.dim_in, a.dim_emb, a.dim_pe = N, K, dim_in, dim_emb, dim_pe
    a.expand_x, a.batch_norm, a.training = expand_x, batch_norm, training
    return a


def _plan(**kw):
    plan = _lib.GpsKernelPePlan()
    rc = _lib.load().gps_kernel_pe_plan(C.byref(_args(**kw)), C.byref(plan))
    return rc, plan


def test_abi_plan():
    rc, p = _plan()
    assert rc == _lib.GPS_OK
    assert p.saved_bytes >= 4 * 4106 * 16                        # zhat
    assert p.fwd_workspace_bytes >= 8 * 2 * 16 * 65              # double column sums of 65 chunks of 64 rows
    assert p.bwd_workspace_bytes >= 4 * 4106 * 16 + 8 * 129 * (20 * 17 + 32)   # gz, the gradient partials
    rc, ev = _plan(training=0)
    assert rc == _lib.GPS_OK and ev.fwd_workspace_bytes == 0
    rc, nn_ = _plan(batch_norm=0)
    assert rc == _lib.GPS_OK and nn_.saved_bytes == 0
    rc, pad = _plan(K=5)
    assert rc == _lib.GPS_OK and pad.saved_bytes >= 4 * 4106 * 8 + 4 * 4 * 8     # padded to 8 columns + parameters
    rc, ex = _plan(dim_in=5, dim_emb=52, dim_pe=24, expand_x=1)
    assert rc == _lib.GPS_OK


@pytest.mark.parametrize("kw,rc", [
    (dict(K=0), _lib.GPS_ERR_ARG), (dict(K=65), _lib.GPS_ERR_UNSUPPORTED), (dict(dim_pe=0), _lib.GPS_ERR_ARG),
    (dict(dim_pe=305), _lib.GPS_ERR_ARG), (dict(dim_emb=4097, dim_in=4077), _lib.GPS_ERR_UNSUPPORTED),
    (dict(dim_in=0), _lib.GPS_ERR_ARG), (dict(dim_in=283), _lib.GPS_ERR_ARG), (dict(expand_x=2), _lib.GPS_ERR_ARG),
    (dict(batch_norm=2), _lib.GPS_ERR_ARG), (dict(N=1), _lib.GPS_ERR_ARG), (dict(N=-1), _lib.GPS_ERR_ARG)])
def test_abi_plan_rejects(kw, rc):
    assert _plan(**kw)[0] == rc
    assert _lib.load().gps_kernel_pe_plan(None, C.byref(_lib.GpsKernelPePlan())) == _lib.GPS_ERR_ARG


def test_abi_rejects_before_any_cuda_call():
    """Bad or NULL arguments return GPS_ERR_ARG / GPS_ERR_UNSUPPORTED without touching the device (these pointers are
    never dereferenced)."""
    lib = _lib.load()
    fake = 1 << 40
    assert lib.gps_kernel_pe_forward(None, None) == _lib.GPS_ERR_ARG
    a = _args()
    assert lib.gps_kernel_pe_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    a.saved, a.saved_bytes, a.workspace, a.workspace_bytes = fake, 16, fake, 1 << 30
    assert lib.gps_kernel_pe_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "saved buffer too small" in lib.gps_last_error().decode()
    a.saved_bytes = 1 << 30
    assert lib.gps_kernel_pe_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "pe_encoder" in lib.gps_last_error().decode()
    a.pe_encoder.weight = a.pe_encoder.bias = fake
    assert lib.gps_kernel_pe_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "raw_norm" in lib.gps_last_error().decode()
    a.raw_norm.weight = a.raw_norm.bias = a.raw_norm.running_mean = a.raw_norm.running_var = fake
    assert lib.gps_kernel_pe_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "required" in lib.gps_last_error().decode()
    a.raw_norm.bias = fake + 4
    assert lib.gps_kernel_pe_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "aligned" in lib.gps_last_error().decode()
    a.raw_norm.bias, a.workspace = fake, fake + 8
    assert lib.gps_kernel_pe_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    a.workspace, a.workspace_bytes = fake, 64
    assert lib.gps_kernel_pe_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    assert "workspace too small" in lib.gps_last_error().decode()
    a.workspace_bytes, a.x, a.pestat = 1 << 30, fake, fake
    assert lib.gps_kernel_pe_backward(C.byref(a), None) == _lib.GPS_ERR_ARG   # no grad_out / grad_x
    a.flags = 1
    assert lib.gps_kernel_pe_forward(C.byref(a), None) == _lib.GPS_ERR_ARG

    g = _lib.GpsGraph(N=300, E=10, B=4)
    ks = (C.c_int32 * 3)(1, 2, 3)
    land = lib.gps_rwse_landing
    assert land(None, ks, 3, 10, fake, fake, 1 << 20, None) == _lib.GPS_ERR_ARG
    assert land(C.byref(g), ks, 3, 10, fake, fake, 1 << 20, None) == _lib.GPS_ERR_ARG   # no graph_ptr
    g.graph_ptr = g.dst_ptr = g.dst_src = g.src_ptr = fake
    assert land(C.byref(g), None, 3, 10, fake, fake, 1 << 20, None) == _lib.GPS_ERR_ARG
    assert land(C.byref(g), ks, 0, 10, fake, fake, 1 << 20, None) == _lib.GPS_ERR_ARG
    assert land(C.byref(g), (C.c_int32 * 65)(), 65, 10, fake, fake, 1 << 20, None) == _lib.GPS_ERR_UNSUPPORTED
    assert land(C.byref(g), (C.c_int32 * 2)(1, 257), 2, 10, fake, fake, 1 << 20, None) == _lib.GPS_ERR_UNSUPPORTED
    assert land(C.byref(g), (C.c_int32 * 2)(1, -1), 2, 10, fake, fake, 1 << 20, None) == _lib.GPS_ERR_ARG
    assert land(C.byref(g), ks, 3, 301, fake, fake, 1 << 20, None) == _lib.GPS_ERR_ARG
    assert land(C.byref(g), ks, 3, 10, 0, fake, 1 << 20, None) == _lib.GPS_ERR_ARG
    assert land(C.byref(g), ks, 3, 10, fake, fake + 4, 1 << 20, None) == _lib.GPS_ERR_ARG
    assert land(C.byref(g), ks, 3, 10, fake, fake, 2399, None) == _lib.GPS_ERR_ARG
    big = _lib.GpsGraph(N=40_000, E=10, B=1)
    big.graph_ptr = big.dst_ptr = big.dst_src = big.src_ptr = fake
    assert land(C.byref(big), ks, 3, 40_000, fake, fake, 1 << 20, None) == _lib.GPS_ERR_UNSUPPORTED
    assert "on chip" in lib.gps_last_error().decode()


def _stub_cfg(pe):
    return types.SimpleNamespace(share=types.SimpleNamespace(dim_in=5), posenc_RWSE=pe, posenc_HKdiagSE=pe,
                                 posenc_ElstaticSE=pe)


@pytest.mark.parametrize("on_device", [False, True])
def test_install_rwse(on_device):
    old = {n: type(n, (), {}) for n in ("RWSENodeEncoder", "HKdiagSENodeEncoder", "ElstaticSENodeEncoder")}
    kmod = types.SimpleNamespace(**old)
    concat2 = type("Concat2NodeEncoder", (), {"enc2_cls": old["RWSENodeEncoder"]})
    concat3 = type("Concat3NodeEncoder", (), {"enc2_cls": object, "enc3_cls": old["RWSENodeEncoder"]})
    other = type("Concat2NodeEncoder", (), {"enc2_cls": object})
    reg = types.SimpleNamespace(node_encoder_dict={"RWSE": old["RWSENodeEncoder"], "Atom+RWSE": concat2,
                                                   "Atom+LapPE+RWSE": concat3, "Atom+LapPE": other,
                                                   "HKdiagSE": old["HKdiagSENodeEncoder"]})
    calls = []
    loader = types.SimpleNamespace(compute_posenc_stats=lambda data, pe_types, is_undirected, cfg: calls.append(
        (data, list(pe_types), is_undirected, cfg)))
    pe = types.SimpleNamespace(dim_pe=20, kernel=types.SimpleNamespace(times=list(range(1, 17))), model="Linear",
                               layers=1, raw_norm_type="BatchNorm", pass_as_var=False)
    stub = types.ModuleType("torch_geometric.graphgym.config")
    stub.cfg = _stub_cfg(pe)
    saved = sys.modules.get("torch_geometric.graphgym.config")
    sys.modules["torch_geometric.graphgym.config"] = stub
    try:
        prev = graphgym.install_rwse(on_device, kernel_module=kmod, register_module=reg, loader_module=loader)
        for n, o in old.items():
            assert prev[n] is o
        new = kmod.RWSENodeEncoder
        assert reg.node_encoder_dict["RWSE"] is new and concat2.enc2_cls is new and concat3.enc3_cls is new
        assert concat3.enc2_cls is object and other.enc2_cls is object
        assert reg.node_encoder_dict["HKdiagSE"] is kmod.HKdiagSENodeEncoder
        e = new(64)                                     # (dim_emb, expand_x=True), as the reference builds it
        assert isinstance(e, graphgps_b200.KernelPENodeEncoder) and e.expand_x and e.dim_in == 5
        assert e.ksteps == (tuple(range(1, 17)) if on_device else None)
        e2 = new(64, expand_x=False)                    # composed: x is the first encoder's dim_emb - dim_pe columns
        assert not e2.expand_x and e2.dim_in == 44
        assert kmod.HKdiagSENodeEncoder(64).ksteps is None and kmod.HKdiagSENodeEncoder(64).kernel_type == "HKdiagSE"
        if on_device:
            loader.compute_posenc_stats("data", pe_types=["LapPE", "RWSE"], is_undirected=True, cfg="cfg")
            assert calls == [("data", ["LapPE"], True, "cfg")]
            assert "compute_posenc_stats" in prev
        else:
            assert "compute_posenc_stats" not in prev
        # a second install replaces the first one's classes everywhere
        graphgym.install_rwse(on_device, kernel_module=kmod, register_module=reg, loader_module=loader)
        assert concat2.enc2_cls is kmod.RWSENodeEncoder is not new
    finally:
        if saved is None:
            del sys.modules["torch_geometric.graphgym.config"]
        else:
            sys.modules["torch_geometric.graphgym.config"] = saved
