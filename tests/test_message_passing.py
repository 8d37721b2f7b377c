"""CPU: (1) the fp64 stage references of tests/mp_reference.py composed with fp64 Linear / BatchNorm / activation equal
the oracle's GatedGCN (with and without the EquivStableLapPE gate), GINE and GCN modules, outputs and every gradient
to 1e-12; (2) the argument contract of the message-passing stage entry points: every call here is rejected before any
CUDA call, so it needs no device memory (the addresses are placeholders that are never dereferenced)."""
import copy
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from graphgps_b200 import _lib
from graphgps_b200.batch import batch_from_lists, make_batch
from oracle.gps_oracle import OracleGatedGCN, OracleGCN, OracleGINE
from eslappe_oracle import OracleGatedGCNESLapPE
from eslappe_util import make_pe
import mp_reference as R

TOL = 1e-12


def _close(a, b, what):
    assert (a is None) == (b is None), what
    if b is None or b.numel() == 0:
        return
    a, b = a.detach(), b.detach()
    err = float((a - b).abs().max() / max(1.0, float(b.abs().max())))
    assert err <= TOL, f"{what}: {err}"


def _batch(d):
    # molecules plus the degenerate cases: self loops, a repeated self loop, duplicate edges, an isolated node, an empty graph
    b = make_batch("zinc-gatedgcn", seed=5, dim=d, num_graphs=3)
    extra = batch_from_lists([4, 0, 3], [[(0, 1), (1, 1), (1, 1), (2, 1), (0, 1)], [], [(0, 2), (2, 0)]], d=d, seed=1)
    n0 = b.x.shape[0]
    ei = torch.cat([b.edge_index, extra.edge_index + n0], dim=1)
    return (torch.cat([b.x, extra.x]).double(), torch.cat([b.edge_attr, extra.edge_attr]).double(), ei)


def _check_grads(out_o, out_s, leaves_o, leaves_s, names, cts):
    for a, b_, n in zip(out_s, out_o, ("out", "out_e")):
        _close(a, b_, n)
    go = torch.autograd.grad(out_o, leaves_o, cts, allow_unused=True)
    gs = torch.autograd.grad(out_s, leaves_s, cts, allow_unused=True)
    for a, b_, n in zip(gs, go, names):
        _close(a, b_, "grad " + n)
    return go


@pytest.mark.parametrize("gate,act", [(False, "relu"), (False, "gelu"), (True, "relu"), (True, "gelu")])
def test_gatedgcn_stages_compose_to_the_oracle(gate, act):
    torch.manual_seed(0)
    d = 16
    x, e, ei = _batch(d)
    src, dst = ei
    ora = (OracleGatedGCNESLapPE if gate else OracleGatedGCN)(d, 0.0, act).double().train()
    pe = make_pe(x.shape[0], 5, 3).double().requires_grad_(True)
    x.requires_grad_(True)
    e.requires_grad_(True)
    mine = copy.deepcopy(ora)
    if gate:
        ora.pe = pe
    out_o = ora(x, e, ei)

    m = mine
    rho = None
    if gate:
        mlp = m.mlp_r_ij
        _, rho = R.eslap_forward(pe, src, dst, mlp[0].weight, mlp[0].bias, mlp[2].weight, mlp[2].bias, act)
    xt, e_ij, _, _ = R.gatedgcn_forward(m.A(x), m.B(x), m.D(x), m.E(x), m.C(e), src, dst, rho)
    act_fn = R.ACTS[act]
    out_s = (x + act_fn(m.bn_node_x(xt)), e + act_fn(m.bn_edge_e(e_ij)))

    g = torch.Generator().manual_seed(1)
    cts = [torch.randn(t.shape, generator=g, dtype=torch.float64) for t in out_o]
    pn = [n for n, _ in ora.named_parameters()]
    names = ["x", "e", "pe"] + pn
    g_ora = _check_grads(out_o, out_s, [x, e, pe] + list(ora.parameters()), [x, e, pe] + list(mine.parameters()),
                         names, cts)

    # the backward references against autograd through the composition: g_Bx, g_Dx, g_Ex, g_e, g_num, g_den, and the
    # gate's grad_pe and mlp_r_ij gradients from g_num / g_den
    Ax, Bx, Dx, Ex, Ce = (t.detach() for t in (m.A(x), m.B(x), m.D(x), m.E(x), m.C(e)))
    leaves = [t.clone().requires_grad_(True) for t in (Bx, Dx, Ex, Ce)]
    xt, e_ij, num, den = R.gatedgcn_forward(Ax, *leaves, src, dst, None if rho is None else rho.detach())
    xt.retain_grad(), e_ij.retain_grad(), num.retain_grad(), den.retain_grad()
    y = (x.detach() + act_fn(copy.deepcopy(m.bn_node_x)(xt)), e.detach() + act_fn(copy.deepcopy(m.bn_edge_e)(e_ij)))
    torch.autograd.backward(y, cts)
    g_xt = xt.grad
    # the BatchNorm_e-path gradient alone: the same composition with the node output cut off
    e_ij2 = e_ij.detach().requires_grad_(True)
    (g_e_bn,) = torch.autograd.grad(e.detach() + act_fn(copy.deepcopy(m.bn_edge_e)(e_ij2)), [e_ij2], [cts[1]])
    ref = R.gatedgcn_backward(Ax, Bx, Dx, Ex, Ce, src, dst, g_xt, g_e_bn, None if rho is None else rho.detach())
    for k, t in (("g_Bx", leaves[0]), ("g_Dx", leaves[1]), ("g_Ex", leaves[2]), ("g_e", leaves[3])):
        _close(ref[k], t.grad, k)
    _close(ref["g_num"], num.grad, "g_num")
    _close(ref["g_den"], den.grad, "g_den")
    if gate:
        mlp = mine.mlp_r_ij
        params = [mlp[0].weight, mlp[0].bias, mlp[2].weight, mlp[2].bias]
        pe2 = pe.detach().clone().requires_grad_(True)
        _, rho2 = R.eslap_forward(pe2, src, dst, *params, act)
        num2, den2 = R.gatedgcn_sums(Bx, e_ij.detach(), src, dst, rho2)
        want = torch.autograd.grad([num2, den2], [pe2] + params, [ref["g_num"], ref["g_den"]])
        got = R.eslap_backward(pe.detach(), src, dst, *(p.detach() for p in params), act, Bx, e_ij.detach(),
                               ref["g_num"], ref["g_den"])
        for k, w in zip(("grad_pe", "gw1", "gb1", "gw2", "gb2"), want):
            _close(got[k], w, k)
        # and the chain through the gate equals the oracle's own gradients of pe and mlp_r_ij
        _close(got["grad_pe"], g_ora[2], "grad_pe vs oracle")


@pytest.mark.parametrize("eps", [0.0, 0.37, -0.5])
def test_gine_stages_compose_to_the_oracle(eps):
    torch.manual_seed(1)
    d = 16
    x, e, ei = _batch(d)
    src, dst = ei
    ora = OracleGINE(d, "gelu").double()
    ora.eps.fill_(eps)
    x.requires_grad_(True)
    e.requires_grad_(True)
    out_o = ora(x, ei, e)
    agg = R.gine_forward(x, e, src, dst, eps)
    out_s = ora.nn(agg)
    g = torch.Generator().manual_seed(2)
    ct = torch.randn(out_o.shape, generator=g, dtype=torch.float64)
    wx, we = _check_grads([out_o], [out_s], [x, e] + list(ora.parameters()), [x, e] + list(ora.parameters()),
                          ["x", "e"] + [n for n, _ in ora.named_parameters()], [ct])[:2]
    # backward reference: g_agg from the nn, then gine_backward; `add` is a second gradient path into x
    agg_l = agg.detach().requires_grad_(True)
    (g_agg,) = torch.autograd.grad(ora.nn(agg_l), [agg_l], [ct])
    add = torch.randn(x.shape, generator=g, dtype=torch.float64)
    g_x, g_e = R.gine_backward(x, e, src, dst, eps, g_agg, add)
    _close(g_x, wx + add, "g_x")
    _close(g_e, we, "g_e")


def test_gcn_stages_compose_to_the_oracle():
    torch.manual_seed(2)
    d = 16
    x, _, ei = _batch(d)
    src, dst = ei
    ora = OracleGCN(d).double()
    with torch.no_grad():
        ora.bias.uniform_(-0.5, 0.5)
    x.requires_grad_(True)
    out_o = ora(x, ei)
    out_s = R.gcn_forward(ora.lin(x), ora.bias, torch.zeros_like(x), src, dst)
    g = torch.Generator().manual_seed(3)
    ct = torch.randn(out_o.shape, generator=g, dtype=torch.float64)
    wx = _check_grads([out_o], [out_s], [x] + list(ora.parameters()), [x] + list(ora.parameters()),
                      ["x"] + [n for n, _ in ora.named_parameters()], [ct])[0]
    Y = ora.lin(x).detach()
    gY = R.gcn_backward(Y, src, dst, ct)
    (wY,) = torch.autograd.grad(R.gcn_forward(Y.requires_grad_(True), ora.bias.detach(), x.detach(), src, dst), [Y], [ct])
    _close(gY, wY, "gY")
    _close(gY @ ora.lin.weight.detach(), wx, "g_x through lin")
    # the degree count: 1 + in-edges from other nodes, each duplicate counted
    deg = R.gcn_dinv(src, dst, x.shape[0]) ** -2
    want = 1 + torch.bincount(dst[src != dst], minlength=x.shape[0]).double()
    assert torch.equal(deg.round(), want)


# ---------------------------------------------------------------------------------------------------- argument contract
P = 1 << 20    # placeholder address: never dereferenced, every call below fails validation first


def _graph(N=8, E=12):
    return _lib.GpsGraph(N, E, 1, P, P, P, P, P, P, P)


def _calls(lib, g, d, null):
    """(name, thunk) for every stage entry point; `null` names the one pointer argument passed as NULL."""
    def a(name):
        return 0 if name == null else P
    nop = C.byref(_lib.GpsPlanes(0, 0, 0))
    return {
        "gps_gatedgcn_aggregate_forward_gated": (
            ["Ax", "Bx", "Dx", "Ex", "Ce", "xt"],
            lambda: lib.gps_gatedgcn_aggregate_forward_gated(C.byref(g), d, a("Ax"), a("Bx"), a("Dx"), a("Ex"), 4 * d,
                                                             a("Ce"), a("xt"), 0, 0, 0, 0)),
        "gps_gatedgcn_aggregate_backward": (
            ["ehat", "Bx", "gY", "g_e", "g_num", "g_den"],
            lambda: lib.gps_gatedgcn_aggregate_backward(C.byref(g), d, a("ehat"), a("Bx"), 4 * d, P, a("gY"), 4 * d,
                                                        a("g_e"), a("g_num"), a("g_den"), nop, nop, 0)),
        "gps_eslap_forward": (
            ["pe", "w1", "b1", "w2", "b2", "r", "rho"],
            lambda: lib.gps_eslap_forward(C.byref(g), a("pe"), 3, d, 0, a("w1"), a("b1"), a("w2"), a("b2"), a("r"),
                                          a("rho"), 0)),
        "gps_eslap_backward": (
            ["pe", "g_num", "g_den", "Bx", "ehat", "r", "rho", "w1", "b1", "w2", "workspace"],
            lambda: lib.gps_eslap_backward(C.byref(g), a("pe"), 3, d, 0, a("g_num"), a("g_den"), a("Bx"), 4 * d,
                                           a("ehat"), a("r"), a("rho"), a("w1"), a("b1"), a("w2"), a("workspace"),
                                           1 << 40, P, P, P, P, P, 0, 0)),
        "gps_gine_aggregate_forward": (
            ["x", "e", "out"],
            lambda: lib.gps_gine_aggregate_forward(C.byref(g), d, a("x"), a("e"), 0.0, a("out"), 0)),
        "gps_gine_aggregate_backward": (
            ["x", "e", "g_out", "g_e", "g_x"],
            lambda: lib.gps_gine_aggregate_backward(C.byref(g), d, a("x"), a("e"), a("g_out"), 0.0, 0, a("g_e"),
                                                    a("g_x"), 0)),
        "gps_gcn_aggregate_forward": (
            ["Y", "bias", "x", "dinv", "xloc"],
            lambda: lib.gps_gcn_aggregate_forward(C.byref(g), d, a("Y"), d, a("bias"), a("x"), a("dinv"), a("xloc"),
                                                  0.0, 1, 0, 0, 0)),
        "gps_gcn_aggregate_backward": (
            ["g_h", "dinv", "gY"],
            lambda: lib.gps_gcn_aggregate_backward(C.byref(g), d, a("g_h"), a("dinv"), a("gY"), d, nop, 0)),
    }


def _entry_points():
    return list(_calls(None, _graph(), 8, None))


@pytest.mark.parametrize("name", _entry_points())
def test_stage_entry_points_reject_null_pointers(name):
    lib = _lib.load()
    g = _graph()
    ptrs, _ = _calls(lib, g, 8, None)[name]
    for p in ptrs:
        rc = _calls(lib, g, 8, p)[name][1]()
        assert rc == _lib.GPS_ERR_ARG, (name, p, rc)
        assert lib.gps_last_error()


@pytest.mark.parametrize("name", _entry_points())
@pytest.mark.parametrize("d", [6, 4100, 0])
def test_stage_entry_points_reject_unsupported_widths(name, d):
    lib = _lib.load()
    rc = _calls(lib, _graph(), d, None)[name][1]()
    assert rc == _lib.GPS_ERR_UNSUPPORTED, (name, d, rc)


def test_eslap_workspace_bytes():
    lib = _lib.load()
    assert lib.gps_eslap_workspace_bytes(0, 64) == 0
    # gz, gr [E] and one part row [3d + 1] per chunk of max(32, ceil(E / 132)) edges
    assert lib.gps_eslap_workspace_bytes(10, 64) == 4 * (2 * 10 + 1 * 193)
    E = 132 * 32 + 1     # chunks of 33 edges: 128 full ones and a last one of 1 edge
    assert lib.gps_eslap_workspace_bytes(E, 8) == 4 * (2 * E + 129 * 25)
