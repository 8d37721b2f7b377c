"""CPU: the PNA local model's oracles, parameter layout and argument contract (tests/pna_oracle.py)."""
import ctypes as C
import os

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from pna_oracle import PNAConvLoop, PNAConvMP, pna_batch, pna_conv, pna_oracle_layer, tie_edge
from local_model_harness import _args, _planes, _plan, _r
from util import GOLDEN_DIR, golden_batch

PNA_DIR = os.path.join(GOLDEN_DIR, "pna")
GLOBALS = ("Transformer", "BiasedTransformer", "Performer", "None")
DEG = [0, 3, 11, 9, 4, 1]


def _load(name):
    return torch.load(os.path.join(PNA_DIR, name + ".pt"), weights_only=False)


def _pair(d, seed):
    torch.manual_seed(seed)
    mp = pna_conv(PNAConvMP, d, DEG).double()
    lp = pna_conv(PNAConvLoop, d, DEG).double()
    lp.load_state_dict(mp.state_dict(), strict=True)
    return mp, lp


def test_batch_has_the_special_structures():
    b = pna_batch("zinc-gine", 3, 16, 5, dtype=torch.float64)
    src, dst = b.edge_index
    deg = torch.bincount(dst, minlength=b.num_nodes)
    assert bool((src == dst).any())                                        # self loops
    pairs = src * b.num_nodes + dst
    assert pairs.unique().numel() < pairs.numel()                          # duplicates
    assert int(deg.max()) >= 40                                            # hub
    assert bool((deg == 0).any())                                          # isolated node
    k, last = tie_edge(b), b.edge_index.shape[1] - 1                       # the exact duplicate
    assert torch.equal(b.edge_index[:, k], b.edge_index[:, last]) and torch.equal(b.edge_attr[k], b.edge_attr[last])
    assert int(deg[dst[k]]) >= 3
    assert pna_batch("zinc-gine", 3, 160, 2).edge_attr.shape[1] == 128    # de = min(128, d)


@pytest.mark.parametrize("d", [16, 36, 132])
def test_restatements_agree(d):
    b = pna_batch("zinc-gine", 3, d, 4, dtype=torch.float64)
    mp, lp = _pair(d, 1)
    ct = torch.randn(b.num_nodes, d, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    res = []
    for m in (mp, lp):
        x, e = b.x.clone().requires_grad_(True), b.edge_attr.clone().requires_grad_(True)
        o = m(x, b.edge_index, e)
        res.append([o] + list(torch.autograd.grad((o * ct).sum(), [x, e] + list(m.parameters()))))
    for a, r in zip(*res):
        assert float((a - r).detach().abs().max()) <= 1e-12 * max(1.0, float(r.detach().abs().max()))
    agg = mp.aggregate(b.x, b.edge_index, b.edge_attr)
    iso = torch.bincount(b.edge_index[1], minlength=b.num_nodes) == 0
    assert bool((agg[iso] == 0).all())


def test_max_gradient_goes_to_the_first_tied_edge():
    """The exact duplicate ties its original in every channel: where the pair holds the segment max, the whole max
    gradient lands on the lower edge id and none on the copy; the mean and sum shares are equal for both."""
    d = 16
    b = pna_batch("zinc-gine", 3, d, 4, dtype=torch.float64)
    k, last = tie_edge(b), b.edge_index.shape[1] - 1
    for cls in (PNAConvMP, PNAConvLoop):
        m = pna_conv(cls, d, DEG).double()
        gz = torch.zeros(b.num_nodes, 3 * d, dtype=torch.float64)
        t = int(b.edge_index[1, k])
        gz[t, d:2 * d] = 1.0            # the max block of the tied pair's target only
        pre = m.pre_nns[0][0]
        # each edge's message gradient g_m, read off its edge_attr gradient g_e = g_m W_e W_enc (W_e W_enc invertible)
        e = b.edge_attr.clone().requires_grad_(True)
        agg = m.aggregate(b.x, b.edge_index, e)
        (agg * gz).sum().backward()
        W = pre.weight[:, 2 * d:] @ m.edge_encoder.weight
        gm = torch.linalg.solve(W.t().detach(), e.grad.t()).t()   # [E, d]
        assert float(gm[last].abs().max()) < 1e-9, cls
        msgs = m.pre_nns[0](torch.cat([b.x[b.edge_index[1]], b.x[b.edge_index[0]],
                                       m.edge_encoder(b.edge_attr)], -1)).detach()
        held = msgs[k] == msgs[b.edge_index[1] == t].max(0).values
        assert bool(held.any())
        assert torch.allclose(gm[k][held], torch.ones(int(held.sum()), dtype=torch.float64), atol=1e-9)


def test_oracle_equals_reference_live_pna():
    """The oracle layer (per-node loop PNA) against the reference's gps_layer.py run verbatim with the message-passing
    PNAConv, fp64: outputs 1e-10, gradients (grad_edge_attr and every local_model.* included) 1e-9, running stats."""
    fix = _load("reference_live_PNA_Transformer")
    cfg = fix["config"]
    ora = pna_oracle_layer(cfg["d"], cfg["glob"], cfg["heads"], cfg["pna_degrees"]).double()
    ora.load_state_dict(fix["state"], strict=True)
    b = golden_batch(fix, dtype=torch.float64)
    b.x.requires_grad_(True)
    b.edge_attr.requires_grad_(True)
    x, e = b.x, b.edge_attr
    out = ora.train()(b)
    (out.x * fix["ct_x"]).sum().backward()
    assert float((out.x - fix["out_x"]).abs().max()) < 1e-10
    assert float((x.grad - fix["grad_x"]).abs().max()) < 1e-9
    assert float((e.grad - fix["grad_e"]).abs().max()) < 1e-9
    got = dict(ora.named_parameters())
    for p in ("edge_encoder", "pre_nns.0.0", "post_nns.0.0", "lin"):
        assert f"local_model.{p}.weight" in fix["grad_params"], p
    for n, g in fix["grad_params"].items():
        assert float((got[n].grad - g).abs().max()) < 1e-9, n
    st = ora.state_dict()
    for n, v in fix["state_after"].items():
        assert torch.equal(st[n], v) if not v.is_floating_point() else float((st[n] - v).abs().max()) < 1e-12, n


def _pna_keys(d):
    de = min(128, d)
    return {"local_model.edge_encoder.weight": (d, de), "local_model.edge_encoder.bias": (d,),
            "local_model.pre_nns.0.0.weight": (d, 3 * d), "local_model.pre_nns.0.0.bias": (d,),
            "local_model.post_nns.0.0.weight": (d, 4 * d), "local_model.post_nns.0.0.bias": (d,),
            "local_model.lin.weight": (d, d), "local_model.lin.bias": (d,)}


@pytest.mark.parametrize("name", ["pna_transformer_relu", "pna_transformer_nonorm", "pna_performer_relu",
                                  "pna_none_relu", "pna_biased_relu"])
def test_state_dict_matches_reference(name):
    """Keys and shapes equal those of the module the reference built for the fixture; strict loads both ways."""
    fix = _load(name)
    cfg = fix["config"]
    ours = graphgps_b200.GPSLayer(cfg["d"], "PNA", cfg["glob"], cfg["heads"], act=cfg["act"],
                                  pna_degrees=cfg["pna_degrees"], batch_norm=cfg["batch_norm"])
    so, sr = ours.state_dict(), fix["state"]
    assert set(so) == set(sr)
    for k in so:
        assert so[k].shape == sr[k].shape, k
    local = {k: tuple(v.shape) for k, v in so.items() if k.startswith("local_model.")}
    assert local == _pna_keys(cfg["d"])
    assert not list(ours.local_model.buffers())
    ours.load_state_dict(sr, strict=True)
    ora = pna_oracle_layer(cfg["d"], cfg["glob"], cfg["heads"], cfg["pna_degrees"], act=cfg["act"],
                           batch_norm=cfg["batch_norm"])
    ora.load_state_dict(ours.state_dict(), strict=True)
    for k, v in ora.state_dict().items():
        assert torch.equal(v, sr[k]), k


def test_state_dict_matches_live_reference_module():
    from oracle.ref_shim import find_reference_layer_dir, load_reference
    if find_reference_layer_dir() is None:
        pytest.skip("reference layer files not present (the fixtures pin the same layout)")
    from pna_oracle import shim_pna
    ref = load_reference()
    for d, glob in ((32, "Transformer"), (160, "None")):
        with shim_pna():
            r = ref.GPSLayer(d, "PNA", glob, 4, pna_degrees=DEG)
        ours = graphgps_b200.GPSLayer(d, "PNA", glob, 4, pna_degrees=DEG)
        sr, so = r.state_dict(), ours.state_dict()
        assert {k: tuple(v.shape) for k, v in sr.items()} == {k: tuple(v.shape) for k, v in so.items()}
        ours.load_state_dict(sr, strict=True)
        r.load_state_dict(ours.state_dict(), strict=True)


@pytest.mark.parametrize("glob", GLOBALS)
@pytest.mark.parametrize("batch_norm", [True, False])
def test_constructs_under_every_global_model(glob, batch_norm):
    layer = graphgps_b200.GPSLayer(64, "PNA", glob, 4, pna_degrees=DEG, batch_norm=batch_norm)
    assert layer.local_model.edge_dim == 64
    assert ("norm1_local.weight" in layer.state_dict()) == batch_norm
    assert graphgps_b200.GPSLayer(304, "PNA", glob, 4, pna_degrees=DEG).local_model.edge_dim == 128


def test_constructor_error_contract():
    G = graphgps_b200.GPSLayer
    for bad in (None, [], [0, 0, 0], [1, -1, 3], torch.zeros(4, dtype=torch.int64)):
        with pytest.raises(NotImplementedError, match="PNA"):
            G(64, "PNA", "Transformer", 4, pna_degrees=bad)
    with pytest.raises(NotImplementedError, match="equivstable_pe"):
        G(64, "PNA", "Transformer", 4, pna_degrees=DEG, equivstable_pe=True)
    G(64, "PNA", "Transformer", 4, pna_degrees=torch.tensor(DEG))   # a tensor histogram is accepted
    with pytest.raises(NotImplementedError):
        G(64, "GIN", "Transformer", 4)


def test_reference_rejects_what_the_constructor_rejects():
    """The reference fails on the histograms the constructor refuses: TypeError for None, ZeroDivisionError for an empty
    or all-zero one (PyG 2.2's average degrees); equivstable_pe=True fails at PNAConv.forward."""
    import numpy as np
    with pytest.raises(TypeError):
        torch.from_numpy(np.array(None))
    for bad in ([], [0, 0]):
        with pytest.raises(ZeroDivisionError):
            pna_conv(PNAConvMP, 8, torch.from_numpy(np.array(bad, dtype=np.int64)))
    m = pna_conv(PNAConvMP, 8, DEG)
    with pytest.raises(TypeError):
        m(torch.zeros(2, 8), torch.zeros(2, 0, dtype=torch.int64), torch.zeros(0, 8), torch.zeros(2, 3))


def test_dp_groups():
    from graphgps_b200.dp import LATE, MID, _group
    for n in _pna_keys(8):
        want = LATE if n.startswith(("local_model.pre_nns.", "local_model.lin.")) else MID
        assert _group(n) == want, n


@pytest.mark.parametrize("N,E,d,glob,norm,prec", [(10, 20, 64, "Transformer", "batch", "fp32"),
                                                  (1000, 5000, 304, "None", "batch", "bf16"),
                                                  (7, 0, 64, "Transformer", "none", "fp32"),
                                                  (33, 80, 36, "Performer", "batch", "fp32")])
def test_plan_size_deltas_against_gine(N, E, d, glob, norm, prec):
    """PNA against GINE (relu), sized with edge_dim = d (the bound):
    saved   + F [d,d], c [d]; arg, h [N,d] instead of agg, h1; planes of e [E,d] (both), F [d,d], Z [N,4d], h [N,d]
            instead of agg, h1 (Z in fp32 without planes); Wcat / bcat / Y1 and their planes grow by 2d rows; weight
            planes of post [d,4d] / lin [d,d] instead of nn.0 / nn.2 (also in wplanes_bytes)
    forward + q [E,d]
    backward + g_Z [N,4d], g_q [E,d] (+ planes), g_F | g_c [d*d + d]; g_h, g_xl as GINE's g_h1, g_xl, no g_agg;
            gY1, gWcat | gbcat and gY1's planes grow by 2d columns"""
    lo = prec == "fp32"
    f = 4
    a_pna, a_gine = _args("PNA", N, E, d, 4, glob, norm), _args("GINE", N, E, d, 4, glob, norm)
    for a in (a_pna, a_gine):
        a.precision = _lib.PRECISION[prec]
        if glob == "Performer":
            a.perf_features, a.perf_dim_head = 266, 64
    rc, pp = _plan(a_pna)
    rc2, pi = _plan(a_gine)
    assert rc == 0 and rc2 == 0
    planes = d % 8 == 0
    P = (lambda rows, cols: _planes(rows, cols, lo) if rows or cols else 0) if planes else (lambda rows, cols: 0)
    wy0 = 3 * d if glob == "Transformer" else 0
    wy1 = wy0 + 2 * d
    Pw = lambda wy: P(wy, d) if wy else 0
    wdelta = Pw(wy1) - Pw(wy0) + P(d, 4 * d) - P(d, d)
    wcat = (_r(f * wy1 * d) - _r(f * wy0 * d) + _r(f * wy1) - _r(f * wy0) + _r(f * N * wy1) - _r(f * N * wy0))
    saved = (_r(f * d * d) + _r(f * d) + P(d, d) + P(N, 4 * d) - P(N, d) + wcat + wdelta
             + (0 if planes else _r(f * N * 4 * d)))
    assert pp.saved_bytes - pi.saved_bytes == saved
    assert pp.wplanes_bytes - pi.wplanes_bytes == wdelta
    assert pp.fwd_workspace_bytes - pi.fwd_workspace_bytes == _r(f * E * d)
    Pg = lambda wy: P(N, wy) if wy else 0
    bwd = (_r(f * N * 4 * d) + _r(f * E * d) + _r(f * (d * d + d)) - _r(f * N * d) + P(E, d)
           + _r(f * N * wy1) - _r(f * N * wy0) + _r(f * (wy1 * d + wy1)) - _r(f * (wy0 * d + wy0)) + Pg(wy1) - Pg(wy0))
    assert pp.bwd_workspace_bytes - pi.bwd_workspace_bytes == bwd


def _full_pna(de=64):
    pna = _lib.GpsPna()
    for lin in (pna.edge_encoder, pna.pre, pna.post, pna.lin):
        lin.weight = lin.bias = 8
    pna.edge_dim = de
    return pna


def _err():
    return _lib.load().gps_last_error().decode()


def test_error_contract_before_any_cuda_call():
    """Every case below returns before the library enqueues anything (the pointers are not device memory)."""
    lib = _lib.load()
    ARG, UNS = _lib.GPS_ERR_ARG, _lib.GPS_ERR_UNSUPPORTED
    a = _args("PNA")
    a.x, a.edge_attr, a.x_out, a.saved, a.saved_bytes, a.workspace, a.workspace_bytes = 8, 8, 8, 8, 1 << 40, 8, 1 << 40
    a.grad_x_out, a.grad_x = 8, 8
    for lin in (a.attn_in, a.attn_out, a.ff1, a.ff2):   # the rest of the layer is complete
        lin.weight = lin.bias = 8
    for bn in (a.norm1_local, a.norm1_attn, a.norm2):
        bn.weight = bn.bias = 8
    # NULL parameters one at a time
    for s, what in (("edge_encoder", "edge_encoder"), ("pre", "pre_nns"), ("post", "post_nns"), ("lin", "local_model.lin")):
        for f in ("weight", "bias"):
            a.pna = _full_pna()
            setattr(getattr(a.pna, s), f, 0)
            for fn in (lib.gps_layer_forward, lib.gps_layer_backward):
                assert fn(C.byref(a), None) == ARG, (s, f)
                assert what in _err(), (s, f, _err())
    a.pna = _full_pna()
    # edge_attr / grad_edge_attr with E > 0
    a.edge_attr = 0
    assert lib.gps_layer_forward(C.byref(a), None) == ARG and "edge_attr" in _err()
    a.edge_attr = 8
    a.grad_edge_attr = 0
    assert lib.gps_layer_backward(C.byref(a), None) == ARG
    assert "grad_edge_attr" in _err()
    # an attention bias needs the Transformer
    n = _args("PNA", glob="None")
    n.pna, n.attn_bias = _full_pna(), _lib.GpsAttnBias(8, 4, 0)
    assert lib.gps_layer_forward(C.byref(n), None) == ARG and "GPS_GLOBAL_TRANSFORMER" in _err()
    # edge widths: 0 < edge_dim <= d, edge_dim % 4 == 0 (0: the GpsPna left empty)
    for de in (0, -4, 6, 68):
        a.pna = _full_pna(de)
        assert lib.gps_layer_forward(C.byref(a), None) == UNS, de
        assert lib.gps_layer_backward(C.byref(a), None) == UNS, de
    assert _plan(_args("PNA", d=66, glob="None"))[0] == UNS
    # stage entry points
    g = _lib.GpsGraph()
    g.N, g.E = 4, 4
    fold = [8, 8, 8, 8, 64, 32, 8, 8, None]
    for i in (0, 1, 2, 3, 6, 7):
        args = list(fold)
        args[i] = None
        assert lib.gps_pna_fold_forward(*args) == ARG, i
    assert lib.gps_pna_fold_forward(*fold[:5], 30, *fold[6:]) == UNS
    assert lib.gps_pna_fold_forward(*fold[:5], 68, *fold[6:]) == UNS
    unfold = [8, 8, 8, 8, 8, 64, 32, None, None, None, None, 0, None]
    for i in (0, 1, 2, 3, 4):
        args = list(unfold)
        args[i] = None
        assert lib.gps_pna_fold_backward(*args) == ARG, i
    assert lib.gps_pna_fold_backward(*unfold[:6], 0, *unfold[7:]) == UNS
    fw = [C.byref(g), 64, 8, 8, 128, 8, 8, 8, None]
    for i in (0, 2, 3, 5, 6, 7):
        args = list(fw)
        args[i] = None
        assert lib.gps_pna_aggregate_forward(*args) == ARG, i
    assert lib.gps_pna_aggregate_forward(*fw[:4], 64, *fw[5:]) == ARG   # ldy < 2d
    assert lib.gps_pna_aggregate_forward(fw[0], 6, *fw[2:]) == UNS
    bw = [C.byref(g), 64, 8, 8, None, 8, 8, 128, 8, None]
    for i in (0, 2, 3, 5, 6, 8):
        args = list(bw)
        args[i] = None
        assert lib.gps_pna_aggregate_backward(*args) == ARG, i
    assert lib.gps_pna_aggregate_backward(bw[0], 8192, *bw[2:]) == UNS
