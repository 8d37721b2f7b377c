"""CPU: the GENConv local model's oracles, parameter layout and argument contract (tests/genconv_oracle.py)."""
import ctypes as C
import math
import os

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from genconv_oracle import GENConvLoop, GENConvMP, dead_node, genconv_batch, genconv_oracle_layer
from local_model_harness import _args, _planes, _plan, _r
from util import GOLDEN_DIR, golden_batch

GEN_DIR = os.path.join(GOLDEN_DIR, "genconv")
GLOBALS = ("Transformer", "BiasedTransformer", "Performer", "None")


def _load(name):
    return torch.load(os.path.join(GEN_DIR, name + ".pt"), weights_only=False)


def _pair(d, seed):
    torch.manual_seed(seed)
    mp = GENConvMP(d, d).double()
    with torch.no_grad():
        bn = mp.mlp[1]
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.3, 0.3)
    lp = GENConvLoop(d, d).double()
    lp.load_state_dict(mp.state_dict(), strict=True)
    return mp, lp


def test_batch_has_the_special_structures():
    b = genconv_batch("zinc-gine", 3, 16, 5, dtype=torch.float64)
    src, dst = b.edge_index
    deg = torch.bincount(dst, minlength=b.num_nodes)
    assert bool((src == dst).any())                                        # self loops
    pairs = src * b.num_nodes + dst
    assert pairs.unique().numel() < pairs.numel()                          # duplicates
    assert int(deg.max()) >= 40                                            # hub
    assert bool((deg == 0).any())                                          # isolated node
    k = dst == dead_node(b)
    assert bool(k.any()) and bool(((b.x[src[k]] + b.edge_attr[k]) <= 0).all())   # all messages 1e-7


@pytest.mark.parametrize("d", [16, 36])
@pytest.mark.parametrize("training", [True, False])
def test_restatements_agree(d, training):
    b = genconv_batch("zinc-gine", 3, d, 5, dtype=torch.float64)
    mp, lp = _pair(d, 1)
    ct = torch.randn(b.num_nodes, d, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    res = []
    for m in (mp, lp):
        m.train(training)
        x, e = b.x.clone().requires_grad_(True), b.edge_attr.clone().requires_grad_(True)
        o = m(x, b.edge_index, e)
        res.append([o] + list(torch.autograd.grad((o * ct).sum(), [x, e] + list(m.parameters()))))
    for a, r in zip(*res):
        assert float((a - r).detach().abs().max()) <= 1e-12 * max(1.0, float(r.detach().abs().max()))
    # the aggregations themselves, the all-1e-7 node and the isolated node
    agg = mp.aggregate(b.x, b.edge_index, b.edge_attr)
    assert float((agg - lp.aggregate(b.x, b.edge_index, b.edge_attr)).abs().max()) <= 1e-12 * float(agg.abs().max())
    assert torch.allclose(agg[dead_node(b)], torch.full((d,), 1e-7, dtype=torch.float64), rtol=1e-12, atol=0)
    iso = torch.bincount(b.edge_index[1], minlength=b.num_nodes) == 0
    assert bool((agg[iso] == 0).all())
    # an edge into the all-1e-7 node gets no gradient (ReLU's derivative at <= 0 is 0)
    k = b.edge_index[1] == dead_node(b)
    assert bool((res[0][2][k] == 0).all()) and bool((res[1][2][k] == 0).all())


def test_four_node_example_matches_hand_computed_alpha():
    """Edges 1->0, 2->0, 0->0 (an ordinary edge), 3->1 with d = 2 and edge_attr 0: node 0's messages are relu(x_1),
    relu(x_2), relu(x_0) (+1e-7), node 1's relu(x_3), nodes 2 and 3 get 0."""
    m = GENConvMP(2, 2).double()
    x = torch.tensor([[-1.0, 5.0], [2.0, 1.0], [0.5, -3.0], [1.0, 7.0]], dtype=torch.float64)
    ei = torch.tensor([[1, 2, 0, 3], [0, 0, 0, 1]])
    agg = m.aggregate(x, ei, torch.zeros(4, 2, dtype=torch.float64))
    eps = 1e-7
    for c, msgs in ((0, [2.0, 0.5, 0.0]), (1, [1.0, 0.0, 5.0])):
        mm = [v + eps for v in msgs]
        w = [math.exp(v) for v in mm]
        alpha = [v / sum(w) for v in w]
        assert abs(float(agg[0, c]) - sum(a * v for a, v in zip(alpha, mm))) < 1e-14
    assert torch.allclose(agg[1], torch.tensor([1.0 + eps, 7.0 + eps], dtype=torch.float64), atol=1e-15)
    assert bool((agg[2:] == 0).all())
    # channel 0 of node 0 by hand: alpha = (e^2, e^0.5, e^0) / (e^2 + e^0.5 + 1)
    s = math.exp(2.0) + math.exp(0.5) + 1.0
    assert abs(float(agg[0, 0]) - (2.0 * math.exp(2.0) + 0.5 * math.exp(0.5)) / s) < 1e-6


def test_oracle_equals_reference_live_genconv():
    """The oracle layer (per-node loop GENConv) against the reference's gps_layer.py run verbatim with the
    message-passing GENConv, fp64: outputs 1e-10, gradients (grad_edge_attr and mlp.* included) 1e-9, running stats."""
    fix = _load("reference_live_GENConv_Transformer")
    cfg = fix["config"]
    ora = genconv_oracle_layer(cfg["d"], cfg["glob"], cfg["heads"]).double()
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
    assert any(n.startswith("local_model.mlp.") for n in fix["grad_params"])
    for n, g in fix["grad_params"].items():
        assert float((got[n].grad - g).abs().max()) < 1e-9, n
    st = ora.state_dict()
    for n, v in fix["state_after"].items():
        assert torch.equal(st[n], v) if not v.is_floating_point() else float((st[n] - v).abs().max()) < 1e-12, n


def _genconv_keys(d):
    return {"local_model.mlp.0.weight": (2 * d, d), "local_model.mlp.1.weight": (2 * d,),
            "local_model.mlp.1.bias": (2 * d,), "local_model.mlp.1.running_mean": (2 * d,),
            "local_model.mlp.1.running_var": (2 * d,), "local_model.mlp.1.num_batches_tracked": (),
            "local_model.mlp.4.weight": (d, 2 * d)}


@pytest.mark.parametrize("name", ["genconv_transformer_relu", "genconv_transformer_nonorm", "genconv_performer_relu",
                                  "genconv_none_relu", "genconv_biased_relu"])
def test_state_dict_matches_reference(name):
    """Keys and shapes equal those of the module the reference built for the fixture; strict loads both ways."""
    fix = _load(name)
    cfg = fix["config"]
    ours = graphgps_b200.GPSLayer(cfg["d"], "GENConv", cfg["glob"], cfg["heads"], act=cfg["act"],
                                  batch_norm=cfg["batch_norm"])
    so, sr = ours.state_dict(), fix["state"]
    assert set(so) == set(sr)
    for k in so:
        assert so[k].shape == sr[k].shape, k
    local = {k: tuple(v.shape) for k, v in so.items() if k.startswith("local_model.")}
    assert local == _genconv_keys(cfg["d"])
    ours.load_state_dict(sr, strict=True)
    ora = genconv_oracle_layer(cfg["d"], cfg["glob"], cfg["heads"], act=cfg["act"], batch_norm=cfg["batch_norm"])
    ora.load_state_dict(ours.state_dict(), strict=True)
    for k, v in ora.state_dict().items():
        assert torch.equal(v, sr[k]), k


def test_state_dict_matches_live_reference_module():
    from oracle.ref_shim import find_reference_layer_dir, load_reference
    if find_reference_layer_dir() is None:
        pytest.skip("reference layer files not present (the fixtures pin the same layout)")
    from genconv_oracle import shim_genconv
    ref = load_reference()
    for glob in ("Transformer", "None"):
        with shim_genconv():
            r = ref.GPSLayer(32, "GENConv", glob, 4)
        ours = graphgps_b200.GPSLayer(32, "GENConv", glob, 4)
        sr, so = r.state_dict(), ours.state_dict()
        assert {k: tuple(v.shape) for k, v in sr.items()} == {k: tuple(v.shape) for k, v in so.items()}
        ours.load_state_dict(sr, strict=True)
        r.load_state_dict(ours.state_dict(), strict=True)


@pytest.mark.parametrize("glob", GLOBALS)
@pytest.mark.parametrize("batch_norm", [True, False])
def test_constructs_under_every_global_model(glob, batch_norm):
    layer = graphgps_b200.GPSLayer(64, "GENConv", glob, 4, batch_norm=batch_norm)
    assert isinstance(layer.local_model.mlp[2], torch.nn.ReLU)
    assert layer.local_model.mlp[0].bias is None and layer.local_model.mlp[4].bias is None
    assert ("norm1_local.weight" in layer.state_dict()) == batch_norm
    gelu = graphgps_b200.GPSLayer(64, "GENConv", glob, 4, act="gelu", batch_norm=batch_norm)
    assert isinstance(gelu.local_model.mlp[2], torch.nn.ReLU)   # the MLP's ReLU does not follow gnn.act


def test_equivstable_pe_raises():
    with pytest.raises(NotImplementedError, match="size"):
        graphgps_b200.GPSLayer(64, "GENConv", "Transformer", 4, equivstable_pe=True)


def test_gin_stays_unbuilt():
    with pytest.raises(NotImplementedError):
        graphgps_b200.GPSLayer(64, "GIN", "Transformer", 4)


def test_mlp_gradients_are_mid():
    from graphgps_b200.dp import MID, _group
    for n in _genconv_keys(8):
        if "running" not in n and "num_batches" not in n:
            assert _group(n) == MID, n


def test_check_params_covers_mlp1_buffers():
    """The library reads mlp.1's running statistics through raw pointers: a CPU (or non-fp32) buffer is refused."""
    layer = graphgps_b200.GPSLayer(16, "GENConv", "None", 4)
    with pytest.raises(TypeError, match=r"local_model\.mlp\.1\.running_mean"):
        layer._check_params({})   # parameters checked elsewhere: only the buffers here


@pytest.mark.parametrize("N,E,d,glob,norm,prec", [(10, 20, 64, "Transformer", "batch", "fp32"),
                                                  (1000, 5000, 304, "None", "batch", "bf16"),
                                                  (7, 0, 64, "Transformer", "none", "fp32"),
                                                  (33, 80, 36, "Performer", "batch", "fp32")])
def test_plan_size_deltas_against_gine(N, E, d, glob, norm, prec):
    """GENConv against GINE (relu, so GINE saves no pre-activation):
    saved   + lse, u [N,d], h1, r [N,2d], mlp.1's statistics slot [4d]; planes of u and r instead of agg, h1 and edge_attr;
            weight planes of mlp.0 [2d,d] / mlp.4 [d,2d] instead of nn.0 / nn.2 [d,d] (also in wplanes_bytes)
    forward + mlp.1's column sums [2][2d] doubles
    backward + mlp.1's column sums, g_r, g_h1 [N,2d], g_u [N,d] instead of GINE's g_h1, g_agg [N,d]; g_h1's planes are
            [N,2d] instead of [N,d]"""
    lo = prec == "fp32"
    f = 4
    a_gen, a_gine = _args("GENConv", N, E, d, 4, glob, norm), _args("GINE", N, E, d, 4, glob, norm)
    for a in (a_gen, a_gine):
        a.precision = _lib.PRECISION[prec]
        if glob == "Performer":
            a.perf_features, a.perf_dim_head = 266, 64
    rc, pg = _plan(a_gen)
    rc2, pi = _plan(a_gine)
    assert rc == 0 and rc2 == 0
    planes = d % 8 == 0
    P = (lambda rows, cols: _planes(rows, cols, lo)) if planes else (lambda rows, cols: 0)
    wdelta = P(2 * d, d) + P(d, 2 * d) - 2 * P(d, d)
    saved = (_r(f * N * d) + 2 * _r(f * N * 2 * d) + _r(f * 4 * d) + P(N, d) + P(N, 2 * d)
             - P(E, d) - 2 * P(N, d) + wdelta)
    assert pg.saved_bytes - pi.saved_bytes == saved
    assert pg.wplanes_bytes - pi.wplanes_bytes == wdelta
    assert pg.fwd_workspace_bytes - pi.fwd_workspace_bytes == _r(8 * 4 * d)
    bwd = _r(8 * 4 * d) + 2 * _r(f * N * 2 * d) + _r(f * N * d) - 2 * _r(f * N * d) + P(N, 2 * d) - P(N, d)
    assert pg.bwd_workspace_bytes - pi.bwd_workspace_bytes == bwd


def test_plan_width_limits():
    assert _plan(_args("GENConv", d=2048, glob="None"))[0] == 0
    assert _plan(_args("GENConv", d=2052, glob="None"))[0] == _lib.GPS_ERR_UNSUPPORTED
    assert _plan(_args("GENConv", d=66, glob="None"))[0] == _lib.GPS_ERR_UNSUPPORTED
    assert _plan(_args("GINE", d=2052, glob="None"))[0] == 0   # the limit is GENConv's own


def _full_gen():
    gen = _lib.GpsGenConv()
    gen.lin0.weight = gen.lin1.weight = 8
    gen.bn.weight = gen.bn.bias = gen.bn.running_mean = gen.bn.running_var = 8
    return gen


def _err():
    return _lib.load().gps_last_error().decode()


def test_error_contract_before_any_cuda_call():
    """Every case below returns before the library enqueues anything (the pointers are not device memory)."""
    lib = _lib.load()
    ARG, UNS = _lib.GPS_ERR_ARG, _lib.GPS_ERR_UNSUPPORTED
    a = _args("GENConv")
    a.x, a.edge_attr, a.x_out, a.saved, a.saved_bytes, a.workspace, a.workspace_bytes = 8, 8, 8, 8, 1 << 40, 8, 1 << 40
    a.grad_x_out, a.grad_x = 8, 8
    for lin in (a.attn_in, a.attn_out, a.ff1, a.ff2):   # the rest of the layer is complete
        lin.weight = lin.bias = 8
    for bn in (a.norm1_local, a.norm1_attn, a.norm2):
        bn.weight = bn.bias = 8
    # NULL parameters: all of them, then one at a time
    assert lib.gps_layer_forward(C.byref(a), None) == ARG and "local_model.mlp.0" in _err()
    assert lib.gps_layer_backward(C.byref(a), None) == ARG and "local_model.mlp.0" in _err()
    for field, what in (("lin0.weight", "mlp.0"), ("bn.weight", "mlp.1"), ("bn.bias", "mlp.1"),
                        ("bn.running_mean", "mlp.1.running"), ("bn.running_var", "mlp.1.running"),
                        ("lin1.weight", "mlp.4")):
        a.genconv = _full_gen()
        s, f = field.split(".")
        setattr(getattr(a.genconv, s), f, 0)
        for fn in (lib.gps_layer_forward, lib.gps_layer_backward):
            assert fn(C.byref(a), None) == ARG, field
            assert what in _err(), (field, _err())
    a.genconv = _full_gen()
    # edge_attr / grad_edge_attr with E > 0
    a.edge_attr = 0
    assert lib.gps_layer_forward(C.byref(a), None) == ARG and "edge_attr" in _err()
    a.edge_attr = 8
    a.grad_edge_attr = 0
    assert lib.gps_layer_backward(C.byref(a), None) == ARG
    assert "grad_edge_attr" in _err()
    # an attention bias needs the Transformer
    n = _args("GENConv", glob="None")
    n.genconv, n.attn_bias = _full_gen(), _lib.GpsAttnBias(8, 4, 0)
    assert lib.gps_layer_forward(C.byref(n), None) == ARG and "GPS_GLOBAL_TRANSFORMER" in _err()
    # widths
    for d in (66, 2052):
        w = _args("GENConv", d=d, H=2)
        w.x, w.edge_attr, w.x_out, w.saved, w.workspace = 8, 8, 8, 8, 8
        w.genconv = _full_gen()
        assert lib.gps_layer_forward(C.byref(w), None) == UNS
    # stage entry points
    g = _lib.GpsGraph()
    g.N, g.E = 4, 4
    fw = [C.byref(g), 64, 8, 8, 8, 8, 8, None]
    for i in (0, 2, 3, 4, 5, 6):
        args = list(fw)
        args[i] = None
        assert lib.gps_genconv_aggregate_forward(*args) == ARG, i
    assert lib.gps_genconv_aggregate_forward(fw[0], 6, *fw[2:]) == UNS
    assert lib.gps_genconv_aggregate_forward(fw[0], 8192, *fw[2:]) == UNS
    bw = [C.byref(g), 64, 8, 8, 8, 8, 8, None, 8, 8, None]
    for i in (0, 2, 3, 4, 5, 6, 8, 9):
        args = list(bw)
        args[i] = None
        assert lib.gps_genconv_aggregate_backward(*args) == ARG, i
    assert lib.gps_genconv_aggregate_backward(bw[0], 6, *bw[2:]) == UNS
