"""GPU: the BiasedTransformer attention bias (gps_layer.py:202-204) in the attention kernels and the layer.

Stages against a float64 torch restatement of dense per-graph attention with the bias added to the scaled scores: the
CUDA-core forward and backward (grad_bias included, exactly 0 at padded entries, bitwise equal in two runs) and the
wgmma forward on batches of large graphs.  The layer against the reference's own fp64 fixtures (tests/golden/biased/),
a finite-difference check with attention dropout along x and attn_bias, and a captured 10-layer GPSStack whose
attn_bias gradient is the sum over the layers."""
import ctypes as C

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import batch_from_lists, make_batch
from graphgps_b200.graph import graph_of
from attention_reference import padded_planes
from biased_oracle import OracleGPSLayerBiased
from biased_util import PAD_VALUE, biased_batch, biased_names, compare_biased, load_biased, make_bias, run_biased
from util import _nan, _stream, pin_dropout_counter, rel_err, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = {"fp32": 1e-3, "bf16": 1e-2}
GRAD_L2 = {"fp32": 5e-3, "bf16": 1e-1}   # the criterion of tests/test_layer_gpu.py (util.compare)


def _ref(QKV, bias, ptr, H, hd):
    """fp64 dense attention per graph: softmax(q k^T / sqrt(hd) + bias[g*H + h, :n, :n]) v, and the log-sum-exp."""
    D = H * hd
    Q, K, V = QKV[:, :D], QKV[:, D:2 * D], QKV[:, 2 * D:]
    outs, lses = [], []
    for g in range(len(ptr) - 1):
        s, e = int(ptr[g]), int(ptr[g + 1])
        if e == s:
            continue
        q, k, v = (t[s:e].view(e - s, H, hd).transpose(0, 1) for t in (Q, K, V))
        sc = q @ k.transpose(1, 2) / hd ** 0.5 + bias[g * H:(g + 1) * H, :e - s, :e - s]
        outs.append((torch.softmax(sc, -1) @ v).transpose(0, 1).reshape(e - s, D))
        lses.append(torch.logsumexp(sc, -1).transpose(0, 1))
    return torch.cat(outs), torch.cat(lses)


def _ptr(b):
    return b.ptr if b.ptr is not None else torch.cat([torch.zeros(1, dtype=torch.int64),
                                                      torch.bincount(b.batch.cpu(), minlength=b.num_graphs).cumsum(0)])


def _stage_batch(case):
    if case == "edge":   # empty graphs, single nodes, a 200-node graph among small ones
        return batch_from_lists([1, 0, 200, 3, 0, 1, 5], [[] for _ in range(7)], d=8)
    shape, B = case
    return make_batch(shape, seed=4, dim=8, num_graphs=B)


def _fwd_cuda_core(gs, H, hd, QKV, ab, nmax):
    lib = _lib.load()
    N, D = QKV.shape[0], H * hd
    O, lse = _nan(N, D), _nan(N, H)
    base = QKV.data_ptr()
    bias = _lib.GpsAttnBias(ab.data_ptr(), nmax, 0)
    _lib.check(lib.gps_attention_forward_biased(C.byref(gs.desc), H, hd, base, base + 4 * D, base + 8 * D, 3 * D,
                                                O.data_ptr(), D, lse.data_ptr(), 0.0, 0, 0, C.byref(bias), _stream()),
               "attention_forward_biased")
    return O, lse


def _bwd_cuda_core(gs, H, hd, QKV, O, lse, dO, ab, nmax):
    lib = _lib.load()
    N, D = QKV.shape[0], H * hd
    dQKV, delta, gb = _nan(N, 3 * D), _nan(N, H), torch.full_like(ab, float("nan"))
    base, g = QKV.data_ptr(), dQKV.data_ptr()
    bias = _lib.GpsAttnBias(ab.data_ptr(), nmax, gb.data_ptr())
    _lib.check(lib.gps_attention_backward_biased(C.byref(gs.desc), H, hd, base, base + 4 * D, base + 8 * D, 3 * D,
                                                 O.data_ptr(), dO.data_ptr(), D, lse.data_ptr(), delta.data_ptr(), g,
                                                 g + 4 * D, g + 8 * D, 3 * D, 0.0, 0, 0, C.byref(bias), _stream()),
               "attention_backward_biased")
    return dQKV, gb


@pytest.mark.parametrize("case,H,hd", [(("zinc-gine", 32), 4, 16), (("pcqm4m-small", 32), 4, 76),
                                       (("pcqm4m-small", 16), 16, 24), (("code2", 6), 4, 64), ("edge", 4, 76),
                                       (("zinc-gine", 8), 1, 64), (("zinc-gine", 8), 2, 192)])
@pytest.mark.parametrize("kind", ["random", "graph_token"])
def test_biased_attention_cuda_core_matches_fp64(case, H, hd, kind):
    b = _stage_batch(case)
    ptr = _ptr(b)
    b = b.to(DEV)
    gs = graph_of(b)
    nmax = gs.nmax
    assert nmax == int((ptr[1:] - ptr[:-1]).max())
    N, D = b.num_nodes, H * hd
    torch.manual_seed(11)
    QKV = torch.randn(N, 3 * D, device=DEV)
    ab = make_bias(b.batch, b.num_graphs, H, 3, kind).to(DEV)
    O, lse = _fwd_cuda_core(gs, H, hd, QKV, ab, nmax)
    qkv64 = QKV.double().cpu().requires_grad_(True)
    ab64 = ab.double().cpu().requires_grad_(True)
    ref, ref_lse = _ref(qkv64, ab64, ptr, H, hd)
    assert rel_err(O.cpu(), ref.detach()) < 2e-5
    assert rel_err(lse.cpu(), ref_lse.detach()) < 2e-5
    dO = torch.randn(N, D, device=DEV)
    ref.backward(dO.double().cpu())
    dQKV, gb = _bwd_cuda_core(gs, H, hd, QKV, O, lse, dO, ab, nmax)
    assert rel_err(dQKV.cpu(), qkv64.grad) < 5e-5
    assert rel_err(gb.cpu(), ab64.grad) < 5e-5
    pad = (ab == PAD_VALUE).cpu()
    assert bool((gb.cpu()[pad] == 0).all())                       # padded entries: exactly 0, not left unwritten
    assert float(ab64.grad.norm()) > 0.1
    _, gb2 = _bwd_cuda_core(gs, H, hd, QKV, O, lse, dO, ab, nmax)
    assert torch.equal(gb, gb2)                                  # no atomics: the same bits in every run


@pytest.mark.parametrize("H,hd", [(4, 16), (4, 64), (2, 128), (4, 76)])
@pytest.mark.parametrize("precision", [0, 1])
def test_biased_attention_tc_matches_fp64(H, hd, precision):
    """Mean graph size >= 64 (the layer's wgmma dispatch) with a 340-node graph spanning three 128-key tiles."""
    lib = _lib.load()
    b = batch_from_lists([340, 64, 130, 1, 0, 90, 200, 17], [[] for _ in range(8)], d=8)
    ptr = _ptr(b)
    b = b.to(DEV)
    gs = graph_of(b)
    N, D = b.num_nodes, H * hd
    assert N >= 64 * b.num_graphs and gs.nmax == 340
    torch.manual_seed(12)
    QKV = torch.randn(N, 3 * D, device=DEV)
    ab = make_bias(b.batch, b.num_graphs, H, 5).to(DEV)
    planes, ld = padded_planes(QKV, H, hd)
    O, lse = _nan(N, D), _nan(N, H)
    bias = _lib.GpsAttnBias(ab.data_ptr(), gs.nmax, 0)
    _lib.check(lib.gps_attention_forward_tc_biased(C.byref(gs.desc), H, hd, planes[0].data_ptr(),
                                                   planes[1].data_ptr() if precision == 0 else 0, ld, O.data_ptr(), D,
                                                   lse.data_ptr(), 0.0, 0, 0, precision, C.byref(bias), _stream()),
               "attention_forward_tc_biased")
    ref, ref_lse = _ref(QKV.double().cpu(), ab.double().cpu(), ptr, H, hd)
    tol = 5e-5 if precision == 0 else 2e-2
    assert rel_err(O.cpu(), ref) < tol
    assert rel_err(lse.cpu(), ref_lse) < tol
    if precision == 0:   # the CUDA-core kernel on the same inputs, with and without attention dropout (same Philox masks)
        base = QKV.data_ptr()
        for p in (0.0, 0.5):
            O1, l1, O2, l2 = _nan(N, D), _nan(N, H), _nan(N, D), _nan(N, H)
            _lib.check(lib.gps_attention_forward_biased(C.byref(gs.desc), H, hd, base, base + 4 * D, base + 8 * D, 3 * D,
                                                        O1.data_ptr(), D, l1.data_ptr(), p, 77, 4096, C.byref(bias),
                                                        _stream()), "attention_forward_biased")
            _lib.check(lib.gps_attention_forward_tc_biased(C.byref(gs.desc), H, hd, planes[0].data_ptr(),
                                                           planes[1].data_ptr(), ld, O2.data_ptr(), D, l2.data_ptr(), p,
                                                           77, 4096, 0, C.byref(bias), _stream()), "tc")
            assert rel_err(O2.cpu(), O1.cpu()) < 5e-5 and rel_err(l2.cpu(), l1.cpu()) < 5e-5, p


# ------------------------------------------------------------------------------- whole layer
def _layer(fix, precision):
    cfg = fix["config"]
    layer = graphgps_b200.GPSLayer(cfg["d"], cfg["local"], "BiasedTransformer", cfg["heads"], act=cfg["act"],
                                   batch_norm=cfg["batch_norm"], precision=precision)
    layer.load_state_dict(fix["state"], strict=True)
    return layer.to(DEV).train(cfg["training"])


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", biased_names())
def test_layer_matches_biased_golden(name, precision):
    fix = load_biased(name)
    res = run_biased(_layer(fix, precision), biased_batch(fix, DEV), fix, backward=fix["config"]["training"])
    errs = compare_biased(res, fix, TOL[precision], f"CUDA {precision} vs biased golden {name}",
                          grad_l2_tol=GRAD_L2[precision])
    print(name, precision, "max err", max(v for k, v in errs.items() if not k.startswith("raw:")))
    # the bias is read: the same layer with a zero bias gives visibly different outputs
    nob = biased_batch(fix, DEV)
    nob.attn_bias = torch.zeros_like(nob.attn_bias)
    with torch.no_grad():
        other = _layer(fix, precision)(nob).x.cpu()
    assert rel_err(other, fix["out_x"]) > 0.1


def test_layer_large_graphs_take_the_wgmma_forward_and_match_the_oracle():
    """A batch of large graphs (mean >= 64 nodes) runs the wgmma forward in the layer; forward and backward match the
    fp64 oracle, the attn_bias gradient included."""
    torch.manual_seed(4)
    d, H = 64, 4
    ora = OracleGPSLayerBiased(d, "GINE", "BiasedTransformer", H)
    ours = graphgps_b200.GPSLayer(d, "GINE", "BiasedTransformer", H)
    ours.load_state_dict(ora.state_dict(), strict=True)
    ours = ours.to(DEV).train()
    ora = ora.double().train()
    sizes = [340, 64, 130, 90, 200, 17]
    b = batch_from_lists(sizes, [[(i, i + 1) for i in range(n - 1)] + [(i + 1, i) for i in range(n - 1)] for n in sizes],
                         d=d, seed=2)
    b.attn_bias = make_bias(b.batch, len(sizes), H, 9)
    ct = torch.randn(b.x.shape, generator=torch.Generator().manual_seed(1))
    res = []
    for layer, dev, dt in ((ours, DEV, torch.float32), (ora, "cpu", torch.float64)):
        bb = b.clone().to(dev)
        bb.x, bb.edge_attr, bb.attn_bias = bb.x.to(dt), bb.edge_attr.to(dt), bb.attn_bias.to(dt).requires_grad_(True)
        bb.x.requires_grad_(True)
        x_in, ab_in = bb.x, bb.attn_bias
        out = layer(bb)
        (out.x * ct.to(dev, dt)).sum().backward()
        res.append((out.x.detach().cpu(), x_in.grad.cpu(), ab_in.grad.cpu()))
    assert rel_err(res[0][0], res[1][0]) < 1e-3
    for a, r in zip(res[0][1:], res[1][1:]):
        assert rel_err(a, r) < 1e-3 or rel_l2(a, r) < 5e-3


def test_biased_dropout_forward_backward_consistent():
    """With the Philox offset pinned, the layer with attention dropout 0.5 is a deterministic smooth (GELU) function of x
    and attn_bias: its backward equals a central finite difference of its forward along a direction in each."""
    torch.manual_seed(5)
    d, H = 64, 4
    layer = graphgps_b200.GPSLayer(d, "CustomGatedGCN", "BiasedTransformer", H, act="gelu", dropout=0.2,
                                   attn_dropout=0.5).to(DEV).train()
    b = make_batch("zinc-gatedgcn", seed=3, dim=d, num_graphs=12).to(DEV)
    ab0 = make_bias(b.batch, 12, H, 4).to(DEV)
    g = torch.Generator().manual_seed(2)
    ct_x = torch.randn(b.x.shape, generator=g).to(DEV)
    ct_e = torch.randn(b.edge_attr.shape, generator=g).to(DEV)
    vx = torch.randn(b.x.shape, generator=g).to(DEV)
    vb = torch.randn(ab0.shape, generator=g).to(DEV)

    def f(x, ab):
        pin_dropout_counter(DEV, 7 * 4096)
        bb = graphgps_b200.GraphBatch(x=x, edge_index=b.edge_index, edge_attr=b.edge_attr.clone(), batch=b.batch,
                                      num_graphs=b.num_graphs, attn_bias=ab)
        out = layer(bb)
        return (out.x * ct_x).sum() + (out.edge_attr * ct_e).sum(), out

    x0, a0 = b.x.clone().requires_grad_(True), ab0.clone().requires_grad_(True)
    loss, out0 = f(x0, a0)
    loss.backward()
    eps = 1e-2
    for which, analytic, dx, db in (("x", float((x0.grad * vx).sum()), eps * vx, 0.0),
                                    ("attn_bias", float((a0.grad * vb).sum()), 0.0, eps * vb)):
        with torch.no_grad():
            lp, _ = f(b.x + dx, ab0 + db)
            lm, _ = f(b.x - dx, ab0 - db)
        numeric = float((lp - lm) / (2 * eps))
        assert abs(numeric - analytic) <= 3e-2 * max(1.0, abs(analytic)), (which, numeric, analytic)
    with torch.no_grad():
        _, again = f(b.x.clone(), ab0.clone())
    assert torch.equal(again.x, out0.x.detach())                 # pinned offset => identical masks


def _eager_step(stack, gb, ct):
    # a function of its own: the eager autograd graph (whose parameter AccumulateGrad nodes belong to the default stream)
    # must be gone before the capture starts
    eb = gb.clone()
    eb.__dict__["_gps_b200_graph"] = graph_of(gb)
    eb.x.requires_grad_(True)
    eb.attn_bias.requires_grad_(True)
    ex, eab = eb.x, eb.attn_bias
    out = stack(eb)
    out.x.backward(ct)
    return out.x.detach().clone(), ex.grad.clone(), eab.grad.clone()


def test_stack_captured_biased_step_matches_eager_and_sums_the_layer_gradients():
    """A 10-layer GINE+BiasedTransformer GPSStack at the zinc-gine shape, captured and replayed: equal to eager
    execution, and grad_attn_bias equals the fp64 oracle's gradient, which sums the ten layers'."""
    torch.manual_seed(6)
    L, d, H = 10, 64, 4
    stack = graphgps_b200.GPSStack(L, d, "GINE", "BiasedTransformer", H).to(DEV).train()
    oras = [OracleGPSLayerBiased(d, "GINE", "BiasedTransformer", H) for _ in range(L)]
    for o, l in zip(oras, stack.layers):
        o.load_state_dict({k: v.cpu() for k, v in l.state_dict().items()}, strict=True)
    b = make_batch("zinc-gine", seed=7, dim=d, num_graphs=32)
    b.attn_bias = make_bias(b.batch, 32, H, 8)
    ct_x = torch.randn(b.x.shape, generator=torch.Generator().manual_seed(3))
    fb0 = _lib.load().gps_fallback_count()

    # fp64 oracle stack (CPU)
    ob = b.clone()
    ob.x, ob.edge_attr = ob.x.double().requires_grad_(True), ob.edge_attr.double()
    ob.attn_bias = ob.attn_bias.double().requires_grad_(True)
    ox, oab = ob.x, ob.attn_bias
    for o in oras:
        ob = o.double().train()(ob)
    (ob.x * ct_x.double()).sum().backward()

    # eager, then captured
    gb = b.clone().to(DEV)
    graph_of(gb)
    ct = ct_x.to(DEV)
    eager = _eager_step(stack, gb, ct)
    for p in stack.parameters():
        p.grad = None
    step = stack.capture(gb, ct)
    step.replay()
    step.replay()
    torch.cuda.synchronize()
    assert rel_err(step.x_out.cpu(), eager[0].cpu()) < 1e-5
    assert rel_err(step.grad_x.cpu(), eager[1].cpu()) < 1e-5
    assert rel_err(step.grad_attn_bias.cpu(), eager[2].cpu()) < 1e-5
    assert rel_err(step.x_out.cpu(), ob.x.detach()) < 1e-3
    ga, gr = step.grad_attn_bias.cpu(), oab.grad
    assert rel_err(ga, gr) < 1e-3 or rel_l2(ga, gr) < 5e-3, (rel_err(ga, gr), rel_l2(ga, gr))
    assert float(gr.norm()) > 1.0
    assert bool((ga[(b.attn_bias == PAD_VALUE)] == 0).all())
    assert _lib.load().gps_fallback_count() == fb0               # no dense product fell back to the CUDA-core kernel


def test_attn_bias_validation():
    torch.manual_seed(0)
    layer = graphgps_b200.GPSLayer(32, "GINE", "BiasedTransformer", 4).to(DEV)
    b = make_batch("zinc-gine", seed=1, dim=32, num_graphs=3).to(DEV)
    with pytest.raises(AttributeError, match="attn_bias"):
        layer(b.clone())
    ab = make_bias(b.batch, 3, 4, 0).to(DEV)
    for bad, exc in ((ab.double(), TypeError), (ab.cpu(), TypeError), (ab[:, :-1], ValueError),
                     (ab[:-1], ValueError), (ab[:, :, :-1], ValueError)):
        bb = b.clone()
        bb.attn_bias = bad
        with pytest.raises(exc):
            layer(bb)
    # no bias (None), or a zero bias, is the Transformer
    t = graphgps_b200.GPSLayer(32, "GINE", "Transformer", 4).to(DEV)
    t.load_state_dict(layer.state_dict(), strict=True)
    with torch.no_grad():
        ref = t(b.clone()).x
        bn = b.clone()
        bn.attn_bias = None
        bz = b.clone()
        bz.attn_bias = torch.zeros_like(ab)
        assert rel_err(layer(bn).x.cpu(), ref.cpu()) < 1e-6    # BatchNorm column sums: atomics, order-dependent
        assert rel_err(layer(bz).x.cpu(), ref.cpu()) < 1e-6
