"""Graphormer layer on the GPU: the fixtures from the reference in fp32-grade and bf16, the attention stage at head dims
10 and 7 against float64, the full zinc-Graphormer and actor-Graphormer shapes against the float64 oracle, dropout at
all four sites, reproducibility, retained graphs, CUDA-graph capture and the launch count."""
import ctypes as C
import os

import pytest
import torch
import torch.nn as nn

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import GraphBatch
from graphgps_b200.graph import graph_of
from graphormer_oracle import attention, graphormer_batch, graphormer_forward, random_bias
from util import GOLDEN_DIR, pin_dropout_counter, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GR_DIR = os.path.join(GOLDEN_DIR, "graphormer")
FIXTURES = sorted(p[:-3] for p in os.listdir(GR_DIR) if p.endswith(".pt") and p != "reference_live.pt")
FWD_TOL = {"fp32": 1e-3, "bf16": 1e-2}
STRICT_GRAD = {"fp32": 1e-3, "bf16": 3e-2}   # the strict max-abs bound of test_nonorm_gpu.py: smooth layer, no L2 fallback
# launches of one layer forward + backward at d % 8 == 0 on the CUDA-core attention (DESIGN.md): forward 8 (weight
# planes, LN_in, QKV, attention, out-projection, LN_mlp, FF1, FF2), backward 16 (dropout / planes of the two upstream
# gradients 2, five data products, four weight products, two LayerNorm backwards 4, attention 2)
LAUNCHES_FWD, LAUNCHES_BWD = 8, 16


def _load(name):
    return torch.load(os.path.join(GR_DIR, name + ".pt"), weights_only=False)


def _batch(x, edge_index, batch, num_graphs):
    return GraphBatch(x=x, edge_index=edge_index, edge_attr=None, batch=batch, num_graphs=num_graphs)


def _run(layer, fix, precision_dtype=torch.float32, bias_grad=True):
    """forward + backward with the fixture's cotangent; outputs and gradients on the CPU."""
    b = _batch(fix["x"].to(DEV).clone().requires_grad_(True), fix["edge_index"].to(DEV), fix["batch"].to(DEV),
               fix["num_graphs"])
    kind = fix["config"]["bias"]
    ab = None
    if kind == "tensor":
        ab = fix["attn_bias"].to(DEV).clone().requires_grad_(bias_grad)
        b.attn_bias = ab
    elif kind == "none":
        b.attn_bias = None
    x_in = b.x
    out = layer(b).x
    (out * fix["ct"].to(DEV)).sum().backward()
    torch.cuda.synchronize()
    res = {"out": out.detach().cpu(), "grad_x": x_in.grad.cpu(),
           "grad_params": {n: p.grad.detach().cpu() for n, p in layer.named_parameters()}}
    if ab is not None and bias_grad:
        res["grad_attn_bias"] = ab.grad.cpu()
    return res


def _layer(fix, precision="fp32", p=(0.0, 0.0, 0.0)):
    cfg = fix["config"]
    layer = graphgps_b200.GraphormerLayer(cfg["d"], cfg["heads"], *p, precision=precision)
    layer.load_state_dict(fix["state"], strict=True)
    layer = layer.to(DEV)
    layer.train(cfg.get("training", True))
    return layer


def _check(res, fix, precision, what):
    bad = {}
    e = rel_err(res["out"], fix["out"])
    if not e <= FWD_TOL[precision]:
        bad["out"] = e
    grads = [("grad_x", res["grad_x"], fix["grad_x"])]
    if fix.get("grad_attn_bias") is not None:
        grads.append(("grad_attn_bias", res["grad_attn_bias"], fix["grad_attn_bias"]))
    grads += [("grad:" + n, res["grad_params"][n], g) for n, g in fix["grad_params"].items()]
    worst = 0.0
    for k, a, g in grads:
        e = rel_err(a, g)
        worst = max(worst, e)
        if not e <= STRICT_GRAD[precision]:
            bad[k] = e
    assert not bad, f"{what}: {bad}"
    return worst


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", FIXTURES)
def test_fixture(name, precision):
    fix = _load(name)
    res = _run(_layer(fix, precision), fix)
    worst = _check(res, fix, precision, f"{name} {precision}")
    print(name, precision, f"out {rel_err(res['out'], fix['out']):.2e} worst grad {worst:.2e}")


# ------------------------------------------------------------------------------------------ attention stage
def _stage(sizes, H, hd, biased, seed=0):
    g = torch.Generator().manual_seed(seed)
    N = sum(sizes)
    D = H * hd
    ld = 3 * D
    Y = (torch.randn(N, ld, generator=g, dtype=torch.float64)).to(DEV)
    dO = torch.randn(N, D, generator=g, dtype=torch.float64).to(DEV)
    batch = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes)).to(DEV)
    ei = torch.zeros(2, 0, dtype=torch.int64, device=DEV)
    b = _batch(torch.zeros(N, 4, device=DEV), ei, batch, len(sizes))
    gs = graph_of(b)
    ab = random_bias(sizes, H, seed, torch.float64).to(DEV) if biased else None
    # float64 reference and its gradients
    q, k, v = (Y[:, i * D:(i + 1) * D].clone().requires_grad_(True) for i in range(3))
    abr = ab.clone().requires_grad_(True) if biased else None
    Oref = attention(q, k, v, batch, len(sizes), H, abr)
    (Oref * dO).sum().backward()
    # the library, fp32
    lib = _lib.load()
    Yf = Y.float().contiguous()
    O = torch.empty(N, D, device=DEV)
    lse = torch.empty(N, H, device=DEV)
    delta = torch.empty(N, H, device=DEV)
    gY = torch.empty(N, ld, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    p = Yf.data_ptr()
    fb = ab.float().contiguous() if biased else None
    gb = torch.empty_like(fb) if biased else None
    if biased:
        bias = _lib.GpsAttnBias(fb.data_ptr(), fb.shape[-1], gb.data_ptr())
        _lib.check(lib.gps_attention_forward_biased(C.byref(gs.desc), H, hd, p, p + 4 * D, p + 8 * D, ld, O.data_ptr(), D,
                                                    lse.data_ptr(), 0.0, 0, 0, C.byref(bias), st), "fwd")
    else:
        _lib.check(lib.gps_attention_forward(C.byref(gs.desc), H, hd, p, p + 4 * D, p + 8 * D, ld, O.data_ptr(), D,
                                             lse.data_ptr(), 0.0, 0, 0, st), "fwd")
    dOf = dO.float().contiguous()
    gp = gY.data_ptr()
    args = (C.byref(gs.desc), H, hd, p, p + 4 * D, p + 8 * D, ld, O.data_ptr(), dOf.data_ptr(), D, lse.data_ptr(),
            delta.data_ptr(), gp, gp + 4 * D, gp + 8 * D, ld, 0.0, 0, 0)
    if biased:
        _lib.check(lib.gps_attention_backward_biased(*args, C.byref(bias), st), "bwd")
    else:
        _lib.check(lib.gps_attention_backward(*args, st), "bwd")
    torch.cuda.synchronize()
    errs = {"O": rel_err(O, Oref.detach()), "dQ": rel_err(gY[:, :D], q.grad), "dK": rel_err(gY[:, D:2 * D], k.grad),
            "dV": rel_err(gY[:, 2 * D:], v.grad)}
    if biased:
        errs["dbias"] = rel_err(gb, abr.grad)
    return errs


@pytest.mark.parametrize("hd", [10, 7])
@pytest.mark.parametrize("biased", [False, True])
@pytest.mark.parametrize("sizes", [[24, 19, 30, 1, 12, 27, 21, 33], [700]], ids=["small", "large"])
def test_attention_stage_head_dims(hd, biased, sizes):
    errs = _stage(sizes, 8 if hd == 10 else 5, hd, biased)
    print(hd, biased, len(sizes), {k: f"{v:.1e}" for k, v in errs.items()})
    assert max(errs.values()) < 2e-5, errs


# ------------------------------------------------------------------------------------------ full size
def _full(sizes, d, H, token, seed, precision="fp32"):
    torch.manual_seed(seed)
    layer = graphgps_b200.GraphormerLayer(d, H, 0.0, 0.0, 0.0, precision=precision).to(DEV)
    with torch.no_grad():
        for m in layer.modules():
            if isinstance(m, nn.LayerNorm):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.3, 0.3)
    b = graphormer_batch(sizes, d, seed, token)
    ab = random_bias(sizes, H, seed).to(DEV)
    g = torch.Generator().manual_seed(seed + 1)
    ct = torch.randn(b.x.shape, generator=g).to(DEV)
    x = b.x.to(DEV)
    batch, ei = b.batch.to(DEV), b.edge_index.to(DEV)
    # float64 oracle on the GPU
    state = {n: p.detach().double().requires_grad_(True) for n, p in layer.named_parameters()}
    xr, abr = x.double().requires_grad_(True), ab.double().requires_grad_(True)
    out_r = graphormer_forward(state, xr, batch, len(sizes), H, abr)
    (out_r * ct.double()).sum().backward()
    ref = {"out": out_r.detach().cpu(), "grad_x": xr.grad.cpu(), "grad_attn_bias": abr.grad.cpu(),
           "grad_params": {n: t.grad.cpu() for n, t in state.items()}}
    del out_r, xr, abr, state
    fix = {"x": x, "edge_index": ei, "batch": batch, "num_graphs": len(sizes), "attn_bias": ab, "ct": ct,
           "config": {"bias": "tensor"}}
    res = _run(layer, fix)
    worst = _check(res, ref, precision, f"full {len(sizes)} graphs, N {x.shape[0]}")
    print(f"N {x.shape[0]} d {d} H {H}: out {rel_err(res['out'], ref['out']):.2e} worst grad {worst:.2e}")


def test_full_size_zinc_graphormer():
    g = torch.Generator().manual_seed(3)
    sizes = (torch.randint(10, 38, (256,), generator=g) + 1).tolist()   # ZINC-sized graphs, one token each
    _full(sizes, 80, 8, True, 11)


def test_full_size_actor_graphormer():
    _full([7600], 64, 4, False, 12)


# ------------------------------------------------------------------------------------------ dropout
def test_dropout_backward_is_derivative_of_forward():
    """All four sites active, offset pinned: the layer is a fixed smooth function; its backward equals a central finite
    difference of its forward along a random direction (x, bias and one weight)."""
    fix = _load("hd10_bias_token_train")
    layer = _layer(fix, "fp32", (0.2, 0.2, 0.2))
    x0 = fix["x"].to(DEV)
    ab0 = fix["attn_bias"].to(DEV)
    ct = fix["ct"].to(DEV)
    ei, batch = fix["edge_index"].to(DEV), fix["batch"].to(DEV)
    w = layer.mlp[1].weight
    g = torch.Generator().manual_seed(9)
    vx, vb, vw = (torch.randn(t.shape, generator=g).to(DEV) for t in (x0, ab0, w))

    def f(eps, grad=False):
        pin_dropout_counter(DEV, 4096 * 77)
        b = _batch((x0 + eps * vx).requires_grad_(grad), ei, batch, fix["num_graphs"])
        b.attn_bias = (ab0 + eps * vb).requires_grad_(grad)
        xin, abin = b.x, b.attn_bias
        with torch.no_grad():
            w.add_(eps * vw)
        try:
            out = layer(b).x
            loss = (out.double() * ct.double()).sum()
            if grad:
                layer.zero_grad()
                loss.backward()
                return float((xin.grad * vx).sum() + (abin.grad * vb).sum() + (w.grad * vw).sum())
            return float(loss)
        finally:
            with torch.no_grad():
                w.sub_(eps * vw)

    dd = f(0.0, grad=True)
    eps = 1e-2
    fd = (f(eps) - f(-eps)) / (2 * eps)
    print("directional derivative", dd, "finite difference", fd)
    assert abs(dd - fd) <= 2e-3 * max(1.0, abs(fd)), (dd, fd)


def test_dropout_kept_fraction_scaling_and_fresh_masks():
    """out_proj and mlp.4 made constant 1: out - x = drop_10(1) + drop_12(1), entries in {0, s, 2s}, s = 1/(1-p)."""
    p = 0.3
    layer = graphgps_b200.GraphormerLayer(80, 8, p, 0.0, 0.0).to(DEV)
    with torch.no_grad():
        for lin in (layer.attention.out_proj, layer.mlp[4]):
            lin.weight.zero_()
            lin.bias.fill_(1.0)
    sizes = [30] * 200
    bb = graphormer_batch(sizes, 80, 5)
    x = bb.x.to(DEV)

    def run(offset):
        pin_dropout_counter(DEV, offset)
        b = _batch(x.clone(), bb.edge_index.to(DEV), bb.batch.to(DEV), len(sizes))
        return (layer(b).x - x).detach()

    r = run(4096)
    s = 1.0 / (1.0 - p)
    vals = torch.tensor([0.0, s, 2 * s], device=DEV)
    assert bool(((r[..., None] - vals).abs().min(-1).values < 1e-4).all())
    zero = float((r.abs() < 1e-4).double().mean())
    mean = float(r.double().mean())
    print("zero fraction", zero, "expected", p * p, "mean", mean)
    assert abs(zero - p * p) < 0.01
    assert abs(mean - 2.0) < 0.01
    r2 = run(4096)
    assert torch.equal(r, r2)
    r3 = run(8192)
    assert not torch.equal(r, r3)


# ------------------------------------------------------------------------------------------ reproducibility
def test_bitwise_reproducible_and_retain_graph():
    fix = _load("hd16_bias_wgmma")
    layer = _layer(fix)
    a = _run(layer, fix)
    layer.zero_grad()
    b = _run(layer, fix)
    assert torch.equal(a["out"], b["out"]) and torch.equal(a["grad_x"], b["grad_x"])
    assert torch.equal(a["grad_attn_bias"], b["grad_attn_bias"])
    for n in a["grad_params"]:
        assert torch.equal(a["grad_params"][n], b["grad_params"][n]), n
    # backward(retain_graph=True) twice: the same result each time
    bt = _batch(fix["x"].to(DEV).clone().requires_grad_(True), fix["edge_index"].to(DEV), fix["batch"].to(DEV),
                fix["num_graphs"])
    bt.attn_bias = fix["attn_bias"].to(DEV)
    xin = bt.x
    out = layer(bt).x
    loss = (out * fix["ct"].to(DEV)).sum()
    g1 = torch.autograd.grad(loss, [xin], retain_graph=True)[0]
    g2 = torch.autograd.grad(loss, [xin])[0]
    assert torch.equal(g1, g2)


# ------------------------------------------------------------------------------------------ capture
def _seq_step(seq, x, b, ct):
    b.x = x
    out = seq(b).x
    return torch.autograd.grad((out * ct).sum(), [x] + list(seq.parameters())), out


@pytest.mark.parametrize("p", [0.0, 0.2])
def test_captured_two_layer_stack(p):
    torch.manual_seed(4)
    seq = nn.Sequential(*[graphgps_b200.GraphormerLayer(80, 8, p, p, p) for _ in range(2)]).to(DEV)
    sizes = [26, 13, 31, 22, 18, 29]
    bb = graphormer_batch(sizes, 80, 6, True)
    ab = random_bias(sizes, 8, 6).to(DEV)
    b = _batch(bb.x.to(DEV), bb.edge_index.to(DEV), bb.batch.to(DEV), len(sizes))
    b.attn_bias = ab
    graph_of(b).nmax   # read before capture (the read synchronises)
    ct = torch.randn(bb.x.shape, device=DEV)
    x = bb.x.to(DEV).clone().requires_grad_(True)
    pin_dropout_counter(DEV, 4096 * 1000)
    eager_g, eager_out = _seq_step(seq, x, b, ct)
    eager_out = eager_out.detach()
    x = x.detach().clone().requires_grad_(True)   # the graph's static input, a fresh leaf
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            _seq_step(seq, x, b, ct)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, capture_error_mode="thread_local"):
        cap_g, cap_out = _seq_step(seq, x, b, ct)
    pin_dropout_counter(DEV, 4096 * 1000)   # the first replay's two layers draw the eager step's offsets
    graph.replay()
    torch.cuda.synchronize()
    first = cap_out.clone()
    if p == 0.0:
        assert torch.equal(first, eager_out)
        for a, e in zip(cap_g, eager_g):
            assert torch.equal(a, e)
    graph.replay()
    torch.cuda.synchronize()
    if p > 0.0:
        assert not torch.equal(first, cap_out)   # fresh masks on every replay
    else:
        assert torch.equal(first, cap_out)


# ------------------------------------------------------------------------------------------ launches
def test_launch_count():
    fix = _load("hd10_bias_token_train")
    layer = _layer(fix)
    _run(layer, fix)
    lib = _lib.load()
    b = _batch(fix["x"].to(DEV).clone().requires_grad_(True), fix["edge_index"].to(DEV), fix["batch"].to(DEV),
               fix["num_graphs"])
    b.attn_bias = fix["attn_bias"].to(DEV).requires_grad_(True)
    graph_of(b)
    c0 = lib.gps_launch_count()
    out = layer(b).x
    c1 = lib.gps_launch_count()
    (out * fix["ct"].to(DEV)).sum().backward()
    c2 = lib.gps_launch_count()
    print("launches: forward", c1 - c0, "backward", c2 - c1)
    assert (c1 - c0, c2 - c1) == (LAUNCHES_FWD, LAUNCHES_BWD)
