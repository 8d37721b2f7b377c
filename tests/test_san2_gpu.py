"""SAN2 layer on the GPU: the fixtures from the reference in fp32-grade and bf16 (gamma's gradient included), the
attention stage at every shipped head dim against float64, dropout at both sites with the library's masks injected into
the oracle, running statistics, reproducibility, retained graphs, a captured step replayed after an in-place change of
gamma, the launch count, and the full zinc-, molpcba- and coco-SAN shapes against the float64 oracle run on the GPU."""
import ctypes as C
import os

import pytest
import torch
import torch.nn as nn

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import GraphBatch
from graphgps_b200.graph import graph_of
from san2_oracle import san2_forward, san2_parts, scores
from san_oracle import dataset_sizes, fake_pairs, san_batch
from util import GOLDEN_DIR, pin_dropout_counter, rel_err, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SAN2_DIR = os.path.join(GOLDEN_DIR, "san2")
FIXTURES = sorted(p[:-3] for p in os.listdir(SAN2_DIR) if p.endswith(".pt") and p != "reference_live.pt")
# Held in fp32-grade only: no_clamp_hd8's scores reach ~108, where bf16's rounding of the projections (2^-9 relative)
# moves each score by ~0.2 and so every softmax weight by ~20 %; two stacked layers on 61 rows make the near-cancelling
# BatchNorm-bias gradients bf16-noise dominated (as for SANLayer's two_layer_shared_hd6)
FP32_ONLY = {"no_clamp_hd8", "two_layer_shared_hd6"}
CASES = [(n, p) for n in FIXTURES for p in ("fp32", "bf16") if p == "fp32" or n not in FP32_ONLY]
FWD_TOL = {"fp32": 1e-3, "bf16": 1e-2}
GRAD_TOL = {"fp32": 1e-3, "bf16": 1e-2}   # max-abs, or the relative-L2 fallback of tests/test_san_gpu.py (the ReLU
GRAD_L2 = {"fp32": 5e-3, "bf16": 1e-1}    # makes the derivative discontinuous)
# In training mode the biases of O_h and FFN_h_layer2 feed a BatchNorm, so their exact gradient is 0 and neither bound
# applies: they are held to an absolute bound at the rounding level of an fp32 column sum over N rows of O(1) values
ZERO_GRADS = ("O_h.bias", "FFN_h_layer2.bias")
ZERO_TOL = {"fp32": 5e-3, "bf16": 5e-2}
# g_gamma is one scalar, sum over every (i, c) of g_attn (F - R) / (gamma + 1)^2, and those terms cancel: in bf16 the
# rounding of g_attn (the bf16-operand O_h product, ~2^-8 relative) moves the sum by a share of the terms' magnitude,
# not of the sum.  Besides the bounds above it may therefore meet GRAD_TOL relative to
# S = sum |g_attn (F - R)| / (gamma + 1)^2, formed by the float64 oracle (fixtures with one layer)
GAMMA = "attention.gamma"
# launches of one layer at d % 8 == 0, training, E > 0, no dropout (DESIGN.md): forward 10, as SANLayer; backward 19,
# SANLayer's 18 and the gamma reduction
LAUNCHES_FWD, LAUNCHES_BWD = 10, 19


def _load(name):
    return torch.load(os.path.join(SAN2_DIR, name + ".pt"), weights_only=False)


def _gb(x, e, ei, batch, num_graphs):
    return GraphBatch(x=x, edge_index=ei, edge_attr=e, batch=batch, num_graphs=num_graphs)


def _module(cfg, precision="fp32", p=0.0):
    emb = nn.Embedding(1, cfg["d"])
    layers = [graphgps_b200.SAN2Layer(0.1, cfg["d"], cfg["d"], cfg["heads"], True, emb, p, precision=precision)
              for _ in range(cfg["layers"])]
    return layers[0] if cfg["layers"] == 1 else nn.Sequential(*layers)


def _layer(fix, precision="fp32", p=0.0):
    mod = _module(fix["config"], precision, p)
    mod.load_state_dict(fix["state"], strict=True)
    mod = mod.to(DEV)
    mod.train(fix["config"]["training"])
    return mod


def _run(mod, fix):
    b = _gb(fix["x"].to(DEV).clone().requires_grad_(True), fix["edge_attr"].to(DEV).clone().requires_grad_(True),
            fix["edge_index"].to(DEV), fix["batch"].to(DEV), fix["num_graphs"])
    x_in, e_in = b.x, b.edge_attr
    out = mod(b).x
    (out * fix["ct"].to(DEV)).sum().backward()
    torch.cuda.synchronize()
    assert b.edge_attr is e_in      # batch.edge_attr is left unchanged
    return {"out": out.detach().cpu(), "grad_x": x_in.grad.cpu(), "grad_edge_attr": e_in.grad.cpu(),
            "grad_params": {n: p.grad.detach().cpu() for n, p in mod.named_parameters()}}


def _gamma_scale(fix):
    """S of the comment at GAMMA for a one-layer fixture, from the float64 oracle."""
    state = {k: (v.double().requires_grad_(True) if v.is_floating_point() else v) for k, v in fix["state"].items()}
    x, e = fix["x"].double(), fix["edge_attr"].double()
    fake = fake_pairs(fix["edge_index"], fix["batch"], fix["num_graphs"])
    taps = {}
    out = san2_forward(state, x, e, fix["edge_index"], fake, fix["config"]["heads"], fix["config"]["training"],
                       taps=taps)
    (out * fix["ct"].double()).sum().backward()
    gp1 = float(state[GAMMA].detach()) + 1.0
    return float((taps["attn"].grad * (taps["F"] - taps["R"]).detach()).abs().sum()) / gp1 ** 2


def _check(res, ref, precision, what, training=True, gamma_scale=None):
    bad, worst = {}, 0.0
    e = rel_err(res["out"], ref["out"])
    if not e <= FWD_TOL[precision]:
        bad["out"] = e
    grads = [("grad_x", res["grad_x"], ref["grad_x"]), ("grad_edge_attr", res["grad_edge_attr"], ref["grad_edge_attr"])]
    grads += [("grad:" + n, res["grad_params"][n], g) for n, g in ref["grad_params"].items()]
    for k, a, g in grads:
        if k.endswith(GAMMA):
            assert a.dtype == torch.float64, k
        e = rel_err(a, g)
        if training and k.endswith(ZERO_GRADS):
            if not float((a.double() - g.double()).abs().max()) <= ZERO_TOL[precision]:
                bad[k] = e
            continue
        worst = max(worst, e)
        if not e <= GRAD_TOL[precision]:
            l2 = rel_l2(a, g)
            gamma_ok = (k.endswith(GAMMA) and gamma_scale is not None
                        and float((a.double() - g.double()).abs()) <= GRAD_TOL[precision] * gamma_scale)
            if not (l2 <= GRAD_L2[precision] or gamma_ok):
                bad[k] = (e, l2)
    assert not bad, f"{what}: {bad}"
    return worst


@pytest.mark.parametrize("name,precision", CASES)
def test_fixture(name, precision):
    fix = _load(name)
    res = _run(_layer(fix, precision), fix)
    scale = _gamma_scale(fix) if fix["config"]["layers"] == 1 else None
    worst = _check(res, fix, precision, f"{name} {precision}", fix["config"]["training"], scale)
    gk = next(k for k in fix["grad_params"] if k.endswith(GAMMA))
    print(name, precision, f"out {rel_err(res['out'], fix['out']):.2e} worst grad max-abs {worst:.2e}",
          f"g_gamma {float(res['grad_params'][gk]):.6e} ref {float(fix['grad_params'][gk]):.6e} S {scale}")


def test_gamma_zero_still_has_a_gradient():
    fix = _load("gamma_zero_hd7")
    res = _run(_layer(fix), fix)
    g, ref = float(res["grad_params"]["attention.gamma"]), float(fix["grad_params"]["attention.gamma"])
    assert abs(ref) > 1e-6 and abs(g - ref) <= 1e-3 * max(1.0, abs(ref))
    # the fake part has weight 0: K_2 gets no gradient
    assert float(res["grad_params"]["attention.K_2.weight"].abs().max()) == 0.0


def test_eval_mode_leaves_running_statistics():
    fix = _load("molhiv_hd16_eval")
    mod = _layer(fix)
    before = {k: v.clone() for k, v in mod.state_dict().items()}
    _run(mod, fix)
    for k, v in mod.state_dict().items():
        assert torch.equal(v, before[k]), k


def test_training_updates_running_statistics():
    fix = _load("zinc_hd7")
    mod = _layer(fix)
    _run(mod, fix)
    x = fix["x"].double()
    st = {k: v.double() for k, v in fix["state"].items()}
    fake = fake_pairs(fix["edge_index"], fix["batch"], fix["num_graphs"])
    emb = st["attention.fake_edge_emb.weight"][0]
    lin = lambda t, n: t @ st[n + ".weight"].t()  # noqa: E731
    R, F = san2_parts(lin(x, "attention.Q"), lin(x, "attention.K"), lin(x, "attention.V"), lin(x, "attention.Q_2"),
                      lin(x, "attention.K_2"), lin(fix["edge_attr"].double(), "attention.E"),
                      st["attention.E_2.weight"] @ emb, fix["edge_index"], fake, fix["config"]["heads"])
    gm = st["attention.gamma"]
    h = ((R + gm * F) / (gm + 1)).reshape(x.shape)
    z1 = x + h @ st["O_h.weight"].t() + st["O_h.bias"]
    rm = 0.9 * st["batch_norm1_h.running_mean"] + 0.1 * z1.mean(0)
    rv = 0.9 * st["batch_norm1_h.running_var"] + 0.1 * z1.var(0, unbiased=True)
    assert rel_err(mod.batch_norm1_h.running_mean.cpu(), rm) < 1e-3
    assert rel_err(mod.batch_norm1_h.running_var.cpu(), rv) < 1e-3
    assert int(mod.batch_norm2_h.num_batches_tracked) == int(fix["state"]["batch_norm2_h.num_batches_tracked"]) + 1


# ------------------------------------------------------------------------------------------ attention stage
def _stage(kind, sizes, H, hd, gamma, seed=0, scale=1.0):
    b = san_batch(kind, sizes, 4, seed)
    N, E, d = b.x.shape[0], b.edge_index.shape[1], H * hd
    g = torch.Generator().manual_seed(seed)
    Y = (torch.randn(N, 5 * d, generator=g, dtype=torch.float64) * scale).to(DEV)
    Ee = (torch.randn(E, d, generator=g, dtype=torch.float64) * scale).to(DEV)
    E2 = (torch.randn(d, generator=g, dtype=torch.float64) * scale).to(DEV)
    dO = torch.randn(N, d, generator=g, dtype=torch.float64).to(DEV)
    bb = _gb(torch.zeros(N, 4, device=DEV), torch.zeros(E, 4, device=DEV), b.edge_index.to(DEV), b.batch.to(DEV),
             len(sizes))
    gs = graph_of(bb)
    fake = fake_pairs(b.edge_index, b.batch, len(sizes)).to(DEV)
    ei = b.edge_index.to(DEV)
    parts = [Y[:, i * d:(i + 1) * d].clone().requires_grad_(True) for i in range(5)]
    Er, E2r = Ee.clone().requires_grad_(True), E2.clone().requires_grad_(True)
    gr = torch.tensor(gamma, dtype=torch.float64, device=DEV, requires_grad=True)
    Rr, Fr = san2_parts(*parts, Er, E2r, ei, fake, H)
    Oref = ((Rr + gr * Fr) / (gr + 1)).reshape(N, d)
    (Oref * dO).sum().backward()
    with torch.no_grad():
        t, u = scores(parts[0], parts[1], parts[3], parts[4], Er, E2r, ei, fake, H)
        top = float(max(t.abs().max(), u.abs().max()))
    lib = _lib.load()
    Yf, Ef, E2f, dOf = (t.float().contiguous() for t in (Y, Ee, E2, dO))
    gdev = torch.tensor(gamma, dtype=torch.float64, device=DEV)
    O = torch.empty(N, d, device=DEV)
    R = torch.empty(N, d, device=DEV)
    F = torch.empty(N, d, device=DEV)
    lse = torch.empty(2, N, H, device=DEV)
    dY = torch.empty(N, 5 * d, device=DEV)
    dE = torch.empty(E, d, device=DEV)
    dE2 = torch.empty(d, device=DEV)
    dg = torch.empty((), dtype=torch.float64, device=DEV)
    nmax = gs.nmax
    ws = torch.empty(lib.gps_san2_attention_workspace_bytes(N, d, H, nmax), dtype=torch.uint8, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.gps_san2_attention_forward(C.byref(gs.desc), H, hd, Yf.data_ptr(), 5 * d, Ef.data_ptr(),
                                              E2f.data_ptr(), gdev.data_ptr(), nmax, ws.data_ptr(), ws.numel(),
                                              O.data_ptr(), d, R.data_ptr(), F.data_ptr(), lse.data_ptr(), st), "fwd")
    _lib.check(lib.gps_san2_attention_backward(C.byref(gs.desc), H, hd, Yf.data_ptr(), 5 * d, Ef.data_ptr(),
                                               E2f.data_ptr(), gdev.data_ptr(), nmax, ws.data_ptr(), ws.numel(),
                                               R.data_ptr(), F.data_ptr(), lse.data_ptr(), dOf.data_ptr(), d,
                                               dY.data_ptr(), 5 * d, dE.data_ptr(), dE2.data_ptr(), dg.data_ptr(), st),
               "bwd")
    torch.cuda.synchronize()
    errs = {"O": rel_err(O, Oref.detach()), "R": rel_err(R, Rr.detach().reshape(N, d)),
            "F": rel_err(F, Fr.detach().reshape(N, d))}
    for i, n in enumerate(("dQ", "dK", "dV", "dQ2", "dK2")):
        errs[n] = rel_err(dY[:, i * d:(i + 1) * d], parts[i].grad)
    errs["dE"] = rel_err(dE, Er.grad)
    errs["dE2(l2)"] = rel_l2(dE2, E2r.grad)
    errs["dgamma"] = rel_err(dg.cpu(), gr.grad.cpu())
    return errs, top


# every shipped head dim: zinc 7, cluster 6, pattern 8, molhiv 16, molpcba 76, coco / voc 11, peptides 21
@pytest.mark.parametrize("hd,H,kind,gamma", [(7, 8, "mol", 0.5), (6, 8, "sbm", 0.0), (8, 10, "sbm", 2.5),
                                             (16, 4, "mol", 0.5), (76, 4, "mol", 1.3), (11, 8, "knn", 0.5),
                                             (21, 4, "chain", 0.05)])
def test_attention_stage_head_dims(hd, H, kind, gamma):
    sizes = dataset_sizes(kind, 3 if kind in ("mol", "sbm") else 1, hd) + [1]
    errs, top = _stage(kind, sizes, H, hd, gamma, seed=hd, scale=1.6)
    print(hd, kind, gamma, {k: f"{v:.1e}" for k, v in errs.items()}, f"max |score| {top:.1f}")
    assert top > 5                          # scores well past SANLayer's clamp
    assert max(errs.values()) < 5e-5, errs


def test_attention_stage_scores_past_exp_overflow():
    # |score| > 88: exp overflows fp32 without the running max
    errs, top = _stage("mol", dataset_sizes("mol", 3, 9), 4, 8, 0.5, seed=9, scale=4.0)
    print({k: f"{v:.1e}" for k, v in errs.items()}, f"max |score| {top:.1f}")
    assert top > 88
    assert max(errs.values()) < 1e-4, errs


# ------------------------------------------------------------------------------------------ dropout
def _mask(rows, cols, p, offset, site):
    m = torch.empty(rows, cols, device=DEV)
    lib = _lib.load()
    _lib.check(lib.gps_dropout_mask(m.data_ptr(), rows, cols, p, int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF, offset,
                                    site, torch.cuda.current_stream().cuda_stream), "mask")
    return m.double() / (1.0 - p)


def _oracle_gpu(mod, b, ct, masks_per_layer=None):
    """float64 oracle of a layer (or stack) on the GPU: output and gradients by name."""
    layers = [mod] if isinstance(mod, graphgps_b200.SAN2Layer) else list(mod)
    params = dict(mod.named_parameters())
    state = {n: p.detach().double().requires_grad_(True) for n, p in params.items()}
    full = {}
    for k, v in mod.state_dict().items():
        full[k] = state[k] if k in state else v.double()
    emb_key = next(k for k in state if k.endswith("attention.fake_edge_emb.weight"))
    fake = fake_pairs(b.edge_index, b.batch, b.num_graphs).to(DEV)
    x = b.x.detach().double().requires_grad_(True)
    e = b.edge_attr.detach().double().requires_grad_(True)
    h = x
    for li, layer in enumerate(layers):
        pre = "" if len(layers) == 1 else f"{li}."
        full[pre + "attention.fake_edge_emb.weight"] = state[emb_key]
        masks = masks_per_layer[li] if masks_per_layer else None
        h = san2_forward(full, h, e, b.edge_index, fake, layer.num_heads, layer.training, masks, pre)
    (h * ct.double()).sum().backward()
    return {"out": h.detach().cpu(), "grad_x": x.grad.cpu(), "grad_edge_attr": e.grad.cpu(),
            "grad_params": {n: t.grad.cpu() for n, t in state.items()}}


def test_dropout_both_sites_with_injected_masks():
    p = 0.3
    torch.manual_seed(7)
    cfg = dict(d=56, heads=8, layers=1, training=True)
    mod = _module(cfg, "fp32", p).to(DEV)
    with torch.no_grad():
        mod.attention.gamma.fill_(0.8)
    sb = san_batch("mol", dataset_sizes("mol", 8, 5), 56, 5).to(DEV)
    b = _gb(sb.x.clone().requires_grad_(True), sb.edge_attr.clone().requires_grad_(True), sb.edge_index, sb.batch, 8)
    ct = torch.randn(sb.x.shape, device=DEV)
    N = sb.x.shape[0]
    pin_dropout_counter(DEV, 4096 * 50)
    off = 4096 * 51                      # the call's snapshot of the counter
    masks = (_mask(N, 56, p, off, 13), _mask(N, 112, p, off, 14))
    x_in, e_in = b.x, b.edge_attr
    out = mod(b).x
    (out * ct).sum().backward()
    res = {"out": out.detach().cpu(), "grad_x": x_in.grad.cpu(), "grad_edge_attr": e_in.grad.cpu(),
           "grad_params": {n: q.grad.cpu() for n, q in mod.named_parameters()}}
    ref = _oracle_gpu(mod, sb, ct, [masks])
    _check(res, ref, "fp32", "dropout")
    kept = [float((m > 0).double().mean()) for m in masks]
    assert all(abs(k - (1 - p)) < 0.02 for k in kept), kept


# ------------------------------------------------------------------------------------------ shared embedding
def test_shared_embedding_gradient_over_two_layers():
    fix = _load("two_layer_shared_hd6")
    mod = _layer(fix)
    res = _run(mod, fix)
    assert mod[1].attention.fake_edge_emb.weight is mod[0].attention.fake_edge_emb.weight
    g = res["grad_params"]["0.attention.fake_edge_emb.weight"]
    assert rel_err(g, fix["grad_params"]["0.attention.fake_edge_emb.weight"]) < GRAD_TOL["fp32"]
    assert float(g.abs().max()) > 0
    for li in (0, 1):   # each layer's own gamma
        k = f"{li}.attention.gamma"
        assert rel_err(res["grad_params"][k], fix["grad_params"][k]) < GRAD_TOL["fp32"], k


# ------------------------------------------------------------------------------------------ reproducibility
def test_bitwise_reproducible_and_retain_graph():
    fix = _load("pattern_dense_hd8")     # d % 8 == 0: every product on the plane-fed GEMM (fixed-order split-K)
    mod = _layer(fix)
    a = _run(mod, fix)
    mod.zero_grad()
    b = _run(mod, fix)
    for k in ("out", "grad_x", "grad_edge_attr"):
        assert torch.equal(a[k], b[k]), k
    for n in a["grad_params"]:
        assert torch.equal(a["grad_params"][n], b["grad_params"][n]), n
    bt = _gb(fix["x"].to(DEV).clone().requires_grad_(True), fix["edge_attr"].to(DEV).clone().requires_grad_(True),
             fix["edge_index"].to(DEV), fix["batch"].to(DEV), fix["num_graphs"])
    xin, ein = bt.x, bt.edge_attr
    out = mod(bt).x
    loss = (out * fix["ct"].to(DEV)).sum()
    g1 = torch.autograd.grad(loss, [xin, ein, mod.attention.gamma], retain_graph=True)
    g2 = torch.autograd.grad(loss, [xin, ein, mod.attention.gamma])
    for u, v in zip(g1, g2):
        assert torch.equal(u, v)


# ------------------------------------------------------------------------------------------ capture
def _seq_step(seq, x, e, b, ct):
    b.x, b.edge_attr = x, e
    out = seq(b).x
    return torch.autograd.grad((out * ct).sum(), [x, e] + list(seq.parameters())), out


@pytest.mark.parametrize("p", [0.0, 0.2])
def test_captured_step_follows_gamma_changed_in_place(p):
    torch.manual_seed(4)
    seq = _module(dict(d=56, heads=8, layers=2), "fp32", p).to(DEV)
    sb = san_batch("mol", dataset_sizes("mol", 6, 6), 56, 6).to(DEV)
    b = _gb(sb.x, sb.edge_attr, sb.edge_index, sb.batch, 6)
    graph_of(b).nmax   # read before capture (the read synchronises)
    ct = torch.randn(sb.x.shape, device=DEV)
    x = sb.x.clone().requires_grad_(True)
    e = sb.edge_attr.clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            _seq_step(seq, x, e, b, ct)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, capture_error_mode="thread_local"):
        cap_g, cap_out = _seq_step(seq, x, e, b, ct)
    pin_dropout_counter(DEV, 4096 * 1000)
    graph.replay()
    torch.cuda.synchronize()
    before = cap_out.clone()
    # an optimiser step on gamma alone, in place
    with torch.no_grad():
        seq[0].attention.gamma.add_(0.9)
        seq[1].attention.gamma.mul_(0.25)
    pin_dropout_counter(DEV, 4096 * 1000)
    graph.replay()
    torch.cuda.synchronize()
    assert not torch.equal(before, cap_out)
    pin_dropout_counter(DEV, 4096 * 1000)
    eager_g, eager_out = _seq_step(seq, x, e, b, ct)
    torch.cuda.synchronize()
    assert torch.equal(cap_out, eager_out)
    for a, r in zip(cap_g, eager_g):
        assert torch.equal(a, r)
    names = [n for n, _ in seq.named_parameters()]
    for li in (0, 1):
        assert cap_g[2 + names.index(f"{li}.attention.gamma")].dtype == torch.float64


# ------------------------------------------------------------------------------------------ launches
def test_launch_count():
    fix = _load("zinc_hd7")
    mod = _layer(fix)
    _run(mod, fix)
    lib = _lib.load()
    b = _gb(fix["x"].to(DEV).clone().requires_grad_(True), fix["edge_attr"].to(DEV).clone().requires_grad_(True),
            fix["edge_index"].to(DEV), fix["batch"].to(DEV), fix["num_graphs"])
    graph_of(b).nmax
    c0 = lib.gps_launch_count()
    out = mod(b).x
    c1 = lib.gps_launch_count()
    (out * fix["ct"].to(DEV)).sum().backward()
    c2 = lib.gps_launch_count()
    print("launches: forward", c1 - c0, "backward", c2 - c1)
    assert (c1 - c0, c2 - c1) == (LAUNCHES_FWD, LAUNCHES_BWD)


# ------------------------------------------------------------------------------------------ full size
def _full(kind, B, d, H, gamma, p, seed):
    torch.manual_seed(seed)
    mod = _module(dict(d=d, heads=H, layers=1), "fp32", p).to(DEV)
    with torch.no_grad():
        mod.attention.gamma.fill_(gamma)
        for bn in (mod.batch_norm1_h, mod.batch_norm2_h):
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.uniform_(-0.3, 0.3)
    sb = san_batch(kind, dataset_sizes(kind, B, seed), d, seed).to(DEV)
    b = _gb(sb.x.clone().requires_grad_(True), sb.edge_attr.clone().requires_grad_(True), sb.edge_index, sb.batch, B)
    ct = torch.randn(sb.x.shape, device=DEV)
    N = sb.x.shape[0]
    masks = None
    if p > 0:
        pin_dropout_counter(DEV, 4096 * 300)
        off = 4096 * 301
        masks = [(_mask(N, d, p, off, 13), _mask(N, 2 * d, p, off, 14))]
    x_in, e_in = b.x, b.edge_attr
    out = mod(b).x
    (out * ct).sum().backward()
    res = {"out": out.detach().cpu(), "grad_x": x_in.grad.cpu(), "grad_edge_attr": e_in.grad.cpu(),
           "grad_params": {n: q.grad.cpu() for n, q in mod.named_parameters()}}
    ref = _oracle_gpu(mod, sb, ct, masks)
    worst = _check(res, ref, "fp32", f"{kind} B {B} d {d}")
    print(f"{kind} B {B} N {N} d {d} H {H}: out {rel_err(res['out'], ref['out']):.2e} worst grad {worst:.2e}")


def test_full_size_zinc_san2():
    _full("mol", 32, 56, 8, 0.5, 0.0, 21)


def test_full_size_molpcba_san2():
    _full("mol", 512, 304, 4, 0.5, 0.2, 22)


def test_full_size_coco_san2():
    _full("knn", 8, 88, 8, 0.5, 0.0, 23)
