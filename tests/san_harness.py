"""SANLayer and SAN2Layer share one orchestration (san.cu; GpsSanArgs.variant tells them apart), and their tests share
these pieces: one spec per variant, the fixtures, the layer runs, the comparison, the attention-stage run, the dropout
masks and the float64 oracle on the GPU."""
import ctypes as C
import math
import os
import types

import pytest
import torch
import torch.nn as nn

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import GraphBatch
from graphgps_b200.graph import graph_of
from san2_oracle import san2_forward, san2_parts, scores
from san_oracle import dataset_sizes, fake_pairs, san_attention, san_batch, san_forward
from util import DEV, GOLDEN_DIR, pin_dropout_counter, rel_err, rel_l2

FWD_TOL = {"fp32": 1e-3, "bf16": 1e-2}
GRAD_TOL = {"fp32": 1e-3, "bf16": 1e-2}   # max-abs, or the relative-L2 fallback of tests/test_layer_gpu.py: the clamp
GRAD_L2 = {"fp32": 5e-3, "bf16": 1e-1}    # and the ReLU make the derivative discontinuous (tests/util.py compare)
# In training mode the biases of O_h and FFN_h_layer2 feed a BatchNorm, so their exact gradient is 0 and neither bound
# applies: they are held to an absolute bound at the rounding level of an fp32 column sum over N rows of O(1) values
ZERO_GRADS = ("O_h.bias", "FFN_h_layer2.bias")
ZERO_TOL = {"fp32": 5e-3, "bf16": 5e-2}
# SAN2's g_gamma is one scalar, sum over every (i, c) of g_attn (F - R) / (gamma + 1)^2, and those terms cancel: in bf16
# the rounding of g_attn (the bf16-operand O_h product, ~2^-8 relative) moves the sum by a share of the terms' magnitude,
# not of the sum.  Besides the bounds above it may therefore meet GRAD_TOL relative to
# S = sum |g_attn (F - R)| / (gamma + 1)^2, formed by the float64 oracle (fixtures with one layer)
GAMMA = "attention.gamma"


def _attention_san(Q, K, V, Q2, K2, E, E2, ei, fake, heads, st, cfg):
    return san_attention(Q, K, V, Q2, K2, E, E2, ei, fake, heads, cfg["gamma"])


def _attention_san2(Q, K, V, Q2, K2, E, E2, ei, fake, heads, st, cfg):
    R, F = san2_parts(Q, K, V, Q2, K2, E, E2, ei, fake, heads)
    gm = st[GAMMA]
    return ((R + gm * F) / (gm + 1)).reshape(Q.shape)


# cls: the layer.  forward(state, h, e, ei, fake, layer, masks, prefix): its float64 oracle.  attention(...): its
# attention block in float64 from the state dict st.  launches: (forward, backward) launches of one layer at
# d % 8 == 0, training, E > 0, no dropout (DESIGN.md), as counted on an H100: forward 10 (planes, bitmap + E2, edge and
# node projections, attention, O_h, BN1, FFN1, FFN2, BN2); backward 18, and SAN2's 19 adds the gamma reduction.
# repro_fixture: a fixture at d % 8 == 0, where every product is on the plane-fed GEMM, whose split-K sums in a fixed
# order.
VARIANTS = {
    "SAN": types.SimpleNamespace(
        name="SAN", cls=graphgps_b200.SANLayer, dir=os.path.join(GOLDEN_DIR, "san"),
        forward=lambda st, h, e, ei, fake, layer, masks, pre: san_forward(
            st, h, e, ei, fake, layer.num_heads, layer.gamma, layer.training, masks, pre),
        attention=_attention_san, launches=(10, 18), repro_fixture="pattern_dense_hd6"),
    "SAN2": types.SimpleNamespace(
        name="SAN2", cls=graphgps_b200.SAN2Layer, dir=os.path.join(GOLDEN_DIR, "san2"),
        forward=lambda st, h, e, ei, fake, layer, masks, pre: san2_forward(
            st, h, e, ei, fake, layer.num_heads, layer.training, masks, pre),
        attention=_attention_san2, launches=(10, 19), repro_fixture="pattern_dense_hd8"),
}


def fixtures(variant):
    d = VARIANTS[variant].dir
    return sorted(p[:-3] for p in os.listdir(d) if p.endswith(".pt") and p != "reference_live.pt")


def _load(variant, name):
    return torch.load(os.path.join(VARIANTS[variant].dir, name + ".pt"), weights_only=False)


def _gb(x, e, ei, batch, num_graphs):
    return GraphBatch(x=x, edge_index=ei, edge_attr=e, batch=batch, num_graphs=num_graphs)


def _module(variant, cfg, precision="fp32", p=0.0):
    """One layer, or an nn.Sequential of cfg["layers"] sharing one fake-edge embedding.  SAN takes cfg["gamma"] as its
    constructor argument; SAN2 ignores that argument, as the reference does, and its learned gamma is set to
    cfg["gamma"] when the configuration has one."""
    emb = nn.Embedding(1, cfg["d"])
    layers = [VARIANTS[variant].cls(cfg.get("gamma", 0.1), cfg["d"], cfg["d"], cfg["heads"], True, emb, p,
                                    precision=precision) for _ in range(cfg["layers"])]
    if variant == "SAN2" and "gamma" in cfg:
        with torch.no_grad():
            for layer in layers:
                layer.attention.gamma.fill_(cfg["gamma"])
    return layers[0] if cfg["layers"] == 1 else nn.Sequential(*layers)


def _layer(variant, fix, precision="fp32", p=0.0):
    mod = _module(variant, fix["config"], precision, p)
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


# ------------------------------------------------------------------------------------------ attention stage
def _stage(variant, kind, sizes, H, hd, gamma, seed=0, scale=1.0):
    """The attention stage against float64.  Returns the errors and, for SAN, the share of scores beyond the clamp and
    the number of nodes excluded for a pair within 1e-4 of a clamp bound; for SAN2, the largest |score|."""
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
    lib = _lib.load()
    Yf, Ef, E2f, dOf = (t.float().contiguous() for t in (Y, Ee, E2, dO))
    O = torch.empty(N, d, device=DEV)
    dY = torch.empty(N, 5 * d, device=DEV)
    dE = torch.empty(E, d, device=DEV)
    dE2 = torch.empty(d, device=DEV)
    nmax = gs.nmax
    st = torch.cuda.current_stream().cuda_stream
    if variant == "SAN":
        # float64 reference, its gradients and each pair's score (to find the pairs at the clamp bounds)
        Oref = san_attention(*parts, Er, E2r, ei, fake, H, gamma)
        (Oref * dO).sum().backward()
        with torch.no_grad():
            v = lambda t: t.reshape(-1, H, hd)  # noqa: E731
            t_real = (v(parts[1])[ei[0]] * v(parts[0])[ei[1]] * v(Er)).sum(-1) / math.sqrt(hd)
            t_fake = (v(parts[4])[fake[0]] * v(parts[3])[fake[1]] * E2r.reshape(1, H, hd)).sum(-1) / math.sqrt(hd)
            near = lambda t: ((t.abs() - 5).abs() < 1e-4)  # noqa: E731
            # nodes touched by a pair within 1e-4 of a clamp bound: their gradients are excluded from the elementwise
            # check
            bad_nodes = torch.zeros(N, dtype=torch.bool, device=DEV)
            bad_edges = near(t_real).any(-1)
            for (s, dd), m in (((ei[0], ei[1]), bad_edges), ((fake[0], fake[1]), near(t_fake).any(-1))):
                bad_nodes[s[m]] = True
                bad_nodes[dd[m]] = True
            saturated = float(((t_real.abs() > 5).double().mean() + (t_fake.abs() > 5).double().mean()) / 2)
        rz = torch.empty(N, H, device=DEV)
        ws = torch.empty(lib.gps_san_attention_workspace_bytes(N, d, H, nmax), dtype=torch.uint8, device=DEV)
        _lib.check(lib.gps_san_attention_forward(C.byref(gs.desc), H, hd, Yf.data_ptr(), 5 * d, Ef.data_ptr(),
                                                 E2f.data_ptr(), gamma, nmax, ws.data_ptr(), ws.numel(), O.data_ptr(),
                                                 d, rz.data_ptr(), st), "fwd")
        _lib.check(lib.gps_san_attention_backward(C.byref(gs.desc), H, hd, Yf.data_ptr(), 5 * d, Ef.data_ptr(),
                                                  E2f.data_ptr(), gamma, nmax, ws.data_ptr(), ws.numel(), O.data_ptr(),
                                                  dOf.data_ptr(), d, rz.data_ptr(), dY.data_ptr(), 5 * d, dE.data_ptr(),
                                                  dE2.data_ptr(), st), "bwd")
        torch.cuda.synchronize()
        ok = ~bad_nodes
        errs = {"O": rel_err(O, Oref.detach())}
        for i, n in enumerate(("dQ", "dK", "dV", "dQ2", "dK2")):
            errs[n] = rel_err(dY[ok, i * d:(i + 1) * d], parts[i].grad[ok])
        okE = ~(bad_edges | bad_nodes[ei[0]] | bad_nodes[ei[1]])
        errs["dE"] = rel_err(dE[okE], Er.grad[okE])
        errs["dE2(l2)"] = rel_l2(dE2, E2r.grad)
        return errs, dict(saturated=saturated, excluded=int(bad_nodes.sum()))
    gr = torch.tensor(gamma, dtype=torch.float64, device=DEV, requires_grad=True)
    Rr, Fr = san2_parts(*parts, Er, E2r, ei, fake, H)
    Oref = ((Rr + gr * Fr) / (gr + 1)).reshape(N, d)
    (Oref * dO).sum().backward()
    with torch.no_grad():
        t, u = scores(parts[0], parts[1], parts[3], parts[4], Er, E2r, ei, fake, H)
        top = float(max(t.abs().max(), u.abs().max()))
    gdev = torch.tensor(gamma, dtype=torch.float64, device=DEV)
    R = torch.empty(N, d, device=DEV)
    F = torch.empty(N, d, device=DEV)
    lse = torch.empty(2, N, H, device=DEV)
    dg = torch.empty((), dtype=torch.float64, device=DEV)
    ws = torch.empty(lib.gps_san2_attention_workspace_bytes(N, d, H, nmax), dtype=torch.uint8, device=DEV)
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
    return errs, dict(top=top)


# ------------------------------------------------------------------------------------------ dropout and the oracle
def _mask(rows, cols, p, offset, site):
    m = torch.empty(rows, cols, device=DEV)
    lib = _lib.load()
    _lib.check(lib.gps_dropout_mask(m.data_ptr(), rows, cols, p, int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF, offset,
                                    site, torch.cuda.current_stream().cuda_stream), "mask")
    return m.double() / (1.0 - p)


def _oracle_gpu(variant, mod, b, ct, masks_per_layer=None):
    """float64 oracle of a layer (or stack) on the GPU: output and gradients by name."""
    spec = VARIANTS[variant]
    layers = [mod] if isinstance(mod, spec.cls) else list(mod)
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
        h = spec.forward(full, h, e, b.edge_index, fake, layer, masks, pre)
    (h * ct.double()).sum().backward()
    return {"out": h.detach().cpu(), "grad_x": x.grad.cpu(), "grad_edge_attr": e.grad.cpu(),
            "grad_params": {n: t.grad.cpu() for n, t in state.items()}}


def _seq_step(seq, x, e, b, ct):
    b.x, b.edge_attr = x, e
    out = seq(b).x
    return torch.autograd.grad((out * ct).sum(), [x, e] + list(seq.parameters())), out


def _full(variant, kind, B, d, H, gamma, p, seed):
    torch.manual_seed(seed)
    mod = _module(variant, dict(d=d, heads=H, gamma=gamma, layers=1), "fp32", p).to(DEV)
    with torch.no_grad():
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
    ref = _oracle_gpu(variant, mod, sb, ct, masks)
    worst = _check(res, ref, "fp32", f"{kind} B {B} d {d}")
    print(f"{kind} B {B} N {N} d {d} H {H}: out {rel_err(res['out'], ref['out']):.2e} worst grad {worst:.2e}")


# ------------------------------------------------------------------------------------------ layer checks (GPU)
def check_fixture(variant, fix, precision, gamma_scale=None):
    """The layer against one of the reference's fixtures; returns the layer's outputs and gradients."""
    res = _run(_layer(variant, fix, precision), fix)
    name = fix["config"]["name"]
    worst = _check(res, fix, precision, f"{name} {precision}", fix["config"]["training"], gamma_scale)
    print(name, precision, f"out {rel_err(res['out'], fix['out']):.2e} worst grad max-abs {worst:.2e}")
    return res


def check_eval_mode_leaves_running_statistics(variant):
    fix = _load(variant, "molhiv_hd16_eval")
    mod = _layer(variant, fix)
    before = {k: v.clone() for k, v in mod.state_dict().items()}
    _run(mod, fix)
    for k, v in mod.state_dict().items():
        assert torch.equal(v, before[k]), k


def check_training_updates_running_statistics(variant):
    fix = _load(variant, "zinc_hd7")
    mod = _layer(variant, fix)
    _run(mod, fix)
    x = fix["x"].double()
    st = {k: v.double() for k, v in fix["state"].items()}
    fake = fake_pairs(fix["edge_index"], fix["batch"], fix["num_graphs"])
    # BN1's input, from the oracle's own steps
    emb = st["attention.fake_edge_emb.weight"][0]
    lin = lambda t, n: t @ st[n + ".weight"].t()  # noqa: E731
    h = VARIANTS[variant].attention(lin(x, "attention.Q"), lin(x, "attention.K"), lin(x, "attention.V"),
                                    lin(x, "attention.Q_2"), lin(x, "attention.K_2"),
                                    lin(fix["edge_attr"].double(), "attention.E"), st["attention.E_2.weight"] @ emb,
                                    fix["edge_index"], fake, fix["config"]["heads"], st, fix["config"])
    z1 = x + h @ st["O_h.weight"].t() + st["O_h.bias"]
    rm = 0.9 * st["batch_norm1_h.running_mean"] + 0.1 * z1.mean(0)
    rv = 0.9 * st["batch_norm1_h.running_var"] + 0.1 * z1.var(0, unbiased=True)
    assert rel_err(mod.batch_norm1_h.running_mean.cpu(), rm) < 1e-3
    assert rel_err(mod.batch_norm1_h.running_var.cpu(), rv) < 1e-3
    assert int(mod.batch_norm2_h.num_batches_tracked) == int(fix["state"]["batch_norm2_h.num_batches_tracked"]) + 1


# ------------------------------------------------------------------------------------------ dropout
def check_dropout_both_sites_with_injected_masks(variant, gamma):
    """Dropout p = 0.3 at both sites against the float64 oracle fed the library's masks.  gamma is SAN's constructor
    argument, or the value SAN2's learned gamma is set to."""
    p = 0.3
    torch.manual_seed(7)
    cfg = dict(d=56, heads=8, gamma=gamma, layers=1, training=True)
    mod = _module(variant, cfg, "fp32", p).to(DEV)
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
    ref = _oracle_gpu(variant, mod, sb, ct, [masks])
    _check(res, ref, "fp32", "dropout")
    kept = [float((m > 0).double().mean()) for m in masks]
    assert all(abs(k - (1 - p)) < 0.02 for k in kept), kept


# ------------------------------------------------------------------------------------------ shared embedding
def check_shared_embedding_gradient_over_two_layers(variant):
    fix = _load(variant, "two_layer_shared_hd6")
    mod = _layer(variant, fix)
    res = _run(mod, fix)
    emb = mod[0].attention.fake_edge_emb.weight
    assert mod[1].attention.fake_edge_emb.weight is emb
    g = res["grad_params"]["0.attention.fake_edge_emb.weight"]
    assert rel_err(g, fix["grad_params"]["0.attention.fake_edge_emb.weight"]) < GRAD_TOL["fp32"]
    # the sum of each layer's own share: layer 1 alone (on layer 0's output) plus layer 0 alone
    assert float(g.abs().max()) > 0
    for k in (k for k in fix["grad_params"] if k.endswith(GAMMA)):   # SAN2: each layer's own gamma
        assert rel_err(res["grad_params"][k], fix["grad_params"][k]) < GRAD_TOL["fp32"], k


# ------------------------------------------------------------------------------------------ reproducibility
def check_bitwise_reproducible_and_retain_graph(variant):
    fix = _load(variant, VARIANTS[variant].repro_fixture)
    mod = _layer(variant, fix)
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
    wrt = [xin, ein] + [q for n, q in mod.named_parameters() if n.endswith(GAMMA)]
    g1 = torch.autograd.grad(loss, wrt, retain_graph=True)
    g2 = torch.autograd.grad(loss, wrt)
    for u, v in zip(g1, g2):
        assert torch.equal(u, v)


# ------------------------------------------------------------------------------------------ launches
def check_launch_count(variant):
    fix = _load(variant, "zinc_hd7")
    mod = _layer(variant, fix)
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
    assert (c1 - c0, c2 - c1) == VARIANTS[variant].launches


# ------------------------------------------------------------------------------------------ CPU side
def _oracle(variant, fix, state, x, e):
    cfg = fix["config"]
    fake = fake_pairs(fix["edge_index"], fix["batch"], fix["num_graphs"])
    prefixes = [""] if cfg["layers"] == 1 else [f"{i}." for i in range(cfg["layers"])]
    layer = types.SimpleNamespace(num_heads=cfg["heads"], gamma=cfg["gamma"], training=cfg["training"])
    h = x
    for p in prefixes:
        if p:   # one embedding shared by the layers (state_dict lists it under each; its gradient is layer 0's entry)
            state[p + "attention.fake_edge_emb.weight"] = state["0.attention.fake_edge_emb.weight"]
        h = VARIANTS[variant].forward(state, h, e, fix["edge_index"], fake, layer, None, p)
    return h


def _check_oracle(variant, fix, tol_out, tol_grad):
    state = {k: (v.double().requires_grad_(True) if v.is_floating_point() else v) for k, v in fix["state"].items()}
    x = fix["x"].double().clone().requires_grad_(True)
    e = fix["edge_attr"].double().clone().requires_grad_(True)
    out = _oracle(variant, fix, state, x, e)
    assert float((out.detach() - fix["out"].double()).abs().max()) < tol_out
    (out * fix["ct"].double()).sum().backward()
    assert float((x.grad - fix["grad_x"].double()).abs().max()) < tol_grad
    assert float((e.grad - fix["grad_edge_attr"].double()).abs().max()) < tol_grad
    for n, g in fix["grad_params"].items():
        assert float((state[n].grad - g.double()).abs().max()) < tol_grad, n


def check_shared_embedding(variant):
    """Layers built with one fake-edge embedding share it, and a stack holds it once."""
    emb = nn.Embedding(1, 24)
    a = VARIANTS[variant].cls(0.1, 24, 24, 4, True, emb)
    b = VARIANTS[variant].cls(0.1, 24, 24, 4, True, emb)
    assert a.attention.fake_edge_emb is emb and b.attention.fake_edge_emb is emb
    assert "attention.fake_edge_emb.weight" in a.state_dict()
    assert sum(1 for p in nn.Sequential(a, b).parameters() if p is emb.weight) == 1


# the reference's options the layers refuse
NOT_BUILT = [dict(full_graph=False), dict(layer_norm=True), dict(batch_norm=False), dict(residual=False),
             dict(use_bias=True)]


def check_constructor_not_built(variant, kw, match=None):
    args = dict(gamma=0.1, in_dim=48, out_dim=48, num_heads=8, full_graph=True, fake_edge_emb=nn.Embedding(1, 48))
    args.update(kw)
    with pytest.raises(NotImplementedError, match=match):
        VARIANTS[variant].cls(**args)


def _args(variant, d=56, heads=8, N=133, E=300, B=6, nmax=30):
    a = _lib.GpsSanArgs()
    a.d, a.heads = d, heads
    a.graph.N, a.graph.E, a.graph.B = N, E, B
    a.nmax = nmax
    a.training = 1
    a.variant = {"SAN": 0, "SAN2": 1}.get(variant, variant)
    return a
