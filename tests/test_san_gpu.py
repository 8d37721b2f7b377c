"""SAN layer on the GPU: the fixtures from the reference in fp32-grade and bf16, the attention stage at every shipped
head dim against float64, dropout at both sites with the library's masks injected into the oracle, the shared
embedding over two layers, reproducibility, retained graphs, CUDA-graph capture, the launch count, and the full
zinc-, molpcba- and coco-SAN shapes against the float64 oracle run on the GPU."""
import ctypes as C
import math
import os

import pytest
import torch
import torch.nn as nn

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import GraphBatch
from graphgps_b200.graph import graph_of
from san_oracle import dataset_sizes, fake_pairs, san_attention, san_batch, san_forward
from util import GOLDEN_DIR, pin_dropout_counter, rel_err, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SAN_DIR = os.path.join(GOLDEN_DIR, "san")
FIXTURES = sorted(p[:-3] for p in os.listdir(SAN_DIR) if p.endswith(".pt") and p != "reference_live.pt")
FWD_TOL = {"fp32": 1e-3, "bf16": 1e-2}
GRAD_TOL = {"fp32": 1e-3, "bf16": 1e-2}   # max-abs, or the relative-L2 fallback of tests/test_layer_gpu.py: the clamp
GRAD_L2 = {"fp32": 5e-3, "bf16": 1e-1}    # and the ReLU make the derivative discontinuous (tests/util.py compare)
# In training mode the biases of O_h and FFN_h_layer2 feed a BatchNorm, so their exact gradient is 0 and neither bound
# applies: they are held to an absolute bound at the rounding level of an fp32 column sum over N rows of O(1) values
ZERO_GRADS = ("O_h.bias", "FFN_h_layer2.bias")
ZERO_TOL = {"fp32": 5e-3, "bf16": 5e-2}
# launches of one layer at d % 8 == 0, training, E > 0, no dropout (DESIGN.md): forward 10 (planes, bitmap + E2, edge
# and node projections, attention, O_h, BN1, FFN1, FFN2, BN2), backward 18 as counted on an H100 (DESIGN.md)
LAUNCHES_FWD, LAUNCHES_BWD = 10, 18


def _load(name):
    return torch.load(os.path.join(SAN_DIR, name + ".pt"), weights_only=False)


def _gb(x, e, ei, batch, num_graphs):
    return GraphBatch(x=x, edge_index=ei, edge_attr=e, batch=batch, num_graphs=num_graphs)


def _module(cfg, precision="fp32", p=0.0):
    emb = nn.Embedding(1, cfg["d"])
    layers = [graphgps_b200.SANLayer(cfg["gamma"], cfg["d"], cfg["d"], cfg["heads"], True, emb, p, precision=precision)
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


def _check(res, ref, precision, what, training=True):
    bad, worst = {}, 0.0
    e = rel_err(res["out"], ref["out"])
    if not e <= FWD_TOL[precision]:
        bad["out"] = e
    grads = [("grad_x", res["grad_x"], ref["grad_x"]), ("grad_edge_attr", res["grad_edge_attr"], ref["grad_edge_attr"])]
    grads += [("grad:" + n, res["grad_params"][n], g) for n, g in ref["grad_params"].items()]
    for k, a, g in grads:
        e = rel_err(a, g)
        if training and k.endswith(ZERO_GRADS):
            if not float((a.double() - g.double()).abs().max()) <= ZERO_TOL[precision]:
                bad[k] = e
            continue
        worst = max(worst, e)
        if not e <= GRAD_TOL[precision]:
            l2 = rel_l2(a, g)
            if not l2 <= GRAD_L2[precision]:
                bad[k] = (e, l2)
    assert not bad, f"{what}: {bad}"
    return worst


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", FIXTURES)
def test_fixture(name, precision):
    if name == "saturate_hd8" and precision == "bf16":
        # scores of |t| ~ 20 carry bf16 rounding of ~2^-9 |t| ~ 0.04: the clamp mask of every pair that close to +-5
        # flips, which moves the fake-pair weight gradients by O(10 %) in L2; fp32-grade holds this fixture instead
        pytest.skip("saturated scores are checked in fp32-grade only")
    if name == "two_layer_shared_hd6" and precision == "bf16":
        # 61 rows per BatchNorm column through two layers: bf16 rounding moves the near-cancelling BatchNorm-bias and
        # FFN1-bias gradients by ~0.2 relative L2; the shared-embedding gradient is held in fp32-grade
        pytest.skip("two stacked layers on 61 rows are checked in fp32-grade only")
    fix = _load(name)
    res = _run(_layer(fix, precision), fix)
    worst = _check(res, fix, precision, f"{name} {precision}", fix["config"]["training"])
    print(name, precision, f"out {rel_err(res['out'], fix['out']):.2e} worst grad max-abs {worst:.2e}")


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
    # BN1's input, from the oracle's own steps
    emb = st["attention.fake_edge_emb.weight"][0]
    lin = lambda t, n: t @ st[n + ".weight"].t()  # noqa: E731
    h = san_attention(lin(x, "attention.Q"), lin(x, "attention.K"), lin(x, "attention.V"), lin(x, "attention.Q_2"),
                      lin(x, "attention.K_2"), lin(fix["edge_attr"].double(), "attention.E"),
                      st["attention.E_2.weight"] @ emb, fix["edge_index"], fake, fix["config"]["heads"],
                      fix["config"]["gamma"])
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
    # float64 reference, its gradients and each pair's score (to find the pairs at the clamp bounds)
    parts = [Y[:, i * d:(i + 1) * d].clone().requires_grad_(True) for i in range(5)]
    Er, E2r = Ee.clone().requires_grad_(True), E2.clone().requires_grad_(True)
    Oref = san_attention(*parts, Er, E2r, ei, fake, H, gamma)
    (Oref * dO).sum().backward()
    with torch.no_grad():
        v = lambda t: t.reshape(-1, H, hd)  # noqa: E731
        t_real = (v(parts[1])[ei[0]] * v(parts[0])[ei[1]] * v(Er)).sum(-1) / math.sqrt(hd)
        t_fake = (v(parts[4])[fake[0]] * v(parts[3])[fake[1]] * E2r.reshape(1, H, hd)).sum(-1) / math.sqrt(hd)
        near = lambda t: ((t.abs() - 5).abs() < 1e-4)  # noqa: E731
        # nodes touched by a pair within 1e-4 of a clamp bound: their gradients are excluded from the elementwise check
        bad_nodes = torch.zeros(N, dtype=torch.bool, device=DEV)
        bad_edges = near(t_real).any(-1)
        for (s, dd), m in (((ei[0], ei[1]), bad_edges), ((fake[0], fake[1]), near(t_fake).any(-1))):
            bad_nodes[s[m]] = True
            bad_nodes[dd[m]] = True
        saturated = float(((t_real.abs() > 5).double().mean() + (t_fake.abs() > 5).double().mean()) / 2)
    lib = _lib.load()
    Yf, Ef, E2f, dOf = (t.float().contiguous() for t in (Y, Ee, E2, dO))
    O = torch.empty(N, d, device=DEV)
    rz = torch.empty(N, H, device=DEV)
    dY = torch.empty(N, 5 * d, device=DEV)
    dE = torch.empty(E, d, device=DEV)
    dE2 = torch.empty(d, device=DEV)
    nmax = gs.nmax
    ws = torch.empty(lib.gps_san_attention_workspace_bytes(N, d, H, nmax), dtype=torch.uint8, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.gps_san_attention_forward(C.byref(gs.desc), H, hd, Yf.data_ptr(), 5 * d, Ef.data_ptr(),
                                             E2f.data_ptr(), gamma, nmax, ws.data_ptr(), ws.numel(), O.data_ptr(), d,
                                             rz.data_ptr(), st), "fwd")
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
    return errs, saturated, int(bad_nodes.sum())


# every shipped head dim: zinc 7, cluster 6, pattern 8, molhiv 16, molpcba 76, coco / voc 11, peptides 21
@pytest.mark.parametrize("hd,H,kind,gamma", [(7, 8, "mol", 1e-5), (6, 8, "sbm", 0.1), (8, 10, "sbm", 1e-5),
                                             (16, 4, "mol", 1e-5), (76, 4, "mol", 1e-5), (11, 8, "knn", 1e-6),
                                             (21, 4, "chain", 0.1)])
def test_attention_stage_head_dims(hd, H, kind, gamma):
    sizes = dataset_sizes(kind, 3 if kind in ("mol", "sbm") else 1, hd) + [1]
    errs, sat, nbad = _stage(kind, sizes, H, hd, gamma, seed=hd, scale=1.6)
    print(hd, kind, {k: f"{v:.1e}" for k, v in errs.items()}, f"saturated {sat:.2f}", "excluded nodes", nbad)
    assert sat > 0.01                       # a share of the scores lies beyond the clamp
    assert max(errs.values()) < 2e-5, errs


# ------------------------------------------------------------------------------------------ dropout
def _mask(rows, cols, p, offset, site):
    m = torch.empty(rows, cols, device=DEV)
    lib = _lib.load()
    _lib.check(lib.gps_dropout_mask(m.data_ptr(), rows, cols, p, int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF, offset,
                                    site, torch.cuda.current_stream().cuda_stream), "mask")
    return m.double() / (1.0 - p)


def _oracle_gpu(mod, b, ct, masks_per_layer=None):
    """float64 oracle of a layer (or stack) on the GPU: output and gradients by name."""
    layers = [mod] if isinstance(mod, graphgps_b200.SANLayer) else list(mod)
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
        h = san_forward(full, h, e, b.edge_index, fake, layer.num_heads, layer.gamma, layer.training, masks, pre)
    (h * ct.double()).sum().backward()
    return {"out": h.detach().cpu(), "grad_x": x.grad.cpu(), "grad_edge_attr": e.grad.cpu(),
            "grad_params": {n: t.grad.cpu() for n, t in state.items()}}


def test_dropout_both_sites_with_injected_masks():
    p = 0.3
    torch.manual_seed(7)
    cfg = dict(d=56, heads=8, gamma=1e-5, layers=1, training=True)
    mod = _module(cfg, "fp32", p).to(DEV)
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
    emb = mod[0].attention.fake_edge_emb.weight
    assert mod[1].attention.fake_edge_emb.weight is emb
    g = res["grad_params"]["0.attention.fake_edge_emb.weight"]
    assert rel_err(g, fix["grad_params"]["0.attention.fake_edge_emb.weight"]) < GRAD_TOL["fp32"]
    # the sum of each layer's own share: layer 1 alone (on layer 0's output) plus layer 0 alone
    assert float(g.abs().max()) > 0


# ------------------------------------------------------------------------------------------ reproducibility
def test_bitwise_reproducible_and_retain_graph():
    # d % 8 == 0: every product on the plane-fed GEMM, whose split-K sums in a fixed order (DESIGN.md)
    fix = _load("pattern_dense_hd6")
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
    g1 = torch.autograd.grad(loss, [xin, ein], retain_graph=True)
    g2 = torch.autograd.grad(loss, [xin, ein])
    assert torch.equal(g1[0], g2[0]) and torch.equal(g1[1], g2[1])


# ------------------------------------------------------------------------------------------ capture
def _seq_step(seq, x, e, b, ct):
    b.x, b.edge_attr = x, e
    out = seq(b).x
    return torch.autograd.grad((out * ct).sum(), [x, e] + list(seq.parameters())), out


@pytest.mark.parametrize("p", [0.0, 0.2])
def test_captured_two_layer_stack(p):
    torch.manual_seed(4)
    seq = _module(dict(d=56, heads=8, gamma=1e-5, layers=2), "fp32", p).to(DEV)
    sb = san_batch("mol", dataset_sizes("mol", 6, 6), 56, 6).to(DEV)
    b = _gb(sb.x, sb.edge_attr, sb.edge_index, sb.batch, 6)
    graph_of(b).nmax   # read before capture (the read synchronises); the eager step below also caches it
    ct = torch.randn(sb.x.shape, device=DEV)
    x = sb.x.clone().requires_grad_(True)
    e = sb.edge_attr.clone().requires_grad_(True)
    pin_dropout_counter(DEV, 4096 * 1000)
    eager_g, eager_out = _seq_step(seq, x, e, b, ct)
    eager_out = eager_out.detach()
    x = x.detach().clone().requires_grad_(True)
    e = e.detach().clone().requires_grad_(True)
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
    first = cap_out.clone()
    assert torch.equal(first, eager_out)
    for a, r in zip(cap_g, eager_g):
        assert torch.equal(a, r)
    graph.replay()
    torch.cuda.synchronize()
    if p > 0.0:
        assert not torch.equal(first, cap_out)   # fresh masks on every replay
    else:
        assert torch.equal(first, cap_out)


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
    mod = _module(dict(d=d, heads=H, gamma=gamma, layers=1), "fp32", p).to(DEV)
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
    ref = _oracle_gpu(mod, sb, ct, masks)
    worst = _check(res, ref, "fp32", f"{kind} B {B} d {d}")
    print(f"{kind} B {B} N {N} d {d} H {H}: out {rel_err(res['out'], ref['out']):.2e} worst grad {worst:.2e}")


def test_full_size_zinc_san():
    _full("mol", 32, 56, 8, 1e-5, 0.0, 21)


def test_full_size_molpcba_san():
    _full("mol", 512, 304, 4, 1e-5, 0.2, 22)


def test_full_size_coco_san():
    _full("knn", 8, 88, 8, 1e-6, 0.0, 23)
