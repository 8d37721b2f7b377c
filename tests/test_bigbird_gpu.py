"""GPU: the BigBird global model (gps_layer.py:115-119,207-208; bigbird_layer.py of the reference).

Stages against float64 restatements: block-sparse attention forward and backward for head dims 7, 8, 16 and 19, block
sizes 2, 3, 4, one and three random blocks and every plan branch, and the row-wise LayerNorm.  Then the layer against
every fixture of tests/golden/bigbird/ (fp32 and bf16), the other local models under BigBird against their oracles,
one graph in two batches of different Nmax, dropout with the library's masks injected into the oracle, bitwise
reproducibility, a captured 3-layer stack against eager execution, and a batch the reference cannot run."""
import copy
import ctypes as C
import glob as _glob
import os
import types

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib, bigbird as bbmod
from graphgps_b200.graph import graph_of
from bigbird_oracle import attach_bigbird, bb_batch, bigbird_cfg, bigbird_oracle_layer, multiplicity
from util import _stream, compare, golden_batch, GOLDEN_DIR, pin_dropout_counter, rel_err, run_layer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = {"fp32": 1e-3, "bf16": 1e-2}
GRAD_L2 = {"fp32": 5e-3, "bf16": 1e-1}
BB_DIR = os.path.join(GOLDEN_DIR, "bigbird")
FIXTURES = sorted(os.path.basename(p)[:-3] for p in _glob.glob(os.path.join(BB_DIR, "*.pt"))
                  if not p.endswith("tables.pt"))


def _load(name):
    return torch.load(os.path.join(BB_DIR, name + ".pt"), weights_only=False)


# ------------------------------------------------------------------------------------------------- stages
def _bb_struct(sizes, bs, r, H):
    nmax = max(sizes)
    nb = bbmod.padded_length(nmax, bs) // bs
    R = bbmod.random_table(nb * bs, bs, H, r)
    lists = [torch.from_numpy(a).to(DEV) for a in bbmod.block_lists(R, nb)]
    b = _lib.GpsBigBird()
    b.block_size, b.num_blocks, b.hidden_act, b.ln_eps = bs, nb, 0, 1e-6
    b.key_ptr, b.key_idx, b.query_ptr, b.query_idx = (t.data_ptr() for t in lists)
    return b, R, nb, lists


def _dense_attention(Q, K, V, sizes, R, nb, bs, H, hd):
    """fp64 restatement over each graph: p = W exp(s) / sum W exp(s) with the block multiplicity W."""
    W = multiplicity(R, nb, bs)
    outs, lses = [], []
    r0 = 0
    for n in sizes:
        q = Q[r0:r0 + n].view(n, H, hd).transpose(0, 1)
        k = K[r0:r0 + n].view(n, H, hd).transpose(0, 1)
        v = V[r0:r0 + n].view(n, H, hd).transpose(0, 1)
        s = q @ k.transpose(1, 2) / hd ** 0.5
        w = W[:, :n, :n]
        s = s.masked_fill(w == 0, float("-inf"))
        m = s.amax(-1, keepdim=True)
        e = w * torch.exp(s - m)
        den = e.sum(-1, keepdim=True)
        outs.append(((e / den) @ v).transpose(0, 1).reshape(n, H * hd))
        lses.append((m + den.log()).squeeze(-1).transpose(0, 1))
        r0 += n
    return torch.cat(outs), torch.cat(lses)


CASES = [(hd, bs, r, sizes) for hd in (7, 8, 16, 19) for bs, r, sizes in (
    (3, 3, [20, 13, 16, 9]),         # one band
    (3, 3, [30, 13, 26, 8]),         # two bands (r // 2, r - r // 2)
    (3, 3, [40, 33, 7]),             # two bands (r, 0)
    (2, 1, [15, 22, 9, 18]),
    (4, 3, [31, 22, 61, 18]),
    (3, 1, [12, 7, 10, 4]),          # nb = 4
)]


@pytest.mark.parametrize("hd,bs,r,sizes", CASES, ids=[f"hd{c[0]}-bs{c[1]}-r{c[2]}-n{max(c[3])}" for c in CASES])
def test_attention_forward_backward_vs_fp64(hd, bs, r, sizes):
    lib = _lib.load()
    H = 3
    d = H * hd
    b = bb_batch(sizes, 4).to(DEV)
    gs = graph_of(b)
    st, R, nb, lists = _bb_struct(sizes, bs, r, H)
    N = sum(sizes)
    gen = torch.Generator().manual_seed(hd * 100 + bs * 10 + r)
    qkv = torch.randn(N, 3 * d + 5, generator=gen, dtype=torch.float64)   # ld = 3d + 5
    Q, K, V = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:3 * d]
    dO = torch.randn(N, d, generator=gen, dtype=torch.float64)
    dqkv = qkv.float().to(DEV)
    O = torch.full((N, d), float("nan"), device=DEV)
    lse = torch.full((N, H), float("nan"), device=DEV)
    ld = 3 * d + 5
    _lib.check(lib.gps_bigbird_attention_forward(C.byref(gs.desc), H, hd, C.byref(st), dqkv.data_ptr(),
                                                 dqkv[:, d:].data_ptr(), dqkv[:, 2 * d:].data_ptr(), ld, O.data_ptr(),
                                                 d, lse.data_ptr(), _stream()), "bb fwd")
    Qr, Kr, Vr = (t.clone().requires_grad_(True) for t in (Q, K, V))
    Oref, lref = _dense_attention(Qr, Kr, Vr, sizes, R, nb, bs, H, hd)
    assert rel_err(O.cpu(), Oref.detach()) <= 2e-5
    assert rel_err(lse.cpu(), lref.detach()) <= 2e-5
    (Oref * dO).sum().backward()
    delta = torch.full((N, H), float("nan"), device=DEV)
    g = torch.full((N, 3 * d), float("nan"), device=DEV)
    dOd = dO.float().to(DEV)
    _lib.check(lib.gps_bigbird_attention_backward(C.byref(gs.desc), H, hd, C.byref(st), dqkv.data_ptr(),
                                                  dqkv[:, d:].data_ptr(), dqkv[:, 2 * d:].data_ptr(), ld, O.data_ptr(),
                                                  dOd.data_ptr(), d, lse.data_ptr(), delta.data_ptr(), g.data_ptr(),
                                                  g[:, d:].data_ptr(), g[:, 2 * d:].data_ptr(), 3 * d, _stream()),
               "bb bwd")
    for name, got, ref in (("dQ", g[:, :d], Qr.grad), ("dK", g[:, d:2 * d], Kr.grad), ("dV", g[:, 2 * d:], Vr.grad)):
        assert not torch.isnan(got).any(), name
        assert rel_err(got.cpu(), ref) <= 5e-5, (name, rel_err(got.cpu(), ref))
    # the same bits in a second run
    g2 = torch.full_like(g, float("nan"))
    _lib.check(lib.gps_bigbird_attention_backward(C.byref(gs.desc), H, hd, C.byref(st), dqkv.data_ptr(),
                                                  dqkv[:, d:].data_ptr(), dqkv[:, 2 * d:].data_ptr(), ld, O.data_ptr(),
                                                  dOd.data_ptr(), d, lse.data_ptr(), delta.data_ptr(), g2.data_ptr(),
                                                  g2[:, d:].data_ptr(), g2[:, 2 * d:].data_ptr(), 3 * d, _stream()),
               "bb bwd")
    assert torch.equal(g, g2)


@pytest.mark.parametrize("rows,d", [(1, 8), (129, 56), (1000, 64), (77, 1024)])
def test_layernorm_forward_backward_vs_fp64(rows, d):
    lib = _lib.load()
    gen = torch.Generator().manual_seed(rows + d)
    z = torch.randn(rows, d, generator=gen, dtype=torch.float64) * 3 + 1.5
    gamma = torch.rand(d, generator=gen, dtype=torch.float64) + 0.5
    beta = torch.randn(d, generator=gen, dtype=torch.float64)
    gy = torch.randn(rows, d, generator=gen, dtype=torch.float64)
    zr, gr, br = (t.clone().requires_grad_(True) for t in (z, gamma, beta))
    y_ref = torch.nn.functional.layer_norm(zr, (d,), gr, br, 1e-6)
    (y_ref * gy).sum().backward()
    zd, gd, bd, gyd = (t.float().to(DEV) for t in (z, gamma, beta, gy))
    y, mean, rstd = torch.empty_like(zd), torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
    _lib.check(lib.gps_layernorm_forward(zd.data_ptr(), rows, d, gd.data_ptr(), bd.data_ptr(), 1e-6, y.data_ptr(),
                                         mean.data_ptr(), rstd.data_ptr(), _stream()), "ln fwd")
    assert rel_err(y.cpu(), y_ref.detach()) <= 2e-5
    dz = torch.empty_like(zd)
    ggam, gbet = torch.full((d,), 7.0, device=DEV), torch.full((d,), 7.0, device=DEV)
    ws = torch.empty(264 * d, device=DEV)
    _lib.check(lib.gps_layernorm_backward(gyd.data_ptr(), zd.data_ptr(), rows, d, gd.data_ptr(), mean.data_ptr(),
                                          rstd.data_ptr(), dz.data_ptr(), ggam.data_ptr(), gbet.data_ptr(),
                                          ws.data_ptr(), 0, _stream()), "ln bwd")
    assert rel_err(dz.cpu(), zr.grad) <= 5e-5
    assert rel_err(ggam.cpu(), gr.grad) <= 5e-5 and rel_err(gbet.cpu(), br.grad) <= 5e-5
    _lib.check(lib.gps_layernorm_backward(gyd.data_ptr(), zd.data_ptr(), rows, d, gd.data_ptr(), mean.data_ptr(),
                                          rstd.data_ptr(), dz.data_ptr(), ggam.data_ptr(), gbet.data_ptr(),
                                          ws.data_ptr(), 1, _stream()), "ln bwd accumulate")
    assert rel_err(gbet.cpu(), 2 * br.grad) <= 5e-5


# ------------------------------------------------------------------------------------------------- layer
def _ours(fix, precision="fp32", **kw):
    c = fix["config"]
    layer = graphgps_b200.GPSLayer(c["d"], c["local"], "BigBird", c["heads"], batch_norm=c["batch_norm"],
                                   bigbird_cfg=types.SimpleNamespace(**c["bigbird"]), precision=precision, **kw)
    layer.load_state_dict(fix["state"], strict=True)
    return layer.to(DEV).train(c["training"])


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", FIXTURES)
def test_layer_matches_fixture(name, precision):
    fix = _load(name)
    layer = _ours(fix, precision)
    res = run_layer(layer, golden_batch(fix, DEV), fix, backward="grad_x" in fix)
    compare(res, fix, TOL[precision], f"{name} {precision}", grad_l2_tol=GRAD_L2[precision])


def _oracle_for(local, d, H, cfg, **kw):
    import gat_oracle
    import genconv_oracle
    import pna_oracle
    if local == "GAT":
        layer = gat_oracle.gat_oracle_layer(d, "None", H, **kw)
    elif local == "GENConv":
        layer = genconv_oracle.genconv_oracle_layer(d, "None", H, **kw)
    elif local == "PNA":
        layer = pna_oracle.pna_oracle_layer(d, "None", H, pna_degrees=[0, 3, 11, 9, 4, 1], **kw)
    else:
        return bigbird_oracle_layer(d, local, H, cfg, **kw)
    return attach_bigbird(layer, d, H, cfg, kw.get("dropout", 0.0))


@pytest.mark.parametrize("local", ["GCN", "GAT", "GENConv", "PNA", "CustomGatedGCN", "None"])
def test_every_local_model_under_bigbird(local):
    d, H = 56, 8
    torch.manual_seed(11)
    cfg = bigbird_cfg()
    ora = _oracle_for(local, d, H, cfg)
    kw = dict(pna_degrees=[0, 3, 11, 9, 4, 1]) if local == "PNA" else {}
    ours = graphgps_b200.GPSLayer(d, local, "BigBird", H, bigbird_cfg=bigbird_cfg(), **kw)
    ours.load_state_dict(ora.state_dict(), strict=True)
    ours = ours.to(DEV).train()
    b = bb_batch([23, 17, 30, 21, 12], d, seed=4)
    if local == "PNA":
        b.edge_attr = b.edge_attr[:, :min(128, d)].contiguous()
    g = torch.Generator().manual_seed(4)
    fix = {"config": dict(local=local), "ct_x": torch.randn(b.x.shape, generator=g)}
    if local == "CustomGatedGCN":
        fix["ct_e"] = torch.randn(b.edge_attr.shape, generator=g)
    o64 = ora.double().train()   # (the GAT oracle wraps its own forward: no deepcopy)
    bb64 = b.clone()
    bb64.x, bb64.edge_attr = bb64.x.double(), bb64.edge_attr.double()
    ref = run_layer(o64, bb64, fix)
    res = run_layer(ours, b.clone().to(DEV), fix)
    tgt = {k: ref[k] for k in ("out_x", "out_e", "grad_x", "grad_e") if k in ref}
    tgt["grad_params"], tgt["state_after"] = ref["grad_params"], ref["state_after"]
    compare(res, tgt, 1e-3, f"{local}+BigBird", grad_l2_tol=5e-3)


def test_same_graph_in_two_batches_differs_and_matches_oracle():
    d, H = 56, 8
    torch.manual_seed(5)
    cfg = bigbird_cfg()
    ora = bigbird_oracle_layer(d, "GINE", H, cfg).eval()
    ours = graphgps_b200.GPSLayer(d, "GINE", "BigBird", H, bigbird_cfg=bigbird_cfg())
    ours.load_state_dict(ora.state_dict(), strict=True)
    ours = ours.to(DEV).eval()
    b1 = bb_batch([20, 13, 16], d, seed=9)      # Nmax 20
    b2 = bb_batch([20, 13, 37], d, seed=9)      # the same first graph, Nmax 37
    outs = []
    for b in (b1, b2):
        with torch.no_grad():
            got = ours(b.clone().to(DEV)).x.cpu()
            o64 = copy.deepcopy(ora).double()
            bb = b.clone()
            bb.x, bb.edge_attr = bb.x.double(), bb.edge_attr.double()
            ref = o64(bb).x
        assert rel_err(got, ref) <= 1e-3
        outs.append(got[:20])
    assert float((outs[0] - outs[1]).abs().max()) > 1e-3


def test_dropout_matches_oracle_with_injected_masks():
    """BigBird's two dropouts (sites 8 and 9) and the GPS dropouts (4: dropout_attn, 5 / 6: the FFN) replayed through
    gps_dropout_mask and injected into the oracle: the comparison is exact up to rounding."""
    lib = _lib.load()
    d, H, p = 56, 8, 0.2
    torch.manual_seed(6)
    cfg = bigbird_cfg()
    ora = bigbird_oracle_layer(d, "None", H, cfg, dropout=p)
    ours = graphgps_b200.GPSLayer(d, "None", "BigBird", H, dropout=p, bigbird_cfg=bigbird_cfg())
    ours.load_state_dict(ora.state_dict(), strict=True)
    ours = ours.to(DEV).train()
    b = bb_batch([23, 17, 30, 21, 12], d, seed=2)
    N = b.x.shape[0]
    base = 33 * 4096
    pin_dropout_counter(DEV, base)
    seed = int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF
    masks = {}
    for site, cols in ((4, d), (5, 2 * d), (6, d), (8, d), (9, d)):
        m = torch.empty(N, cols, device=DEV)
        _lib.check(lib.gps_dropout_mask(m.data_ptr(), N, cols, p, seed, base + 4096, site, _stream()), "mask")
        masks[site] = m.cpu().double()

    class Fixed(torch.nn.Module):
        def __init__(self, m):
            super().__init__()
            self.m = m

        def forward(self, t):
            return t * self.m / (1.0 - p)

    o64 = copy.deepcopy(ora).double().train()
    o64.dropout_attn, o64.ff_dropout1, o64.ff_dropout2 = Fixed(masks[4]), Fixed(masks[5]), Fixed(masks[6])
    o64.self_attn.masks = {"self_out": masks[8], "output": masks[9]}
    g = torch.Generator().manual_seed(4)
    fix = {"config": dict(local="None"), "ct_x": torch.randn(b.x.shape, generator=g)}
    bb = b.clone()
    bb.x, bb.edge_attr = bb.x.double(), bb.edge_attr.double()
    ref = run_layer(o64, bb, fix)
    res = run_layer(ours, b.clone().to(DEV), fix)
    tgt = {k: ref[k] for k in ("out_x", "grad_x")}
    tgt["grad_params"], tgt["state_after"] = ref["grad_params"], ref["state_after"]
    compare(res, tgt, 1e-3, "BigBird with dropout masks injected", grad_l2_tol=5e-3)
    o_plain = copy.deepcopy(o64)
    o_plain.self_attn.masks = {"self_out": torch.ones_like(masks[8]) * (1 - p),
                               "output": torch.ones_like(masks[9]) * (1 - p)}
    with torch.no_grad():
        plain = o_plain(bb.clone()).x
    assert rel_err(res["out_x"], plain.float()) > 1e-2


def test_two_runs_are_bitwise_identical():
    fix = _load("gine_bigbird_relu")
    outs = []
    for _ in range(2):
        layer = _ours(fix)
        outs.append(run_layer(layer, golden_batch(fix, DEV), fix))
    a, b = outs
    assert torch.equal(a["out_x"], b["out_x"]) and torch.equal(a["grad_x"], b["grad_x"])
    for n in a["grad_params"]:
        assert torch.equal(a["grad_params"][n], b["grad_params"][n]), n


def test_captured_stack_replay_equals_eager():
    """A 3-layer GINE+BigBird stack at the shipped shape: two eager steps give the same bits, and a captured step
    replays them exactly; no dense product leaves the tensor-core kernels."""
    from graphgps_b200.batch import make_batch
    torch.manual_seed(7)
    d, H = 56, 8
    stack = graphgps_b200.GPSStack(3, d, "GINE", "BigBird", H, bigbird_cfg=bigbird_cfg()).to(DEV).train()
    fb0 = _lib.load().gps_fallback_count()
    gb = make_batch("zinc-gine", seed=3, dim=d).to(DEV)
    graph_of(gb)
    ct = torch.randn(gb.x.shape, generator=torch.Generator().manual_seed(3)).to(DEV)
    runs = []
    for _ in range(2):
        state = {k: v.clone() for k, v in stack.state_dict().items()}
        eb = gb.clone()
        eb.__dict__["_gps_b200_graph"] = graph_of(gb)
        eb.x.requires_grad_(True)
        eb.edge_attr.requires_grad_(True)
        ex, ee = eb.x, eb.edge_attr
        out = stack(eb)
        out.x.backward(ct)
        runs.append((out.x.detach().clone(), ex.grad.clone(), ee.grad.clone(),
                     [p.grad.clone() for p in stack.parameters()]))
        for p in stack.parameters():
            p.grad = None
        stack.load_state_dict(state)
        del out, eb
    for a, c in zip(runs[0][:3], runs[1][:3]):
        assert torch.equal(a, c)
    for a, c in zip(runs[0][3], runs[1][3]):
        assert torch.equal(a, c)
    eager = runs[0]
    step = stack.capture(gb, ct)
    step.replay()
    step.replay()
    torch.cuda.synchronize()
    assert torch.equal(step.x_out, eager[0]) and torch.equal(step.grad_x, eager[1])
    assert torch.equal(step.grad_e, eager[2])
    for (n, p), g in zip(stack.named_parameters(), eager[3]):
        assert torch.equal(p.grad, g), n
    assert _lib.load().gps_fallback_count() == fb0


def test_batch_the_reference_cannot_run_raises_before_any_launch():
    lib = _lib.load()
    layer = graphgps_b200.GPSLayer(56, "GINE", "BigBird", 8, bigbird_cfg=bigbird_cfg()).to(DEV)
    b = bb_batch([9, 7, 5], 56).to(DEV)          # Nmax 9: 3 blocks of 3
    graph_of(b).nmax                             # the batch's own structure (built once per batch, for every layer)
    torch.cuda.synchronize()
    n0 = lib.gps_launch_count()
    with pytest.raises(NotImplementedError):
        layer(b)
    assert lib.gps_launch_count() == n0
    layer5 = graphgps_b200.GPSLayer(56, "GINE", "BigBird", 8, bigbird_cfg=bigbird_cfg(num_random_blocks=5)).to(DEV)
    with pytest.raises(NotImplementedError):
        layer5(bb_batch([36, 7, 5], 56).to(DEV))  # nb = 12 with r = 5: the plan cannot fill a row
