"""The node-prediction heads and losses on the GPU: the reference's fixtures in fp32 and bf16, training and eval; the row
normalisation and the loss stages alone against float64; bitwise reproducibility; CUDA-graph capture of head + loss;
pinned launch counts; no synchronising call on a cached batch; and two layer chains into a head and its loss against
float64 oracle chains."""
import math
import os
import types

import pytest
import torch
import torch.nn.functional as F

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import GraphBatch
from custom_gnn_oracle import oracle_layer, run_stack
from node_head_oracle import LOSSES, ambiguous_rows, fixture_ct, fixture_labels, fixture_x, mlp, oracle, weighted_cross_entropy
from oracle.gps_oracle import OracleGPSLayer
from util import GOLDEN_DIR, rel_err, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NH_DIR = os.path.join(GOLDEN_DIR, "node_head")
FIXTURES = sorted(p[:-3] for p in os.listdir(NH_DIR) if p.endswith(".pt") and p != "reference_live.pt")
TOL = {"fp32": 1e-3, "bf16": 1e-2}
FN = {"weighted_cross_entropy": graphgps_b200.weighted_cross_entropy, "cross_entropy": graphgps_b200.cross_entropy}


def _load(name):
    return torch.load(os.path.join(NH_DIR, name + ".pt"), weights_only=False)


def _head(fix, precision="fp32"):
    c = fix["config"]
    cls = graphgps_b200.NodeHead if c["head"] == "node" else graphgps_b200.InductiveNodeHead
    h = cls(c["d"], c["dout"], layers_post_mp=c["L"], dim_inner=c["dim_inner"], precision=precision)
    h.load_state_dict({k: v.float() for k, v in fix["state"].items()}, strict=True)
    return h.to(DEV)


def _batch(fix, x):
    c = fix["config"]
    b = types.SimpleNamespace(x=x, y=fixture_labels(fix).to(DEV))
    if c["head"] == "node":
        b.split = c["split"]
        for k, m in fix["masks"].items():
            setattr(b, f"{k}_mask", m.to(DEV))
    return b


def _step(head, fix, mode, data=None):
    """loss, pred_score, grad_x and the parameter gradients of the library's head and loss on the fixture."""
    head.zero_grad(set_to_none=True)
    x = fixture_x(fix).float().to(DEV).requires_grad_(True)
    data = _batch(fix, x) if data is None else data
    data.x = x
    pred, true = head(data)
    if fix["config"]["dout"] == 1:
        pred = pred.squeeze(-1)
    loss, score = FN[fix["config"]["loss"]](pred, true)
    out = loss if mode == "loss" else (score * fixture_ct(fix).float().to(DEV)).sum()
    out.backward()
    torch.cuda.synchronize()
    gx = x.grad if x.grad is not None else torch.zeros_like(x)
    return (loss.detach().cpu(), score.detach().cpu(), gx.cpu(),
            {n: (p.grad if p.grad is not None else torch.zeros_like(p)).cpu() for n, p in head.named_parameters()})


def _err(a, r):
    """Largest deviation over the largest reference entry; NaN patterns must agree exactly."""
    a, r = a.double(), r.double()
    if not torch.equal(torch.isnan(a), torch.isnan(r)):
        return math.inf
    fin = ~torch.isnan(r)
    if not fin.any():
        return 0.0
    return float((a[fin] - r[fin]).abs().max()) / max(float(r[fin].abs().max()), 1e-30)


@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", FIXTURES)
def test_fixture(name, precision, mode):
    """fp32 against the reference's values (the oracle where a fixture stores no grad_x or pred_score); bf16 against
    the float64 oracle with the bf16-rounded product operands of that mode.  Both upstream gradients: loss.backward()
    and a cotangent on pred_score.  In fp32, a hidden pre-activation within 2^-16 of its term scale of zero (about 1 %
    of the rows at VOC shapes) can take the other side of the ReLU under the three-MMA bf16 hi / lo products (two VOC
    rows do); those rows' grad_x is left out, and the first layers' gradients are held to 5e-3 in relative L2 there."""
    fix = _load(name)
    head = _head(fix, precision).train(mode == "train")
    fallbacks = _lib.load().gps_fallback_count()
    tol = TOL[precision]
    for grad_mode, sfx in (("loss", ""), ("ct", "_ct")):
        loss, score, gx, grads = _step(head, fix, grad_mode)
        o_loss, o_score, o_gx, o_grads = oracle(fix, grad_mode, bf16=precision == "bf16")
        if precision == "fp32":
            o_loss = torch.tensor(fix["loss"], dtype=torch.float64)
            o_score = fix.get("pred_score", o_score)
            o_gx = fix.get("grad_x" + sfx, o_gx)
            o_grads = fix["grads" + sfx]
        amb = ambiguous_rows(fix) if precision == "fp32" else torch.zeros(gx.shape[0], dtype=torch.bool)
        assert int(amb.sum()) <= max(2, gx.shape[0] // 50)
        checks = [("loss", loss.reshape(1), o_loss.reshape(1)), ("pred_score", score, o_score),
                  ("grad_x", gx[~amb], o_gx[~amb])]
        for what, a, r in checks:
            e = _err(a, r)
            assert e <= tol, (grad_mode, what, e)
        for k, g in o_grads.items():   # a flipped ReLU (amb rows) moves one unit's share of the first layers' grads
            e = _err(grads[k], g)
            assert e <= tol or (amb.any() and not torch.isnan(g).any() and rel_l2(grads[k], g) <= 5e-3), \
                (grad_mode, k, e)
    assert _lib.load().gps_fallback_count() == fallbacks   # every product ran on the TMA GEMM


# ------------------------------------------------------------------------------------------ stages
@pytest.mark.parametrize("d,ld", [(96, 96), (40, 48), (1024, 1024), (4096, 4096)])
def test_l2norm_stage_against_float64(d, ld):
    """The normalisation alone through its stage entries: ReLU'd rows with zero rows (the 1e-12 branch) and rows of
    tiny norm, forward and backward against float64 at 1e-5 relative."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(d)
    rows = 777
    r64 = torch.relu(torch.randn(rows, d, generator=g, dtype=torch.float64))
    r64[[0, 5, 400]] = 0.0
    r64[7] *= 1e-20
    r = torch.zeros(rows, ld, device=DEV)
    r[:, :d] = r64.float().to(DEV)
    out = torch.full((rows, ld), 7.0, device=DEV)
    norm = torch.empty(rows, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.gps_row_l2norm_forward(r.data_ptr(), rows, d, ld, out.data_ptr(), norm.data_ptr(), st), "fwd")
    rr = r[:, :d].double().cpu().requires_grad_(True)
    ref = rr / rr.norm(dim=1, keepdim=True).clamp_min(1e-12)
    assert rel_err(out[:, :d].cpu(), ref.detach()) < 1e-5
    assert (out[:, d:] == 7.0).all()
    assert rel_err(norm.cpu(), rr.detach().norm(dim=1)) < 1e-5
    gg = torch.randn(rows, d, generator=g, dtype=torch.float64)
    gpad = torch.zeros(rows, ld, device=DEV)
    gpad[:, :d] = gg.float().to(DEV)
    gin = torch.full((rows, ld), 7.0, device=DEV)
    _lib.check(lib.gps_row_l2norm_backward(gpad.data_ptr(), out.data_ptr(), norm.data_ptr(), rows, d, ld, gin.data_ptr(),
                                           st), "bwd")
    (ref * gg).sum().backward()
    want = rr.grad * (rr.detach() > 0)   # times the ReLU mask
    got = gin[:, :d].cpu().double()
    big = rr.detach().norm(dim=1) >= 1e-12
    assert rel_err(got[big], want[big]) < 1e-5
    assert torch.allclose(got[~big], (gg * (rr.detach() > 0) / 1e-12)[~big], rtol=1e-5)
    # in place, as the head runs it
    _lib.check(lib.gps_row_l2norm_forward(r.data_ptr(), rows, d, ld, r.data_ptr(), norm.data_ptr(), st), "in place")
    torch.cuda.synchronize()
    assert torch.equal(r[:, :d], out[:, :d])


def _loss_stage(pred, true, weighted, g_loss, g_score):
    loss, score = (graphgps_b200.weighted_cross_entropy if weighted else graphgps_b200.cross_entropy)(
        pred.requires_grad_(True), true)
    (gp,) = torch.autograd.grad([loss, score], [pred], [g_loss, g_score])
    torch.cuda.synchronize()
    return loss.cpu(), score.detach().cpu(), gp.cpu()


@pytest.mark.parametrize("M,Cn,weighted", [(15000, 21, 1), (7742, 81, 1), (3000, 2, 1), (900, 1, 1), (7600, 5, 0),
                                           (300, 4096, 0), (300, 4096, 1), (1, 3, 0), (50000, 40, 1)])
def test_loss_stage_against_float64(M, Cn, weighted):
    """The loss alone: loss, pred_score and grad_pred from both the scalar gradient and a gradient of pred_score,
    against float64 at 1e-5 relative."""
    g = torch.Generator().manual_seed(M + Cn)
    pred64 = torch.randn(M, Cn, generator=g, dtype=torch.float64) * 3
    if Cn == 1:
        pred64 = pred64.flatten()
    true = torch.randint(0, max(Cn, 2), (M,), generator=g)
    g_loss = torch.tensor(1.7, dtype=torch.float64)
    g_score = torch.randn(pred64.shape, generator=g, dtype=torch.float64)
    loss, score, gp = _loss_stage(pred64.float().to(DEV), true.to(DEV), weighted, g_loss.float().to(DEV),
                                  g_score.float().to(DEV))
    pr = pred64.float().double().requires_grad_(True)
    rl, rs = (weighted_cross_entropy if weighted else LOSSES["cross_entropy"])(pr, true)
    (rg,) = torch.autograd.grad([rl, rs], [pr], [g_loss, g_score])
    assert abs(float(loss.detach()) - float(rl)) <= 1e-5 * abs(float(rl))
    assert rel_err(score, rs.detach()) < 1e-5
    assert rel_err(gp, rg) < 1e-5


def test_loss_edge_cases_follow_torch():
    """A one-class batch (weights sum to 0) and an empty selection give NaN as torch does; the pred_score path alone
    stays finite."""
    p = torch.randn(10, 4, device=DEV)
    loss, score = graphgps_b200.weighted_cross_entropy(p.clone().requires_grad_(True), torch.full((10,), 2, device=DEV))
    assert math.isnan(float(loss)) and torch.isfinite(score).all()
    loss, _ = graphgps_b200.cross_entropy(torch.zeros(0, 4, device=DEV), torch.zeros(0, dtype=torch.int64, device=DEV))
    assert math.isnan(float(loss))
    with pytest.raises(IndexError):
        graphgps_b200.cross_entropy(p, torch.full((10,), 4, device=DEV))
    with pytest.raises(NotImplementedError):
        graphgps_b200.cross_entropy(p, torch.full((10,), -100, device=DEV))
    with pytest.raises(TypeError):
        graphgps_b200.cross_entropy(p, torch.zeros(10, dtype=torch.int32, device=DEV))
    with pytest.raises(NotImplementedError):
        graphgps_b200.cross_entropy(torch.randn(2, 4097, device=DEV), torch.zeros(2, dtype=torch.int64, device=DEV))


# ------------------------------------------------------------------------------------------ determinism and capture
@pytest.mark.parametrize("name", ["voc_d96_L3", "actor_d64_C5_train", "binary_d64_L3"])
def test_bitwise_reproducible(name):
    fix = _load(name)
    head = _head(fix).train()
    a, b = _step(head, fix, "loss"), _step(head, fix, "loss")
    for u, v in zip(a[:3], b[:3]):
        assert torch.equal(u.nan_to_num(), v.nan_to_num())
    for k in a[3]:
        assert torch.equal(a[3][k], b[3][k]), k


@pytest.mark.parametrize("name", ["pattern_d64_L3", "webkb_d64_C5_val", "binary_d64_L3"])
def test_capture_head_and_loss(name):
    """After one warm-up call on the batch, head + loss forward + backward records into one CUDA graph and replays to
    the eager result bit for bit."""
    fix = _load(name)
    head = _head(fix).train()
    x = fixture_x(fix).float().to(DEV).requires_grad_(True)
    data = _batch(fix, x)
    ct = fixture_ct(fix).float().to(DEV)
    params = [x] + list(head.parameters())
    fn = FN[fix["config"]["loss"]]

    def step():
        data.x = x
        pred, true = head(data)
        if pred.dim() == 2 and pred.shape[1] == 1:
            pred = pred.squeeze(-1)
        loss, score = fn(pred, true)
        grads = torch.autograd.grad(loss + 0.5 * (score * ct).sum(), params)
        return (loss.detach(), score.detach()) + grads

    eager = step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap = step()
    g.replay()
    torch.cuda.synchronize()
    for i, (a, e) in enumerate(zip(cap, eager)):
        assert torch.equal(a, e), (i, float((a - e).abs().max()))


@pytest.mark.parametrize("name,counts", [
    # pad weights + x, 2 x (product, normalise), product, unpad + select | loss rows, partials, final
    # || loss' | seed, 3 x (weight product, data product), 2 x normalise', unpad
    ("voc_d96_L3", (7, 3, 1, 10)),
    # pad, product, unpad + select | loss: rows, partials, final || loss' | seed, rows, weight and data products, unpad
    ("actor_d64_C5_train", (3, 3, 1, 5)),
    ("odd_d37_inner40_L2", (5, 3, 1, 7))])
def test_launch_count(name, counts):
    fix = _load(name)
    head = _head(fix).train()
    _step(head, fix, "loss")
    lib = _lib.load()
    x = fixture_x(fix).float().to(DEV).requires_grad_(True)
    data = _batch(fix, x)
    fn = FN[fix["config"]["loss"]]
    f0, c0 = lib.gps_fallback_count(), lib.gps_launch_count()
    pred, true = head(data)
    c1 = lib.gps_launch_count()
    loss, score = fn(pred, true)
    c2 = lib.gps_launch_count()
    (gp,) = torch.autograd.grad(loss, [pred], retain_graph=True)
    c3 = lib.gps_launch_count()
    pred.backward(gp)
    c4 = lib.gps_launch_count()
    print("launches: head", c1 - c0, "loss", c2 - c1, "loss'", c3 - c2, "head'", c4 - c3)
    assert (c1 - c0, c2 - c1, c3 - c2, c4 - c3) == counts
    assert lib.gps_fallback_count() == f0


@pytest.mark.parametrize("head_kind,loss_fun", [("inductive_node", "weighted_cross_entropy"),
                                                ("node", "cross_entropy"), ("inductive_node", "cross_entropy"),
                                                ("node", "weighted_cross_entropy")])
def test_no_sync_on_a_cached_batch(head_kind, loss_fun):
    """Once the batch's rows and the labels have been read once, head + loss forward and backward make no synchronising
    call: torch's sync debug mode raises on any."""
    fix = _load("actor_d64_C5_train")
    fix = dict(fix, config=dict(fix["config"], head=head_kind, L=3 if head_kind == "inductive_node" else 1))
    torch.manual_seed(0)
    cls = graphgps_b200.NodeHead if head_kind == "node" else graphgps_b200.InductiveNodeHead
    head = cls(64, 5, layers_post_mp=fix["config"]["L"]).to(DEV)
    x = fixture_x(fix).float().to(DEV).requires_grad_(True)
    data = _batch(dict(fix, config=dict(fix["config"], head="node")), x)
    fn = FN[loss_fun]

    def step():
        data.x = x
        pred, true = head(data)
        loss, _ = fn(pred, true)
        loss.backward()

    step()
    torch.cuda.synchronize()
    data.x = x
    labels = data.y if head_kind == "inductive_node" else head(data)[1]
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
        if head_kind == "node":
            data.x = x
            assert head(data)[1] is labels   # the cached label tensor is returned again
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ chains
def test_chain_gatedgcn_inductive_head_weighted_ce_against_oracle():
    """GatedGCNLayer x 2 at d 108 -> InductiveNodeHead(L = 3) -> weighted cross-entropy -> backward, against the
    float64 chain."""
    torch.manual_seed(7)
    d, C = 108, 21
    layers = [graphgps_b200.GatedGCNLayer(d, d, dropout=0.0, residual=True, act="relu").to(DEV).train()
              for _ in range(2)]
    head = graphgps_b200.InductiveNodeHead(d, C, layers_post_mp=3).to(DEV).train()
    oracles = [oracle_layer("gatedgcn", d).double().train() for _ in range(2)]
    for o, layer in zip(oracles, layers):
        o.load_state_dict({k: v.detach().cpu() for k, v in layer.state_dict().items()}, strict=True)
    b = graphgps_b200.make_batch("zinc-gatedgcn", seed=3, dim=d, num_graphs=12)
    y = torch.randint(0, C, (b.x.shape[0],), generator=torch.Generator().manual_seed(1))
    x = b.x.to(DEV).clone().requires_grad_(True)
    data = GraphBatch(x=x, edge_index=b.edge_index.to(DEV), edge_attr=b.edge_attr.to(DEV), batch=b.batch.to(DEV),
                      num_graphs=12)
    data.y = y.to(DEV)
    for layer in layers:
        data = layer(data)
    pred, true = head(data)
    loss, _ = graphgps_b200.weighted_cross_entropy(pred, true)
    loss.backward()
    xr = b.x.double().clone().requires_grad_(True)
    hr, _ = run_stack(oracles, xr, b.edge_attr.double(), b.edge_index)
    hp = {k: v.detach().cpu().double().requires_grad_(True) for k, v in head.state_dict().items()}
    names = [n[:-7] for n in hp if n.endswith(".weight")]
    pr = mlp(hr, [hp[n + ".weight"] for n in names], [hp[n + ".bias"] for n in names])
    rl, _ = weighted_cross_entropy(pr, y)
    rl.backward()
    assert abs(float(loss) - float(rl)) < 1e-3 * abs(float(rl))
    assert rel_err(x.grad.cpu(), xr.grad) < 1e-3 or rel_l2(x.grad.cpu(), xr.grad) < 5e-3
    for n, p in head.named_parameters():
        assert rel_err(p.grad.cpu(), hp[n].grad) < 1e-3 or rel_l2(p.grad.cpu(), hp[n].grad) < 5e-3, n
    for layer, o in zip(layers, oracles):
        qs = dict(o.named_parameters())
        for n, p in layer.named_parameters():
            q = qs[n]
            if q.grad is None:   # the last layer's edge branch does not reach the loss
                continue
            assert rel_err(p.grad.cpu(), q.grad) < 1e-3 or rel_l2(p.grad.cpu(), q.grad) < 5e-3, n


def test_chain_gcn_transformer_node_head_ce_against_oracle():
    """A GCN+Transformer GPSLayer without normalisation -> NodeHead -> cross-entropy on a masked single graph ->
    backward, against the float64 chain."""
    torch.manual_seed(9)
    d, heads, C = 64, 4, 5
    layer = graphgps_b200.GPSLayer(d, "GCN", "Transformer", heads, act="gelu", batch_norm=False).to(DEV).train()
    ora = OracleGPSLayer(d, "GCN", "Transformer", heads, act="gelu", batch_norm=False).double().train()
    ora.load_state_dict({k: v.detach().cpu() for k, v in layer.state_dict().items()}, strict=True)
    head = graphgps_b200.NodeHead(d, C).to(DEV).train()
    b = graphgps_b200.make_batch("zinc-gine", seed=5, dim=d, num_graphs=1)
    N = b.x.shape[0]
    g = torch.Generator().manual_seed(2)
    y = torch.randint(0, C, (N,), generator=g)
    mask = torch.rand(N, generator=g) < 0.6
    bd = b.clone().to(DEV)
    x = bd.x.requires_grad_(True)
    bd.y, bd.split, bd.train_mask = y.to(DEV), "train", mask.to(DEV)
    bd = layer(bd)
    pred, true = head(bd)
    loss, _ = graphgps_b200.cross_entropy(pred, true)
    loss.backward()
    bo = b.clone()
    bo.x, bo.edge_attr = bo.x.double().requires_grad_(True), bo.edge_attr.double()
    xr = bo.x
    bo = ora(bo)
    w = head.layer_post_mp.model[0].model
    wr, br = w.weight.detach().cpu().double().requires_grad_(True), w.bias.detach().cpu().double().requires_grad_(True)
    pr = (bo.x @ wr.t() + br)[mask]
    rl = F.nll_loss(F.log_softmax(pr, -1), y[mask])
    rl.backward()
    assert abs(float(loss) - float(rl)) < 1e-3 * abs(float(rl))
    assert rel_err(x.grad.cpu(), xr.grad) < 1e-3 or rel_l2(x.grad.cpu(), xr.grad) < 5e-3
    for a, r in ((w.weight.grad, wr.grad), (w.bias.grad, br.grad)):
        assert rel_err(a.cpu(), r) < 1e-3 or rel_l2(a.cpu(), r) < 5e-3
    qs = dict(ora.named_parameters())
    for n, p in layer.named_parameters():
        if qs[n].grad is None:
            continue
        assert rel_err(p.grad.cpu(), qs[n].grad) < 1e-3 or rel_l2(p.grad.cpu(), qs[n].grad) < 5e-3, n
