"""The graph-prediction heads on the GPU: the reference's fixtures in fp32 and bf16, training and eval; the pooling
stages against float64; bitwise reproducibility; CUDA-graph capture; pinned launch counts; the error paths; and layer
stacks chained into each head and an L1 loss, against float64 oracle chains."""
import ctypes as C
import os
import types

import pytest
import torch
import torch.nn.functional as F

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.graph import GraphStructure, graph_of
from graph_head_oracle import fixture_batch, fixture_ct, fixture_x, graphormer_head, oracle, pool, san_head
from graphormer_oracle import graphormer_batch, graphormer_forward
from oracle.gps_oracle import OracleGPSLayer
from util import GOLDEN_DIR, rel_err, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GH_DIR = os.path.join(GOLDEN_DIR, "graph_head")
FIXTURES = sorted(p[:-3] for p in os.listdir(GH_DIR) if p.endswith(".pt") and p != "reference_live.pt")
TOL = {"fp32": 1e-3, "bf16": 1e-2}
POOLINGS = ("mean", "add", "graph_token")


def _load(name):
    return torch.load(os.path.join(GH_DIR, name + ".pt"), weights_only=False)


def _head(fix, precision="fp32"):
    c = fix["config"]
    if c["kind"] == "san_graph":
        h = graphgps_b200.SANGraphHead(c["d"], c["dout"], L=c["L"], graph_pooling=c["pooling"], act=c["act"],
                                       precision=precision)
    else:
        h = graphgps_b200.GraphormerHead(c["d"], c["dout"], graph_pooling=c["pooling"], precision=precision)
    h.load_state_dict({k: v.float() for k, v in fix["state"].items()}, strict=True)
    return h.to(DEV)


def _batch(fix, x):
    bvec = fixture_batch(fix).to(DEV)
    return types.SimpleNamespace(x=x, edge_index=torch.zeros(2, 0, dtype=torch.int64, device=DEV), batch=bvec,
                                 num_graphs=fix["num_graphs"], y=torch.zeros(fix["num_graphs"], device=DEV))


def _step(head, fix, data=None):
    head.zero_grad(set_to_none=True)
    x = fixture_x(fix).float().to(DEV).requires_grad_(True)
    data = _batch(fix, x) if data is None else data
    data.x = x
    pred, y = head(data)
    assert y is data.y and data.graph_feature is pred
    (pred * fixture_ct(fix).float().to(DEV)).sum().backward()
    torch.cuda.synchronize()
    return pred.detach().cpu(), x.grad.cpu(), {n: p.grad.cpu() for n, p in head.named_parameters()}


def _err(a, r):
    return float((a.double() - r.double()).abs().max()) / max(float(r.abs().max()), 1e-30)


@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", FIXTURES)
def test_fixture(name, precision, mode):
    """fp32 against the reference's values.  bf16 against the float64 oracle with the bf16-rounded product operands
    of that mode: single-pass bf16 products move these heads' input gradients by up to 14 % of their largest entry
    against exact arithmetic (ReLU masks flip, the sums over a few hidden units cancel), which the oracle shows too."""
    fix = _load(name)
    head = _head(fix, precision).train(mode == "train")
    fallbacks = _lib.load().gps_fallback_count()
    pred, gx, grads = _step(head, fix)
    assert _lib.load().gps_fallback_count() == fallbacks   # every product ran on the TMA GEMM
    if precision == "fp32":
        ref_pred, ref_gx, ref_grads = fix["pred"], fix["grad_x"] if "grad_x" in fix else oracle(fix)[1], fix["grads"]
    else:
        ref_pred, ref_gx, ref_grads = oracle(fix, bf16=True)
    tol = TOL[precision]
    for what, a, r in [("pred", pred, ref_pred), ("grad_x", gx, ref_gx)] + \
            [(k, grads[k], g) for k, g in ref_grads.items()]:
        e = _err(a, r)
        assert e <= tol, (what, e)
    if fix["config"]["pooling"] == "graph_token":   # zero off the token rows
        off = torch.ones(gx.shape[0], dtype=torch.bool)
        off[fix["ptr"][:-1][torch.diff(fix["ptr"]) > 0]] = False
        assert not gx[off].any()


def _pool_stage(gs, pooling, x, d, ldo=None):
    lib = _lib.load()
    ldo = ldo or d
    out = torch.full((gs.B, ldo), 7.0, device=DEV)
    ws = torch.empty(8 * -(-gs.N // 64) * (-(-d // 4) * 4) + 16, dtype=torch.uint8, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.gps_graph_pool_forward(C.byref(gs.desc), _lib.POOLING[pooling], x.data_ptr(), d, out.data_ptr(), ldo,
                                          ws.data_ptr(), ws.numel(), st), "gps_graph_pool_forward")
    g = torch.randn(gs.B, d, device=DEV, dtype=torch.float32)
    gx = torch.full((gs.N, d), 7.0, device=DEV)
    _lib.check(lib.gps_graph_pool_backward(C.byref(gs.desc), _lib.POOLING[pooling], g.data_ptr(), d, d, gx.data_ptr(),
                                           st), "gps_graph_pool_backward")
    torch.cuda.synchronize()
    return out.cpu(), g.cpu(), gx.cpu()


@pytest.mark.parametrize("pooling", POOLINGS)
@pytest.mark.parametrize("case", ["edge_cases_L0_add", "edge_cases_L3_mean", "one_large_graph", "pcqm4m_d304_mean",
                                  "odd_width"])
def test_pool_stage_against_float64(case, pooling):
    """Forward and backward of each pooling alone, through the stage entries, against float64: empty and one-node
    graphs, graphs across many 64-row chunks, one graph of 20 000 nodes, and a width that is not a multiple of 4 at a
    wider output pitch (whose extra columns stay untouched)."""
    ldo = None
    if case == "odd_width":
        sizes = [3, 0, 130, 1, 64, 65, 0, 7]
        ptr = torch.zeros(len(sizes) + 1, dtype=torch.int64)
        ptr[1:] = torch.cumsum(torch.tensor(sizes), 0)
        fix = {"ptr": ptr, "num_graphs": len(sizes)}
        x64 = torch.randn(int(ptr[-1]), 13, dtype=torch.float64)
        ldo = 16
    else:
        fix = _load(case)
        x64 = fixture_x(fix)
    x = x64.float().to(DEV)
    d = x.shape[1]
    gs = GraphStructure(torch.zeros(2, 0, dtype=torch.int64, device=DEV), fixture_batch(fix).to(DEV), fix["num_graphs"])
    out, g, gx = _pool_stage(gs, pooling, x, d, ldo)
    ref = pool(x.double().cpu(), fix["ptr"], pooling)
    assert rel_err(out[:, :d], ref) < 1e-5
    if ldo:
        assert (out[:, d:] == 7.0).all()
    xr = x.double().cpu().requires_grad_(True)
    (pool(xr, fix["ptr"], pooling) * g.double()).sum().backward()
    assert rel_err(gx, xr.grad) < 1e-6


def test_pool_stage_bitwise_reproducible():
    fix = _load("one_large_graph")
    x = fixture_x(fix).float().to(DEV) * 1.37
    gs = GraphStructure(torch.zeros(2, 0, dtype=torch.int64, device=DEV), fixture_batch(fix).to(DEV), 1)
    a, b = _pool_stage(gs, "mean", x, x.shape[1]), _pool_stage(gs, "mean", x, x.shape[1])
    assert torch.equal(a[0], b[0])


@pytest.mark.parametrize("name", ["pcqm4m_d304_mean", "one_large_graph", "zinc_graphormer_d80_token"])
def test_bitwise_reproducible(name):
    fix = _load(name)
    head = _head(fix).train()
    a, b = _step(head, fix), _step(head, fix)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    for k in a[2]:
        assert torch.equal(a[2][k], b[2][k]), k


@pytest.mark.parametrize("name", ["pcqm4m_d304_mean", "zinc_graphormer_d80_token"])
def test_capture_forward_backward(name):
    """After one warm-up call a forward + backward records into a CUDA graph and replays to the eager result."""
    fix = _load(name)
    head = _head(fix).train()
    x = fixture_x(fix).float().to(DEV).requires_grad_(True)
    data = _batch(fix, x)
    ct = fixture_ct(fix).float().to(DEV)
    params = [x] + list(head.parameters())

    def step():
        pred, _ = head(data)
        data.graph_feature = None   # a graph kept alive from the previous step would tie the capture to its stream
        return (pred.detach(),) + torch.autograd.grad((pred * ct).sum(), params)

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
    # pad weights, pool (chunks + finish), 3 products, unpad | pad grad_pred, 3 weight and 3 data products, pool', unpad
    ("pcqm4m_d304_mean", (7, 9)),
    # the same with a gather in place of the two pooling launches
    ("zinc_vn_d64_token", (6, 9)),
    # pad weight, gather, LayerNorm, empty-graph rows, product, unpad | pad grad_pred, weight and data products,
    # empty-graph rows, LayerNorm' (2), pool', unpad
    ("zinc_graphormer_d80_token", (6, 8)),
    ("graphormer_edge_d76_token", (6, 8))])
def test_launch_count(name, counts):
    fix = _load(name)
    head = _head(fix).train()
    _step(head, fix)
    lib = _lib.load()
    x = fixture_x(fix).float().to(DEV).requires_grad_(True)
    data = _batch(fix, x)
    graph_of(data)   # the batch's graph structure, as the layers before the head build it
    f0, c0 = lib.gps_fallback_count(), lib.gps_launch_count()
    pred, _ = head(data)
    c1 = lib.gps_launch_count()
    pred.sum().backward()
    c2 = lib.gps_launch_count()
    print("launches: forward", c1 - c0, "backward", c2 - c1)
    assert (c1 - c0, c2 - c1) == counts
    assert lib.gps_fallback_count() == f0


def test_errors():
    fix = _load("zinc_d64_add")
    head = _head(fix)
    x = fixture_x(fix).float().to(DEV)
    b = _batch(fix, x.double())
    with pytest.raises(TypeError):
        head(b)
    b = _batch(fix, x[:, :32].contiguous())
    with pytest.raises(ValueError):
        head(b)
    for bad in (lambda v: v.int(), lambda v: v[:-1], lambda v: v.cpu()):
        b = _batch(fix, x)
        b.batch = bad(b.batch)
        with pytest.raises(ValueError):
            head(b)
    b = _batch(fix, x.cpu())
    with pytest.raises(RuntimeError, match="CUDA"):
        head(b)
    head.FC_layers[0].weight.data = head.FC_layers[0].weight.data.double()
    with pytest.raises(TypeError):
        head(_batch(fix, x))


def test_empty_graph_rows_are_zero_and_receive_nothing():
    fix = _load("edge_cases_L3_mean")
    h = graphgps_b200.SANGraphHead(24, 5, L=0, graph_pooling="mean").to(DEV)
    x = fixture_x(fix).float().to(DEV).requires_grad_(True)
    pred, _ = h(_batch(fix, x))
    empty = (torch.diff(fix["ptr"]) == 0).to(DEV)
    assert torch.equal(pred[empty], h.FC_layers[0].bias.detach().expand(int(empty.sum()), 5))
    g = torch.zeros_like(pred)
    g[empty] = 1.0
    (gx,) = torch.autograd.grad((pred * g).sum(), [x])
    assert not gx.any()


def test_chain_gps_layers_san_head_l1_against_oracle():
    """GatedGCN + Transformer GPSLayer x 2 -> SANGraphHead (mean) -> L1 loss -> backward, against the float64 chain."""
    torch.manual_seed(3)
    d, heads = 64, 4
    layers = [graphgps_b200.GPSLayer(d, "CustomGatedGCN", "Transformer", heads).to(DEV).train() for _ in range(2)]
    head = graphgps_b200.SANGraphHead(d, 1, graph_pooling="mean").to(DEV).train()
    oracles = []
    for layer in layers:
        o = OracleGPSLayer(d, "CustomGatedGCN", "Transformer", heads).double().train()
        o.load_state_dict({k: v.detach().cpu() for k, v in layer.state_dict().items()}, strict=True)
        oracles.append(o)
    b = graphgps_b200.make_batch("zinc-gatedgcn", seed=2, dim=d, num_graphs=12)
    y = torch.randn(12, 1, dtype=torch.float64)
    # the library
    bd = b.clone().to(DEV)
    x = bd.x.requires_grad_(True)
    bd.y = y.float().to(DEV)
    for layer in layers:
        bd = layer(bd)
    pred, label = head(bd)
    F.l1_loss(pred, label).backward()
    # float64 oracle chain
    bo = b.clone()
    bo.x, bo.edge_attr = bo.x.double().requires_grad_(True), bo.edge_attr.double()
    xr = bo.x
    for o in oracles:
        bo = o(bo)
    ws = [m.weight.detach().cpu().double().requires_grad_(True) for m in head.FC_layers]
    bs = [m.bias.detach().cpu().double().requires_grad_(True) for m in head.FC_layers]
    ptr = torch.zeros(13, dtype=torch.int64)
    ptr[1:] = torch.cumsum(torch.bincount(b.batch, minlength=12), 0)
    pr = san_head(bo.x, ptr, "mean", "relu", ws, bs)
    F.l1_loss(pr, y).backward()
    assert rel_err(pred.detach().cpu(), pr.detach()) < 1e-3
    assert rel_err(x.grad.cpu(), xr.grad) < 1e-3 or rel_l2(x.grad.cpu(), xr.grad) < 5e-3
    for m, w, bb in zip(head.FC_layers, ws, bs):
        for a, r in ((m.weight.grad, w.grad), (m.bias.grad, bb.grad)):
            assert rel_err(a.cpu(), r) < 1e-3 or rel_l2(a.cpu(), r) < 5e-3
    for layer, o in zip(layers, oracles):
        qs = dict(o.named_parameters())
        for n, p in layer.named_parameters():
            q = qs[n]
            if q.grad is None:   # the last layer's edge branch does not reach the loss: the library writes zeros
                assert not p.grad.any(), n
                continue
            assert rel_err(p.grad.cpu(), q.grad) < 1e-3 or rel_l2(p.grad.cpu(), q.grad) < 5e-3, n


def test_chain_graphormer_layers_head_l1_against_oracle():
    """GraphormerLayer x 2 -> GraphormerHead (graph_token) -> L1 loss -> backward, against the float64 chain."""
    torch.manual_seed(5)
    d, heads, sizes = 80, 8, [26, 13, 31, 22, 18, 29]
    layers = [graphgps_b200.GraphormerLayer(d, heads, 0.0, 0.0, 0.0).to(DEV).train() for _ in range(2)]
    head = graphgps_b200.GraphormerHead(d, 1).to(DEV).train()
    with torch.no_grad():
        head.ln.weight.uniform_(0.5, 1.5)
        head.ln.bias.uniform_(-0.5, 0.5)
    bb = graphormer_batch(sizes, d, 6, True)
    y = torch.randn(len(sizes), 1, dtype=torch.float64)
    x = bb.x.to(DEV).clone().requires_grad_(True)
    data = types.SimpleNamespace(x=x, edge_index=bb.edge_index.to(DEV), batch=bb.batch.to(DEV),
                                 num_graphs=len(sizes), y=y.float().to(DEV))
    h = data
    for layer in layers:
        h = layer(h)
    pred, label = head(h)
    F.l1_loss(pred, label).backward()
    xr = bb.x.double().clone().requires_grad_(True)
    hr = xr
    states = [{k: v.detach().cpu().double().requires_grad_(True) for k, v in layer.state_dict().items()}
              for layer in layers]
    for s in states:
        hr = graphormer_forward(s, hr, bb.batch, len(sizes), heads)
    hp = {k: v.detach().cpu().double().requires_grad_(True) for k, v in head.state_dict().items()}
    ptr = torch.zeros(len(sizes) + 1, dtype=torch.int64)
    ptr[1:] = torch.cumsum(torch.tensor(sizes), 0)
    pr = graphormer_head(hr, ptr, "graph_token", hp["ln.weight"], hp["ln.bias"], hp["layers.0.weight"],
                         hp["layers.0.bias"])
    F.l1_loss(pr, y).backward()
    assert rel_err(pred.detach().cpu(), pr.detach()) < 1e-3
    assert rel_err(x.grad.cpu(), xr.grad) < 1e-3 or rel_l2(x.grad.cpu(), xr.grad) < 5e-3
    for n, p in head.named_parameters():
        assert rel_err(p.grad.cpu(), hp[n].grad) < 1e-3 or rel_l2(p.grad.cpu(), hp[n].grad) < 5e-3, n
    for layer, s in zip(layers, states):
        for n, p in layer.named_parameters():
            assert rel_err(p.grad.cpu(), s[n].grad) < 1e-3 or rel_l2(p.grad.cpu(), s[n].grad) < 5e-3, n


def test_head_synchronises_nothing_on_a_cached_batch():
    """Once the batch's graph structure is cached (as the layers before the head leave it), forward and backward make
    no synchronising call: torch's sync debug mode raises on any."""
    fix = _load("pcqm4m_d304_mean")
    for head in (_head(fix), graphgps_b200.GraphormerHead(304, 1).to(DEV)):
        x = fixture_x(fix).float().to(DEV).requires_grad_(True)
        data = _batch(fix, x)
        ct = torch.randn(fix["num_graphs"], 1, device=DEV)
        pred, _ = head(data)   # plans, workspaces and the graph structure
        (pred * ct).sum().backward()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            pred, _ = head(data)
            (pred * ct).sum().backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
