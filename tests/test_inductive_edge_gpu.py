"""The inductive link-prediction head on the GPU: the reference's fixtures in fp32 and bf16, training (pred and the
gradients) and eval (the ranking statistics); the tie rule through gps_link_rank_metrics; IndexError and ValueError;
bitwise reproducibility; CUDA-graph capture of a training step; pinned launch counts; and two GatedGCNLayers chained
into the head and binary_cross_entropy_with_logits against the float64 oracle chain."""
import ctypes as C
import os
import types

import pytest
import torch
import torch.nn.functional as F

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import GraphBatch
from graphgps_b200.graph import GraphStructure
from custom_gnn_oracle import OracleGatedGCN, run_stack
from inductive_edge_oracle import STATS, fixture_x, head_forward, rank_stats
from san_oracle import san_batch
from util import GOLDEN_DIR, rel_err, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
IE_DIR = os.path.join(GOLDEN_DIR, "inductive_edge")
FIXTURES = sorted(p[:-3] for p in os.listdir(IE_DIR) if p.endswith(".pt") and p != "reference_live.pt")
W, B = "layer_post_mp.model.0.model.weight", "layer_post_mp.model.0.model.bias"
TOL = {"fp32": 1e-3, "bf16": 1e-2}
STATS_TOL = {"fp32": 1e-6, "bf16": 1e-2}


def _load(name):
    fix = torch.load(os.path.join(IE_DIR, name + ".pt"), weights_only=False)
    fix["x"] = fixture_x(fix)
    return fix


def _head(fix, precision="fp32"):
    h = graphgps_b200.InductiveEdgeHead(fix["config"]["d"], 1, precision=precision)
    h.load_state_dict(fix["state"], strict=True)
    return h.to(DEV)


def _batch(fix, x=None, label_dtype=torch.int64):
    x = fix["x"].float().to(DEV) if x is None else x
    return types.SimpleNamespace(x=x, edge_index_labeled=fix["edge_index_labeled"].to(DEV),
                                 edge_label=fix["edge_label"].to(device=DEV, dtype=label_dtype),
                                 batch=fix["batch"].to(DEV), num_graphs=fix["num_graphs"])


def _train_step(head, fix, label_dtype=torch.int64):
    head.train()
    head.zero_grad(set_to_none=True)
    x = fix["x"].float().to(DEV).requires_grad_(True)
    pred, label = head(_batch(fix, x, label_dtype))
    assert label.dtype == label_dtype
    (pred * fix["ct"].float().to(DEV)).sum().backward()
    torch.cuda.synchronize()
    lin = head.layer_post_mp.model[0].model
    return pred.detach().cpu(), x.grad.cpu(), lin.weight.grad.cpu(), lin.bias.grad.cpu()


def _err(a, r):
    return float((a.double() - r.double()).abs().max()) / max(float(r.abs().max()), 1e-30)


def _oracle_grad_x(fix):
    x = fix["x"].double().requires_grad_(True)
    _, pred = head_forward(x, fix["state"][W].double(), fix["state"][B].double(), fix["edge_index_labeled"])
    (pred * fix["ct"].double()).sum().backward()
    return x.grad


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", FIXTURES)
def test_fixture(name, precision):
    fix = _load(name)
    head = _head(fix, precision)
    pred, gx, gw, gb = _train_step(head, fix, torch.int32 if name.startswith("tiny") else torch.int64)
    tol = TOL[precision]
    ref_gx = fix["grad_x"] if "grad_x" in fix else _oracle_grad_x(fix)
    for what, a, r in (("pred", pred, fix["pred"]), ("grad_x", gx, ref_gx), ("grad_weight", gw, fix["grad_weight"]),
                       ("grad_bias", gb, fix["grad_bias"])):
        e = _err(a, r)
        assert e <= tol, (what, e)
    head.eval()
    with torch.no_grad():
        pred_e, label, stats = head(_batch(fix))
    assert torch.equal(pred_e.cpu(), pred) or _err(pred_e.cpu(), fix["pred"]) <= tol
    assert set(stats) == set(STATS) and all(isinstance(v, float) for v in stats.values())
    for k in STATS:
        assert abs(stats[k] - fix["stats"][k]) <= STATS_TOL[precision], (k, stats[k], fix["stats"][k])


def test_tie_rule_through_rank_metrics():
    """Duplicated rows give bitwise-equal scores, and a tie counts in the positive's favour, also for a positive whose
    target is its source and one whose target duplicates its source."""
    rows = [[1.0, 0.0, 0.0], [1.0, 0.0, 0.0], [1.0, 0.0, 0.0], [2.0, 0.0, 0.0], [0.5, 0.0, 0.0],
            [0.3, 1.0, 0.0], [0.3, 1.0, 0.0], [0.7, -1.0, 2.0]]
    y = torch.tensor(rows, dtype=torch.float64)
    batch = torch.tensor([0, 0, 0, 0, 0, 1, 1, 1])
    eli = torch.tensor([[0, 0, 2, 0, 4, 5, 5, 6],
                        [1, 0, 1, 4, 3, 6, 7, 7]])
    label = torch.tensor([1, 1, 1, 1, 0, 1, 0, 0])
    ref = rank_stats(y, eli, label, torch.tensor([0, 5, 8]))
    # graph 0: (0,1), (0,0), (2,1) rank 2 (node 3 above, the duplicates tie); (0,4) rank 5.  graph 1: (5,6) rank 1
    assert ref["mrr"] == pytest.approx(((3 * 0.5 + 0.2) / 4 + 1.0) / 2)
    gs = GraphStructure(eli.to(DEV), batch.to(DEV), 2)
    yd = y.float().to(DEV)
    stats = torch.empty(4, dtype=torch.float64, device=DEV)
    ws = torch.empty(64, dtype=torch.uint8, device=DEV)
    lab = label.to(DEV)
    lib = _lib.load()
    rc = lib.gps_link_rank_metrics(C.byref(gs.desc), yd.data_ptr(), 3, 3, lab.data_ptr(), 8, stats.data_ptr(),
                                   ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "gps_link_rank_metrics")
    got = stats.tolist()
    for k, v in zip(STATS, got):
        assert v == pytest.approx(ref[k], abs=1e-12), k


def test_index_and_value_errors():
    fix = _load("no_positives_d64")
    head = _head(fix)
    N = fix["x"].shape[0]
    for pos, value in (((1, 3), N), ((0, 0), -1), ((1, 0), 10 ** 6)):
        b = _batch(fix)
        b.edge_index_labeled = b.edge_index_labeled.clone()
        b.edge_index_labeled[pos] = value
        with pytest.raises(IndexError):
            head(b)
    b = _batch(fix)
    b.edge_index_labeled = b.edge_index_labeled.to(torch.int32)
    with pytest.raises(IndexError):
        head(b)
    # a positive whose nodes lie in different graphs: refused in eval (its candidates are undefined), fine in training
    b = _batch(fix)
    k = int((fix["edge_label"] == 1).nonzero()[0])
    b.edge_index_labeled = b.edge_index_labeled.clone()
    b.edge_index_labeled[1, k] = N - 1
    head.eval()
    with pytest.raises(ValueError):
        head(b)
    head.train()
    head(b)
    b = _batch(fix)
    b.edge_label = b.edge_label[:-1]
    with pytest.raises(ValueError):
        head(b)


def test_bitwise_reproducible():
    fix = _load("contact_d138")
    head = _head(fix)
    a, b = _train_step(head, fix), _train_step(head, fix)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    head.eval()
    with torch.no_grad():
        s1, s2 = head(_batch(fix))[2], head(_batch(fix))[2]
    assert s1 == s2


def test_capture_training_step():
    """After the first call on a batch the pair structure is cached: a training forward + backward records into a CUDA
    graph and replays to the eager result."""
    fix = _load("contact_d138")
    head = _head(fix).train()
    x = fix["x"].float().to(DEV).requires_grad_(True)
    data = _batch(fix, x)
    ct = fix["ct"].float().to(DEV)
    params = [x] + list(head.parameters())

    def step():
        pred, _ = head(data)
        data.x = x   # the head replaced batch.x with y
        return torch.autograd.grad((pred * ct).sum(), params)

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
    for a, e in zip(cap, eager):
        assert torch.equal(a, e)


def test_launch_count():
    """fp32 training: pad, projection, pair scores, unpad forward; pair gradient, dW | db, grad_x, unpad backward.  Eval
    adds the ranking and the mean over graphs."""
    fix = _load("contact_d138")
    head = _head(fix)
    _train_step(head, fix)   # first call: pair structure
    lib = _lib.load()
    x = fix["x"].float().to(DEV).requires_grad_(True)
    b = _batch(fix, x)
    head(b)   # builds this batch's pair structure
    b.x = x
    c0 = lib.gps_launch_count()
    pred, _ = head(b)
    c1 = lib.gps_launch_count()
    pred.sum().backward()
    c2 = lib.gps_launch_count()
    head.eval()
    with torch.no_grad():
        b.x = x.detach()
        c3 = lib.gps_launch_count()
        head(b)
        c4 = lib.gps_launch_count()
    print("launches: forward", c1 - c0, "backward", c2 - c1, "eval", c4 - c3)
    assert (c1 - c0, c2 - c1, c4 - c3) == (4, 4, 6)


def test_chain_gatedgcn_head_bce_against_oracle():
    """GatedGCNLayer x 2 -> head -> binary_cross_entropy_with_logits -> backward, against the float64 oracle chain."""
    torch.manual_seed(3)
    d, sizes = 138, [20, 31, 17, 25, 1, 2]
    sb = san_batch("mol", sizes, d, 4)
    g = torch.Generator().manual_seed(5)
    eli, lab, off = [], [], 0
    for n in sizes:
        K = 3 * n
        eli.append(torch.randint(0, n, (2, K), generator=g) + off)
        lab.append((torch.rand(K, generator=g) < 0.3).long())
        off += n
    eli, lab = torch.cat(eli, 1), torch.cat(lab)
    layers = [graphgps_b200.GatedGCNLayer(d, d, 0.0, True).to(DEV).train() for _ in range(2)]
    head = graphgps_b200.InductiveEdgeHead(d, 1).to(DEV).train()
    oracles = []
    for layer in layers:
        o = OracleGatedGCN(d).double().train()
        o.load_state_dict({k: v.detach().cpu() for k, v in layer.state_dict().items()}, strict=True)
        oracles.append(o)
    # the library
    x = sb.x.to(DEV).requires_grad_(True)
    b = GraphBatch(x=x, edge_index=sb.edge_index.to(DEV), edge_attr=sb.edge_attr.to(DEV), batch=sb.batch.to(DEV),
                   num_graphs=len(sizes), edge_index_labeled=eli.to(DEV), edge_label=lab.to(DEV))
    for layer in layers:
        b = layer(b)
    pred, label = head(b)
    F.binary_cross_entropy_with_logits(pred, label.float()).backward()
    # float64 oracle chain
    xr = sb.x.double().requires_grad_(True)
    h, _ = run_stack(oracles, xr, sb.edge_attr.double(), sb.edge_index)
    w = head.layer_post_mp.model[0].model.weight.detach().cpu().double().requires_grad_(True)
    bb = head.layer_post_mp.model[0].model.bias.detach().cpu().double().requires_grad_(True)
    _, pr = head_forward(h, w, bb, eli)
    F.binary_cross_entropy_with_logits(pr, lab.double()).backward()
    assert rel_err(pred.detach().cpu(), pr.detach()) < 1e-3
    assert rel_err(x.grad.cpu(), xr.grad) < 1e-3 or rel_l2(x.grad.cpu(), xr.grad) < 5e-3
    lin = head.layer_post_mp.model[0].model
    for a, r in ((lin.weight.grad, w.grad), (lin.bias.grad, bb.grad)):
        assert rel_err(a.cpu(), r) < 1e-3 or rel_l2(a.cpu(), r) < 5e-3
    for layer, o in zip(layers, oracles):
        for (n, p), (_, q) in zip(layer.named_parameters(), o.named_parameters()):
            if q.grad is None:   # the last layer's edge branch does not reach the loss: the library writes zeros
                assert not p.grad.any(), n
                continue
            assert rel_err(p.grad.cpu(), q.grad) < 1e-3 or rel_l2(p.grad.cpu(), q.grad) < 5e-3, n
