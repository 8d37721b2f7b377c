"""Graphormer's attention-bias encoder on the GPU: the reference's fixtures, bitwise reproducibility, IndexError on
out-of-range types, an actor-sized spatial-only batch against the float64 oracle, and the encoder chained into two
GraphormerLayers (graph token) and into GPSLayer's BiasedTransformer (no token) against the float64 oracle chain, so
the attn_bias layout and the gradient summed over the consuming layers are checked end to end."""
import os
import types

import pytest
import torch

import graphgps_b200
from graphgps_b200.batch import GraphBatch, batch_from_lists
from biased_oracle import OracleGPSLayerBiased
from graphormer_bias_oracle import bias_forward
from graphormer_oracle import graphormer_batch, graphormer_forward
from util import GOLDEN_DIR, rel_err, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GB_DIR = os.path.join(GOLDEN_DIR, "graphormer_bias")
FIXTURES = sorted(p[:-3] for p in os.listdir(GB_DIR) if p.endswith(".pt"))


def _load(name):
    return torch.load(os.path.join(GB_DIR, name + ".pt"), weights_only=False)


def _encoder(cfg, state=None):
    enc = graphgps_b200.BiasEncoder(cfg["heads"], cfg["num_spatial_types"], cfg["num_edge_types"],
                                    cfg["use_graph_token"])
    if state is not None:
        enc.load_state_dict(state, strict=True)
    return enc.to(DEV)


def _data(st, gi, batch, spt=None, ptr=None):
    d = types.SimpleNamespace(spatial_types=st.to(DEV), graph_index=gi.to(DEV), batch=batch.to(DEV))
    if spt is not None:
        d.shortest_path_types = spt.to(DEV)
    if ptr is not None:
        d.ptr = ptr.to(DEV)
    return d


def _run(enc, data, ct):
    out = enc(data).attn_bias
    enc.zero_grad(set_to_none=True)
    (out * ct).sum().backward()
    torch.cuda.synchronize()
    return out.detach().cpu(), {n: None if p.grad is None else p.grad.cpu() for n, p in enc.named_parameters()}


def _fixture_data(fix, with_ptr):
    return _data(fix["spatial_types"], fix["graph_index"], fix["batch"], fix.get("shortest_path_types"),
                 fix["ptr"] if with_ptr else None)


@pytest.mark.parametrize("with_ptr", [True, False], ids=["ptr", "batch"])
@pytest.mark.parametrize("name", FIXTURES)
def test_fixture(name, with_ptr):
    fix = _load(name)
    enc = _encoder(fix["config"], fix["state"])
    out, grads = _run(enc, _fixture_data(fix, with_ptr), fix["ct"].float().to(DEV))
    assert out.shape == fix["out"].shape
    err = float((out.double() - fix["out"].double()).abs().max())
    assert err <= 1e-5, err
    for n, g in fix["grad_params"].items():
        if g is None:   # no shortest_path_types: the edge tables are not read, as in the reference
            assert grads[n] is None, n
            continue
        e = float((grads[n].double() - g.double()).abs().max()) / max(float(g.abs().max()), 1e-30)
        assert e <= 1e-4, (n, e)


def test_bitwise_reproducible():
    fix = _load("zinc_token")
    enc = _encoder(fix["config"], fix["state"])
    ct = fix["ct"].float().to(DEV)
    a = _run(enc, _fixture_data(fix, True), ct)
    b = _run(enc, _fixture_data(fix, True), ct)
    assert torch.equal(a[0], b[0])
    for n in a[1]:
        assert torch.equal(a[1][n], b[1][n]), n


def test_out_of_range_indices_raise_index_error():
    fix = _load("zinc_token")
    enc = _encoder(fix["config"], fix["state"])
    S, T = fix["config"]["num_spatial_types"], fix["config"]["num_edge_types"]
    for field, pos, value in (("spatial_types", (5,), S + 1), ("spatial_types", (0,), -1),
                              ("shortest_path_types", (7, 3), T), ("shortest_path_types", (2, 0), -2),
                              ("graph_index", (1, 4), 10 ** 6), ("graph_index", (1, 0), 30)):
        d = _fixture_data(fix, True)
        t = getattr(d, field).clone()
        t[pos] = value
        setattr(d, field, t)
        with pytest.raises(IndexError):
            enc(d)


# ------------------------------------------------------------------------------------------------ synthetic batches
def random_pairs(sizes, S, T, seed, edges=True):
    """graphormer_pre_processing-shaped attributes of a batch: every ordered pair of each graph once, in a random
    order, with random spatial types in [0, S] and path types in [0, T)."""
    g = torch.Generator().manual_seed(seed)
    gis, off = [], 0
    for n in sizes:
        i = torch.arange(n).repeat_interleave(n)
        j = torch.arange(n).repeat(n)
        gis.append(torch.stack([i, j]) + off)
        off += n
    gi = torch.cat(gis, 1)
    gi = gi[:, torch.randperm(gi.shape[1], generator=g)]
    P = gi.shape[1]
    st = torch.randint(0, S + 1, (P,), generator=g)
    spt = torch.randint(0, T, (P, S), generator=g) if edges else None
    batch = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))
    return st, gi, batch, spt


def _state(enc):
    return {n: p.detach().double().requires_grad_(True) for n, p in enc.named_parameters()}


def test_actor_sized_spatial_only_matches_oracle():
    torch.manual_seed(0)
    cfg = dict(heads=4, num_spatial_types=20, num_edge_types=0, use_graph_token=False)
    enc = _encoder(cfg)
    st, gi, batch, _ = random_pairs([3000], 20, 0, 1, edges=False)
    ct = torch.randn(4, 3000, 3000, device=DEV)
    out, grads = _run(enc, _data(st, gi, batch), ct)
    state = _state(enc)
    ref = bias_forward(state, st.to(DEV), gi.to(DEV), batch.to(DEV), 4, None, False)
    (ref * ct.double()).sum().backward()
    assert float((out.double() - ref.detach().cpu()).abs().max()) <= 1e-6
    g = state["spatial_encoder.weight"].grad.cpu()
    assert float((grads["spatial_encoder.weight"].double() - g).abs().max()) <= 1e-4 * float(g.abs().max())
    assert grads["edge_dis_encoder.weight"] is None and grads["edge_encoder.weight"] is None


def test_chain_into_two_graphormer_layers_with_graph_token():
    """BiasEncoder -> GraphormerLayer x 2 on graphs with a prepended token node (N' = Nmax + 1); attn_bias's gradient is
    the sum over both layers."""
    torch.manual_seed(1)
    sizes, d, H = [21, 9, 30, 14, 1, 25], 80, 8
    enc = _encoder(dict(heads=H, num_spatial_types=20, num_edge_types=4, use_graph_token=True))
    with torch.no_grad():   # O(1) bias so it moves the attention visibly
        for p in enc.parameters():
            p.normal_(std=0.5)
    layers = [graphgps_b200.GraphormerLayer(d, H, 0.0, 0.0, 0.0).to(DEV) for _ in range(2)]
    st, gi, batch, spt = random_pairs(sizes, 20, 4, 2)
    lb = graphormer_batch([n + 1 for n in sizes], d, 3, token=True)
    ct = torch.randn(lb.x.shape, generator=torch.Generator().manual_seed(4))
    # the library
    data = _data(st, gi, batch, spt)
    x = lb.x.to(DEV).requires_grad_(True)
    b = GraphBatch(x=x, edge_index=lb.edge_index.to(DEV), edge_attr=None, batch=lb.batch.to(DEV), num_graphs=len(sizes))
    b.attn_bias = enc(data).attn_bias
    assert tuple(b.attn_bias.shape) == (len(sizes) * H, max(sizes) + 1, max(sizes) + 1)
    for layer in layers:
        b = layer(b)
    (b.x * ct.to(DEV)).sum().backward()
    # float64 oracle chain
    est = _state(enc)
    ab = bias_forward(est, st.to(DEV), gi.to(DEV), batch.to(DEV), H, spt.to(DEV), True)
    xr = lb.x.to(DEV).double().requires_grad_(True)
    h = xr
    for layer in layers:
        h = graphormer_forward({n: p.detach() for n, p in layer.named_parameters()}, h, lb.batch.to(DEV), len(sizes),
                               H, ab)
    (h * ct.to(DEV).double()).sum().backward()
    assert rel_err(b.x.detach(), h.detach()) < 1e-3
    assert rel_err(x.grad, xr.grad) < 1e-3
    for n, p in enc.named_parameters():
        r = est[n].grad
        assert rel_err(p.grad, r) < 1e-3 or rel_l2(p.grad, r) < 5e-3, n


def test_chain_into_gps_layer_biased_transformer_without_token():
    torch.manual_seed(2)
    sizes, d, H = [18, 27, 11, 23], 64, 4
    enc = _encoder(dict(heads=H, num_spatial_types=20, num_edge_types=4, use_graph_token=False))
    with torch.no_grad():
        for p in enc.parameters():
            p.normal_(std=0.5)
    ora = OracleGPSLayerBiased(d, "GINE", "BiasedTransformer", H)
    ours = graphgps_b200.GPSLayer(d, "GINE", "BiasedTransformer", H)
    ours.load_state_dict(ora.state_dict(), strict=True)
    ours, ora = ours.to(DEV).train(), ora.double().train()
    st, gi, batch, spt = random_pairs(sizes, 20, 4, 5)
    lb = batch_from_lists(sizes, [[(i, i + 1) for i in range(n - 1)] + [(i + 1, i) for i in range(n - 1)]
                                  for n in sizes], d=d, seed=6)
    ct = torch.randn(lb.x.shape, generator=torch.Generator().manual_seed(7))
    # the library
    bb = lb.clone().to(DEV)
    bb.x.requires_grad_(True)
    x_in = bb.x
    bb.attn_bias = enc(_data(st, gi, batch, spt)).attn_bias
    (ours(bb).x * ct.to(DEV)).sum().backward()
    # float64 oracle chain on the CPU
    est = {n: p.detach().cpu().double().requires_grad_(True) for n, p in enc.named_parameters()}
    ob = lb.clone()
    ob.x, ob.edge_attr = ob.x.double().requires_grad_(True), ob.edge_attr.double()
    ob.attn_bias = bias_forward(est, st, gi, batch, H, spt, False)
    xo = ob.x
    out = ora(ob).x
    (out * ct.double()).sum().backward()
    assert rel_err(bb.x.detach().cpu(), out.detach()) < 1e-3
    assert rel_err(x_in.grad.cpu(), xo.grad) < 1e-3 or rel_l2(x_in.grad.cpu(), xo.grad) < 5e-3
    for n, p in enc.named_parameters():
        r = est[n].grad
        assert rel_err(p.grad.cpu(), r) < 1e-3 or rel_l2(p.grad.cpu(), r) < 5e-3, n


def test_capture_after_first_read():
    """The host read is cached on the batch: a forward + backward step records into a CUDA graph and replays to the
    eager result."""
    fix = _load("zinc_token")
    enc = _encoder(fix["config"], fix["state"])
    data = _fixture_data(fix, True)
    ct = fix["ct"].float().to(DEV)
    params = list(enc.parameters())

    def step():
        out = enc(data).attn_bias
        del data.attn_bias   # a batch holding the last step's output would keep its autograd graph alive
        return torch.autograd.grad((out * ct).sum(), params)

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
