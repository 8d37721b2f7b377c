"""RWSE on the H100: the landing probabilities against the reference's float64 results and the float64 oracle on every
fixture, the kernel-PE encoder in training and eval against float64, determinism, capture, launch counts, the size
limit, and one chain encoder -> GPSLayers -> SANGraphHead against float64."""
import types

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.rwse import cached_rw_landing_probs
from rwse_oracle import encoder as oracle_encoder, fixture_inputs, fixture_names, landing as oracle_landing, load

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FIXTURES = fixture_names()


def _batch(fix, x=None):
    ptr = fix["ptr"]
    N = int(ptr[-1])
    bvec = torch.repeat_interleave(torch.arange(ptr.numel() - 1), torch.diff(ptr))
    return types.SimpleNamespace(edge_index=fix["edge_index"].long().to(DEV), batch=bvec.to(DEV),
                                 num_graphs=ptr.numel() - 1, x=x if x is not None else torch.zeros(N, 1, device=DEV))


def _oracle_rw(fix):
    return torch.from_numpy(oracle_landing(fix["edge_index"].long().numpy(), fix["ptr"].numpy(),
                                           fix["config"]["ksteps"]))


def _rel(a, r):
    a, r = a.detach().double().cpu(), r.detach().double().cpu()
    return float((a - r).abs().max() / max(float(r.abs().max()), 1e-30)) if r.numel() else 0.0


def _encoder(fix, **kw):
    c = fix["config"]
    enc = graphgps_b200.KernelPENodeEncoder(c["dim_in"], c["dim_emb"], len(c["ksteps"]), c["dim_pe"],
                                            raw_norm_type="batchnorm" if c["batch_norm"] else "none",
                                            expand_x=c["expand_x"], **kw)
    enc.load_state_dict(fix["state"])
    return enc.to(DEV).train(c["training"])


@pytest.mark.parametrize("name", FIXTURES)
def test_landing_probabilities(name):
    fix = load(name)
    ks = fix["config"]["ksteps"]
    ours = graphgps_b200.rw_landing_probs(_batch(fix), ks).cpu().double()
    ref = _oracle_rw(fix)
    rows = fix["rw64"].shape[0]
    assert float((ref[:rows] - fix["rw64"]).abs().max()) < 1e-12   # the oracle is the reference here
    err = (ours - ref).abs()
    assert bool((err <= 1e-5 * ref.abs() + 1e-7).all()), f"max abs err {float(err.max()):.3e}"
    assert bool((ours[ref == 0] == 0).all())   # exact zeros stay exact (odd k of bipartite graphs, sinks, no edges)
    rel = float((err / (ref.abs() + 1e-7)).max())
    print(f"{name}: ours max rel dev {rel:.2e}, the reference's own float32 {fix['ref32_rel_dev']:.2e}")


def test_block_diagonal_batch_equals_graph_by_graph():
    fix = load("edge_cases_k3183")
    b = _batch(fix)
    ptr = fix["ptr"].tolist()
    whole = graphgps_b200.rw_landing_probs(b, [3, 1, 8, 3]).cpu()
    ei = fix["edge_index"].long()
    for g in range(len(ptr) - 1):
        m = (ei[0] >= ptr[g]) & (ei[0] < ptr[g + 1])
        n = ptr[g + 1] - ptr[g]
        one = types.SimpleNamespace(edge_index=(ei[:, m] - ptr[g]).to(DEV), batch=torch.zeros(n, dtype=torch.long,
                                                                                               device=DEV),
                                    num_graphs=1)
        assert torch.equal(graphgps_b200.rw_landing_probs(one, [3, 1, 8, 3]).cpu(), whole[ptr[g]:ptr[g + 1]])


def test_oversized_graph_is_refused_before_any_launch():
    n = 30_000
    b = types.SimpleNamespace(edge_index=torch.stack([torch.arange(n), (torch.arange(n) + 1) % n]).to(DEV),
                              batch=torch.zeros(n, dtype=torch.long, device=DEV), num_graphs=1)
    graphgps_b200.graph.graph_of(b).nmax
    torch.cuda.synchronize()
    before = _lib.load().gps_launch_count()
    with pytest.raises(NotImplementedError, match="does not fit on chip"):
        graphgps_b200.rw_landing_probs(b, [1, 2])
    with pytest.raises(NotImplementedError):
        graphgps_b200.rw_landing_probs(_batch(load("edge_cases_k3183")), [257])
    assert _lib.load().gps_launch_count() == before


def _run(enc, fix, x, g, pestat, steps=1):
    for _ in range(steps):
        xx = x.clone().requires_grad_(True)
        b = _batch(fix, xx)
        b.pestat_RWSE = pestat
        out = enc(b).x
        for p in enc.parameters():
            p.grad = None
        out.backward(g)
    return out, xx.grad, {k: p.grad for k, p in enc.named_parameters()}


@pytest.mark.parametrize("name", FIXTURES)
def test_encoder_matches_float64(name):
    fix = load(name)
    c = fix["config"]
    x, g, pestat = fixture_inputs(fix)
    for training in ([True, False] if c["training"] else [False]):
        enc = _encoder(fix).train(training)
        out, gx, grads = _run(enc, fix, x.to(DEV), g.to(DEV), pestat.to(DEV))
        o_out, o_gx, o_grads, o_run = oracle_encoder(fix["state"], c, x, pestat, g, training)
        assert _rel(out, o_out) < 1e-5 and _rel(gx, o_gx) < 1e-5, name
        for k, v in grads.items():
            assert _rel(v, o_grads[k]) < 1e-5, (name, k)
            if training == c["training"]:
                assert _rel(v, fix["grads"][k]) < 1e-5, (name, k)   # the reference's own float64 gradients
        if c["batch_norm"]:
            assert _rel(enc.raw_norm.running_mean, o_run[0]) < 1e-6 and _rel(enc.raw_norm.running_var, o_run[1]) < 1e-6


@pytest.mark.parametrize("name", ["zinc_k20_pe28", "edge_cases_range5"])
def test_running_statistics_after_three_steps(name):
    fix = load(name)
    c = fix["config"]
    x, g, pestat = fixture_inputs(fix)
    enc = _encoder(fix).train(True)
    _run(enc, fix, x.to(DEV), g.to(DEV), pestat.to(DEV), steps=3)
    run = (fix["state"]["raw_norm.running_mean"], fix["state"]["raw_norm.running_var"])
    for _ in range(3):
        *_, run = oracle_encoder(fix["state"], c, x, pestat, g, True, running=run)
    assert _rel(enc.raw_norm.running_mean, run[0]) < 1e-6 and _rel(enc.raw_norm.running_var, run[1]) < 1e-6
    assert int(enc.raw_norm.num_batches_tracked) == int(fix["state"]["raw_norm.num_batches_tracked"]) + 3


def test_bitwise_reproducible():
    for name in ("malnet_hubs_5000", "pcqm4m_k16_pe20_d304"):
        fix = load(name)
        x, g, pestat = fixture_inputs(fix)
        runs = []
        for _ in range(2):
            rw = graphgps_b200.rw_landing_probs(_batch(fix), fix["config"]["ksteps"])
            runs.append((rw,) + _run(_encoder(fix).train(True), fix, x.to(DEV), g.to(DEV), pestat.to(DEV))[:2]
                        + tuple(_run(_encoder(fix).train(True), fix, x.to(DEV), g.to(DEV), pestat.to(DEV))[2].values()))
        for a, b in zip(*runs):
            assert torch.equal(a, b), name


def test_ksteps_mode_equals_pestat_mode():
    fix = load("pcqm4m_k16_pe20_d304")
    x, g, _ = fixture_inputs(fix)
    ks = fix["config"]["ksteps"]
    pestat = graphgps_b200.rw_landing_probs(_batch(fix), ks)
    a = _run(_encoder(fix), fix, x.to(DEV), g.to(DEV), pestat)
    enc = _encoder(fix, ksteps=ks)
    xx = x.to(DEV).clone().requires_grad_(True)
    b = _batch(fix, xx)
    out = enc(b).x
    out.backward(g.to(DEV))
    assert torch.equal(b.pestat_RWSE, pestat)
    assert torch.equal(out, a[0]) and torch.equal(xx.grad, a[1])
    for k, p in enc.named_parameters():
        assert torch.equal(p.grad, a[2][k]), k
    # cached per batch object and ksteps: a second call launches nothing
    torch.cuda.synchronize()
    before = _lib.load().gps_launch_count()
    assert cached_rw_landing_probs(b, ks) is b.pestat_RWSE
    assert _lib.load().gps_launch_count() == before


def test_launch_counts():
    lib = _lib.load()
    for name, fwd_train, fwd_eval in (("zinc_k20_pe28", 4, 2), ("edge_cases_range5", 6, 3),
                                      ("edge_cases_no_norm", 1, 1)):
        fix = load(name)
        x, g, pestat = fixture_inputs(fix)
        b = _batch(fix, x.to(DEV))
        graphgps_b200.graph.graph_of(b).nmax
        torch.cuda.synchronize()
        c0 = lib.gps_launch_count()
        graphgps_b200.rw_landing_probs(b, fix["config"]["ksteps"])
        c1 = lib.gps_launch_count()
        assert c1 - c0 == 2, name                          # inverse degrees, walks
        for training, n_fwd in ((True, fwd_train), (False, fwd_eval)):
            enc = _encoder(fix).train(training)
            xx = x.to(DEV).requires_grad_(True)
            bb = _batch(fix, xx)
            bb.pestat_RWSE = pestat.to(DEV)
            c0 = lib.gps_launch_count()
            out = enc(bb).x
            c1 = lib.gps_launch_count()
            out.backward(g.to(DEV))
            c2 = lib.gps_launch_count()
            assert (c1 - c0, c2 - c1) == (n_fwd, 3), (name, training)


def test_cached_batch_makes_no_synchronising_call():
    fix = load("zinc_k20_pe28")
    x, g, _ = fixture_inputs(fix)
    enc = _encoder(fix, ksteps=fix["config"]["ksteps"])
    xx = x.to(DEV).requires_grad_(True)
    b = _batch(fix, xx)
    g = g.to(DEV)
    enc(b).x.backward(g)   # builds and caches the graph structure, Nmax and the statistics
    b.x = xx
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = enc(b).x
        out.backward(g)
        graphgps_b200.rw_landing_probs(b, [1, 2, 3])
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_cuda_graph_capture():
    fix = load("pcqm4m_k16_pe20_d304")
    x, g, _ = fixture_inputs(fix)
    ks = fix["config"]["ksteps"]
    enc = _encoder(fix).train(True)
    x, g = x.to(DEV), g.to(DEV)
    b = _batch(fix, x)
    params = list(enc.parameters())

    def step():
        b.x = x
        b.pestat_RWSE = graphgps_b200.rw_landing_probs(b, ks)
        out = enc(b).x
        return [out, b.pestat_RWSE] + list(torch.autograd.grad(out, [x] + params, g))

    x.requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            eager = step()
    torch.cuda.current_stream().wait_stream(s)
    eager = [t.clone() for t in eager]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize()
    for a, e in zip(captured, eager):
        assert torch.equal(a, e)


def test_chain_encoder_gps_layers_head_matches_float64():
    """Encoder (expand_x False, on a stand-in previous encoder's output) -> two GatedGCN+Transformer GPSLayers ->
    SANGraphHead under an L1 loss, against the same chain in float64 (the reference layer oracle and head oracle)."""
    from oracle.gps_oracle import OracleGPSLayer
    fix = load("zinc_k20_pe28")
    c = fix["config"]
    torch.manual_seed(0)
    N, d = int(fix["ptr"][-1]), c["dim_emb"]
    ei = fix["edge_index"].long()
    h_prev = torch.randn(N, c["dim_in"])
    edge_attr = torch.randn(ei.shape[1], d)
    y = torch.randn(fix["ptr"].numel() - 1, 1)
    x, g, pestat = fixture_inputs(fix)
    enc = _encoder(fix).train(True)
    layers = [graphgps_b200.GPSLayer(d, "CustomGatedGCN", "Transformer", 4) for _ in range(2)]
    oras = [OracleGPSLayer(d, "CustomGatedGCN", "Transformer", 4) for _ in range(2)]
    for lay, ora in zip(layers, oras):
        lay.load_state_dict(ora.state_dict())
    head = graphgps_b200.SANGraphHead(d, 1)
    ref_head = torch.nn.ModuleList([torch.nn.Linear(d >> l, d >> (l + 1)) for l in range(2)] +
                                   [torch.nn.Linear(d >> 2, 1)])
    head.FC_layers.load_state_dict(ref_head.state_dict())

    def chain(dev, dtype, mods):
        enc_m, lays, hd = mods
        hp = h_prev.to(dev, dtype).requires_grad_(True)
        bvec = torch.repeat_interleave(torch.arange(fix["ptr"].numel() - 1), torch.diff(fix["ptr"])).to(dev)
        if dev == "cpu":
            o_out, *_ = oracle_encoder(fix["state"], c, hp, pestat, torch.zeros(N, d), True)
            hx = torch.cat([hp, o_out[:, c["dim_in"]:].to(dtype)], 1)
        else:
            b0 = types.SimpleNamespace(x=hp, pestat_RWSE=pestat.to(dev), edge_index=ei.to(dev), batch=bvec,
                                       num_graphs=fix["ptr"].numel() - 1)
            hx = enc_m(b0).x
        b = graphgps_b200.GraphBatch(x=hx, edge_index=ei.to(dev), edge_attr=edge_attr.to(dev, dtype), batch=bvec,
                                     num_graphs=fix["ptr"].numel() - 1)
        for lay in lays:
            b = lay(b)
        if dev == "cpu":
            pooled = torch.zeros(b.num_graphs, d, dtype=dtype).index_add_(0, bvec, b.x)
            pooled = pooled / torch.bincount(bvec, minlength=b.num_graphs).clamp(min=1).unsqueeze(1).to(dtype)
            h = pooled
            for l, lin in enumerate(hd):
                h = lin(h)
                if l < 2:
                    h = torch.relu(h)
            pred = h
        else:
            pred, _ = hd(types.SimpleNamespace(x=b.x, batch=bvec, edge_index=ei.to(dev), num_graphs=b.num_graphs,
                                               y=y.to(dev)))
        loss = (pred - y.to(dev, dtype)).abs().mean()
        loss.backward()
        return pred.detach().cpu().double(), hp.grad.cpu().double()

    ours = chain(DEV, torch.float32, (enc, [lay.to(DEV).train() for lay in layers], head.to(DEV)))
    ref = chain("cpu", torch.float64, (None, [o.double().train() for o in oras], ref_head.double()))
    assert _rel(ours[0], ref[0]) < 1e-3
    assert _rel(ours[1], ref[1]) < 1e-3
