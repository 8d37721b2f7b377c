"""GPU: GPSLayer with the GatedGCN local model at the pcqm4m-small shape, where the backward runs as two concurrent
branches: the attention-branch backward forks at g_s, next to norm1_local's backward, and the grad_edge_attr product
runs on the edge stream, off the local branch.  Results must not depend on that schedule: parity with
the float64 oracle (with and without the EquivStableLapPE gate, relu and gelu, dropout with the library's masks
injected, eval mode), bitwise equality across runs, retained graphs, CUDA-graph capture and a 3-layer stack with the
plane hand-off, and the launch count of one step."""
import copy

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import make_batch
from graphgps_b200.graph import graph_of
from oracle.gps_oracle import OracleGPSLayer
from eslappe_oracle import OracleGPSLayerESLapPE
from eslappe_util import calibrate_gate, compare_eslap, make_pe, run_eslap
from util import _stream, compare, pin_dropout_counter, run_layer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPE = "pcqm4m-small"


def _batch(seed=7, pe=False):
    b = make_batch(SHAPE, seed=seed)
    if pe:
        b.pe_EquivStableLapPE = make_pe(b.x.shape[0], 8, seed)
    return b


def _cts(b, seed=9):
    g = torch.Generator().manual_seed(seed)
    return {"config": dict(local="CustomGatedGCN"), "ct_x": torch.randn(b.x.shape, generator=g),
            "ct_e": torch.randn(b.edge_attr.shape, generator=g)}


def _to64(b):
    b = b.clone()
    for k in ("x", "edge_attr", "pe_EquivStableLapPE"):
        if hasattr(b, k):
            setattr(b, k, getattr(b, k).double())
    return b


def _target(ref, keys=("out_x", "out_e", "grad_x", "grad_e")):
    t = {k: ref[k] for k in keys if k in ref}
    t["grad_params"], t["state_after"] = ref["grad_params"], ref["state_after"]
    return t


@pytest.mark.parametrize("act", ["relu", "gelu"])
def test_matches_oracle_fp64(act):
    d = graphgps_b200.SHAPES[SHAPE].dim
    torch.manual_seed(0)
    ora = OracleGPSLayer(d, "CustomGatedGCN", "Transformer", 4, act=act)
    ours = graphgps_b200.GPSLayer(d, "CustomGatedGCN", "Transformer", 4, act=act)
    ours.load_state_dict(ora.state_dict())
    ours = ours.to(DEV)
    b = _batch()
    fix = _cts(b)
    ref = run_layer(copy.deepcopy(ora).double(), _to64(b), fix)
    res = run_layer(ours, b.clone().to(DEV), fix)
    compare(res, _target(ref), 1e-3, f"GatedGCN+Transformer {act} @ {SHAPE}", grad_l2_tol=5e-3)


@pytest.mark.parametrize("act", ["relu", "gelu"])
def test_equivstable_pe_matches_oracle_fp64(act):
    d = graphgps_b200.SHAPES[SHAPE].dim
    b = _batch(pe=True)
    torch.manual_seed(0)
    ora = OracleGPSLayerESLapPE(d, "CustomGatedGCN", "Transformer", 4, act=act)
    calibrate_gate(ora, b.pe_EquivStableLapPE, b.edge_index)
    ours = graphgps_b200.GPSLayer(d, "CustomGatedGCN", "Transformer", 4, act=act, equivstable_pe=True)
    ours.load_state_dict(ora.state_dict(), strict=True)
    ours = ours.to(DEV)
    fix = _cts(b)
    ref = run_eslap(copy.deepcopy(ora).double(), _to64(b), fix)
    res = run_eslap(ours, b.clone().to(DEV), fix)
    compare_eslap(res, _target(ref, ("out_x", "out_e", "grad_x", "grad_e", "grad_pe")), 1e-3,
                  f"GatedGCN+Transformer with EquivStableLapPE {act} @ {SHAPE}", grad_l2_tol=5e-3)


def test_dropout_matches_oracle_with_injected_masks():
    """dropout = 0.2 at every GPSLayer site, GatedGCN's node and edge outputs included: the library's Philox masks
    are replayed through gps_dropout_mask and injected into the float64 oracle."""
    from test_layer_gpu import _inject_gatedgcn_dropout
    lib = _lib.load()
    d, p = graphgps_b200.SHAPES[SHAPE].dim, 0.2
    torch.manual_seed(3)
    ora = OracleGPSLayer(d, "CustomGatedGCN", "Transformer", 4, dropout=0.0, attn_dropout=0.0)
    ours = graphgps_b200.GPSLayer(d, "CustomGatedGCN", "Transformer", 4, dropout=p, attn_dropout=0.0)
    ours.load_state_dict(ora.state_dict())
    ours = ours.to(DEV).train()
    b = _batch(seed=8)
    N, E = b.num_nodes, b.num_edges
    base = 23 * 4096
    pin_dropout_counter(DEV, base)
    seed = int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF
    masks = {}
    for site, (rows, cols) in ((1, (N, d)), (2, (E, d)), (4, (N, d)), (5, (N, 2 * d)), (6, (N, d))):
        m = torch.empty(rows, cols, device=DEV)
        _lib.check(lib.gps_dropout_mask(m.data_ptr(), rows, cols, p, seed, base + 4096, site, _stream()), "mask")
        masks[site] = m.cpu().double() / (1.0 - p)

    class Fixed(torch.nn.Module):
        def __init__(self, m):
            super().__init__()
            self.m = m

        def forward(self, t):
            return t * self.m

    o64 = copy.deepcopy(ora).double()
    o64.dropout_attn = Fixed(masks[4])
    _inject_gatedgcn_dropout(o64.local_model, masks[1], masks[2])
    o64.ff_dropout1, o64.ff_dropout2 = Fixed(masks[5]), Fixed(masks[6])
    fix = _cts(b, seed=4)
    ref = run_layer(o64, _to64(b), fix)
    res = run_layer(ours, b.clone().to(DEV), fix)
    compare(res, _target(ref), 1e-3, f"GatedGCN+Transformer with dropout masks injected @ {SHAPE}", grad_l2_tol=5e-3)


def test_eval_mode_matches_oracle_fp64():
    """Eval mode: running statistics, so the BatchNorm backward applies drop the batch-statistics terms."""
    d = graphgps_b200.SHAPES[SHAPE].dim
    torch.manual_seed(5)
    ora = OracleGPSLayer(d, "CustomGatedGCN", "Transformer", 4)
    with torch.no_grad():
        for name, buf in ora.named_buffers():
            if name.endswith("running_mean"):
                buf.copy_(0.1 * torch.randn_like(buf))
            elif name.endswith("running_var"):
                buf.copy_(0.5 + torch.rand_like(buf))
    ours = graphgps_b200.GPSLayer(d, "CustomGatedGCN", "Transformer", 4)
    ours.load_state_dict(ora.state_dict())
    ours = ours.to(DEV).eval()
    b = _batch(seed=10)
    fix = _cts(b)
    ref = run_layer(copy.deepcopy(ora).double().eval(), _to64(b), fix)
    res = run_layer(ours, b.clone().to(DEV), fix)
    compare(res, _target(ref), 1e-3, f"GatedGCN+Transformer eval @ {SHAPE}", grad_l2_tol=5e-3)


def _layer(dropout=0.2, precision="fp32"):
    torch.manual_seed(1)
    d = graphgps_b200.SHAPES[SHAPE].dim
    return graphgps_b200.GPSLayer(d, "CustomGatedGCN", "Transformer", 4, dropout=dropout, attn_dropout=0.5,
                                  precision=precision).to(DEV).train()


def _step(layer, b, ct_x, ct_e, retain=False):
    """One forward + backward; returns every output and gradient (cloned)."""
    bb = b.clone()
    bb.x.requires_grad_(True)
    bb.edge_attr.requires_grad_(True)
    x_in, e_in = bb.x, bb.edge_attr
    for p in layer.parameters():
        p.grad = None
    out = layer(bb)
    torch.autograd.backward([out.x, out.edge_attr], [ct_x, ct_e], retain_graph=retain)
    res = [out.x.detach().clone(), out.edge_attr.detach().clone(), x_in.grad.clone(), e_in.grad.clone()]
    res += [p.grad.clone() for p in layer.parameters()]
    if retain:
        x_in.grad, e_in.grad = None, None
        for p in layer.parameters():
            p.grad = None
        torch.autograd.backward([out.x, out.edge_attr], [ct_x, ct_e])
        again = [x_in.grad.clone(), e_in.grad.clone()] + [p.grad.clone() for p in layer.parameters()]
        return res, again
    return res


def _assert_equal(a, b, what):
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        assert torch.equal(u, v), (what, i, float((u - v).abs().max()))


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_two_runs_are_bitwise_identical(precision):
    layer = _layer(precision=precision)
    b = _batch().to(DEV)
    ct_x, ct_e = torch.randn_like(b.x), torch.randn_like(b.edge_attr)
    state = copy.deepcopy(layer.state_dict())
    pin_dropout_counter(DEV, 5 * 4096)
    r1 = _step(layer, b, ct_x, ct_e)
    layer.load_state_dict(state)   # the running statistics as before the first run
    pin_dropout_counter(DEV, 5 * 4096)
    r2 = _step(layer, b, ct_x, ct_e)
    _assert_equal(r1, r2, "run to run")


def test_retain_graph_second_backward_is_identical():
    layer = _layer()
    b = _batch().to(DEV)
    ct_x, ct_e = torch.randn_like(b.x), torch.randn_like(b.edge_attr)
    first, again = _step(layer, b, ct_x, ct_e, retain=True)
    _assert_equal(first[2:], again, "retain_graph")


def test_captured_step_matches_eager():
    layer = _layer()
    b = _batch().to(DEV)
    graph_of(b)
    ct_x, ct_e = torch.randn_like(b.x), torch.randn_like(b.edge_attr)
    x = b.x.clone().requires_grad_(True)
    e = b.edge_attr.clone().requires_grad_(True)
    params = list(layer.parameters())

    def body():
        bb = graphgps_b200.GraphBatch(x=x, edge_index=b.edge_index, edge_attr=e, batch=b.batch, num_graphs=b.num_graphs)
        bb.__dict__["_gps_b200_graph"] = b.__dict__["_gps_b200_graph"]
        x.grad, e.grad = None, None
        for p in params:
            p.grad = None
        out = layer(bb)
        torch.autograd.backward([out.x, out.edge_attr], [ct_x, ct_e])
        return out

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            body()
    torch.cuda.current_stream().wait_stream(side)
    state = copy.deepcopy(layer.state_dict())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = body()
    layer.load_state_dict(state)
    pin_dropout_counter(DEV, 7 * 4096)
    g.replay()
    torch.cuda.synchronize()
    got = [out.x.clone(), out.edge_attr.clone(), x.grad.clone(), e.grad.clone()] + [p.grad.clone() for p in params]
    layer.load_state_dict(state)
    pin_dropout_counter(DEV, 7 * 4096)
    o = body()
    torch.cuda.synchronize()
    want = [o.x.detach(), o.edge_attr.detach(), x.grad, e.grad] + [p.grad for p in params]
    _assert_equal(got, want, "captured vs eager")


def test_three_layer_stack_with_plane_handoff():
    """Each layer's e_out and its planes are the next layer's edge input, and each backward's grad_edge_attr (written
    on the edge stream) is the previous layer's grad_edge_out: with the hand-off the next layer reads those planes,
    without it it converts e_out itself."""
    d = graphgps_b200.SHAPES[SHAPE].dim
    torch.manual_seed(2)
    stack = graphgps_b200.GPSStack(3, d, "CustomGatedGCN", "Transformer", 4).to(DEV).train()
    b = _batch(seed=3).to(DEV)
    ct_x, ct_e = torch.randn_like(b.x), torch.randn_like(b.edge_attr)
    state = copy.deepcopy(stack.state_dict())

    def run(handoff):
        stack.load_state_dict(state)
        for layer in stack.layers:
            layer.__dict__["plane_handoff"] = handoff
            layer.__dict__.pop("_wplanes", None)
        bb = b.clone()
        bb.x.requires_grad_(True)
        bb.edge_attr.requires_grad_(True)
        x_in, e_in = bb.x, bb.edge_attr
        for p in stack.parameters():
            p.grad = None
        out = stack(bb)
        torch.autograd.backward([out.x, out.edge_attr], [ct_x, ct_e])
        return [out.x.detach().clone(), out.edge_attr.detach().clone(), x_in.grad.clone(), e_in.grad.clone()] + \
            [p.grad.clone() for p in stack.parameters()]

    _assert_equal(run(True), run(False), "stack with vs without plane hand-off")


# Kernel launches of one pcqm4m-small GatedGCN+Transformer step (fp32, training, dropout 0, attn_dropout 0.5): moving
# work between streams adds or removes none
FWD_LAUNCHES, BWD_LAUNCHES = 18, 25


def test_launch_count():
    lib = _lib.load()
    layer = _layer(dropout=0.0)
    b = _batch().to(DEV)
    graph_of(b)
    ct_x, ct_e = torch.randn_like(b.x), torch.randn_like(b.edge_attr)
    _step(layer, b, ct_x, ct_e)
    torch.cuda.synchronize()
    bb = b.clone()
    bb.x.requires_grad_(True)
    bb.edge_attr.requires_grad_(True)
    c0 = lib.gps_launch_count()
    out = layer(bb)
    c1 = lib.gps_launch_count()
    torch.autograd.backward([out.x, out.edge_attr], [ct_x, ct_e])
    c2 = lib.gps_launch_count()
    print("launches: forward", c1 - c0, "backward", c2 - c1)
    assert (c1 - c0, c2 - c1) == (FWD_LAUNCHES, BWD_LAUNCHES)
