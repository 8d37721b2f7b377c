"""CPU: the GAT local model's oracles, parameter layout and argument contract (tests/gat_oracle.py)."""
import ctypes as C
import math
import os

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from gat_oracle import GATConvDense, GATConvMP, gat_batch, gat_oracle_layer
from local_model_harness import _args, _plan
from util import GOLDEN_DIR, golden_batch

GAT_DIR = os.path.join(GOLDEN_DIR, "gat")


def _pair(d, H, seed):
    torch.manual_seed(seed)
    mp = GATConvMP(d, d // H, heads=H, edge_dim=d).double()
    with torch.no_grad():
        for p in (mp.att_src, mp.att_dst, mp.att_edge):
            p.mul_(3.0)
        mp.bias.normal_()
    dn = GATConvDense(d, d // H, heads=H, edge_dim=d).double()
    dn.load_state_dict(mp.state_dict(), strict=True)
    return mp, dn


@pytest.mark.parametrize("d,H", [(16, 4), (36, 4), (32, 1)])
def test_restatements_agree(d, H):
    b = gat_batch("zinc-gine", 3, d, 5, dtype=torch.float64)
    mp, dn = _pair(d, H, 1)
    n = torch.bincount(b.batch, minlength=b.num_graphs)
    dn.ptr = torch.cat([torch.zeros(1, dtype=torch.int64), n.cumsum(0)])
    ct = torch.randn(b.num_nodes, d, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    res = []
    for m in (mp, dn):
        x, e = b.x.clone().requires_grad_(True), b.edge_attr.clone().requires_grad_(True)
        o = m(x, b.edge_index, e)
        res.append([o] + list(torch.autograd.grad((o * ct).sum(), [x, e] + list(m.parameters()))))
    for a, r in zip(*res):
        assert float((a - r).detach().abs().max()) <= 1e-12 * max(1.0, float(r.detach().abs().max()))
    selfe = b.edge_index[0] == b.edge_index[1]
    assert bool(selfe.any()) and bool((res[0][2][selfe] == 0).all())   # removed self loops get no gradient


def test_four_node_example_matches_hand_computed_alpha():
    """Edges 1->0, 2->0, 0->0 (removed), 3->1; H = 1, C = 2.  With lin_src = I, lin_edge = 0 (edge scores 0),
    att_src = (1, 0), att_dst = 0: z_j0 = leaky_relu(x_j[0]); node 0 attends over {1, 2, self}; node 2 and 3 only over
    themselves."""
    m = GATConvMP(2, 2, heads=1, edge_dim=2).double()
    with torch.no_grad():
        m.lin_src.weight.copy_(torch.eye(2))
        m.lin_edge.weight.zero_()
        m.att_src.copy_(torch.tensor([[[1.0, 0.0]]]))
        m.att_dst.zero_()
        m.att_edge.zero_()
        m.bias.zero_()
    x = torch.tensor([[-1.0, 5.0], [2.0, 1.0], [0.5, -3.0], [1.0, 7.0]], dtype=torch.float64)
    ei = torch.tensor([[1, 2, 0, 3], [0, 0, 0, 1]])
    out = m(x, ei, torch.randn(4, 2, dtype=torch.float64))
    z = [0.2 * -1.0, 2.0, 0.5]                    # self (node 0), node 1, node 2
    w = [math.exp(t) for t in z]
    a = [t / sum(w) for t in w]
    exp0 = a[0] * x[0] + a[1] * x[1] + a[2] * x[2]
    z1 = [2.0, 1.0]                               # node 1: self, node 3
    w1 = [math.exp(t) for t in z1]
    exp1 = (w1[0] * x[1] + w1[1] * x[3]) / sum(w1)
    assert torch.allclose(out[0], exp0, atol=1e-14) and torch.allclose(out[1], exp1, atol=1e-14)
    assert torch.allclose(out[2], x[2], atol=1e-15) and torch.allclose(out[3], x[3], atol=1e-15)


def test_oracle_equals_reference_live_gat():
    """The oracle layer (dense GATConv) against the reference's gps_layer.py run verbatim with the message-passing
    GATConv, fp64: outputs 1e-10, gradients (grad_edge_attr included) 1e-9."""
    fix = torch.load(os.path.join(GAT_DIR, "reference_live_GAT_Transformer.pt"), weights_only=False)
    cfg = fix["config"]
    ora = gat_oracle_layer(cfg["d"], cfg["glob"], cfg["heads"]).double()
    ora.load_state_dict(fix["state"], strict=True)
    b = golden_batch(fix, dtype=torch.float64)
    b.x.requires_grad_(True)
    b.edge_attr.requires_grad_(True)
    x, e = b.x, b.edge_attr
    out = ora.train()(b)
    (out.x * fix["ct_x"]).sum().backward()
    assert float((out.x - fix["out_x"]).abs().max()) < 1e-10
    assert float((x.grad - fix["grad_x"]).abs().max()) < 1e-9
    assert float((e.grad - fix["grad_e"]).abs().max()) < 1e-9
    got = dict(ora.named_parameters())
    for n, g in fix["grad_params"].items():
        assert float((got[n].grad - g).abs().max()) < 1e-9, n


def test_state_dict_parity_with_alias_key():
    ours = graphgps_b200.GPSLayer(64, "GAT", "Transformer", 4)
    ref = gat_oracle_layer(64, "Transformer", 4)
    so, sr = ours.state_dict(), ref.state_dict()
    assert set(so) == set(sr)
    assert "local_model.lin_dst.weight" in so and "local_model.lin_src.weight" in so
    names = [n for n, _ in ours.named_parameters()]
    assert "local_model.lin_src.weight" in names and "local_model.lin_dst.weight" not in names
    for k in so:
        assert so[k].shape == sr[k].shape, k
    ours.load_state_dict(sr, strict=True)
    ref.load_state_dict(ours.state_dict(), strict=True)
    assert ours.local_model.lin_dst.weight is ours.local_model.lin_src.weight
    assert ours.local_model.att_edge.shape == (1, 4, 16) and float(ours.local_model.bias.abs().sum()) == 0.0


def test_constructor_contract():
    with pytest.raises(ValueError):
        graphgps_b200.GPSLayer(30, "GAT", "Transformer", 4)
    with pytest.raises(ValueError):
        graphgps_b200.GPSLayer(30, "GAT", "None", 4)
    for glob in ("Transformer", "Performer", "None", "BiasedTransformer"):
        graphgps_b200.GPSLayer(64, "GAT", glob, 4)


def test_bucket_groups():
    from graphgps_b200.dp import LATE, MID, _group
    assert _group("local_model.lin_src.weight") == LATE
    for n in ("local_model.att_src", "local_model.att_dst", "local_model.att_edge", "local_model.bias",
              "local_model.lin_edge.weight"):
        assert _group(n) == MID, n


def test_plan_sizes():
    lib = _lib.load()
    r = lambda n: (n + 255) // 256 * 256
    for N, E, d, H, glob in ((10, 20, 64, 4, "Transformer"), (1000, 5000, 36, 4, "None"), (7, 0, 64, 1, "Transformer")):
        rc, pg = _plan(_args("GAT", N, E, d, H, glob))
        rc2, pc = _plan(_args("GCN", N, E, d, H, glob))
        assert rc == 0 and rc2 == 0
        # GCN saves dinv [N]; GAT saves v [H, d] and the scores [(4N + E) H]
        assert pg.saved_bytes - pc.saved_bytes == r(4 * H * d) + r(4 * (4 * N + E) * H) - r(4 * N)
        assert pg.bwd_workspace_bytes - pc.bwd_workspace_bytes == r(4 * H * d + lib.gps_gat_workspace_bytes(N, E, H, d))
        assert pg.fwd_workspace_bytes == pc.fwd_workspace_bytes and pg.wplanes_bytes == pc.wplanes_bytes
    rc, _ = _plan(_args("GAT", d=64, H=3))
    assert rc == _lib.GPS_ERR_ARG


def test_error_contract_before_any_cuda_call():
    lib = _lib.load()
    a = _args("GAT")
    a.x, a.edge_attr, a.x_out, a.saved, a.saved_bytes, a.workspace, a.workspace_bytes = 8, 8, 8, 8, 1 << 40, 8, 1 << 40
    a.grad_x_out, a.grad_x = 8, 8
    assert lib.gps_layer_forward(C.byref(a), None) == _lib.GPS_ERR_ARG   # null parameters
    assert lib.gps_layer_backward(C.byref(a), None) == _lib.GPS_ERR_ARG

    def full_gat():
        gat = _lib.GpsGat()
        gat.lin_src.weight = gat.lin_src.bias = gat.lin_edge.weight = gat.att_src = gat.att_dst = gat.att_edge = 8
        return gat

    for field, what in (("lin_src.weight", "lin_src"), ("lin_src.bias", "lin_src"), ("lin_edge.weight", "lin_edge"),
                        ("att_src", "att_"), ("att_dst", "att_"), ("att_edge", "att_")):
        a.gat = full_gat()
        obj, f = (getattr(a.gat, field.split(".")[0]), field.split(".")[1]) if "." in field else (a.gat, field)
        setattr(obj, f, 0)
        for fn in (lib.gps_layer_forward, lib.gps_layer_backward):
            assert fn(C.byref(a), None) == _lib.GPS_ERR_ARG, field
            assert what in lib.gps_last_error().decode(), field
    a.gat = full_gat()
    a.edge_attr = 0
    assert lib.gps_layer_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    a.edge_attr = 8
    a.grad_edge_attr = 0
    assert lib.gps_layer_backward(C.byref(a), None) == _lib.GPS_ERR_ARG
    n = _args("GAT", glob="None")   # an attention bias needs the Transformer
    n.gat, n.attn_bias = full_gat(), _lib.GpsAttnBias(8, 4, 0)
    assert lib.gps_layer_forward(C.byref(n), None) == _lib.GPS_ERR_ARG
    a.heads = 3
    assert lib.gps_layer_forward(C.byref(a), None) == _lib.GPS_ERR_ARG
    g = _lib.GpsGraph()
    g.N, g.E = 4, 4
    assert lib.gps_gat_fold_forward(None, 8, 64, 4, 8, None) == _lib.GPS_ERR_ARG
    assert lib.gps_gat_fold_forward(8, 8, 64, 3, 8, None) == _lib.GPS_ERR_ARG
    assert lib.gps_gat_fold_forward(8, 8, 6, 2, 8, None) == _lib.GPS_ERR_UNSUPPORTED
    assert lib.gps_gat_fold_backward(8, 8, None, 64, 4, 8, 8, 0, None) == _lib.GPS_ERR_ARG
    assert lib.gps_gat_fold_backward(8, 8, 8, 8192, 4, 8, 8, 0, None) == _lib.GPS_ERR_UNSUPPORTED
    fw = [C.byref(g), 64, 4, 8, 64, 8, 8, 8, 8, 8, 8, 8, 8, 0.0, 0, 0, None, None]
    assert lib.gps_gat_forward(*fw[:5], None, *fw[6:]) == _lib.GPS_ERR_ARG
    assert lib.gps_gat_forward(*fw[:2], 5, *fw[3:]) == _lib.GPS_ERR_ARG
    assert lib.gps_gat_forward(*fw[:1], 6, 2, *fw[3:]) == _lib.GPS_ERR_UNSUPPORTED
    bw = [C.byref(g), 64, 4, 8, 64, 8, 8, 8, 8, 8, 8, 8, 1 << 40, 8, 64, None, 8, 8, 8, 8, 8, 0, None]
    assert lib.gps_gat_backward(*bw[:7], None, *bw[8:]) == _lib.GPS_ERR_ARG
    assert lib.gps_gat_backward(*bw[:12], 4, *bw[13:]) == _lib.GPS_ERR_ARG
    assert lib.gps_gat_backward(*bw[:1], 6, 2, *bw[3:]) == _lib.GPS_ERR_UNSUPPORTED
