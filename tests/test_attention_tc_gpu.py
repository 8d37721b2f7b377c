"""GPU: the wgmma attention forward (csrc/attention_tc.cu) against float64 dense per-graph softmax attention and against
the CUDA-core kernel (same Philox dropout stream => identical masks), at the head dims of the BASELINE configs
(hd 76 C3, 16 zinc, 24 C4-Transformer, 64 code2 incl. graphs far longer than one 128-key tile)."""
import ctypes as C

import pytest
import torch

from graphgps_b200 import _lib
from graphgps_b200.batch import batch_from_lists, make_batch
from graphgps_b200.graph import graph_of
from util import _stream, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _padded_planes(QKV, H, hd, lo=True):
    """[N, 3*H*hd] fp32 -> bf16 hi/lo planes [2, N, 3*H*hd_pad] in the per-head padded layout (pads zero)."""
    N = QKV.shape[0]
    hp = (hd + 15) // 16 * 16
    x = torch.zeros(N, 3 * H, hp, device=QKV.device)
    x[:, :, :hd] = QKV.view(N, 3 * H, hd)
    x = x.view(N, 3 * H * hp)
    hi = x.to(torch.bfloat16)
    lo_t = (x - hi.float()).to(torch.bfloat16)
    buf = torch.stack([hi, lo_t]).contiguous()
    return buf, 3 * H * hp


def _ref(QKV, ptr, H, hd):
    N = QKV.shape[0]
    D = H * hd
    Q, K, V = QKV[:, :D].double(), QKV[:, D:2 * D].double(), QKV[:, 2 * D:].double()
    outs, lses = [], []
    for g in range(len(ptr) - 1):
        s, e = int(ptr[g]), int(ptr[g + 1])
        if e == s:
            continue
        q = Q[s:e].view(e - s, H, hd).transpose(0, 1)
        k = K[s:e].view(e - s, H, hd).transpose(0, 1)
        v = V[s:e].view(e - s, H, hd).transpose(0, 1)
        sc = q @ k.transpose(1, 2) / hd ** 0.5
        outs.append((torch.softmax(sc, -1) @ v).transpose(0, 1).reshape(e - s, D))
        lses.append(torch.logsumexp(sc, -1).transpose(0, 1))
    return torch.cat(outs), torch.cat(lses)


@pytest.mark.parametrize("shape,H,hd,B", [("pcqm4m-small", 4, 76, 256), ("zinc-gatedgcn", 4, 16, 32),
                                          ("pcqm4m-small", 16, 24, 40), ("code2", 4, 64, 12), ("code2", 2, 128, 5)])
@pytest.mark.parametrize("precision", [0, 1])
def test_attention_tc_forward_matches_fp64(shape, H, hd, B, precision):
    lib = _lib.load()
    b = make_batch(shape, seed=4, dim=8, num_graphs=B).to(DEV)
    gs = graph_of(b)
    N, D = b.num_nodes, H * hd
    QKV = torch.randn(N, 3 * D, device=DEV)
    planes, ld = _padded_planes(QKV, H, hd)
    O = torch.full((N, D), float("nan"), device=DEV)
    lse = torch.empty(N, H, device=DEV)
    rc = lib.gps_attention_forward_tc(C.byref(gs.desc), H, hd, planes[0].data_ptr(), planes[1].data_ptr() if precision == 0 else 0,
                                      ld, O.data_ptr(), D, lse.data_ptr(), 0.0, 0, 0, precision, _stream())
    _lib.check(rc, "attention_forward_tc")
    ref, ref_lse = _ref(QKV, b.ptr, H, hd)
    tol = 5e-5 if precision == 0 else 2e-2
    assert rel_err(O.cpu(), ref.cpu()) < tol
    assert rel_err(lse.cpu(), ref_lse.cpu()) < tol


def test_attention_tc_edge_cases_and_dropout_match_cuda_core_kernel():
    lib = _lib.load()
    H, hd = 4, 76
    D = H * hd
    # empty graphs, single-node graphs, a graph straddling two 128-row tiles
    b = batch_from_lists([1, 0, 130, 3, 0, 1, 200], [[] for _ in range(7)], d=8).to(DEV)
    gs = graph_of(b)
    N = b.num_nodes
    QKV = torch.randn(N, 3 * D, device=DEV)
    planes, ld = _padded_planes(QKV, H, hd)
    for p_drop in (0.0, 0.5):
        O1 = torch.empty(N, D, device=DEV)
        O2 = torch.empty(N, D, device=DEV)
        l1 = torch.empty(N, H, device=DEV)
        l2 = torch.empty(N, H, device=DEV)
        base = QKV.data_ptr()
        _lib.check(lib.gps_attention_forward(C.byref(gs.desc), H, hd, base, base + 4 * D, base + 8 * D, 3 * D, O1.data_ptr(), D,
                                             l1.data_ptr(), p_drop, 77, 4096, _stream()), "attention_forward")
        _lib.check(lib.gps_attention_forward_tc(C.byref(gs.desc), H, hd, planes[0].data_ptr(), planes[1].data_ptr(), ld,
                                                O2.data_ptr(), D, l2.data_ptr(), p_drop, 77, 4096, 0, _stream()), "tc")
        assert rel_err(O2.cpu(), O1.cpu()) < 5e-5, p_drop     # same Philox stream: identical dropout masks
        assert rel_err(l2.cpu(), l1.cpu()) < 5e-5
