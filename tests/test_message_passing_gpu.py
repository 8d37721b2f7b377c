"""GPU: every message-passing kernel of csrc/scatter.cu and csrc/eslap.cu, called through its stage entry point,
against the float64 stage references of tests/mp_reference.py, on the BASELINE shapes, heavy-tailed graphs with hubs of
thousands of in-edges, hand-built degenerate graphs, an in-degree sweep over the two-edge loop's odd tail, graphs large
enough for the grid-stride loops to wrap, and a width sweep up to the declared limit d = 4096.

Every output buffer starts as NaN, and every strided input carries NaN in the columns past its block, so an element a
kernel never writes, or a read outside its block, fails the comparison.  Tolerances (no relative-L2 fallback here):
  * sums over edges: the forward-error bound of recursive fp32 summation (`sum_bound`), computed from the fp64
    reference, plus a few ulps per term for __expf, the sigmoid and the division;
  * per-edge outputs (Ce, g_e, r, rho): 1e-5 max-abs, scaled by max(1, max|ref|) as util.rel_err does;
  * structural cases on small integers, where fp32 arithmetic is exact: bitwise equality.
The worst error seen as a fraction of its bound is printed per test (pytest -s)."""
import copy
import ctypes as C

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from graphgps_b200.batch import GraphBatch, batch_from_lists, make_batch
from graphgps_b200.graph import graph_of
from oracle.gps_oracle import OracleGPSLayer
from eslappe_oracle import OracleGPSLayerESLapPE
from eslappe_util import calibrate_gate, compare_eslap, make_pe, run_eslap
from nonorm_util import node_graph
from util import _nan, _stream, compare, rel_err, run_layer
import mp_reference as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F64 = torch.float64
U = 2.0 ** -24          # unit roundoff of fp32 (round to nearest)
EDGE_TOL = 1e-5         # per-edge outputs, scaled by max(1, max|ref|)
NUM_SMS = 132
WORST = {}              # stage -> worst error / bound seen


def gamma(m):
    """gamma_m = m u / (1 - m u): |fl(sum of m + 1 terms) - sum| <= gamma_m sum|t| for any summation order."""
    return m * U / (1 - m * U)


def sum_bound(index, size, mag, depth):
    """Bound on the error of the fp32 per-segment sums out[index[t]] = sum_t term_t, computed from the fp64 reference.

    mag [T, d]: |term_t| (for a term that is itself a product or sum: the sum of the magnitudes of its parts);
    depth [T, d] or [T, 1] or a number: roundings inside the term, in ulps (the 'few ulps per term': 1 per product or
    addition, 2 + 1.2 |x| for __expf(x), 2 for the reciprocal of the sigmoid).  Each segment of n terms adds gamma_n:
        bound_i = sum_{t in segment i} |term_t| gamma_(n_i + depth_t)."""
    n = torch.bincount(index, minlength=size).to(F64)
    g = gamma(n[index].unsqueeze(1) + depth)
    return torch.zeros(size, mag.shape[1], dtype=F64, device=mag.device).index_add_(0, index, mag * g)


def check(name, got, ref, bound):
    """|got - ref| <= bound elementwise (NaN in got fails)."""
    got, ref = got.double(), ref.double()
    err = (got - ref).abs()
    assert not bool(torch.isnan(got).any()), f"{name}: NaN in the output (an element never written)"
    frac = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
    WORST[name] = max(WORST.get(name, 0.0), frac)
    assert frac <= 1.0, f"{name}: error {frac:.3g} x its bound (max err {float(err.max()):.3g})"


def check_edge(name, got, ref):
    assert not bool(torch.isnan(got).any()), f"{name}: NaN in the output"
    e = rel_err(got, ref) if ref.numel() else 0.0
    WORST[name] = max(WORST.get(name, 0.0), e / EDGE_TOL)
    assert e <= EDGE_TOL, f"{name}: {e:.3g}"


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):
        print(f"worst error / bound  {k:28s} {WORST[k]:.3e}")


# ------------------------------------------------------------------------------------------------ graphs
def _malnet(d, seed=0):
    """8 function-call-like graphs of 500-5000 nodes, each with Pareto (tail 1.5) in-degrees: hubs of 1000+ in-edges."""
    sizes = [500, 800, 1200, 1800, 2500, 3200, 4000, 5000]
    xs, eis, eas, off = [], [], [], 0
    for k, n in enumerate(sizes):
        g = node_graph(n, 2 * n, d, seed=seed + k)
        xs.append(g.x), eis.append(g.edge_index + off), eas.append(g.edge_attr)
        off += n
    ptr = torch.tensor([0] + sizes).cumsum(0)
    return GraphBatch(x=torch.cat(xs), edge_index=torch.cat(eis, 1), edge_attr=torch.cat(eas), num_graphs=len(sizes),
                      batch=torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes)), ptr=ptr)


def _degenerate(d):
    """isolated nodes, in-edges without out-edges and the reverse, a self loop repeated three times, duplicate edges,
    empty graphs and a graph of one node"""
    return batch_from_lists([1, 0, 5, 4, 0, 3], [[], [], [(0, 1), (0, 2), (3, 3), (3, 3), (3, 3), (1, 2), (1, 2)],
                                                 [(0, 1), (1, 0), (2, 2)], [], [(0, 1), (0, 1), (0, 1)]], d=d, seed=3)


def _degree_sweep(d):
    """one star per in-degree k in (0, 1, 2, 3, 4, 5, 64, 65): the odd tail of the two-edge loop and long segments"""
    ks = (0, 1, 2, 3, 4, 5, 64, 65)
    return batch_from_lists([k + 1 for k in ks], [[(j, 0) for j in range(1, k + 1)] for k in ks], d=d, seed=4)


def _large(d, N=40000):
    """N above 2112 RY rows (RY = 256 / (d / 4) = 16 at d = 64) so every thread of the grid-stride loops loops more
    than once, with and without the statistics epilogue (132 RY rows per sweep)"""
    return node_graph(N, 2 * N, d, seed=5, tail=3.0)


def _widths(d):
    b = make_batch("zinc-gatedgcn", seed=6, dim=d, num_graphs=6)
    x = _degenerate(d)
    n0 = b.x.shape[0]
    return GraphBatch(x=torch.cat([b.x, x.x]), edge_index=torch.cat([b.edge_index, x.edge_index + n0], 1),
                      edge_attr=torch.cat([b.edge_attr, x.edge_attr]), num_graphs=b.num_graphs + x.num_graphs,
                      batch=torch.cat([b.batch, x.batch + b.num_graphs]), ptr=None)


FAMILIES = {
    "pcqm4m": (304, lambda d: make_batch("pcqm4m-small", seed=2, dim=d)),
    "zinc": (64, lambda d: make_batch("zinc-gatedgcn", seed=2, dim=d)),
    "code2": (256, lambda d: make_batch("code2", seed=2, dim=d)),
    "squirrel": (64, lambda d: node_graph(5201, 217073, d, seed=1)),
    "malnet": (64, _malnet),
    "degenerate": (12, _degenerate),
    "e0": (8, lambda d: batch_from_lists([3, 0, 2], [[], [], []], d=d)),
    "n1": (8, lambda d: batch_from_lists([1], [[(0, 0)]], d=d)),
    "degsweep": (52, _degree_sweep),
    "large": (64, _large),
}
WIDTHS = (4, 12, 48, 52, 64, 76, 96, 256, 304, 384, 1024, 4096)
CASES = [(f, FAMILIES[f][0]) for f in FAMILIES] + [("widths", d) for d in WIDTHS]
_CACHE = {}


def _graph(fam, d):
    key = (fam, d)
    if key not in _CACHE:
        b = _widths(d) if fam == "widths" else FAMILIES[fam][1](d)
        if b.ptr is None:
            b.ptr = torch.cat([torch.zeros(1, dtype=torch.int64), torch.bincount(b.batch, minlength=b.num_graphs).cumsum(0)])
        b = b.to(DEV)
        _CACHE[key] = (b, graph_of(b))
    return _CACHE[key]


def _ids(c):
    return f"{c[0]}-d{c[1]}"


def _rand(gen, *shape, scale=1.0):
    return (torch.randn(*shape, generator=gen) * scale).to(DEV)


def _strided(blocks, pad=8):
    """[N, k d + pad] buffer holding the given [N, d] blocks side by side and NaN in the gap past them"""
    N, d = blocks[0].shape
    buf = _nan(N, len(blocks) * d + pad)
    for i, t in enumerate(blocks):
        buf[:, i * d:(i + 1) * d] = t
    return buf


def _geom(N, d, nstat):
    """scatter.cu node_geom: rows per CTA (RY) and the number of CTAs"""
    C4 = d // 4
    if nstat:
        RY = min(1 if C4 >= 1024 else 1024 // C4, 16)
        RY = min(RY, max(48 * 1024 // (nstat * C4 * 16), 1))
        cap = NUM_SMS
    else:
        RY, cap = (1 if C4 >= 256 else 256 // C4), NUM_SMS * 16
    return RY, min(-(-max(N, 1) // (2 * RY)), cap)


def _ld8(n):
    return (n + 7) // 8 * 8


def _bf16_planes_exact(name, v, hi, lo):
    """hi = bf16_rn(v), lo = bf16_rn(v - hi), bitwise"""
    want_hi = v.to(torch.bfloat16)
    want_lo = (v - want_hi.float()).to(torch.bfloat16)
    assert torch.equal(hi.view(torch.int16), want_hi.view(torch.int16)), f"{name}: hi plane"
    assert torch.equal(lo.view(torch.int16), want_lo.view(torch.int16)), f"{name}: lo plane"


# ------------------------------------------------------------------------------------------------ GatedGCN
def _gated_inputs(b, d, gate, seed=0, scale=1.0):
    gen = torch.Generator().manual_seed(seed)
    N, E = b.num_nodes, b.num_edges
    A, B, D, Ex = (_rand(gen, N, d, scale=scale) for _ in range(4))
    Ce = _rand(gen, E, d, scale=scale)
    rho = (0.05 + 0.9 * torch.rand(E, generator=gen)).to(DEV) if gate else None
    return A, B, D, Ex, Ce, rho


def _gated_fwd(b, gs, d, A, B, D, Ex, Ce, rho, stats):
    lib = _lib.load()
    Y = _strided([A, B, D, Ex])
    ce = Ce.clone()
    xt = _nan(b.num_nodes, d)
    sx = torch.zeros(2, d, device=DEV, dtype=F64) if stats else None
    se = torch.zeros(2, d, device=DEV, dtype=F64) if stats else None
    p = Y.data_ptr()
    _lib.check(lib.gps_gatedgcn_aggregate_forward_gated(C.byref(gs.desc), d, p, p + 4 * d, p + 8 * d, p + 12 * d,
                                                        Y.shape[1], ce.data_ptr(), xt.data_ptr(), _lib.ptr(sx),
                                                        _lib.ptr(se), _lib.ptr(rho), _stream()), "gatedgcn fwd")
    return xt, ce, sx, se


def _sigmoid_ulps(e_ij, Dx, Ex, Ce, src, dst):
    """relative error of the fp32 sigma_ij in ulps: __expf (2 + 1.2 |x|), the reciprocal and the add (2), and the two
    roundings of e_ij = Ce + (Dx + Ex) amplified by the sigmoid's slope, (1 - s) 2 (|Ce| + |Dx| + |Ex|) <= that sum"""
    return 4.0 + 1.2 * e_ij.abs() + 2.0 * (Ce.abs() + Dx[dst].abs() + Ex[src].abs())


def _gated_fwd_bounds(A, B, D, Ex, Ce, rho, src, dst, N):
    e_ij = D[dst] + Ex[src] + Ce
    s = torch.sigmoid(e_ij) * (1.0 if rho is None else rho.unsqueeze(1))
    k = _sigmoid_ulps(e_ij, D, Ex, Ce, src, dst) + (1 if rho is not None else 0)
    num_b = sum_bound(dst, N, (s * B[src]).abs(), k + 1)
    den_b = sum_bound(dst, N, s, k)
    den = torch.zeros(N, s.shape[1], dtype=F64, device=s.device).index_add_(0, dst, s) + 1e-6
    agg = torch.zeros_like(den).index_add_(0, dst, s * B[src]) / den
    agg_abs = torch.zeros_like(den).index_add_(0, dst, (s * B[src]).abs()) / den
    agg_b = (num_b + agg.abs() * den_b) / den + 2 * U * agg_abs
    return e_ij, s, k, den, agg, agg_b


@pytest.mark.parametrize("stats", [False, True])
@pytest.mark.parametrize("gate", [False, True])
@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_gatedgcn_forward(case, gate, stats):
    b, gs = _graph(*case)
    d = case[1]
    A, B, D, Ex, Ce, rho = _gated_inputs(b, d, gate, seed=1)
    xt, ce, sx, se = _gated_fwd(b, gs, d, A, B, D, Ex, Ce, rho, stats)
    src, dst = b.edge_index
    N = b.num_nodes
    A, B, D, Ex, Ce = (t.double() for t in (A, B, D, Ex, Ce))
    rho64 = None if rho is None else rho.double()
    xt_ref, e_ref, _, _ = R.gatedgcn_forward(A, B, D, Ex, Ce, src, dst, rho64)
    e_ij, s, k, den, agg, agg_b = _gated_fwd_bounds(A, B, D, Ex, Ce, rho64, src, dst, N)
    xt_b = agg_b + 2 * U * (A.abs() + agg.abs())
    check("gatedgcn_fwd xt", xt, xt_ref, xt_b)
    check_edge("gatedgcn_fwd Ce", ce, e_ref)
    if stats:
        RY, blocks = _geom(N, d, 4)
        rows = -(-N // (blocks * RY)) + RY + 2
        thread = ((torch.arange(N, device=DEV) // RY) % blocks) * RY + torch.arange(N, device=DEV) % RY
        per_t = torch.bincount(thread[dst], minlength=blocks * RY) if dst.numel() else torch.zeros(1, device=DEV)
        erows = int(per_t.max()) + RY + 2
        e_b = 2 * U * (D[dst].abs() + Ex[src].abs() + Ce.abs())
        check("gatedgcn_fwd stats_x sum", sx[0], xt_ref.sum(0), xt_b.sum(0) + gamma(rows) * xt_ref.abs().sum(0))
        check("gatedgcn_fwd stats_x sumsq", sx[1], (xt_ref ** 2).sum(0),
              (2 * xt_ref.abs() * xt_b + xt_b ** 2).sum(0) + gamma(rows + 1) * (xt_ref ** 2).sum(0))
        check("gatedgcn_fwd stats_e sum", se[0], e_ref.sum(0), e_b.sum(0) + gamma(erows) * e_ref.abs().sum(0))
        check("gatedgcn_fwd stats_e sumsq", se[1], (e_ref ** 2).sum(0),
              (2 * e_ref.abs() * e_b + e_b ** 2).sum(0) + gamma(erows + 1) * (e_ref ** 2).sum(0))


@pytest.mark.parametrize("gate", [False, True])
@pytest.mark.parametrize("fam", ["malnet", "degenerate", "degsweep"])
def test_gatedgcn_forward_saturated(fam, gate):
    """logits of std 20: sigmoids of exactly 0 or 1 in fp32 and nodes with den ~ 0, where the 1e-6 dominates"""
    b, gs = _graph(fam, FAMILIES[fam][0])
    d = FAMILIES[fam][0]
    A, B, D, Ex, Ce, rho = _gated_inputs(b, d, gate, seed=2, scale=20.0 / 3 ** 0.5)
    A, B = A / 20 * 3 ** 0.5, B / 20 * 3 ** 0.5     # only the logits are wide
    xt, ce, _, _ = _gated_fwd(b, gs, d, A, B, D, Ex, Ce, rho, False)
    src, dst = b.edge_index
    A, B, D, Ex, Ce = (t.double() for t in (A, B, D, Ex, Ce))
    rho64 = None if rho is None else rho.double()
    xt_ref, e_ref, _, den = R.gatedgcn_forward(A, B, D, Ex, Ce, src, dst, rho64)
    if fam == "malnet":
        assert bool((den[dst] < 1e-6).any()), "no node with den below 1e-6"
    _, s, _, _, agg, agg_b = _gated_fwd_bounds(A, B, D, Ex, Ce, rho64, src, dst, b.num_nodes)
    check("gatedgcn_fwd_saturated xt", xt, xt_ref, agg_b + 2 * U * (A.abs() + agg.abs()))
    check_edge("gatedgcn_fwd_saturated Ce", ce, e_ref)


def _gated_bwd(b, gs, d, ehat, B, rho, g_xt, g_e_in, planes):
    lib = _lib.load()
    N, E = b.num_nodes, b.num_edges
    Y = _strided([_nan(N, d), B, _nan(N, d), _nan(N, d)])     # only Bx may be read
    gY = _strided([g_xt, _nan(N, d), _nan(N, d), _nan(N, d)])
    g_e = g_e_in.clone()
    g_num, g_den = _nan(N, d), _nan(N, d)
    ldp = 4 * d + 8
    yp = [_nan(N, ldp, dtype=torch.bfloat16) for _ in range(2)] if planes else None
    lde = _ld8(d)
    ep = [_nan(E, lde, dtype=torch.bfloat16) for _ in range(2)] if planes else None
    ypl = _lib.GpsPlanes(yp[0].data_ptr(), yp[1].data_ptr(), ldp) if planes else _lib.GpsPlanes(0, 0, 0)
    epl = _lib.GpsPlanes(ep[0].data_ptr(), ep[1].data_ptr(), lde) if planes else _lib.GpsPlanes(0, 0, 0)
    p = Y.data_ptr()
    _lib.check(lib.gps_gatedgcn_aggregate_backward(C.byref(gs.desc), d, ehat.data_ptr(), p + 4 * d, Y.shape[1],
                                                   _lib.ptr(rho), gY.data_ptr(), gY.shape[1], g_e.data_ptr(),
                                                   g_num.data_ptr(), g_den.data_ptr() if rho is not None else 0,
                                                   C.byref(ypl), C.byref(epl), _stream()), "gatedgcn bwd")
    assert torch.equal(gY[:, :d], g_xt), "block 0 (g_xt) must only be read"
    gated = _lib.ptr(rho) != 0        # an empty rho (E = 0) is NULL: no gate, g_den is not written
    out = {"g_Bx": gY[:, d:2 * d], "g_Dx": gY[:, 2 * d:3 * d], "g_Ex": gY[:, 3 * d:4 * d], "g_e": g_e,
           "g_num": g_num, "g_den": g_den if gated else None}
    if planes:
        for k, c0 in (("g_Bx", d), ("g_Dx", 2 * d), ("g_Ex", 3 * d)):
            _bf16_planes_exact(k, out[k], yp[0][:, c0:c0 + d], yp[1][:, c0:c0 + d])
        _bf16_planes_exact("g_e", g_e, ep[0][:, :d], ep[1][:, :d])
    return out


@pytest.mark.parametrize("planes", [False, True])
@pytest.mark.parametrize("gate", [False, True])
@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_gatedgcn_backward(case, gate, planes):
    b, gs = _graph(*case)
    d = case[1]
    N, E = b.num_nodes, b.num_edges
    A, B, D, Ex, Ce, rho = _gated_inputs(b, d, gate, seed=3)
    src, dst = b.edge_index
    ehat = (D[dst] + Ex[src] + Ce).contiguous()        # e_ij as the forward stored it (an fp32 input here)
    gen = torch.Generator().manual_seed(4)
    g_xt, g_e_in = _rand(gen, N, d), _rand(gen, E, d)
    got = _gated_bwd(b, gs, d, ehat, B, rho, g_xt, g_e_in, planes)

    # reference: e_ij = ehat exactly (Dx = Ex = 0, Ce = ehat), so the fp32 ehat is the exact input
    z = torch.zeros(N, d, dtype=F64, device=DEV)
    B64, eh, gx, ge = B.double(), ehat.double(), g_xt.double(), g_e_in.double()
    rho64 = None if rho is None else rho.double()
    ref = R.gatedgcn_backward(z, B64, z, z, eh, src, dst, gx, ge, rho64)

    # bounds from the fp64 reference (see sum_bound)
    _, s, k, den, agg, agg_b = _gated_fwd_bounds(z, B64, z, z, eh, rho64, src, dst, N)
    den_b = sum_bound(dst, N, s, k)
    g_num = gx / den
    gn_b = g_num.abs() * (den_b / den + 2 * U)
    gd_b = gn_b * agg.abs() + g_num.abs() * agg_b + U * (g_num * agg).abs()
    sig = torch.sigmoid(eh)
    r = 1.0 if rho64 is None else rho64.unsqueeze(1)
    ds = sig * (1 - sig)
    k_e = 4.0 + 1.2 * eh.abs() + 4                                   # __expf, reciprocal, 1 - s, the products
    term_mag = (g_num[dst].abs() * B64[src].abs() + (g_num * agg)[dst].abs())
    ge_b = (r * (gn_b[dst] * B64[src].abs() + gd_b[dst]) * ds + r * term_mag * (gamma(k_e) * ds + 2 * U * sig * sig)
            + U * (ref["g_e"].abs() + ge.abs()))
    check_edge("gatedgcn_bwd g_e", got["g_e"], ref["g_e"])
    check("gatedgcn_bwd g_num", got["g_num"], ref["g_num"], gn_b)
    if got["g_den"] is not None:
        check("gatedgcn_bwd g_den", got["g_den"], ref["g_den"], gd_b)
    ge_abs = ref["g_e"].abs()
    check("gatedgcn_bwd g_Dx", got["g_Dx"], ref["g_Dx"],
          torch.zeros_like(z).index_add_(0, dst, ge_b) + sum_bound(dst, N, ge_abs + ge_b, 1))
    check("gatedgcn_bwd g_Ex", got["g_Ex"], ref["g_Ex"],
          torch.zeros_like(z).index_add_(0, src, ge_b) + sum_bound(src, N, ge_abs + ge_b, 1))
    sr = sig * r
    check("gatedgcn_bwd g_Bx", got["g_Bx"], ref["g_Bx"],
          torch.zeros_like(z).index_add_(0, src, gn_b[dst] * sr)
          + sum_bound(src, N, (g_num[dst] * sr).abs(), 4.0 + 1.2 * eh.abs() + 2))


def test_gatedgcn_backward_structural_sums_are_exact():
    """g_xt = 0 and small-integer g_e: g_Dx = sum of in-edge g_e, g_Ex = sum of out-edge g_e, g_Bx = 0, all bitwise,
    at every degree (5000-edge hubs included): a dropped or doubled edge in either walk shows up"""
    for fam in ("squirrel", "malnet", "degenerate", "degsweep", "large"):
        d = FAMILIES[fam][0]
        b, gs = _graph(fam, d)
        N, E = b.num_nodes, b.num_edges
        src, dst = b.edge_index
        gen = torch.Generator().manual_seed(5)
        for gate in (False, True):
            A, B, D, Ex, Ce, rho = _gated_inputs(b, d, gate, seed=6)
            g_e_in = torch.randint(-3, 4, (E, d), generator=gen).float().to(DEV)
            got = _gated_bwd(b, gs, d, Ce, B, rho, torch.zeros(N, d, device=DEV), g_e_in, False)
            z = torch.zeros(N, d, dtype=F64, device=DEV)
            assert torch.equal(got["g_e"], g_e_in), fam
            assert torch.equal(got["g_Dx"].double(), z.clone().index_add_(0, dst, g_e_in.double())), fam
            assert torch.equal(got["g_Ex"].double(), z.clone().index_add_(0, src, g_e_in.double())), fam
            assert not bool(got["g_Bx"].any()), fam


# ------------------------------------------------------------------------------------------------ EquivStableLapPE
def _eslap_params(d, act, seed):
    gen = torch.Generator().manual_seed(seed)
    w1, b1 = torch.randn(d, 1, generator=gen), torch.randn(d, generator=gen) * 0.5
    w2, b2 = torch.randn(1, d, generator=gen) / d ** 0.5, torch.randn(1, generator=gen) * 0.1
    return [t.to(DEV) for t in (w1, b1, w2, b2)]


def _eslap_graph(kind):
    if kind == "small":       # E below one chunk of 32 edges
        return batch_from_lists([4, 3, 0, 2], [[(0, 1), (1, 0), (2, 1), (3, 3), (0, 1)], [(0, 2), (1, 2)], [], []], d=4)
    if kind == "chunks":      # E = 132 * 32 + 1: 128 chunks of 33 edges and a last one of 1 edge
        b = node_graph(600, NUM_SMS * 32 + 1, 4, seed=7)
        return b
    if kind == "e0":
        return batch_from_lists([3, 2], [[], []], d=4)
    return _malnet(4, seed=8)


@pytest.mark.parametrize("kind", ["small", "chunks", "e0", "malnet"])
@pytest.mark.parametrize("k", [1, 7, 37])
@pytest.mark.parametrize("act", ["relu", "gelu"])
def test_eslap_forward_backward(act, k, kind):
    lib = _lib.load()
    d = 64
    key = ("eslap", kind)
    if key not in _CACHE:
        bb = _eslap_graph(kind)
        bb.x = torch.zeros(bb.x.shape[0], d)
        _CACHE[key] = (bb.to(DEV), None)
    b = _CACHE[key][0]
    gs = graph_of(b)
    N, E = b.num_nodes, b.num_edges
    src, dst = b.edge_index
    pe = make_pe(N, k, seed=k).to(DEV)
    w1, b1, w2, b2 = _eslap_params(d, act, seed=k)
    a = _lib.ACT[act]
    r, rho = _nan(E), _nan(E)
    _lib.check(lib.gps_eslap_forward(C.byref(gs.desc), pe.data_ptr(), k, d, a, w1.data_ptr(), b1.data_ptr(),
                                     w2.data_ptr(), b2.data_ptr(), r.data_ptr(), rho.data_ptr(), _stream()), "eslap fwd")
    P64 = [t.double() for t in (w1, b1, w2, b2)]
    r_ref, rho_ref = R.eslap_forward(pe.double(), src, dst, *P64, act)
    check_edge(f"eslap_fwd r", r, r_ref)
    check_edge(f"eslap_fwd rho", rho, rho_ref)

    # backward from fp32 inputs: g_num, g_den, Bx, ehat, and r / rho rounded from the fp64 reference
    gen = torch.Generator().manual_seed(10 + k)
    g_num, g_den, Bx = _rand(gen, N, d), _rand(gen, N, d), _rand(gen, N, d)
    ehat = _rand(gen, E, d)
    r32, rho32 = r_ref.float(), rho_ref.float()
    Y = _strided([Bx])
    ws_bytes = lib.gps_eslap_workspace_bytes(E, d)
    ws = _nan(max(ws_bytes // 4, 1))
    outs = {}
    for acc in (0, 1):
        base = {n: _rand(gen, *shape) if acc else _nan(*shape)
                for n, shape in (("grad_pe", (N, k)), ("gw1", (d, 1)), ("gb1", (d,)), ("gw2", (1, d)), ("gb2", (1,)))}
        base["grad_pe"] = _nan(N, k)     # grad_pe is always written
        o = {n: t.clone() for n, t in base.items()}
        _lib.check(lib.gps_eslap_backward(C.byref(gs.desc), pe.data_ptr(), k, d, a, g_num.data_ptr(), g_den.data_ptr(),
                                          Y.data_ptr(), Y.shape[1], ehat.data_ptr(), r32.data_ptr(), rho32.data_ptr(),
                                          w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), ws.data_ptr(), ws_bytes,
                                          o["grad_pe"].data_ptr(), o["gw1"].data_ptr(), o["gb1"].data_ptr(),
                                          o["gw2"].data_ptr(), o["gb2"].data_ptr(), acc, _stream()), "eslap bwd")
        outs[acc] = (base, o)
    ref = R.eslap_backward(pe.double(), src, dst, *P64, act, Bx.double(), ehat.double(), g_num.double(), g_den.double())

    # bounds (fp64): gz_e = rho(1-rho) sum_c (g_num_i Bx_j + g_den_i) s_c over d columns, gr_e = gz_e sum_m w2 act' w1
    eh = ehat.double()
    s = torch.sigmoid(eh)
    ks = 8.0 + 1.2 * float(eh.abs().max()) if E else 0.0
    T = ((g_num.double()[dst] * Bx.double()[src]).abs() + g_den.double()[dst].abs()) * s
    rr = rho_ref * (1 - rho_ref)
    g_rho = ((g_num.double()[dst] * Bx.double()[src] + g_den.double()[dst]) * s).sum(1)
    gz = g_rho * rr
    # rho enters rounded to fp32: 1 - rho loses relative precision as rho -> 1, a perturbation of the input
    gz_b = (rr * gamma(d + ks) * T.sum(1) + gamma(6) * gz.abs() + rr * 4 * U * T.sum(1)
            + g_rho.abs() * (rho32.double() - rho_ref).abs() * (1 - 2 * rho_ref).abs())
    pre = r_ref.unsqueeze(1) * P64[0].reshape(1, -1) + P64[1]
    if act == "relu":
        h, dact, dact_mag, h_mag = pre.relu(), (pre > 0).double(), (pre > 0).double(), pre.relu()
    else:
        cdf = 0.5 * (1 + torch.erf(pre / 2 ** 0.5))
        pdf = torch.exp(-0.5 * pre * pre) / (2 * torch.pi) ** 0.5
        h, dact, dact_mag, h_mag = pre * cdf, cdf + pre * pdf, cdf + (pre * pdf).abs(), (pre * cdf).abs() + pre.abs()
    w1r, w2r = P64[0].reshape(1, -1), P64[2].reshape(1, -1)
    S = (w2r * dact * w1r).sum(1)
    Sabs = (w2r.abs() * dact_mag * w1r.abs()).sum(1)
    gr = gz * S
    ka = 16.0                                        # erff, __expf and the products of act / act'
    gr_b = gz_b * S.abs() + gz.abs() * gamma(d + ka) * Sabs
    pn = pe.double()
    dp_in, dp_out = pn[dst] - pn[src], pn[src] - pn[dst]
    pe_b = (torch.zeros(N, k, dtype=F64, device=DEV).index_add_(0, dst, 2 * dp_in.abs() * gr_b.unsqueeze(1))
            .index_add_(0, src, 2 * dp_out.abs() * gr_b.unsqueeze(1)))
    n_pe = (torch.bincount(dst, minlength=N) + torch.bincount(src, minlength=N)).double().unsqueeze(1)
    pe_mag = (torch.zeros(N, k, dtype=F64, device=DEV).index_add_(0, dst, 2 * (dp_in * gr.unsqueeze(1)).abs())
              .index_add_(0, src, 2 * (dp_out * gr.unsqueeze(1)).abs()))
    pe_b = pe_b + gamma(n_pe + 4) * pe_mag
    chunk = max(32, -(-E // NUM_SMS))
    depth = chunk + -(-E // chunk) + ka if E else 0
    gze, gzb = gz.unsqueeze(1), gz_b.unsqueeze(1)
    gpre_mag = (gze * w2r).abs() * dact_mag
    bounds = {
        "gw2": ((gzb * h_mag).sum(0) + gamma(depth) * (gze.abs() * h_mag).sum(0)).reshape(1, -1),
        "gw1": ((gzb * w2r.abs() * dact_mag * r_ref.unsqueeze(1)).sum(0)
                + gamma(depth) * (gpre_mag * r_ref.unsqueeze(1)).sum(0)).reshape(-1, 1),
        "gb1": (gzb * w2r.abs() * dact_mag).sum(0) + gamma(depth) * gpre_mag.sum(0),
        "gb2": (gz_b.sum() + gamma(depth) * gz.abs().sum()).reshape(1),
    }
    for acc, (base, o) in outs.items():
        tag = f"eslap_bwd{'+acc' if acc else ''}"
        check(f"{tag} grad_pe", o["grad_pe"], ref["grad_pe"], pe_b)
        for n in ("gw1", "gb1", "gw2", "gb2"):
            want = ref[n].reshape(base[n].shape)
            bound = bounds[n].reshape(base[n].shape)
            if acc:
                want = want + base[n].double()
                bound = bound + U * want.abs()
            check(f"{tag} {n}", o[n], want, bound)
        if E == 0:
            assert not bool(o["grad_pe"].any())
            if not acc:
                assert all(not bool(o[n].any()) for n in ("gw1", "gb1", "gw2", "gb2"))


# ------------------------------------------------------------------------------------------------ GINE
def _gine(b, gs, d, x, e, eps, g_out, add):
    lib = _lib.load()
    N, E = b.num_nodes, b.num_edges
    out, g_e, g_x = _nan(N, d), _nan(E, d), _nan(N, d)
    _lib.check(lib.gps_gine_aggregate_forward(C.byref(gs.desc), d, x.data_ptr(), e.data_ptr(), eps, out.data_ptr(),
                                              _stream()), "gine fwd")
    _lib.check(lib.gps_gine_aggregate_backward(C.byref(gs.desc), d, x.data_ptr(), e.data_ptr(), g_out.data_ptr(), eps,
                                               _lib.ptr(add), g_e.data_ptr(), g_x.data_ptr(), _stream()), "gine bwd")
    return out, g_e, g_x


@pytest.mark.parametrize("eps", [0.0, 0.37, -0.5])
@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_gine(case, eps):
    b, gs = _graph(*case)
    d = case[1]
    N, E = b.num_nodes, b.num_edges
    src, dst = b.edge_index
    gen = torch.Generator().manual_seed(11)
    x, e, g_out = _rand(gen, N, d), _rand(gen, E, d), _rand(gen, N, d)
    if E:   # the kink: messages of exactly 0 get gradient 0, as torch's relu backward gives
        e[::3] = -x[src[::3]]
    add = _rand(gen, N, d) if eps != 0.0 else None
    out, g_e, g_x = _gine(b, gs, d, x, e, eps, g_out, add)
    eps = float(torch.tensor(eps, dtype=torch.float32))      # the kernel's eps is the fp32 value
    x64, e64 = x.double(), e.double()
    ref = R.gine_forward(x64, e64, src, dst, eps)
    rgx, rge = R.gine_backward(x64, e64, src, dst, eps, g_out.double(), None if add is None else add.double())
    msg = (x64[src] + e64).relu()
    onep = abs(1 + eps)
    check("gine_fwd out", out, ref, sum_bound(dst, N, msg, 1) + gamma(torch.bincount(dst, minlength=N).double()
                                                                        .unsqueeze(1) + 3) * onep * x64.abs())
    assert torch.equal(g_e.double(), rge), "gine_bwd g_e: exact (a selection of g_out)"
    base = onep * g_out.double().abs() + (0 if add is None else add.double().abs())
    n_out = torch.bincount(src, minlength=N).double().unsqueeze(1)
    check("gine_bwd g_x", g_x, rgx, sum_bound(src, N, rge.abs(), 2) + gamma(n_out + 3) * base)


def test_gine_structural_degree_count_is_exact():
    """x = 0, e = 1, eps = 0: out_i = in-degree of i, bitwise, hubs included"""
    for fam in ("squirrel", "malnet", "degenerate", "degsweep", "large"):
        d = FAMILIES[fam][0]
        b, gs = _graph(fam, d)
        N, E = b.num_nodes, b.num_edges
        x, e = torch.zeros(N, d, device=DEV), torch.ones(E, d, device=DEV)
        out, g_e, g_x = _gine(b, gs, d, x, e, 0.0, torch.ones(N, d, device=DEV), None)
        deg = torch.bincount(b.edge_index[1], minlength=N).float().unsqueeze(1).expand(N, d)
        assert torch.equal(out, deg), fam
        outdeg = torch.bincount(b.edge_index[0], minlength=N).float().unsqueeze(1).expand(N, d)
        assert torch.equal(g_x, outdeg + 1), fam


# ------------------------------------------------------------------------------------------------ GCN
def _gcn(b, gs, d, Y, bias, x, p, seed, offset, stats, g_h, planes):
    lib = _lib.load()
    N = b.num_nodes
    Ys = _strided([Y])
    dinv, xloc = _nan(N), _nan(N, d)
    st = torch.zeros(2, d, device=DEV, dtype=F64) if stats else None
    _lib.check(lib.gps_gcn_aggregate_forward(C.byref(gs.desc), d, Ys.data_ptr(), Ys.shape[1], bias.data_ptr(),
                                             x.data_ptr(), dinv.data_ptr(), xloc.data_ptr(), p, seed, offset,
                                             _lib.ptr(st), _stream()), "gcn fwd")
    gY = _nan(N, d + 8)
    ldp = _ld8(d) + 8
    pl = [_nan(N, ldp, dtype=torch.bfloat16) for _ in range(2)] if planes else None
    gp = _lib.GpsPlanes(pl[0].data_ptr(), pl[1].data_ptr(), ldp) if planes else _lib.GpsPlanes(0, 0, 0)
    _lib.check(lib.gps_gcn_aggregate_backward(C.byref(gs.desc), d, g_h.data_ptr(), dinv.data_ptr(), gY.data_ptr(),
                                              gY.shape[1], C.byref(gp), _stream()), "gcn bwd")
    assert bool(torch.isnan(gY[:, d:]).all()), "gcn bwd wrote past its block"
    if planes:
        _bf16_planes_exact("gcn gY", gY[:, :d], pl[0][:, :d], pl[1][:, :d])
    return dinv, xloc, st, gY[:, :d]


@pytest.mark.parametrize("p", [0.0, 0.3])
@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_gcn(case, p):
    lib = _lib.load()
    b, gs = _graph(*case)
    d = case[1]
    N = b.num_nodes
    src, dst = b.edge_index
    gen = torch.Generator().manual_seed(12)
    Y, x, g_h = _rand(gen, N, d), _rand(gen, N, d), _rand(gen, N, d)
    bias = _rand(gen, d, scale=0.5)
    seed, offset = 1234, 8 * 4096
    dinv, xloc, st, gY = _gcn(b, gs, d, Y, bias, x, p, seed, offset, True, g_h, p == 0.0)
    keep = None
    if p > 0:
        keep = torch.empty(N, d, device=DEV)
        _lib.check(lib.gps_dropout_mask(keep.data_ptr(), N, d, p, seed, offset, 3, _stream()), "mask")
        keep = keep.double()
    dref = R.gcn_dinv(src, dst, N)
    check("gcn dinv", dinv, dref, 6 * U * dref)
    ref = R.gcn_forward(Y.double(), bias.double(), x.double(), src, dst, keep, p)
    # bound: dinv_i (dinv_i |Y_i| + sum_j dinv_j |Y_j|) with the rsqrtf error (2 ulps) and the products in each term
    nsl = src != dst
    Ya = Y.double().abs()
    mag = dref.unsqueeze(1) * Ya
    agg = torch.zeros(N, d, dtype=F64, device=DEV).index_add_(0, dst[nsl], dref[src[nsl]].unsqueeze(1) * Ya[src[nsl]])
    n_in = torch.bincount(dst[nsl], minlength=N).double().unsqueeze(1)
    h_b = dref.unsqueeze(1) * gamma(n_in + 8) * (mag + agg) + 2 * U * bias.double().abs()
    scale = 1.0 if keep is None else keep / (1 - p)
    h = ref - x.double()
    x_b = scale * h_b + 4 * U * (h.abs() + ref.abs())
    check("gcn_fwd xloc", xloc, ref, x_b)
    RY, blocks = _geom(N, d, 2)
    rows = -(-N // (blocks * RY)) + RY + 2
    check("gcn_fwd stats sum", st[0], ref.sum(0), x_b.sum(0) + gamma(rows) * ref.abs().sum(0))
    check("gcn_fwd stats sumsq", st[1], (ref ** 2).sum(0),
          (2 * ref.abs() * x_b + x_b ** 2).sum(0) + gamma(rows + 1) * (ref ** 2).sum(0))
    gref = R.gcn_backward(Y.double(), src, dst, g_h.double())
    ga = g_h.double().abs()
    bmag = dref.unsqueeze(1) * ga
    bagg = torch.zeros(N, d, dtype=F64, device=DEV).index_add_(0, src[nsl], dref[dst[nsl]].unsqueeze(1) * ga[dst[nsl]])
    n_out = torch.bincount(src[nsl], minlength=N).double().unsqueeze(1)
    check("gcn_bwd gY", gY, gref, dref.unsqueeze(1) * gamma(n_out + 8) * (bmag + bagg))


def test_gcn_structural_degree_count_is_exact():
    """(1 / dinv^2) rounds to 1 + #non-self in-edges exactly: self loops replaced, duplicates counted, hubs included"""
    for fam in ("squirrel", "malnet", "degenerate", "degsweep", "n1"):
        d = FAMILIES[fam][0]
        b, gs = _graph(fam, d)
        N = b.num_nodes
        z = torch.zeros(N, d, device=DEV)
        dinv = _gcn(b, gs, d, z, torch.zeros(d, device=DEV), z, 0.0, 0, 0, False, z, False)[0]
        src, dst = b.edge_index
        want = 1 + torch.bincount(dst[src != dst], minlength=N)
        assert torch.equal((1.0 / dinv.double() ** 2).round().long(), want), fam


# ------------------------------------------------------------------------------------------------ determinism
def test_two_runs_give_the_same_bits():
    """scatter.cu and eslap.cu reduce in a fixed order: every feature output and the gate's gradients repeat bitwise
    (the double-atomic column statistics are exempt)"""
    lib = _lib.load()
    b, gs = _graph("malnet", 64)
    d, N, E = 64, b.num_nodes, b.num_edges
    src, dst = b.edge_index
    runs = []
    for _ in range(2):
        A, B, D, Ex, Ce, rho = _gated_inputs(b, d, True, seed=13)
        xt, ce, _, _ = _gated_fwd(b, gs, d, A, B, D, Ex, Ce, rho, True)
        gen = torch.Generator().manual_seed(14)
        bw = _gated_bwd(b, gs, d, ce, B, rho, _rand(gen, N, d), _rand(gen, E, d), True)
        x, e, g_out = _rand(gen, N, d), _rand(gen, E, d), _rand(gen, N, d)
        gi = _gine(b, gs, d, x, e, 0.37, g_out, g_out)
        gc = _gcn(b, gs, d, x, g_out[0], e[:N], 0.3, 7, 4096, True, g_out, True)
        k = 7
        pe = make_pe(N, k, seed=1).to(DEV)
        w1, b1, w2, b2 = _eslap_params(d, "gelu", seed=1)
        r, rh = _nan(E), _nan(E)
        _lib.check(lib.gps_eslap_forward(C.byref(gs.desc), pe.data_ptr(), k, d, 1, w1.data_ptr(), b1.data_ptr(),
                                         w2.data_ptr(), b2.data_ptr(), r.data_ptr(), rh.data_ptr(), _stream()), "fwd")
        ws_bytes = lib.gps_eslap_workspace_bytes(E, d)
        ws = torch.empty(ws_bytes // 4, device=DEV)
        grads = [_nan(N, k), _nan(d, 1), _nan(d), _nan(1, d), _nan(1)]
        Y = _strided([B])
        _lib.check(lib.gps_eslap_backward(C.byref(gs.desc), pe.data_ptr(), k, d, 1, bw["g_num"].data_ptr(),
                                          bw["g_den"].data_ptr(), Y.data_ptr(), Y.shape[1], ce.data_ptr(), r.data_ptr(),
                                          rh.data_ptr(), w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), ws.data_ptr(),
                                          ws_bytes, *(t.data_ptr() for t in grads), 0, _stream()), "bwd")
        runs.append([xt, ce, *(v for v in bw.values() if v is not None), *gi, *gc[:2], gc[3], r, rh, *grads])
    for i, (a, c) in enumerate(zip(*runs)):
        assert torch.equal(a.view(torch.int32), c.view(torch.int32)), f"output {i} differs between two runs"


# ------------------------------------------------------------------------------------------------ whole layer at hubs
def _to64(b, keys=("x", "edge_attr")):
    b = b.clone()
    for k in keys:
        setattr(b, k, getattr(b, k).double())
    return b


def _cts(b, seed=9):
    g = torch.Generator().manual_seed(seed)
    return {"config": dict(local="CustomGatedGCN"), "ct_x": torch.randn(b.x.shape, generator=g),
            "ct_e": torch.randn(b.edge_attr.shape, generator=g)}


@pytest.mark.parametrize("eslap", [False, True])
def test_gatedgcn_layer_at_hub_degrees_strict(eslap):
    """GatedGCN+Transformer, GELU, BatchNorm, training, fp32, on the MalNet-like batch against the fp64 oracle (run on
    the GPU): every output and gradient within 1e-3 max-abs, no L2 fallback"""
    d = 64
    b = _malnet(d, seed=20)
    torch.manual_seed(0)
    if eslap:
        b.pe_EquivStableLapPE = make_pe(b.x.shape[0], 8, seed=3)
        ora = OracleGPSLayerESLapPE(d, "CustomGatedGCN", "Transformer", 4, act="gelu")
        calibrate_gate(ora, b.pe_EquivStableLapPE, b.edge_index)
    else:
        ora = OracleGPSLayer(d, "CustomGatedGCN", "Transformer", 4, act="gelu")
    ours = graphgps_b200.GPSLayer(d, "CustomGatedGCN", "Transformer", 4, act="gelu", equivstable_pe=eslap)
    ours.load_state_dict(ora.state_dict(), strict=True)
    ours = ours.to(DEV).train()
    fix = _cts(b)
    keys = ("x", "edge_attr", "pe_EquivStableLapPE") if eslap else ("x", "edge_attr")
    run = run_eslap if eslap else run_layer
    ref = run(copy.deepcopy(ora).double().to(DEV).train(), _to64(b, keys).to(DEV), fix)
    res = run(ours, b.clone().to(DEV), fix)
    for k in ("out_x", "out_e"):
        assert rel_err(res[k], ref[k]) < 1e-3, (k, rel_err(res[k], ref[k]))
    tgt = {k: ref[k] for k in ("grad_x", "grad_e", "grad_pe") if k in ref}
    tgt["grad_params"], tgt["state_after"] = ref["grad_params"], ref["state_after"]
    errs = (compare_eslap if eslap else compare)(res, tgt, 1e-3, f"GatedGCN layer at hubs (eslap={eslap})")
    print("layer at hubs, eslap", eslap, "max err", max(errs.values()))


def test_gine_layer_at_hub_degrees():
    """GINE+Transformer on the same batch; GINE's inner ReLU has kinks, hence the relative-L2 fallback on gradients"""
    d = 64
    b = _malnet(d, seed=20)
    torch.manual_seed(0)
    ora = OracleGPSLayer(d, "GINE", "Transformer", 4)
    ours = graphgps_b200.GPSLayer(d, "GINE", "Transformer", 4)
    ours.load_state_dict(ora.state_dict(), strict=True)
    ours = ours.to(DEV).train()
    fix = _cts(b)
    fix["config"] = dict(local="GINE")
    ref = run_layer(copy.deepcopy(ora).double().to(DEV).train(), _to64(b).to(DEV), fix)
    res = run_layer(ours, b.clone().to(DEV), fix)
    tgt = {k: ref[k] for k in ("out_x", "grad_x", "grad_e") if k in ref}
    tgt["grad_params"], tgt["state_after"] = ref["grad_params"], ref["state_after"]
    compare(res, tgt, 1e-3, "GINE layer at hubs", grad_l2_tol=5e-3)
