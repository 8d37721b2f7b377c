"""Per-product times of the TMA-fed GEMM at the GPSLayer shapes of one workload (CUDA events, warm L2).

    python tools/gemm_products.py [workload] [precision fp32|bf16] [force_bn | sN ...]

Each product runs as the layer issues it (forward Linears also write the operand planes of their output) for 200
back-to-back launches; the time is the mean per launch.  A time marked * belongs to a result that is not bitwise equal
to the one of the first column.  With force_bn values the tile width is forced (0 = the launch policy's choice); a
width the kernel does not instantiate for that operand layout is reported as such.  sN forces N K-splits on the
products that run their epilogue (split-K 1 below; the policy's width), s0 the policy's split."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import graphgps_b200  # noqa: E402
from graphgps_b200 import _lib  # noqa: E402

wl = sys.argv[1] if len(sys.argv) > 1 else "pcqm4m-small"
prec = {"fp32": 0, "bf16": 1}[sys.argv[2] if len(sys.argv) > 2 else "fp32"]
# columns: (label, forced width or 0 = the policy's, forced K-splits or 0 = the policy's)
COLS = [(f, 0, int(f[1:])) if f.startswith("s") else ("policy" if f == "0" else "bn=" + f, int(f), 0)
        for f in sys.argv[3:] or ["0"]]
batch = graphgps_b200.make_batch(wl, seed=0)
Nn, E, d = batch.num_nodes, batch.num_edges, graphgps_b200.SHAPES[wl].dim
lib = _lib.load()
dev = "cuda:0"
st = torch.cuda.current_stream().cuda_stream

# (name, M, N, K, ta, tb, splitk, plane output)
PRODUCTS = [
    ("edge projection fwd", E, d, d, 0, 0, 1, True),
    ("g_edge_attr", E, d, d, 0, 1, 1, False),
    ("node projection Ax..Ex", Nn, 4 * d, d, 0, 0, 1, True),
    ("QKV projection", Nn, 3 * d, d, 0, 0, 1, True),
    ("FF1 fwd", Nn, 2 * d, d, 0, 0, 1, True),
    ("FF2 dgrad", Nn, 2 * d, d, 0, 1, 1, False),
    ("FF2 fwd", Nn, d, 2 * d, 0, 0, 1, True),
    ("FF1 dgrad", Nn, d, 2 * d, 0, 1, 1, False),
    ("out-proj fwd", Nn, d, d, 0, 0, 1, True),
    ("out-proj dgrad", Nn, d, d, 0, 1, 1, False),
    ("g_x", Nn, d, 7 * d, 0, 1, 1, False),
    ("edge wgrad", d, d, E, 1, 1, 8, False),
    ("node wgrad d x d", d, d, Nn, 1, 1, 8, False),
    ("FF1 wgrad", 2 * d, d, Nn, 1, 1, 8, False),
    ("FF2 wgrad", d, 2 * d, Nn, 1, 1, 8, False),
    ("QKV wgrad", 3 * d, d, Nn, 1, 1, 8, False),
    ("dWcat", 7 * d, d, Nn, 1, 1, 8, False),
]


def planes(r, c):
    ld = (c + 7) // 8 * 8
    x = torch.randn(r, c, device=dev)
    buf = torch.zeros(2, r, ld, dtype=torch.bfloat16, device=dev)
    _lib.check(lib.gps_to_planes(x.data_ptr(), x.stride(0), r, c, buf[0].data_ptr(), buf[1].data_ptr(), ld, st), "planes")
    return buf, ld


def lo(buf):
    return buf[1].data_ptr() if prec == 0 else 0


torch.manual_seed(0)
print(f"{wl} {'fp32-grade' if prec == 0 else 'bf16'}: N={Nn} E={E} d={d}; mean us per launch over 200 launches")
print(f"{'product':24s} {'M x N x K':>16s} " + " ".join(f"{label:>8s}" for label, _, _ in COLS))
for name, M, N, K, ta, tb, sk, pout in PRODUCTS:
    Ap, lda = planes(K, M) if ta else planes(M, K)
    db = torch.zeros(M, device=dev) if ta and prec == 0 else None
    Bp, ldb = planes(K, N) if tb else planes(N, K)
    C = torch.zeros(M, N, device=dev)
    Cp = torch.zeros(2, M, (N + 7) // 8 * 8, dtype=torch.bfloat16, device=dev) if pout else None

    def run():
        rc = lib.gps_gemm_planes(Ap[0].data_ptr(), lo(Ap), lda, ta, Bp[0].data_ptr(), lo(Bp), ldb, tb, C.data_ptr(), N,
                                 Cp[0].data_ptr() if pout else 0, lo(Cp) if pout else 0, Cp.shape[2] if pout else 0,
                                 M, N, K, sk, prec, db.data_ptr() if db is not None else 0, st)
        return rc

    cells = []
    ref = None
    for _, fbn, fsplits in COLS:
        lib.gps_debug_tma(fbn, 0)
        lib.gps_debug_tma_splits(fsplits)
        C.zero_()
        if run() != 0:
            cells.append(f"{'n/a':>8s}")
            continue
        same = ""
        if ref is None:
            ref = C.clone()
        elif not torch.equal(C, ref):
            same = "*"   # not bitwise equal to the first column's result
        for _ in range(10):
            run()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(200):
            run()
        e1.record()
        torch.cuda.synchronize()
        cells.append(f"{e0.elapsed_time(e1) * 1e3 / 200:7.1f}{same or ' '}")
    lib.gps_debug_tma(0, 0)
    lib.gps_debug_tma_splits(0)
    print(f"{name:24s} {f'{M}x{N}x{K}':>16s} " + " ".join(cells), flush=True)
