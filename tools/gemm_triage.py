"""Perf triage of the wgmma GEMM: times the kernel with parts switched off (gps_debug_set)."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from graphgps_b200 import _lib
lib = _lib.load()
lib.gps_debug_set.argtypes = [ctypes.c_int]
dev = "cuda:0"
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

def t(M, N, K, ta, tb, splitk, prec, dbg, flush_l2=True, reps=10):
    A = torch.randn((K, M) if ta else (M, K), device=dev)
    B = torch.randn((K, N) if tb else (N, K), device=dev)
    C = torch.zeros(M, N, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    lib.gps_debug_set(dbg)
    f = lambda: lib.gps_gemm(A.data_ptr(), A.shape[1], ta, B.data_ptr(), B.shape[1], tb, C.data_ptr(), N, M, N, K, splitk, prec, 2, st)
    for _ in range(3): f()
    tot = 0
    for _ in range(reps):
        if flush_l2: flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(400000)   # keep the GPU busy while the host enqueues: events then bracket only the kernel
        e0.record(); f(); e1.record(); torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    lib.gps_debug_set(0)
    return tot / reps * 1e3

lib.gps_debug_trace.argtypes = [ctypes.c_void_p]
for (M, N, K, prec) in [(3620, 2128, 304, 0), (3620, 304, 2128, 1)]:
    tr = torch.zeros(8, 64, dtype=torch.int64, device=dev)
    lib.gps_debug_trace(tr.data_ptr())
    us = t(M, N, K, 0, 0, 1, prec, 0, reps=1)
    lib.gps_debug_trace(None)
    tr = tr.cpu()
    base = int(tr[tr > 0].min())
    print(f"M={M} N={N} K={K} prec={prec} {us:.1f} us; CTA0 clock64 deltas: it | mma_full mma_commit | p_top p_empty p_data p_arrive | epi_start epi_end (by tile)")
    for i in range(0, 24):
        f = lambda r: int(tr[r, i]) - base if tr[r, i] > 0 else -1
        print(i, "|", f(0), f(1), "|", f(4), f(2), f(5), f(3), "|", f(6), f(7))
