"""Tile-width / split-K sweep of the wgmma GEMM at the layer's shapes (forces BN through gps_debug_set)."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from graphgps_b200 import _lib
lib = _lib.load()
lib.gps_debug_set.argtypes = [ctypes.c_int]
dev = "cuda:0"
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

def t(M, N, K, ta, tb, splitk, bn, reps=6):
    A = torch.randn((K, M) if ta else (M, K), device=dev)
    B = torch.randn((K, N) if tb else (N, K), device=dev)
    C = torch.zeros(M, N, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    lib.gps_debug_set(bn << 8)
    f = lambda: lib.gps_gemm(A.data_ptr(), A.shape[1], ta, B.data_ptr(), B.shape[1], tb, C.data_ptr(), N, M, N, K, splitk, 0, 2, st)
    if f() != 0:
        lib.gps_debug_set(0); return float("nan")
    f()
    tot = 0
    for _ in range(reps):
        torch.cuda._sleep(200000)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); f(); e1.record(); torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    lib.gps_debug_set(0)
    return tot / reps * 1e3

shapes = [("fwd Y1", 3624, 2128, 304, 0, 0), ("fwd ABDE", 3624, 1216, 304, 0, 0), ("fwd QKV", 3624, 912, 304, 0, 0),
          ("fwd edge", 7456, 304, 304, 0, 0), ("fwd FFN1", 3624, 608, 304, 0, 0), ("fwd FFN2", 3624, 304, 608, 0, 0),
          ("dgrad hid", 3624, 608, 304, 0, 1), ("dgrad s", 3624, 304, 608, 0, 1), ("dgrad O", 3624, 304, 304, 0, 1),
          ("dgrad e", 7456, 304, 304, 0, 1), ("dgrad x", 3624, 304, 2128, 0, 1),
          ("wgrad W2", 304, 608, 3624, 1, 1), ("wgrad W1", 608, 304, 3624, 1, 1), ("wgrad Wo", 304, 304, 3624, 1, 1),
          ("wgrad C", 304, 304, 7456, 1, 1), ("wgrad Wcat", 2128, 304, 3624, 1, 1)]
for name, M, N, K, ta, tb in shapes:
    sks = [1] if not ta else [4, 8, 14, 28]
    if name == "dgrad x":
        sks = [1, 2, 4]
    for sk in sks:
        row = []
        for bn in (0, 48, 64, 80, 112, 128, 160, 208, 256):
            if bn > max(64, N):
                continue
            row.append(f"{bn or 'auto'}:{t(M, N, K, ta, tb, sk, bn):.1f}")
        print(f"{name:11s} M={M} N={N} K={K} sk={sk}: " + "  ".join(row), flush=True)
