"""Bring-up probe for the wgmma GEMM: prints the error of each orientation/precision separately."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch
from test_gemm_gpu import _run
for (M, N, K) in [(128, 128, 64), (128, 64, 128), (256, 256, 304), (3624, 2128, 304)]:
    for ta, tb in [(0, 0), (0, 1), (1, 0), (1, 1)]:
        for prec in (1, 0):
            try:
                e = _run(M, N, K, ta, tb, 1, prec, 2)
                print(f"M={M} N={N} K={K} ta={ta} tb={tb} prec={'bf16' if prec else 'fp32x3'} err={e:.3e}", flush=True)
            except Exception as ex:
                print(f"M={M} N={N} K={K} ta={ta} tb={tb} prec={prec} EXC {type(ex).__name__}: {ex}", flush=True)
                sys.exit(1)
