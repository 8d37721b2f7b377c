"""Phase timeline of the TMA-fed GEMM (gemm_tma.cu) for one shape: per-CTA globaltimer stamps + CUDA-event time.

    python tools/gemm_trace.py M N K [ta tb splitk force_bn]
slots: 0 start, 1 setup done, 2 first TMA issued, 9 last TMA issued, 3 first stage landed, 10 last stage landed,
       4 last MMA retired, 5 bias-gradient sums done, 6 epilogue done, 7 all warps done"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from graphgps_b200 import _lib  # noqa: E402

M, N, K = (int(v) for v in sys.argv[1:4])
ta, tb, splitk, fbn = (int(v) for v in (sys.argv[4:8] + ["0", "0", "1", "0"][len(sys.argv) - 4:]))
lib = _lib.load()
dev = "cuda:0"
st = torch.cuda.current_stream().cuda_stream


def planes(x):
    r, c = x.shape
    ld = (c + 7) // 8 * 8
    buf = torch.zeros(2, r, ld, dtype=torch.bfloat16, device=dev)
    _lib.check(lib.gps_to_planes(x.data_ptr(), x.stride(0), r, c, buf[0].data_ptr(), buf[1].data_ptr(), ld, st), "to_planes")
    return buf, ld


A = torch.randn((K, M) if ta else (M, K), device=dev)
B = torch.randn((K, N) if tb else (N, K), device=dev)
Ap, lda = planes(A)
Bp, ldb = planes(B)
C = torch.zeros(M, N, device=dev)
trace = torch.zeros(256 * 16, dtype=torch.int64, device=dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def run():
    _lib.check(lib.gps_gemm_planes(Ap[0].data_ptr(), Ap[1].data_ptr(), lda, ta, Bp[0].data_ptr(), Bp[1].data_ptr(), ldb, tb,
                                   C.data_ptr(), N, 0, 0, 0, M, N, K, splitk, 0, 0, st), "gemm")


lib.gps_debug_tma(fbn, 0)
for _ in range(3):
    run()
ts = []
for _ in range(10):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run()
    e1.record()
    torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1) * 1e3)
print(f"M={M} N={N} K={K} ta={ta} tb={tb} splitk={splitk} force_bn={fbn}: event time us min={min(ts):.1f} med={sorted(ts)[5]:.1f}")
lib.gps_debug_tma(fbn, trace.data_ptr())
flush.zero_()
run()
torch.cuda.synchronize()
lib.gps_debug_tma(0, 0)
t = trace.view(256, 16).cpu()
t = t[t[:, 0] > 0]
t0 = int(t[:, 0].min())
print(f"{t.shape[0]} traced CTAs; kernel span {(int(t[:, 7].max()) - t0) / 1e3:.1f} us")
print("cta  sm  start setup tma0 tmaN land0 landN mmaN accum epi  end   (us from first CTA start)")
for i in list(range(0, min(8, t.shape[0]))) + list(range(max(8, t.shape[0] - 4), t.shape[0])):
    r = t[i]
    f = lambda s: f"{(int(r[s]) - t0) / 1e3:5.1f}" if int(r[s]) else "  -  "   # noqa: E731
    print(f"{i:3d} {int(r[8]):3d}  " + " ".join(f(s) for s in (0, 1, 2, 9, 3, 10, 4, 5, 6, 7)))
d = lambda a, b: (t[:, a] - t[:, b]).float().mean().item() / 1e3   # noqa: E731
print(f"mean per CTA: setup {d(1, 0):.2f}  first-land {d(3, 1):.2f}  mainloop {d(4, 3):.2f}  drain {d(5, 4):.2f}  "
      f"epilogue {d(6, 5):.2f}  tail {d(7, 6):.2f}  total {d(7, 0):.2f} us")
