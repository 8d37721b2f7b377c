"""Emits the wgmma wrapper specialisations of graphgps_b200/csrc/wgmma_ops.cuh (body after the declarations):

    python tools/gen_wgmma.py
"""
out = []
def ss(N, TA, TB):
    n = N // 2
    regs = ",".join(f"%{i}" for i in range(n))
    cons = ", ".join(f'"+f"(d[{i}])' for i in range(n))
    out.append(f"""template <>
__device__ __forceinline__ void wgmma_ss<{N}, {TA}, {TB}>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {{
  asm volatile(
      "{{\\n\\t.reg .pred p;\\n\\tsetp.ne.b32 p, %{n+2}, 0;\\n\\t"
      "wgmma.mma_async.sync.aligned.m64n{N}k16.f32.bf16.bf16 {{{regs}}}, %{n}, %{n+1}, p, 1, 1, {TA}, {TB};\\n\\t}}"
      : {cons}
      : "l"(da), "l"(db), "r"(scale_d));
}}""")
def rs(N, TB):
    n = N // 2
    regs = ",".join(f"%{i}" for i in range(n))
    cons = ", ".join(f'"+f"(d[{i}])' for i in range(n))
    out.append(f"""template <>
__device__ __forceinline__ void wgmma_rs<{N}, {TB}>(float* d, const uint32_t* a, uint64_t db, uint32_t scale_d) {{
  asm volatile(
      "{{\\n\\t.reg .pred p;\\n\\tsetp.ne.b32 p, %{n+5}, 0;\\n\\t"
      "wgmma.mma_async.sync.aligned.m64n{N}k16.f32.bf16.bf16 {{{regs}}}, {{%{n},%{n+1},%{n+2},%{n+3}}}, %{n+4}, p, 1, 1, {TB};\\n\\t}}"
      : {cons}
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}}""")
for N in (64, 128, 256):
    for TA in (0, 1):
        for TB in (0, 1):
            ss(N, TA, TB)
for N in (64, 128):
    rs(N, 1)
print("\n".join(out))
