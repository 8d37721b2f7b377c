// tc_ptx.cuh — inline-PTX wrappers shared by the tensor-core kernels (gemm_tc.cu, gemm_tma.cu, attention_tc.cu):
// mbarrier, bulk / tensor-map TMA, wgmma fence / commit / wait and shared-memory descriptors (the MMAs themselves are in
// wgmma_ops.cuh).  sm_90a.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

#include "wgmma_ops.cuh"

namespace gps {
namespace tc {

constexpr uint32_t kSpinLimit = 1u << 28;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0, spins = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) break;
    if (++spins > kSpinLimit) __trap();  // never hang the GPU: a protocol bug becomes an error
  }
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// tensor-map TMA (SASS: UTMALDG): one box of a rank-3 tensor {c0 innermost, c1, c2} -> shared
__device__ __forceinline__ void tma_tile_3d(uint32_t dst_smem, const void* tmap, int c0, int c1, int c2, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(dst_smem), "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tma_tile_2d(uint32_t dst_smem, const void* tmap, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(dst_smem), "l"(tmap), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// wgmma: fence before the first MMA that touches freshly written accumulator registers, group commit, and a wait that
// leaves at most N committed groups in flight (their accumulators must not be read, their shared memory not rewritten)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads/writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void reg_fence(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// wgmma shared-memory matrix descriptor, SWIZZLE_128B (cute::GMMA::GmmaDescriptor bit layout).  K-major: rows of 128 B
// (64 bf16 of K), 8-row groups sbo apart.  MN-major: 64-element MN blocks lbo apart, 8-k-row groups sbo apart.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= 1ull << 62;   // layout type SWIZZLE_128B (base offset 0: every tile is 1024-byte aligned)
  return d;
}

// fp32 x8 -> bf16 hi (and residual lo) packed as 16 bytes each
__device__ __forceinline__ void split8(const float* v, uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __nv_bfloat162 hb = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    float r0 = v[2 * i] - __low2float(hb), r1 = v[2 * i + 1] - __high2float(hb);
    __nv_bfloat162 lb = __floats2bfloat162_rn(r0, r1);
    h[i] = *reinterpret_cast<uint32_t*>(&hb);
    l[i] = *reinterpret_cast<uint32_t*>(&lb);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}

}  // namespace tc
}  // namespace gps
