// common.cuh — shared device/host helpers for libgps_b200 (sm_90a).
#pragma once

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "../../include/gps_b200.h"

namespace gps {

// ------------------------------------------------------------------------------------ errors
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);
void count_launch();  // every kernel launch of the library is counted (gps_launch_count)

#define GPS_CUDA(expr)                                                             \
  do {                                                                             \
    cudaError_t _e = (expr);                                                       \
    if (_e != cudaSuccess) return ::gps::cuda_fail(_e, #expr, __FILE__, __LINE__); \
  } while (0)

#define GPS_LAUNCH_CHECK()            \
  do {                                \
    ::gps::count_launch();            \
    GPS_CUDA(cudaGetLastError());     \
  } while (0)

#define GPS_REQUIRE(cond, code, ...)   \
  do {                                 \
    if (!(cond)) {                     \
      ::gps::set_error(__VA_ARGS__);   \
      return (code);                   \
    }                                  \
  } while (0)

#define GPS_TRY(expr)            \
  do {                           \
    int _rc = (expr);            \
    if (_rc != GPS_OK) return _rc; \
  } while (0)

constexpr int kNumSMs = 132;  // H100 SXM
constexpr float kBnEps = 1e-5f;
constexpr float kBnMomentum = 0.1f;

static inline int64_t round_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }
static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Bump allocator over a caller-owned buffer; with base == nullptr it only counts bytes.
struct Arena {
  char* base;
  int64_t cap;
  int64_t used = 0;
  bool overflow = false;
  Arena(void* b, int64_t c) : base(reinterpret_cast<char*>(b)), cap(c) {}
  template <typename T>
  T* alloc(int64_t n) {
    int64_t bytes = round_up(n * (int64_t)sizeof(T), 256);
    int64_t off = used;
    used += bytes;
    if (base == nullptr) return nullptr;
    if (used > cap) {
      overflow = true;
      return nullptr;
    }
    return reinterpret_cast<T*>(base + off);
  }
};

// bf16 "planes" of an fp32 tensor: plain row-major bf16 matrices holding hi = bf16(v) and lo = bf16(v - hi)
// (lo == nullptr in precision="bf16" mode).  Written once by the producing kernel, read by the TMA-fed GEMM
// (gemm_tma.cu) in any operand orientation.  ld is in elements (multiple of 8: 16-byte row pitch for TMA).
struct Planes {
  __nv_bfloat16* hi = nullptr;
  __nv_bfloat16* lo = nullptr;
  int64_t ld = 0;
  Planes cols(int64_t c0) const { Planes q = *this; if (q.hi) q.hi += c0; if (q.lo) q.lo += c0; return q; }
  Planes rows(int64_t r0) const { Planes q = *this; if (q.hi) q.hi += r0 * ld; if (q.lo) q.lo += r0 * ld; return q; }
};

// ------------------------------------------------------------------------------------ device
#ifdef __CUDACC__

// hi/lo split of 4 consecutive values of row r starting at column c (c % 4 == 0): one 8-byte store per plane
__device__ __forceinline__ void planes_store4(const Planes& p, int64_t r, int64_t c, float4 v) {
  __nv_bfloat162 h0 = __floats2bfloat162_rn(v.x, v.y), h1 = __floats2bfloat162_rn(v.z, v.w);
  uint2 hw = make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
  *reinterpret_cast<uint2*>(p.hi + r * p.ld + c) = hw;
  if (p.lo) {
    __nv_bfloat162 l0 = __floats2bfloat162_rn(v.x - __low2float(h0), v.y - __high2float(h0));
    __nv_bfloat162 l1 = __floats2bfloat162_rn(v.z - __low2float(h1), v.w - __high2float(h1));
    *reinterpret_cast<uint2*>(p.lo + r * p.ld + c) = make_uint2(*reinterpret_cast<uint32_t*>(&l0), *reinterpret_cast<uint32_t*>(&l1));
  }
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float4 f4zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ float4 f4add(float4 a, float4 b) {
  return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}
__device__ __forceinline__ float4 f4mul(float4 a, float4 b) {
  return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w);
}
__device__ __forceinline__ float4 f4fma(float4 a, float4 b, float4 c) {
  return make_float4(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y), fmaf(a.z, b.z, c.z), fmaf(a.w, b.w, c.w));
}
__device__ __forceinline__ float4 f4scale(float4 a, float s) {
  return make_float4(a.x * s, a.y * s, a.z * s, a.w * s);
}

__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + __expf(-v)); }

// activation and derivative (act: GPS_ACT_RELU / GPS_ACT_GELU; gelu = exact erf form of nn.GELU())
template <int ACT>
__device__ __forceinline__ float act_fwd(float v) {
  if (ACT == GPS_ACT_RELU) return v > 0.f ? v : 0.f;
  return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
}
template <int ACT>
__device__ __forceinline__ float act_bwd(float v) {  // d act / d v at pre-activation v
  if (ACT == GPS_ACT_RELU) return v > 0.f ? 1.f : 0.f;
  float cdf = 0.5f * (1.f + erff(v * 0.70710678118654752f));
  float pdf = 0.3989422804014327f * __expf(-0.5f * v * v);
  return cdf + v * pdf;
}
__device__ __forceinline__ float act_fwd_rt(int act, float v) {
  return act == GPS_ACT_RELU ? act_fwd<GPS_ACT_RELU>(v) : act_fwd<GPS_ACT_GELU>(v);
}
__device__ __forceinline__ float act_bwd_rt(int act, float v) {
  return act == GPS_ACT_RELU ? act_bwd<GPS_ACT_RELU>(v) : act_bwd<GPS_ACT_GELU>(v);
}

// ---- Philox4x32-10 counter RNG: one call yields 4 x 32 random bits for 4 consecutive columns.
struct Philox4 {
  uint32_t v[4];
};
__device__ __forceinline__ Philox4 philox4x32(uint64_t seed, uint64_t ctr_hi, uint64_t ctr_lo) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
  uint32_t c0 = (uint32_t)ctr_lo, c1 = (uint32_t)(ctr_lo >> 32), c2 = (uint32_t)ctr_hi,
           c3 = (uint32_t)(ctr_hi >> 32);
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
    uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += W0; k1 += W1;
  }
  Philox4 o;
  o.v[0] = c0; o.v[1] = c1; o.v[2] = c2; o.v[3] = c3;
  return o;
}
// Dropout keep-scale for the 4 consecutive elements starting at flat index `idx4*4` of dropout
// site `site`.  keep iff u >= p where u = bits * 2^-32.  Returns 0 or 1/(1-p) per element.
__device__ __forceinline__ float4 dropout_scale4(float p, uint64_t seed, uint64_t offset, int site,
                                                 uint64_t idx4) {
  Philox4 r = philox4x32(seed, offset + (uint64_t)site, idx4);
  uint32_t thr = (uint32_t)fminf(p * 4294967296.f, 4294967295.f);
  float s = 1.f / (1.f - p);
  return make_float4(r.v[0] >= thr ? s : 0.f, r.v[1] >= thr ? s : 0.f, r.v[2] >= thr ? s : 0.f,
                     r.v[3] >= thr ? s : 0.f);
}

// dropout sites (Philox stream ids); attention uses GPS_SITE_ATTN_P + head
enum {
  GPS_SITE_GCN_X = 1, GPS_SITE_GCN_E = 2, GPS_SITE_LOCAL = 3, GPS_SITE_ATTN_OUT = 4,
  GPS_SITE_FF1 = 5, GPS_SITE_FF2 = 6, GPS_SITE_PERF_OUT = 7,
  GPS_SITE_BB_SELF_OUT = 8,   // BigBird attention.output.dropout, on dense(ctx) before LayerNorm 1
  GPS_SITE_BB_OUTPUT = 9,     // BigBird output.dropout, on dense(u) before LayerNorm 2
  GPS_SITE_GR_ATTN = 10,      // Graphormer layer: dropout on the attention output projection
  GPS_SITE_GR_MLP = 11,       // Graphormer layer: mlp.3, on GELU(mlp.1(.))
  GPS_SITE_GR_OUT = 12,       // Graphormer layer: mlp.5, on mlp.4(.)
  GPS_SITE_SAN_ATTN = 13,     // SAN layer: dropout on the concatenated attention heads, before O_h
  GPS_SITE_SAN_FFN = 14,      // SAN layer: dropout on relu(FFN_h_layer1(.))
  GPS_SITE_CG_X = 15,         // CustomGNN layers (custom_gnn.cu): GatedGCN's node output, GINE's output
  GPS_SITE_ATTN_P = 16,       // + head: the attention probabilities
  // CustomGNN GatedGCN's edge output: its own id, the last of the 4096 a call's Philox counter window holds (the layers
  // advance the dropout offset by 4096 per call), far above any attention head's 16 + head
  GPS_SITE_CG_E = 4095
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void atomic_add_f64(double* p, double v) { atomicAdd(p, v); }

#endif  // __CUDACC__

}  // namespace gps
