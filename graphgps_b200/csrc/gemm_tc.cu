// gemm_tc.cu — wgmma (Hopper warpgroup MMA) dense product for every Linear of the GPS layer and
// their data/weight gradients, with the layer's fused epilogues.
//
//   C[M,N] (+)= epi( Aop[M,K] * Bop[K,N] ),  fp32 in HBM, bf16 operands on the tensor cores,
//   fp32 accumulation in registers.  precision FP32: split-bf16 x3 (hi*hi + hi*lo + lo*hi, ~2^-16
//   relative), precision BF16: a single bf16 pass.
//
// One 128 x BN output tile per CTA (BN = 64 or 128, the wgmma instruction shape):
//   * warps 0-7 stage operands: coalesced 128-bit global loads of the fp32 tiles -> bf16 hi/lo split in
//     registers -> 16-byte st.shared into the canonical SWIZZLE_128B layout (K-major when the
//     reduction dim is contiguous in HBM, MN-major when it is the row dim, e.g. weight gradients
//     dW = G^T X) -> fence.proxy.async -> one mbarrier arrive per warp.  All per-chunk addresses are
//     (value for chunk 0) + q * constant, computed once per CTA.  No transposes, no separate conversion
//     pass; the fp32->bf16 split costs no extra HBM bytes.
//   * warps 8-15: two consumer warpgroups, each issuing wgmma m64 x BN x k16 for its 64 rows of the tile per
//     16-wide K step, one commit group per k-block; a stage is released once its group has retired.  After the
//     last k-block the accumulators go to a shared staging tile (the operand stages are free by then).
//   * epilogue (warps 0-7): staging tile -> bias / activation / act' mask / dropout /
//     residuals / 128-bit stores; BatchNorm column sums by a warp butterfly reduce-scatter + double
//     atomics; split-K partials by fp32 atomics; bias-gradient column sums from the staged A tile.
// Smem stages form an mbarrier ring (full: one arrival per producer warp; empty: one arrival per consumer warp).
// Per-thread mbarrier arrivals (256 per stage) serialise on the barrier unit, hence per-warp arrivals; per-chunk
// integer divisions make the producers issue-bound, hence the precomputed addressing.
#include <cuda_bf16.h>

#include <algorithm>

#include "gemm.cuh"
#include "tc_ptx.cuh"

namespace gps {

namespace {

constexpr int BM = 128;          // two wgmma M = 64 warpgroups
constexpr int BK = 64;           // k-block: one 128-byte swizzle row of bf16
constexpr int kProducerWarps = 8;           // operand staging + epilogue
constexpr int kProducerThreads = kProducerWarps * 32;
constexpr int kConsumerWarps = 8;           // two MMA warpgroups
constexpr int kThreads = (kProducerWarps + kConsumerWarps) * 32;
constexpr int kATileBytes = BM * BK * 2;       // 16 KB
constexpr int kBBlockBytes = 64 * BK * 2;      // 8 KB per 64 columns of B
using namespace tc;   // PTX wrappers: tc_ptx.cuh

// Byte offset of chunk `c` inside an operand tile stored in the canonical SWIZZLE_128B layout.
//  K-major : rows of 128 B (64 bf16 of K), 8-row groups of 1024 B.
//  MN-major: 64-column blocks of kBBlockBytes; inside a block 8-k-row groups of 1024 B, each k-row 128 B.
template <bool MN>
__device__ __forceinline__ uint32_t chunk_offset(int c, int tile_rows) {
  if (!MN) {
    const int r = c >> 3, ck = c & 7;
    return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((ck ^ (r & 7)) << 4));
  }
  const int rc = tile_rows >> 3;
  const int k = c / rc, cm = c % rc;
  const int blk = cm >> 3, cc = cm & 7;
  return (uint32_t)(blk * kBBlockBytes + (k >> 3) * 1024 + (k & 7) * 128 + ((cc ^ (k & 7)) << 4));
}

struct TcArgs {
  GemmParams p;
  int BN;          // tile width (64 or 128)
  int nb_blocks;   // BN / 64
  int stages;
  int kb_per_split;
};

// BN_T = tile width; a producer thread stages BN_T / 32 B chunks per k-block.
template <bool A_MN, bool B_MN, bool SPLIT, int BN_T>
__global__ void __launch_bounds__(kThreads, 1) k_gemm_tc(const TcArgs a) {
  constexpr int NBC = BN_T / 32;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const GemmParams& p = a.p;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int b_tile_bytes = a.nb_blocks * kBBlockBytes;
  const int plane = SPLIT ? 2 : 1;
  const int stage_bytes = plane * (kATileBytes + b_tile_bytes);
  const int S = a.stages;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)S * stage_bytes);
  // bars[0..S) full, bars[S..2S) empty
  float* red = reinterpret_cast<float*>(bars + 2 * S + 2);  // 16 x 16 x 8 floats (bias-gradient partials)
  float* stage = reinterpret_cast<float*>(smem);            // epilogue staging tile [128][BN + 4], over the stages
  const int sld = a.BN + 4;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * a.BN;
  const int nkb_total = (p.K + BK - 1) / BK;
  const int kb_begin = blockIdx.z * a.kb_per_split;
  const int kb_end = min(nkb_total, kb_begin + a.kb_per_split);
  const int nkb = kb_end - kb_begin;

  if (tid == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(smem_u32(&bars[s]), kProducerWarps);
      mbar_init(smem_u32(&bars[S + s]), kConsumerWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kProducerWarps) {
    // =========================================================== MMA warpgroups
    // warpgroup wg owns accumulator rows [64 wg, 64 wg + 64): its A operand starts 8 KB into every A plane
    // (eight 1 KB K-major row groups, or the second 64-row MN-major block)
    const int wg = (warp - kProducerWarps) >> 2;
    float acc[BN_T / 2];
#pragma unroll
    for (int e = 0; e < BN_T / 2; ++e) acc[e] = 0.f;
    constexpr uint32_t a_lbo = A_MN ? kBBlockBytes : 16, b_lbo = B_MN ? kBBlockBytes : 16;
    constexpr uint32_t a_kstep = A_MN ? 2048 : 32, b_kstep = B_MN ? 2048 : 32;
    for (int i = 0; i < nkb; ++i) {
      const int s = i % S;
      if (lane == 0) mbar_wait(smem_u32(&bars[s]), (uint32_t)(i / S) & 1u);
      __syncwarp();
      const uint32_t sa_hi = smem_u32(smem + (size_t)s * stage_bytes) + (uint32_t)wg * 8192u;
      const uint32_t sb_hi = smem_u32(smem + (size_t)s * stage_bytes) + plane * kATileBytes;
      const uint32_t sa_lo = sa_hi + kATileBytes;
      const uint32_t sb_lo = sb_hi + b_tile_bytes;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk) {
        const uint64_t da_hi = make_desc(sa_hi + kk * a_kstep, a_lbo, 1024);
        const uint64_t db_hi = make_desc(sb_hi + kk * b_kstep, b_lbo, 1024);
        if (SPLIT) {
          const uint64_t da_lo = make_desc(sa_lo + kk * a_kstep, a_lbo, 1024);
          const uint64_t db_lo = make_desc(sb_lo + kk * b_kstep, b_lbo, 1024);
          wgmma_ss<BN_T, A_MN, B_MN>(acc, da_lo, db_hi, 1u);
          wgmma_ss<BN_T, A_MN, B_MN>(acc, da_hi, db_lo, 1u);
        }
        wgmma_ss<BN_T, A_MN, B_MN>(acc, da_hi, db_hi, 1u);
      }
      wgmma_commit();
      // at most one group in flight: the previous k-block's MMAs have retired, so its stage goes back to the producers
      wgmma_wait<1>();
      reg_fence<BN_T / 2>(acc);
      __syncwarp();
      if (i > 0 && lane == 0) mbar_arrive(smem_u32(&bars[S + (i - 1) % S]));
    }
    wgmma_wait<0>();
    reg_fence<BN_T / 2>(acc);
    asm volatile("bar.sync 2, 256;" ::: "memory");   // both warpgroups are done with the operand stages
    // wgmma fragment: lane of warp w holds rows 16 (w & 3) + lane / 4 (+ 8), columns 8 j + 2 (lane % 4) (+ 1)
    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int c = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN_T / 8; ++j) {
      *reinterpret_cast<float2*>(stage + r * sld + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(stage + (r + 8) * sld + 8 * j + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
    asm volatile("barrier.sync 3, %0;" ::"n"(kThreads) : "memory");   // staging tile complete -> epilogue
  } else {
    // =========================================================== operand producers
    // chunk c = tid + 256 q: every per-q quantity is (value at q = 0) + q * constant
    //   K-major : row (tid>>3) + 32 q, k-chunk (tid&7)            -> global += 32 rows,   smem += 4096 B
    //   MN-major: k-row (tid>>rcs) + (256>>rcs) q, row chunk tid & (rc-1) -> global += (256>>rcs) k-rows
    const int b_rows = a.nb_blocks * 64;
    const int nb_chunks = a.nb_blocks * 2;  // per thread: (nb_blocks*64 rows * 8 chunks) / 256
    const int a_rcs = 4;
    const int b_rcs = a.nb_blocks == 1 ? 3 : a.nb_blocks == 2 ? 4 : 5;   // log2(b_rows / 8); nb_blocks in {1,2,4}
    const int k_end = min(p.K, kb_end * BK);
    const int64_t a_kstride = A_MN ? (int64_t)BK * p.lda : BK;   // floats per k-block
    const int64_t b_kstride = B_MN ? (int64_t)BK * p.ldb : BK;
    const int a_row0 = A_MN ? m0 + (tid & 15) * 8 : m0 + (tid >> 3);
    const int a_k0 = A_MN ? (tid >> a_rcs) : (tid & 7) * 8;
    const float* a_g0 = A_MN ? p.A + ((int64_t)kb_begin * BK + a_k0) * p.lda + a_row0
                             : p.A + (int64_t)a_row0 * p.lda + (int64_t)kb_begin * BK + a_k0;
    const int64_t a_gq = A_MN ? (int64_t)(kProducerThreads >> a_rcs) * p.lda : (int64_t)32 * p.lda;
    const uint32_t a_s0 = chunk_offset<A_MN>(tid, BM);
    const uint32_t a_sq = A_MN ? (uint32_t)((kProducerThreads >> a_rcs) / 8) * 1024u : 4096u;
    const int b_row0 = B_MN ? n0 + (tid & ((1 << b_rcs) - 1)) * 8 : n0 + (tid >> 3);
    const int b_k0 = B_MN ? (tid >> b_rcs) : (tid & 7) * 8;
    const float* b_g0 = B_MN ? p.B + ((int64_t)kb_begin * BK + b_k0) * p.ldb + b_row0
                             : p.B + (int64_t)b_row0 * p.ldb + (int64_t)kb_begin * BK + b_k0;
    const int64_t b_gq = B_MN ? (int64_t)(kProducerThreads >> b_rcs) * p.ldb : (int64_t)32 * p.ldb;
    const uint32_t b_s0 = chunk_offset<B_MN>(tid, b_rows);
    const uint32_t b_sq = B_MN ? (uint32_t)((kProducerThreads >> b_rcs) / 8) * 1024u : 4096u;
    float csum[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) csum[e] = 0.f;
    const bool do_colsum = A_MN && p.colsum_a != nullptr && blockIdx.x == 0;

    for (int i = 0; i < nkb; ++i) {
      const int s = i % S;
      const uint32_t ph = (uint32_t)(i / S) & 1u;
      const int krem = k_end - (kb_begin + i) * BK;     // valid k extent of this k-block (<= 64 on the tail)
      float4 va[4][2], vb[NBC][2];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const bool ok = A_MN ? (a_row0 < p.M && a_k0 + q * (kProducerThreads >> a_rcs) < krem)
                             : (a_row0 + 32 * q < p.M && a_k0 < krem);
        const float* src = a_g0 + (int64_t)i * a_kstride + q * a_gq;
        va[q][0] = ok ? ld4(src) : f4zero();
        va[q][1] = ok ? ld4(src + 4) : f4zero();
      }
#pragma unroll
      for (int q = 0; q < NBC; ++q) {
        const bool ok = q < nb_chunks && (B_MN ? (b_row0 < p.N && b_k0 + q * (kProducerThreads >> b_rcs) < krem)
                                               : (b_row0 + 32 * q < p.N && b_k0 < krem));
        const float* src = b_g0 + (int64_t)i * b_kstride + q * b_gq;
        vb[q][0] = ok ? ld4(src) : f4zero();
        vb[q][1] = ok ? ld4(src + 4) : f4zero();
      }
      if (do_colsum) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          csum[0] += va[q][0].x; csum[1] += va[q][0].y; csum[2] += va[q][0].z; csum[3] += va[q][0].w;
          csum[4] += va[q][1].x; csum[5] += va[q][1].y; csum[6] += va[q][1].z; csum[7] += va[q][1].w;
        }
      }
      // one lane per warp polls / arrives: per-thread mbarrier traffic serialises on the barrier unit
      if (lane == 0) mbar_wait(smem_u32(&bars[S + s]), ph ^ 1u);   // slot free (first pass returns at once)
      __syncwarp();
      uint8_t* st = smem + (size_t)s * stage_bytes;
      uint8_t* sa_hi = st;
      uint8_t* sa_lo = st + kATileBytes;
      uint8_t* sb_hi = st + plane * kATileBytes;
      uint8_t* sb_lo = sb_hi + b_tile_bytes;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        uint4 hi, lo;
        split8(reinterpret_cast<const float*>(va[q]), hi, lo);
        *reinterpret_cast<uint4*>(sa_hi + a_s0 + q * a_sq) = hi;
        if (SPLIT) *reinterpret_cast<uint4*>(sa_lo + a_s0 + q * a_sq) = lo;
      }
#pragma unroll
      for (int q = 0; q < NBC; ++q)
        if (q < nb_chunks) {
          uint4 hi, lo;
          split8(reinterpret_cast<const float*>(vb[q]), hi, lo);
          *reinterpret_cast<uint4*>(sb_hi + b_s0 + q * b_sq) = hi;
          if (SPLIT) *reinterpret_cast<uint4*>(sb_lo + b_s0 + q * b_sq) = lo;
        }
      fence_proxy_async();          // generic-proxy smem writes -> visible to the tensor core (async proxy)
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&bars[s]));
    }

    // bias gradient: thread t always owns MN chunk (t % 16) of A^T -> reduce the 16 owners in smem
    if (do_colsum) {
      const int cm = tid & 15, owner = tid >> 4;
#pragma unroll
      for (int e = 0; e < 8; ++e) red[(owner * 16 + cm) * 8 + e] = csum[e];
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (do_colsum && tid < 128) {
      const int cm = tid >> 3, e = tid & 7;
      float tot = 0.f;
#pragma unroll
      for (int o = 0; o < 16; ++o) tot += red[(o * 16 + cm) * 8 + e];
      const int gm = m0 + cm * 8 + e;
      if (gm < p.M) atomicAdd(&p.colsum_a[gm], tot);
    }

    // =========================================================== epilogue
    asm volatile("barrier.sync 3, %0;" ::"n"(kThreads) : "memory");
    const int q = warp & 3, half = warp >> 2;
    const int row = m0 + q * 32 + lane;
    const bool row_ok = row < p.M;
    const int nchunks = a.BN >> 4;
    for (int c = half; c < nchunks; c += 2) {
      const int gn = n0 + c * 16;
      if (gn >= p.N) break;
      float v[16];
#pragma unroll
      for (int e = 0; e < 16; e += 4) {
        const float4 t = *reinterpret_cast<const float4*>(stage + (q * 32 + lane) * sld + c * 16 + e);
        v[e] = t.x; v[e + 1] = t.y; v[e + 2] = t.z; v[e + 3] = t.w;
      }
        if (p.splitk > 1) {
          if (row_ok) {
            float* dst = p.C + (int64_t)row * p.ldc + gn;
#pragma unroll
            for (int e = 0; e < 16; e += 4) {  // N % 4 == 0: whole 16-byte groups; red.global.add.v4.f32
              if (gn + e >= p.N) continue;
              float4 w4 = make_float4(v[e], v[e + 1], v[e + 2], v[e + 3]);
              if (blockIdx.z == 0) {           // the first split also carries the residual terms
                if (p.R1) w4 = f4add(w4, ld4(p.R1 + (int64_t)row * p.ldr1 + gn + e));
                if (p.R2) w4 = f4add(w4, ld4(p.R2 + (int64_t)row * p.ldr2 + gn + e));
              }
              atomicAdd(reinterpret_cast<float4*>(dst + e), w4);
            }
          }
          continue;
        }
#pragma unroll
        for (int g4 = 0; g4 < 4; ++g4) {
          const int col = gn + g4 * 4;
          const bool ok = row_ok && col < p.N;
          float* w = v + g4 * 4;
          if (p.bias && col < p.N) {
            float4 bb = ld4(p.bias + col);
            w[0] += bb.x; w[1] += bb.y; w[2] += bb.z; w[3] += bb.w;
          }
          if (ok && p.C_pre) st4(p.C_pre + (int64_t)row * p.ldpre + col, make_float4(w[0], w[1], w[2], w[3]));
          if (p.act >= 0) {
#pragma unroll
            for (int e = 0; e < 4; ++e) w[e] = act_fwd_rt(p.act, w[e]);
          }
          if (ok && p.mask_src) {
            float4 ms = ld4(p.mask_src + (int64_t)row * p.ldmask + col);
            float mv[4] = {ms.x, ms.y, ms.z, ms.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) w[e] *= p.mask_is_post ? (mv[e] > 0.f ? 1.f : 0.f) : act_bwd_rt(p.mask_act, mv[e]);
          }
          if (ok && p.p_drop2 > 0.f) {
            float4 sc = dropout_scale4(p.p_drop2, p.seed, p.offset + (p.offset_dev ? *p.offset_dev : 0ull), p.site2,
                                     ((uint64_t)row * (uint64_t)p.N + col) >> 2);
            w[0] *= sc.x; w[1] *= sc.y; w[2] *= sc.z; w[3] *= sc.w;
          }
          if (ok && p.p_drop > 0.f) {
            float4 sc = dropout_scale4(p.p_drop, p.seed, p.offset + (p.offset_dev ? *p.offset_dev : 0ull), p.site,
                                     ((uint64_t)row * (uint64_t)p.N + col) >> 2);
            w[0] *= sc.x; w[1] *= sc.y; w[2] *= sc.z; w[3] *= sc.w;
          }
          if (ok && p.R1) {
            float4 r = ld4(p.R1 + (int64_t)row * p.ldr1 + col);
            w[0] += r.x; w[1] += r.y; w[2] += r.z; w[3] += r.w;
          }
          if (ok && p.R2) {
            float4 r = ld4(p.R2 + (int64_t)row * p.ldr2 + col);
            w[0] += r.x; w[1] += r.y; w[2] += r.z; w[3] += r.w;
          }
          if (ok) st4(p.C + (int64_t)row * p.ldc + col, make_float4(w[0], w[1], w[2], w[3]));
          if (!ok) { w[0] = w[1] = w[2] = w[3] = 0.f; }
        }
        if (p.stats) {
          // column sums over the warp's 32 rows: butterfly reduce-scatter, 16 columns x {sum, sumsq}
          float s1[16], s2[16];
#pragma unroll
          for (int e = 0; e < 16; ++e) { s1[e] = v[e]; s2[e] = v[e] * v[e]; }
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const bool up = (lane & 16) != 0;
            float send1 = up ? s1[e] : s1[e + 8], send2 = up ? s2[e] : s2[e + 8];
            float keep1 = up ? s1[e + 8] : s1[e], keep2 = up ? s2[e + 8] : s2[e];
            s1[e] = keep1 + __shfl_xor_sync(0xffffffffu, send1, 16);
            s2[e] = keep2 + __shfl_xor_sync(0xffffffffu, send2, 16);
          }
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const bool up = (lane & 8) != 0;
            float send1 = up ? s1[e] : s1[e + 4], send2 = up ? s2[e] : s2[e + 4];
            float keep1 = up ? s1[e + 4] : s1[e], keep2 = up ? s2[e + 4] : s2[e];
            s1[e] = keep1 + __shfl_xor_sync(0xffffffffu, send1, 8);
            s2[e] = keep2 + __shfl_xor_sync(0xffffffffu, send2, 8);
          }
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const bool up = (lane & 4) != 0;
            float send1 = up ? s1[e] : s1[e + 2], send2 = up ? s2[e] : s2[e + 2];
            float keep1 = up ? s1[e + 2] : s1[e], keep2 = up ? s2[e + 2] : s2[e];
            s1[e] = keep1 + __shfl_xor_sync(0xffffffffu, send1, 4);
            s2[e] = keep2 + __shfl_xor_sync(0xffffffffu, send2, 4);
          }
          {
            const bool up = (lane & 2) != 0;
            float send1 = up ? s1[0] : s1[1], send2 = up ? s2[0] : s2[1];
            float keep1 = up ? s1[1] : s1[0], keep2 = up ? s2[1] : s2[0];
            s1[0] = keep1 + __shfl_xor_sync(0xffffffffu, send1, 2);
            s2[0] = keep2 + __shfl_xor_sync(0xffffffffu, send2, 2);
          }
          s1[0] += __shfl_xor_sync(0xffffffffu, s1[0], 1);
          s2[0] += __shfl_xor_sync(0xffffffffu, s2[0], 1);
          const int colj = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
          if ((lane & 1) == 0 && gn + colj < p.N) {
            atomic_add_f64(&p.stats[gn + colj], (double)s1[0]);
            atomic_add_f64(&p.stats[(int64_t)p.N + gn + colj], (double)s2[0]);
          }
        }
    }
  }

}

int g_tc_force_bn = 0;

inline bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

template <bool A_MN, bool B_MN, bool SPLIT, int BN_T>
int launch1(const TcArgs& a, dim3 grid, size_t smem, cudaStream_t stream) {
  static bool attr_done = false;
  if (!attr_done) {
    GPS_CUDA(cudaFuncSetAttribute(k_gemm_tc<A_MN, B_MN, SPLIT, BN_T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  227 * 1024));
    attr_done = true;
  }
  k_gemm_tc<A_MN, B_MN, SPLIT, BN_T><<<grid, kThreads, smem, stream>>>(a);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}
template <bool A_MN, bool B_MN, bool SPLIT>
int launch(const TcArgs& a, dim3 grid, size_t smem, cudaStream_t stream) {
  return a.nb_blocks == 1 ? launch1<A_MN, B_MN, SPLIT, 64>(a, grid, smem, stream)
                          : launch1<A_MN, B_MN, SPLIT, 128>(a, grid, smem, stream);
}

}  // namespace

void gemm_tc_set_debug(int v) {   // bits 8.. : forced tile width (0 = heuristic)
  g_tc_force_bn = (v >> 8) & 0x1FF;
}

int gemm_tc(const GemmParams& p, cudaStream_t stream) {
  if (p.M <= 0 || p.N <= 0) return GPS_OK;
  if (p.K <= 0) return GPS_ERR_UNSUPPORTED;
  // 128-bit paths: aligned bases, leading dimensions and N multiples of 4
  if (!aligned16(p.A) || !aligned16(p.B) || !aligned16(p.C) || p.lda % 4 || p.ldb % 4 || p.ldc % 4 || p.N % 4)
    return GPS_ERR_UNSUPPORTED;
  if ((p.bias && !aligned16(p.bias)) || (p.R1 && (!aligned16(p.R1) || p.ldr1 % 4)) ||
      (p.R2 && (!aligned16(p.R2) || p.ldr2 % 4)) || (p.mask_src && (!aligned16(p.mask_src) || p.ldmask % 4)) ||
      (p.C_pre && (!aligned16(p.C_pre) || p.ldpre % 4)))
    return GPS_ERR_UNSUPPORTED;
  // lean producer loop: whole 8-element chunks are either inside or outside the operand
  if ((!p.ta && p.K % 8) || (!p.tb && p.K % 8) || (p.ta && p.M % 8) || (p.tb && p.N % 8)) return GPS_ERR_UNSUPPORTED;
  if (p.splitk > 1 && (p.bias || p.act >= 0 || p.mask_src || p.stats || p.C_pre || p.p_drop != 0.f || p.p_drop2 != 0.f)) {
    set_error("gemm: split-K supports the plain product (+ residuals) only");
    return GPS_ERR_ARG;
  }
  if (p.colsum_a && !p.ta) {
    set_error("gemm: colsum_a needs ta == 1");
    return GPS_ERR_ARG;
  }
  const bool split = p.precision == GPS_PREC_FP32;
  const int plane = split ? 2 : 1;
  const int mt = (int)ceil_div(p.M, BM);
  const int nkb = (int)ceil_div(p.K, BK);

  // tile width: BN in {64, 128} (1 or 2 staged 64-column blocks; the two warpgroups hold 128 x BN fp32 accumulators
  // beside the producers' staging registers); the kernel is bound by operand traffic ~ tiles x (128 + staged B rows),
  // so minimise waves x staged rows, wider on ties
  int bestBN = 128;
  long bestCost = -1;
  for (int bn = 128; bn >= 64; bn >>= 1) {
    const int nb = bn / 64;
    const long tiles = (long)mt * ceil_div(p.N, bn);
    const long waves = ceil_div(tiles, (long)kNumSMs);
    const long cost = waves * (BM + nb * 64L);
    if (bestCost < 0 || cost < bestCost) { bestCost = cost; bestBN = bn; }
  }
  if (g_tc_force_bn == 64 || g_tc_force_bn == 128) bestBN = g_tc_force_bn;   // tuning hook (tools/gemm_tune.py)
  TcArgs a;
  a.p = p;
  a.BN = bestBN;
  a.nb_blocks = a.BN / 64;
  const int stage_bytes = plane * (kATileBytes + a.nb_blocks * kBBlockBytes);
  int stages = (200 * 1024) / stage_bytes;
  if (stages > 4) stages = 4;
  if (stages < 2) return GPS_ERR_UNSUPPORTED;   // (two stages also hold the epilogue's fp32 staging tile)
  a.stages = stages;
  // splitk > 1 keeps its meaning "add into the pre-zeroed C", but the reduction is not split across CTAs: every
  // element then has a single adder and the result does not depend on the order in which CTAs finish (the TMA
  // kernel, which the layer uses, splits K deterministically within a cluster)
  const int splitk = 1;
  a.kb_per_split = nkb;
  a.p.splitk = p.splitk > 1 ? 2 : 1;   // "accumulate atomically" flag
  const size_t smem = (size_t)stages * stage_bytes + 1024 /*align*/ + (2 * stages + 1) * 8 + 16 + 16 * 16 * 8 * 4;
  dim3 grid((unsigned)ceil_div(p.N, a.BN), (unsigned)mt, (unsigned)splitk);
  const bool amn = p.ta != 0, bmn = p.tb != 0;
#define GPS_TC_CASE(AM, BMN)                                                        \
  if (amn == AM && bmn == BMN)                                                      \
    return split ? launch<AM, BMN, true>(a, grid, smem, stream) : launch<AM, BMN, false>(a, grid, smem, stream);
  GPS_TC_CASE(false, false)
  GPS_TC_CASE(false, true)
  GPS_TC_CASE(true, false)
  GPS_TC_CASE(true, true)
#undef GPS_TC_CASE
  return GPS_ERR_UNSUPPORTED;
}

}  // namespace gps
