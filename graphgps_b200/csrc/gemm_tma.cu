// gemm_tma.cu — TMA-fed wgmma dense product: the plane operand path of every Linear of the GPS layer.
//
//   C[M,N] (+)= epi( Aop[M,K] * Bop[K,N] )
//
// Both operands live in HBM as bf16 "planes": plain row-major bf16 matrices holding the hi part of the fp32 value
// and (fp32-grade mode) its bf16 residual lo, written ONCE by the kernel that produced the tensor (GEMM epilogues,
// the row-wise BatchNorm kernels, the gather-reduce kernels, attention) or by k_to_planes for layer inputs and
// weights.  The consumer therefore never converts anything: one thread issues tensor-map TMA
// (cp.async.bulk.tensor) boxes that land in shared memory already in the canonical wgmma SWIZZLE_128B image --
// a {64 x rows} box is a K-major tile, a {64 x 64} box is one MN-major block -- so the same planes serve
// y = x W^T (K-major), g_x = g_y W (B MN-major) and dW = G^T X (both MN-major, reduction over rows) without
// transposes or per-layout copies.  Out-of-range rows/columns are zero-filled by the TMA unit.
//
// Warp roles (288 threads): warps 0-7 are two consumer warpgroups, each issuing wgmma m64 x BN x k16 for its 64 rows of
// the 128-row tile (fp32 accumulators in registers; fp32-grade mode issues lo*hi + hi*lo + hi*hi) and then running the
// epilogue (bias / act / act' / dropout / residuals / fp32 store / bf16 hi-lo plane store / BatchNorm column sums /
// split-K atomics); warp 8 is the TMA producer (one lane).  Stages form an mbarrier ring: full = expect_tx bytes,
// empty = one arrival per consumer warp once the wgmma group reading the stage has retired.
// Narrow tiles (BN = 64) are launched two CTAs per SM so one CTA's epilogue overlaps the other's main loop.
// Split-K: the K-splits of one output tile form a thread-block cluster (at most 8).  Each split stages its fp32 partial
// tile in shared memory; rank r then sums rows [r RB, (r + 1) RB) of all ranks' tiles in rank order through
// distributed shared memory (RB a multiple of 16, the row classes of the column sums), so the result does not depend on
// the order in which the splits finish.  A caller-requested split (splitk > 1) adds the summed rows (and the residuals)
// into the pre-zeroed C; a split the launch policy chooses runs the full epilogue on them instead, rank r being the
// only writer of its rows.  The bias-gradient partials of the splits are combined the same way.
#include <cooperative_groups.h>
#include <cuda.h>
#include <cuda_bf16.h>

#include <mutex>
#include <unordered_map>

#include "gemm.cuh"
#include "tc_ptx.cuh"

namespace gps {

namespace {

using namespace tc;
namespace cgrp = cooperative_groups;

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kEpiWarps = 8;
constexpr int kTmaWarp = 8;
constexpr int kThreads = 288;
constexpr int kATile = BM * BK * 2;     // 16 KB per plane
constexpr int kBlock = 64 * BK * 2;     // 8 KB: one 64-column MN-major block / 64 K-major rows
constexpr int kMaxSplits = 8;           // split-K splits of a tile = cluster size (portable limit)

struct TmaArgs {
  GemmParams p;
  int BN, nb_blocks, stages, kb_per_split, planes;
  unsigned long long* trace;   // bring-up: 16 globaltimer stamps per CTA (first 256 CTAs), see tools/gemm_trace.py
};

__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// Rows [x, y) of the tile that this CTA's K-split owns after the cluster's reduction (the whole tile without split-K).
// RB is a multiple of 16, so a rank's rows start on row class 0 of the column sums; trailing ranks may own no rows
// (5-7 splits).  Read from the special registers at each use (volatile), so that the epilogue keeps no extra registers
// live across its row loop.
__device__ __forceinline__ int2 split_rows() {
  int z, nz;
  asm volatile("mov.u32 %0, %%ctaid.z;" : "=r"(z));
  asm volatile("mov.u32 %0, %%nctaid.z;" : "=r"(nz));
  const int RB = ((BM + nz - 1) / nz + 15) & ~15;
  const int lo = min(BM, z * RB);
  return make_int2(lo, min(BM, lo + RB));
}

#define GPS_TRACE(slot)                                                                         \
  do {                                                                                          \
    if (a.trace && cta_lin < 256) a.trace[cta_lin * 16 + (slot)] = gtimer();                    \
  } while (0)

template <bool A_MN, bool B_MN, int BN_T, bool SPLIT>
__global__ void __launch_bounds__(kThreads, BN_T == 64 ? 2 : 1)
k_gemm_tma(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TmaArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const GemmParams& p = a.p;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int planes = a.planes;
  const int b_tile = B_MN ? a.nb_blocks * kBlock : BN_T * 128;   // K-major B: BN rows of 128 bytes
  const int stage_bytes = planes * (kATile + b_tile);
  const int S = a.stages;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)S * stage_bytes);   // full[S], empty[S]
  float* red = reinterpret_cast<float*>(bars + 2 * S + 2);   // 16 x 16 x 8 floats (bias-gradient partials)
  float* ctot = red + 16 * 16 * 8;                           // [128] this split's bias-gradient sums (split-K)
  const int nsplit = (int)gridDim.z;                         // = cluster size when > 1

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * a.BN;
  const int nkb_total = (p.K + BK - 1) / BK;
  const int kb_begin = blockIdx.z * a.kb_per_split;
  const int kb_end = min(nkb_total, kb_begin + a.kb_per_split);
  const int nkb = kb_end - kb_begin;
  const bool do_colsum = A_MN && p.colsum_a != nullptr && blockIdx.x == 0;
  const int cta_lin = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;

  if (tid == 0) {
    GPS_TRACE(0);
    if (a.trace && cta_lin < 256) {
      unsigned smid;
      asm volatile("mov.u32 %0, %smid;" : "=r"(smid));
      a.trace[cta_lin * 16 + 8] = smid;
    }
    for (int s = 0; s < S; ++s) {
      mbar_init(smem_u32(&bars[s]), 1);
      mbar_init(smem_u32(&bars[S + s]), kEpiWarps);
    }
    fence_barrier_init();
  }
  if (warp == kTmaWarp && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  __syncthreads();
  if (tid == 0) GPS_TRACE(1);

  if (warp == kTmaWarp) {
    // =========================================================== TMA producer
    if (lane == 0 && nkb > 0) {
      // blocks of an MN-major tile that lie completely outside the matrix are not fetched (their smem content only
      // reaches accumulator rows / columns that are never stored)
      int a_blocks = 2, b_blocks = a.nb_blocks;
      if (A_MN) a_blocks = min(2, (p.M - m0 + 63) / 64);
      if (B_MN) b_blocks = min(a.nb_blocks, (p.N - n0 + 63) / 64);
      const uint32_t tx = (uint32_t)planes * ((A_MN ? a_blocks * kBlock : kATile) +
                                              (B_MN ? b_blocks * kBlock : a.BN * 128));
      for (int i = 0; i < nkb; ++i) {
        const int s = i % S;
        if (i >= S) mbar_wait(smem_u32(&bars[S + s]), (uint32_t)((i / S) - 1) & 1u);
        const uint32_t full = smem_u32(&bars[s]);
        mbar_arrive_expect_tx(full, tx);
        const int k0 = (kb_begin + i) * BK;
        const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes);
        const uint32_t sb = sa + planes * kATile;
        for (int pl = 0; pl < planes; ++pl) {
          if (!A_MN) {
            tma_tile_3d(sa + pl * kATile, &tmA, k0, m0, pl, full);
          } else {
            for (int b = 0; b < a_blocks; ++b) tma_tile_3d(sa + pl * kATile + b * kBlock, &tmA, m0 + 64 * b, k0, pl, full);
          }
          if (!B_MN) {
            tma_tile_3d(sb + pl * b_tile, &tmB, k0, n0, pl, full);
          } else {
            for (int b = 0; b < b_blocks; ++b) tma_tile_3d(sb + pl * b_tile + b * kBlock, &tmB, n0 + 64 * b, k0, pl, full);
          }
        }
        if (i == 0) GPS_TRACE(2);
      }
      GPS_TRACE(9);
    }
    __syncwarp();
    if (nsplit > 1) {   // the cluster barriers of the split-K reduction count every thread
      cgrp::this_cluster().sync();
      cgrp::this_cluster().sync();
    }
  } else {
    // =========================================================== consumer warpgroups: wgmma main loop
    // warpgroup wg owns accumulator rows [64 wg, 64 wg + 64) of the tile: its A operand starts 8 KB into every A plane
    // (eight 1 KB K-major row groups, or the second 64-row MN-major block)
    const int wg = warp >> 2;
    float acc[BN_T / 2];
#pragma unroll
    for (int e = 0; e < BN_T / 2; ++e) acc[e] = 0.f;
    // bias gradient db[m] = sum_k Aop[m,k]: the n-tile-0 CTAs sum the staged (MN-major) A tiles while the tensor
    // core works on them.  Thread t owns the 8-column chunk (t & 15) and k-rows 4 (t >> 4) .. +3 of every k-block.
    float csum[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) csum[e] = 0.f;
    const int cm = tid & 15, kq = tid >> 4;
    constexpr uint32_t a_lbo = A_MN ? kBlock : 16, b_lbo = B_MN ? kBlock : 16;
    constexpr uint32_t a_kstep = A_MN ? 2048 : 32, b_kstep = B_MN ? 2048 : 32;
    for (int i = 0; i < nkb; ++i) {
      const int s = i % S;
      if (lane == 0) mbar_wait(smem_u32(&bars[s]), (uint32_t)(i / S) & 1u);
      __syncwarp();
      if (i == 0 && tid == 0) GPS_TRACE(3);
      if (i == nkb - 1 && tid == 0) GPS_TRACE(10);
      const uint8_t* st = smem + (size_t)s * stage_bytes;
      const uint32_t sa_hi = smem_u32(st) + (uint32_t)wg * 8192u;
      const uint32_t sb_hi = smem_u32(st) + planes * kATile;
      const uint32_t sa_lo = sa_hi + kATile;
      const uint32_t sb_lo = sb_hi + b_tile;
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
      if (do_colsum) {
        const uint32_t blk_off = (uint32_t)(cm >> 3) * kBlock;
        const int cc = cm & 7;
        for (int pl = 0; pl < planes; ++pl) {
#pragma unroll
          for (int rr = 0; rr < 4; ++rr) {
            const int r = kq * 4 + rr;
            const uint4 q = *reinterpret_cast<const uint4*>(st + pl * kATile + blk_off + (r >> 3) * 1024 + (r & 7) * 128 +
                                                            ((cc ^ (r & 7)) << 4));
            const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              csum[2 * e] += __uint_as_float(w[e] << 16);
              csum[2 * e + 1] += __uint_as_float(w[e] & 0xFFFF0000u);
            }
          }
        }
      }
      // at most one group in flight: the previous k-block's MMAs have retired, so its stage goes back to the producer
      wgmma_wait<1>();
      reg_fence<BN_T / 2>(acc);
      __syncwarp();
      if (i > 0 && lane == 0) mbar_arrive(smem_u32(&bars[S + (i - 1) % S]));
    }
    wgmma_wait<0>();
    reg_fence<BN_T / 2>(acc);
    if (tid == 0) GPS_TRACE(4);
    if (do_colsum) {
#pragma unroll
      for (int e = 0; e < 8; ++e) red[(kq * 16 + cm) * 8 + e] = csum[e];
    }
    // every wgmma of both warpgroups has retired: the operand stages are free and become the staging tile
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (do_colsum && tid < 128) {
      const int cmr = tid >> 3, e = tid & 7;
      float tot = 0.f;
#pragma unroll
      for (int o = 0; o < 16; ++o) tot += red[(o * 16 + cmr) * 8 + e];
      const int gm = m0 + cmr * 8 + e;
      if (nsplit > 1) ctot[cmr * 8 + e] = tot;   // combined across the cluster below
      else if (gm < p.M) atomicAdd(&p.colsum_a[gm], tot);
    }
    if (tid == 0) GPS_TRACE(5);
    // ---- phase 1: accumulator registers -> shared staging tile [128][BN + 4] fp32.  wgmma fragment: thread lane of warp
    // w holds rows 16 (w & 3) + lane / 4 (+ 8) and columns 8 j + 2 (lane % 4) (+ 1) of its warpgroup's 64 rows.
    float* stage = reinterpret_cast<float*>(smem);
    const int sld = a.BN + 4;
    {
      const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);
      const int c = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BN_T / 8; ++j) {
        *reinterpret_cast<float2*>(stage + r * sld + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(stage + (r + 8) * sld + 8 * j + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    // ---- split-K: rank r replaces rows [lo, hi) of its staging tile by the rank-ordered sum over the cluster and owns
    // them for the rest of the epilogue
    const int lo = split_rows().x, hi = split_rows().y;
    if (nsplit > 1) {
      cgrp::cluster_group cluster = cgrp::this_cluster();
      cluster.sync();   // every split's staging tile (and bias-gradient sums) is complete
      // Each thread keeps U float4s of every rank in flight at once: a distributed shared memory load costs a round
      // trip, and one element at a time the pass is that latency times the element count.  Only the rows below M are
      // summed (the epilogue reads no others).  The 64-wide kernels (96 registers) sum one element at a time.
      const int c4n = a.BN >> 2;
      const int n4 = max(0, min(hi, p.M - m0) - lo) * c4n;
      constexpr int U = BN_T == 64 ? 1 : 4, kStep = kEpiWarps * 32;
      if constexpr (U == 1) {
        for (int idx = tid; idx < n4; idx += kStep) {
          const int o = (lo + idx / c4n) * sld + (idx % c4n) * 4;
          float4 sum = f4zero();
          for (int k = 0; k < nsplit; ++k)
            sum = f4add(sum, *reinterpret_cast<const float4*>(cluster.map_shared_rank(stage, k) + o));
          *reinterpret_cast<float4*>(stage + o) = sum;
        }
      } else {
        for (int b = tid; b < n4; b += U * kStep) {
          int off[U];
          float4 sum[U];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int idx = min(b + u * kStep, n4 - 1);   // past the end: re-reads a valid element, not stored
            off[u] = (lo + idx / c4n) * sld + (idx % c4n) * 4;
            sum[u] = f4zero();
          }
          for (int k = 0; k < nsplit; ++k) {
            const float* src = cluster.map_shared_rank(stage, k);
            float4 v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) v[u] = *reinterpret_cast<const float4*>(src + off[u]);
#pragma unroll
            for (int u = 0; u < U; ++u) sum[u] = f4add(sum[u], v[u]);
          }
#pragma unroll
          for (int u = 0; u < U; ++u)
            if (b + u * kStep < n4) *reinterpret_cast<float4*>(stage + off[u]) = sum[u];
        }
      }
      if (do_colsum && blockIdx.z == 0 && tid < 128 && m0 + tid < p.M) {
        float tot = 0.f;
        for (int k = 0; k < nsplit; ++k) tot += cluster.map_shared_rank(ctot, k)[tid];
        atomicAdd(&p.colsum_a[m0 + tid], tot);   // the only adder of this element
      }
      cluster.sync();   // no rank leaves while another still reads its shared memory
    }
    // ---- phase 2: G = BN/4 threads per row, each owning 4 consecutive columns for all of its rows: every global access
    // (bias, residuals, act' mask, fp32 / plane stores, split-K atomics) is a contiguous row segment and the per-column
    // constants live in registers.  When BatchNorm column sums are wanted, w goes back into the staging tile for them.
    // The pass covers this CTA's rows [lo, row_end) of the tile: all of them without split-K.
    const int G = a.BN >> 2;
    const int rpp = kEpiWarps * 32 / G;            // rows per pass
    const int rip = tid / G, cg = tid - rip * G;
    const int col = n0 + cg * 4;
    const bool col_ok = rip < rpp && col < p.N;
    const int rows_here = min(BM, p.M - m0);
    const int row_end = min(hi, rows_here);
    const bool colstats = p.stats != nullptr;
    if (col_ok) {
      // rows of this thread: r = lo + rip + k * rpp, k < nrows.  Everything is addressed through per-thread base pointers
      // advanced by a constant stride, and the loop is unrolled by 4 rows so that the shared/global loads of a group are
      // in flight together: with 2 epilogue warps per scheduler the pass is instruction-latency bound otherwise
      // (even with the global stores off the critical path).
      const int nrows = lo + rip < row_end ? (row_end - lo - rip + rpp - 1) / rpp : 0;
      const int64_t row0 = m0 + lo + rip;
      float* sp = stage + (lo + rip) * sld + cg * 4;
      const int s_st = rpp * sld;
      float* cp = p.C ? p.C + row0 * p.ldc + col : nullptr;
      const int64_t c_st = (int64_t)rpp * p.ldc;
      const float* r1 = p.R1 ? p.R1 + row0 * p.ldr1 + col : nullptr;
      const int64_t r1_st = (int64_t)rpp * p.ldr1;
      const float* r2 = p.R2 ? p.R2 + row0 * p.ldr2 + col : nullptr;
      const int64_t r2_st = (int64_t)rpp * p.ldr2;
      if (p.splitk > 1) {
        // accumulate into the pre-zeroed C: this CTA is the only adder of rows [lo, hi) (the whole tile without split)
        for (int r = lo + rip; r < min(hi, rows_here); r += rpp) {
          const int64_t row = m0 + r;
          float4 w = *reinterpret_cast<const float4*>(stage + r * sld + cg * 4);
          if (p.R1) w = f4add(w, ld4(p.R1 + row * p.ldr1 + col));
          if (p.R2) w = f4add(w, ld4(p.R2 + row * p.ldr2 + col));
          atomicAdd(reinterpret_cast<float4*>(p.C + row * p.ldc + col), w);   // red.global.add.v4.f32
        }
      } else {
        const bool fast = !p.C_pre && !(p.mask_src && !p.mask_is_post) && p.p_drop == 0.f && p.p_drop2 == 0.f &&
                          (p.act < 0 || p.act == GPS_ACT_RELU);
        const float4 bb = p.bias ? ld4(p.bias + col) : f4zero();
        const float* mk = p.mask_src ? p.mask_src + row0 * p.ldmask + col : nullptr;
        const int64_t mk_st = (int64_t)rpp * p.ldmask;
        // plane column: identity, or the per-head padded layout of the attention operands (cp_hd)
        int pcol = col, npad = 0;
        if (p.cp_hd > 0) {
          const int hq = col / p.cp_hd, cw = col - hq * p.cp_hd;
          pcol = hq * p.cp_hd_pad + cw;
          npad = (cw + 4 == p.cp_hd) ? p.cp_hd_pad - p.cp_hd : 0;   // this thread also zeroes the head's pad columns
        }
        __nv_bfloat16* ph = p.Cp.hi ? p.Cp.hi + row0 * p.Cp.ld + pcol : nullptr;
        __nv_bfloat16* pl = p.Cp.lo ? p.Cp.lo + row0 * p.Cp.ld + pcol : nullptr;
        const int64_t p_st = (int64_t)rpp * p.Cp.ld;
        const bool relu = p.act == GPS_ACT_RELU;
        if (fast) {
          for (int k = 0; k < nrows; k += 4) {
            float4 w[4];
#pragma unroll
            for (int u = 0; u < 4; ++u)
              w[u] = f4add(k + u < nrows ? *reinterpret_cast<const float4*>(sp + (k + u) * s_st) : f4zero(), bb);
            if (relu) {
#pragma unroll
              for (int u = 0; u < 4; ++u)
                w[u] = make_float4(fmaxf(w[u].x, 0.f), fmaxf(w[u].y, 0.f), fmaxf(w[u].z, 0.f), fmaxf(w[u].w, 0.f));
            }
            if (mk) {   // relu': the saved post-activation value is positive
              float4 m[4];
#pragma unroll
              for (int u = 0; u < 4; ++u) m[u] = k + u < nrows ? ld4(mk + (k + u) * mk_st) : f4zero();
#pragma unroll
              for (int u = 0; u < 4; ++u)
                w[u] = make_float4(m[u].x > 0.f ? w[u].x : 0.f, m[u].y > 0.f ? w[u].y : 0.f, m[u].z > 0.f ? w[u].z : 0.f,
                                   m[u].w > 0.f ? w[u].w : 0.f);
            }
            if (r1) {
#pragma unroll
              for (int u = 0; u < 4; ++u) if (k + u < nrows) w[u] = f4add(w[u], ld4(r1 + (k + u) * r1_st));
            }
            if (r2) {
#pragma unroll
              for (int u = 0; u < 4; ++u) if (k + u < nrows) w[u] = f4add(w[u], ld4(r2 + (k + u) * r2_st));
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              if (k + u >= nrows) continue;
              if (colstats) *reinterpret_cast<float4*>(sp + (k + u) * s_st) = w[u];
              if (cp) st4(cp + (k + u) * c_st, w[u]);
              if (ph) {
                __nv_bfloat162 h0 = __floats2bfloat162_rn(w[u].x, w[u].y), h1 = __floats2bfloat162_rn(w[u].z, w[u].w);
                *reinterpret_cast<uint2*>(ph + (k + u) * p_st) =
                    make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
                if (pl) {
                  __nv_bfloat162 l0 = __floats2bfloat162_rn(w[u].x - __low2float(h0), w[u].y - __high2float(h0));
                  __nv_bfloat162 l1 = __floats2bfloat162_rn(w[u].z - __low2float(h1), w[u].w - __high2float(h1));
                  *reinterpret_cast<uint2*>(pl + (k + u) * p_st) =
                      make_uint2(*reinterpret_cast<uint32_t*>(&l0), *reinterpret_cast<uint32_t*>(&l1));
                }
                for (int z = 0; z < npad; z += 4) {
                  *reinterpret_cast<uint2*>(ph + (k + u) * p_st + 4 + z) = make_uint2(0u, 0u);
                  if (pl) *reinterpret_cast<uint2*>(pl + (k + u) * p_st + 4 + z) = make_uint2(0u, 0u);
                }
              }
            }
          }
        } else {
          // general path: pre-activation copy, GELU and its derivative, dropout (two chained sites for the Performer)
          const uint64_t drop_off = p.offset + ((p.p_drop > 0.f || p.p_drop2 > 0.f) && p.offset_dev ? *p.offset_dev : 0ull);
          for (int k = 0; k < nrows; ++k) {
            const int64_t row = row0 + (int64_t)k * rpp;
            float4 w = f4add(*reinterpret_cast<const float4*>(sp + k * s_st), bb);
            if (p.C_pre) st4(p.C_pre + row * p.ldpre + col, w);
            if (p.act >= 0) w = make_float4(act_fwd_rt(p.act, w.x), act_fwd_rt(p.act, w.y), act_fwd_rt(p.act, w.z), act_fwd_rt(p.act, w.w));
            if (mk) {
              const float4 ms = ld4(mk + k * mk_st);
              if (p.mask_is_post) {
                w.x = ms.x > 0.f ? w.x : 0.f; w.y = ms.y > 0.f ? w.y : 0.f; w.z = ms.z > 0.f ? w.z : 0.f; w.w = ms.w > 0.f ? w.w : 0.f;
              } else {
                w.x *= act_bwd_rt(p.mask_act, ms.x); w.y *= act_bwd_rt(p.mask_act, ms.y);
                w.z *= act_bwd_rt(p.mask_act, ms.z); w.w *= act_bwd_rt(p.mask_act, ms.w);
              }
            }
            if (p.p_drop2 > 0.f) w = f4mul(w, dropout_scale4(p.p_drop2, p.seed, drop_off, p.site2, ((uint64_t)row * (uint64_t)p.N + col) >> 2));
            if (p.p_drop > 0.f) w = f4mul(w, dropout_scale4(p.p_drop, p.seed, drop_off, p.site, ((uint64_t)row * (uint64_t)p.N + col) >> 2));
            if (r1) w = f4add(w, ld4(r1 + k * r1_st));
            if (r2) w = f4add(w, ld4(r2 + k * r2_st));
            if (cp) st4(cp + k * c_st, w);
            if (ph) {
              planes_store4(p.Cp, row, pcol, w);
              for (int z = 0; z < npad; z += 4) planes_store4(p.Cp, row, pcol + 4 + z, f4zero());
            }
            if (colstats) *reinterpret_cast<float4*>(sp + k * s_st) = w;
          }
        }
      }
    }
    const int2 own = split_rows();
    const int slo = own.x, send = min(own.y, min(BM, p.M - m0));
    if (colstats && slo < send) {
      // BatchNorm column sums over this CTA's rows, in the same order for every tile width: task (y, g) sums rows
      // lo + y, lo + y + 16, ... of column group g (sum w, sum w^2) and leaves the two partials in rows y, y + 16 of its
      // own row class (lo is a multiple of 16, and after the cluster's last barrier the whole staging tile is this
      // CTA's); then one thread per column group adds the 16 classes in order: one double atomic per column per CTA and
      // statistic.
      asm volatile("bar.sync 1, 256;" ::: "memory");
      for (int t = tid; t < 16 * G; t += kEpiWarps * 32) {
        const int y = t / G, g = t - y * G, c = n0 + g * 4;
        if (c >= p.N) continue;
        float4 s1 = f4zero(), s2 = f4zero();
        for (int r = slo + y; r < send; r += 16) {
          const float4 w = *reinterpret_cast<const float4*>(stage + r * sld + g * 4);
          s1 = f4add(s1, w);
          s2 = f4fma(w, w, s2);
        }
        float* o = stage + y * sld + g * 4;
        *reinterpret_cast<float4*>(o) = s1;
        *reinterpret_cast<float4*>(o + 16 * sld) = s2;
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (tid < G && n0 + tid * 4 < p.N) {
        float4 t[2] = {f4zero(), f4zero()};
        for (int y = 0; y < 16; ++y) {
          t[0] = f4add(t[0], *reinterpret_cast<const float4*>(stage + y * sld + tid * 4));
          t[1] = f4add(t[1], *reinterpret_cast<const float4*>(stage + (y + 16) * sld + tid * 4));
        }
        const int c0 = n0 + tid * 4;
        auto add4 = [&](double* dst, float4 v) {
          atomic_add_f64(dst + 0, (double)v.x); atomic_add_f64(dst + 1, (double)v.y);
          atomic_add_f64(dst + 2, (double)v.z); atomic_add_f64(dst + 3, (double)v.w);
        };
        add4(p.stats + c0, t[0]);
        add4(p.stats + (int64_t)p.N + c0, t[1]);
      }
    }
  }

  if (tid == 0) GPS_TRACE(6);
  if (a.trace) {
    __syncthreads();
    if (tid == 0) GPS_TRACE(7);
  }
}

// ------------------------------------------------------------------------------------ tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      f = nullptr;
    return reinterpret_cast<EncodeTiledFn>(f);
  }();
  return fn;
}

struct MapKey {
  const void* base; int64_t cols, rows, ld, plane_stride; int planes, box_rows;
  bool operator==(const MapKey& o) const {
    return base == o.base && cols == o.cols && rows == o.rows && ld == o.ld && plane_stride == o.plane_stride &&
           planes == o.planes && box_rows == o.box_rows;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.base);
    auto mix = [&](int64_t v) { h ^= (size_t)v + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
    mix(k.cols); mix(k.rows); mix(k.ld); mix(k.plane_stride); mix(k.planes); mix(k.box_rows);
    return h;
  }
};

// rank-3 map over {cols (contiguous), rows, planes} of bf16 with a {64, box_rows, 1} SWIZZLE_128B box
int tensor_map(const __nv_bfloat16* hi, const __nv_bfloat16* lo, int planes, int64_t rows, int64_t cols, int64_t ld,
               int box_rows, CUtensorMap* out) {
  static std::mutex mu;
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  const int64_t plane_stride = planes == 2 ? (int64_t)(lo - hi) : rows * ld;
  GPS_REQUIRE(planes == 1 || plane_stride > 0, GPS_ERR_ARG, "gemm_tma: the lo plane must follow the hi plane in memory");
  MapKey key{hi, cols, rows, ld, plane_stride, planes, box_rows};
  {
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find(key);
    if (it != cache.end()) {
      *out = it->second;
      return GPS_OK;
    }
  }
  EncodeTiledFn enc = encode_fn();
  GPS_REQUIRE(enc, GPS_ERR_UNSUPPORTED, "cuTensorMapEncodeTiled is not available from this driver");
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)planes};
  cuuint64_t strides[2] = {(cuuint64_t)ld * 2, (cuuint64_t)(plane_stride > 0 ? plane_stride : 8) * 2};
  cuuint32_t box[3] = {64, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUtensorMap m;
  CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<__nv_bfloat16*>(hi), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  GPS_REQUIRE(r == CUDA_SUCCESS, GPS_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d): rows %lld cols %lld ld %lld box %d",
              (int)r, (long long)rows, (long long)cols, (long long)ld, box_rows);
  {
    std::lock_guard<std::mutex> lk(mu);
    if (cache.size() > 4096) cache.clear();
    cache[key] = m;
  }
  *out = m;
  return GPS_OK;
}

}  // namespace

int make_tensor_map(const __nv_bfloat16* hi, const __nv_bfloat16* lo, int planes, int64_t rows, int64_t cols, int64_t ld,
                    int box_rows, CUtensorMap* out) {
  return tensor_map(hi, lo, planes, rows, cols, ld, box_rows, out);
}

namespace {

inline bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

template <bool A_MN, bool B_MN, int BN_T, bool SPLIT>
int launch1(const CUtensorMap& tA, const CUtensorMap& tB, const TmaArgs& a, dim3 grid, size_t smem, cudaStream_t stream) {
  static bool attr_done = false;
  if (!attr_done) {
    GPS_CUDA(cudaFuncSetAttribute(k_gemm_tma<A_MN, B_MN, BN_T, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  227 * 1024));
    attr_done = true;
  }
  if (grid.z == 1) {
    k_gemm_tma<A_MN, B_MN, BN_T, SPLIT><<<grid, kThreads, smem, stream>>>(tA, tB, a);
  } else {   // the K-splits of a tile are one cluster
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 1;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = grid.z;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    GPS_CUDA(cudaLaunchKernelEx(&cfg, k_gemm_tma<A_MN, B_MN, BN_T, SPLIT>, tA, tB, a));
  }
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}
template <bool A_MN, bool B_MN, int BN_T>
int launch(const CUtensorMap& tA, const CUtensorMap& tB, const TmaArgs& a, dim3 grid, size_t smem, cudaStream_t stream) {
  return a.planes == 2 ? launch1<A_MN, B_MN, BN_T, true>(tA, tB, a, grid, smem, stream)
                       : launch1<A_MN, B_MN, BN_T, false>(tA, tB, a, grid, smem, stream);
}

int g_tma_force_bn = 0;
int g_tma_force_splits = 0;
unsigned long long* g_tma_trace = nullptr;

}  // namespace

void gemm_tma_set_force_bn(int bn) { g_tma_force_bn = bn; }
void gemm_tma_set_force_splits(int s) { g_tma_force_splits = s; }
void gemm_tma_set_trace(unsigned long long* buf) { g_tma_trace = buf; }

int gemm_tma(const GemmParams& p, cudaStream_t stream) {
  if (p.M <= 0 || p.N <= 0) return GPS_OK;
  if (p.K <= 0 || !p.Ap.hi || !p.Bp.hi) return GPS_ERR_UNSUPPORTED;
  const bool split = p.precision == GPS_PREC_FP32;
  const int planes = split ? 2 : 1;
  if (split && (!p.Ap.lo || !p.Bp.lo)) return GPS_ERR_UNSUPPORTED;
  // TMA: 16-byte aligned bases and row pitches; the epilogue's 128-bit paths as in the register-staged kernel
  if (!aligned16(p.Ap.hi) || !aligned16(p.Bp.hi) || p.Ap.ld % 8 || p.Bp.ld % 8 || p.N % 4) return GPS_ERR_UNSUPPORTED;
  if (split && (!aligned16(p.Ap.lo) || !aligned16(p.Bp.lo))) return GPS_ERR_UNSUPPORTED;
  if ((p.C && (!aligned16(p.C) || p.ldc % 4)) || (!p.C && !p.Cp.hi)) return GPS_ERR_UNSUPPORTED;
  if (p.Cp.hi && (p.Cp.ld % 4 || (reinterpret_cast<uintptr_t>(p.Cp.hi) & 7) || (p.Cp.lo && (reinterpret_cast<uintptr_t>(p.Cp.lo) & 7))))
    return GPS_ERR_UNSUPPORTED;
  if ((p.bias && !aligned16(p.bias)) || (p.R1 && (!aligned16(p.R1) || p.ldr1 % 4)) ||
      (p.R2 && (!aligned16(p.R2) || p.ldr2 % 4)) || (p.mask_src && (!aligned16(p.mask_src) || p.ldmask % 4)) ||
      (p.C_pre && (!aligned16(p.C_pre) || p.ldpre % 4)))
    return GPS_ERR_UNSUPPORTED;
  if (p.splitk > 1 && (p.bias || p.act >= 0 || p.mask_src || p.stats || p.C_pre || p.p_drop != 0.f || p.p_drop2 != 0.f ||
                       p.Cp.hi || !p.C)) {
    set_error("gemm: split-K supports the plain fp32 product (+ residuals) only");
    return GPS_ERR_ARG;
  }
  if (p.colsum_a && !p.ta) {
    set_error("gemm: colsum_a needs ta == 1");
    return GPS_ERR_ARG;
  }
  const int mt = (int)ceil_div(p.M, BM);
  const int nkb = (int)ceil_div(p.K, BK);
  // K-splits actually launched for a requested count s: every split but the last takes ceil(nkb / s) k-blocks
  const auto splits_of = [&](int s) {
    s = max(1, min(kMaxSplits, min(s, nkb)));
    return (int)ceil_div(nkb, ceil_div(nkb, s));
  };
  // Tile width.  Measured at the layer's shapes, a launch takes time in proportion to the MMA columns its busiest SM
  // issues: waves x BN, where zero-padded columns count (they cost MMAs and staging like real ones) and
  // waves = ceil(tiles / CTA slots).  The epilogue's stores and the operand loads of a tile grow with BN as well, and
  // the fixed cost of a tile is small, so this one product ranks the widths.  64-wide tiles run two CTAs per SM; each
  // stages its own copy of the A tile (1.5x the L2 -> SM operand bytes of one 128-wide tile), which costs them a
  // quarter: a wave of them counts as 2 x 64 x 1.25 columns, unless every CTA has an SM of its own (64 columns).
  // Ties go to the wider tile (fewer CTAs re-read A).
  // 152 = 304 / 2 divides every column count of the d = 304 layer; it exists for a K-major B only (an MN-major B is
  // staged in 64-column SWIZZLE_128B blocks).  256 exists for a K-major A only: with an MN-major A (the weight
  // gradients dW = G^T X, split-K clusters) it never costs less than 128 and was measured 20-60 % slower on ties.
  const auto width_ok = [&](int bn) {
    return bn == 64 || bn == 128 || (bn == 152 && !p.tb) || (bn == 256 && !p.ta);
  };
  //
  // K-splits of a launch that runs the epilogue (splitk <= 1).  A CTA's time is a fixed part (launch, prologue, the
  // first operand fetch, staging, the epilogue pass) plus its k-blocks, both per column; a split adds the cluster's
  // barriers and the rank-ordered sum of the staged partial tiles through distributed shared memory.  Fitted to the
  // per-launch times at d = 304 with the layer's epilogues (H100 SXM, 700 W; 58 tiles of 152 columns: 15.6 us at 5
  // k-blocks, 22.3 us at 10, 18.8 and 22.8 us for the same launches in 2 splits), the fixed part is worth about 7
  // k-blocks and a split about 5 more.  So a launch costs waves x BN x (k-blocks per split + 7 (+ 5 when split)), in
  // quarter k-blocks below.  A split is considered only while the split tiles still fit on the SMs at one CTA each
  // (tiles <= 132 / splits; a second wave lost every time it was measured) and every split keeps at least 2 k-blocks;
  // ties go to fewer splits.  At d = 304 no product of the layer is split (10 k-blocks is the break-even); the split
  // pays for long reductions over few row tiles (g_x at d = 256, M = 4000: 2 splits).  The split depends on the shape alone, never on a forced tile
  // width, so every width still computes each element with the same wgmma sequence.
  const auto wave_cost = [&](int bn, long ctas) -> long {
    return bn != 64 ? ceil_div(ctas, (long)kNumSMs) * bn : ctas <= kNumSMs ? 64 : ceil_div(ctas, 2L * kNumSMs) * 160;
  };
  const auto best_width = [&](int s, long* cost_out) {
    int best = 0;
    long best_cost = 0;
    for (const int bn : {64, 128, 152, 256}) {
      if (!width_ok(bn)) continue;
      const long cost = wave_cost(bn, (long)mt * ceil_div(p.N, bn) * s);
      if (!best || cost <= best_cost) { best_cost = cost; best = bn; }
    }
    if (cost_out) *cost_out = best_cost;
    return best;
  };
  int nsplit = 1;
  if (p.splitk > 1) {
    nsplit = splits_of(p.splitk);
  } else if (g_tma_force_splits > 0) {
    nsplit = splits_of(g_tma_force_splits);
  } else {
    long best_cost = 0;
    for (int s = 1; s <= kMaxSplits; ++s) {
      if (splits_of(s) != s) continue;
      const int kbps = (int)ceil_div(nkb, s);
      if (s > 1 && nkb - (s - 1) * kbps < 2) continue;
      long wc = 0;
      const int bn = best_width(s, &wc);
      if (s > 1 && (long)mt * ceil_div(p.N, bn) * s > kNumSMs) continue;
      // a 64-wide CTA with an SM to itself streams the same A tile per k-block as a 128-wide one and was measured no
      // faster over a long K (g_x at M = 4000, d = 256: 64 us against 49 us fp32-grade, and 35 us in 2 splits of 128)
      if (bn == 64) wc = max(wc, 128L);
      const long cost = wc * (4L * kbps + 28 + (s > 1 ? 20 : 0));
      if (s == 1 || cost < best_cost) { best_cost = cost; nsplit = s; }
    }
  }
  int bestBN = best_width(p.splitk > 1 ? min(kMaxSplits, min(p.splitk, nkb)) : nsplit, nullptr);
  if (g_tma_force_bn) {
    if (!width_ok(g_tma_force_bn)) return GPS_ERR_UNSUPPORTED;
    bestBN = g_tma_force_bn;
  }
  TmaArgs a;
  a.p = p;
  a.BN = bestBN;
  a.nb_blocks = a.BN / 64;
  a.planes = planes;
  const bool narrow = a.nb_blocks == 1;
  const int stage_bytes = planes * (kATile + (p.tb ? a.nb_blocks * kBlock : a.BN * 128));
  const int fixed = 1024 /*align*/ + 1024 /*barriers*/ + 16 * 16 * 8 * 4 + 128 * 4;
  int stages = ((narrow ? 112 : 226) * 1024 - fixed) / stage_bytes;
  if (stages > 8) stages = 8;
  if (stages < 2) return GPS_ERR_UNSUPPORTED;
  // the operand stages also hold the epilogue's fp32 staging tile [BM][BN + 4]
  GPS_REQUIRE((size_t)stages * stage_bytes >= (size_t)BM * (a.BN + 4) * 4, GPS_ERR_ARG,
              "gemm_tma: BN %d: the staging tile does not fit the operand stages", a.BN);
  a.stages = stages;
  a.kb_per_split = (int)ceil_div(nkb, nsplit);
  a.p.splitk = p.splitk > 1 ? 2 : 1;   // "accumulate atomically" flag
  a.trace = g_tma_trace;
  const bool amn = p.ta != 0, bmn = p.tb != 0;
  // planes are addressed as stored: Aop[m,k] = A[m, k] (ta = 0: rows = M, cols = K) or A[k, m] (ta = 1: rows = K, cols = M)
  CUtensorMap tA, tB;
  GPS_TRY(tensor_map(p.Ap.hi, p.Ap.lo, planes, amn ? p.K : p.M, amn ? p.M : p.K, p.Ap.ld, amn ? 64 : BM, &tA));
  GPS_TRY(tensor_map(p.Bp.hi, p.Bp.lo, planes, bmn ? p.K : p.N, bmn ? p.N : p.K, p.Bp.ld, bmn ? 64 : a.BN, &tB));
  const size_t smem = (size_t)stages * stage_bytes + fixed;
  dim3 grid((unsigned)ceil_div(p.N, a.BN), (unsigned)mt, (unsigned)nsplit);
#define GPS_TMA_CASE(AM, BMN)                                                                              \
  if (amn == AM && bmn == BMN) {                                                                           \
    if (a.BN == 64) return launch<AM, BMN, 64>(tA, tB, a, grid, smem, stream);                            \
    if (a.BN == 128) return launch<AM, BMN, 128>(tA, tB, a, grid, smem, stream);                          \
  }
  GPS_TMA_CASE(false, false)
  GPS_TMA_CASE(false, true)
  GPS_TMA_CASE(true, false)
  GPS_TMA_CASE(true, true)
#undef GPS_TMA_CASE
  if (a.BN == 152 && !bmn)
    return amn ? launch<true, false, 152>(tA, tB, a, grid, smem, stream) : launch<false, false, 152>(tA, tB, a, grid, smem, stream);
  if (a.BN == 256 && !amn)
    return bmn ? launch<false, true, 256>(tA, tB, a, grid, smem, stream) : launch<false, false, 256>(tA, tB, a, grid, smem, stream);
  return GPS_ERR_UNSUPPORTED;
}

// ------------------------------------------------------------------------------------ fp32 -> planes
namespace {
struct ToPlanesDesc {
  ToPlanesItem it[16];
  int start[17];   // first 8-element chunk row-block of each item in the 1-D grid
  int n;
};
// one thread per 8 consecutive elements of a row: 2 x 128-bit loads, one 128-bit store per plane
__global__ void k_to_planes(ToPlanesDesc d) {
  int item = 0;
  while (item + 1 < d.n && (int)blockIdx.x >= d.start[item + 1]) ++item;
  const ToPlanesItem& it = d.it[item];
  const int cpr = (it.cols + 7) >> 3;                               // chunks per row
  const int64_t total = (int64_t)it.rows * cpr;
  const int64_t idx = ((int64_t)blockIdx.x - d.start[item]) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int64_t r = idx / cpr;
  const int c = (int)(idx - r * cpr) * 8;
  const float* src = it.src + r * it.ld + c;
  float v[8];
  if (c + 8 <= it.cols) {
    const float4 x = ld4(src), y = ld4(src + 4);
    v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w; v[4] = y.x; v[5] = y.y; v[6] = y.z; v[7] = y.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = c + i < it.cols ? src[i] : 0.f;
  }
  uint4 hi, lo;
  tc::split8(v, hi, lo);
  *reinterpret_cast<uint4*>(it.dst.hi + r * it.dst.ld + c) = hi;
  if (it.dst.lo) *reinterpret_cast<uint4*>(it.dst.lo + r * it.dst.ld + c) = lo;
}
}  // namespace

int to_planes(const ToPlanesItem* items, int n, cudaStream_t stream) {
  if (n <= 0) return GPS_OK;
  GPS_REQUIRE(n <= 16, GPS_ERR_ARG, "to_planes: at most 16 matrices per call");
  ToPlanesDesc d;
  d.n = 0;
  int total = 0;
  for (int i = 0; i < n; ++i) {
    const ToPlanesItem& it = items[i];
    if (it.rows <= 0 || it.cols <= 0) continue;
    GPS_REQUIRE(it.src && it.dst.hi && it.ld % 4 == 0 && it.dst.ld % 8 == 0 && it.dst.ld >= round_up(it.cols, 8) &&
                    (reinterpret_cast<uintptr_t>(it.src) & 15) == 0 && (reinterpret_cast<uintptr_t>(it.dst.hi) & 15) == 0 &&
                    (!it.dst.lo || (reinterpret_cast<uintptr_t>(it.dst.lo) & 15) == 0),
                GPS_ERR_ARG, "to_planes: operands must be 16-byte aligned, ld %% 4 == 0, plane ld %% 8 == 0");
    d.it[d.n] = it;
    d.start[d.n] = total;
    total += (int)ceil_div((int64_t)it.rows * ((it.cols + 7) >> 3), 256);
    ++d.n;
  }
  d.start[d.n] = total;
  if (total == 0) return GPS_OK;
  k_to_planes<<<(unsigned)total, 256, 0, stream>>>(d);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

}  // namespace gps
