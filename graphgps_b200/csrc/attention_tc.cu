// attention_tc.cu — softmax attention over each graph's own nodes on the Hopper tensor cores (wgmma + TMA).
//
// Replaces to_dense_batch -> nn.MultiheadAttention core -> [mask] (graphgps/layer/gps_layer.py:199-201, 234-241) like
// attention.cu, but as two warpgroup MMAs per key tile:  S = Q K^T  and  O += P V.
//
//   * Packing instead of padding: a CTA owns 128 CONSECUTIVE node rows of the packed batch (several small graphs, or a
//     slice of a large one) and one head.  Its keys are the contiguous node range [start of the first row's graph, end
//     of the last row's graph), walked in tiles of 128.  The dense batch of the reference (B x Nmax, 1.7x - 3x padding)
//     never exists; the per-graph "key padding mask" is the block-diagonal range test  graph_start(i) <= j < graph_end(i)
//     applied to the S accumulator registers.
//   * Operands: Q, K, V arrive by tensor-map TMA from the bf16 hi/lo planes that the node-projection GEMM's epilogue wrote
//     in a per-head layout padded to a multiple of 16 columns (zero pad), already in the wgmma SWIZZLE_128B image:
//     Q and K K-major ({64 x 128} boxes), V as an MN-major B operand ({64 x 64} boxes).  fp32-grade mode runs every
//     product as lo*hi + hi*lo + hi*hi (the probabilities are split hi/lo as well); bf16 mode is a single pass.
//   * Each of the two consumer warpgroups owns 64 query rows: S (64 x 128) and O (64 x 64 or 64 x 128) stay in its
//     registers.  Online softmax in fp32 with the running row max / sum per thread (a row is spread over the 4 lanes of
//     a quad); when a row's max moves, O is rescaled in registers.  P goes straight from the S registers into the
//     register A operand of the P V product (the accumulator fragment of S is the A fragment of P).  Dropout on the
//     probabilities uses the same Philox stream as attention.cu (site GPS_SITE_ATTN_P + head, one draw per 4 keys).
// 256 threads = two MMA / softmax warpgroups; thread 0 also issues the TMA loads.  The K and V tiles have their own
// full / empty barriers, so the next K tile loads while the softmax and P V of the current one run.  (A separate
// producer warp would make the CTA count as three warpgroups and cap the registers that S, O and P need.)
// The CUDA-core kernel in attention.cu serves batches of small graphs (mean below 64 nodes) and head dims above 128.
// BIAS (BiasedTransformer): after the range mask, each valid S element becomes S * scale + bias[g, h, i - gs, j - gs]
// (the caller's dense [B*H, nmax, nmax] bias) before the row max, and the softmax then runs with scale 1.
#include <cuda.h>
#include <cuda_bf16.h>

#include "gemm.cuh"
#include "kernels.cuh"
#include "tc_ptx.cuh"

namespace gps {

namespace {

using namespace tc;

constexpr int kTile = 128;
constexpr int kSoftWarps = 8;
constexpr int kThreadsA = 256;

struct AttnTcArgs {
  const int* gptr; int B; int N; int H; int hd; int hd_pad; int planes;
  float* O; int64_t ldo; Planes Op; float* lse;
  float scale; float p_drop; uint64_t seed, offset;
  const unsigned long long* offset_dev;
  float* dbg;   // bring-up: CTA (0,0) dumps S [128x128], P [128x128] and the raw O accumulator [128x128] of its first tile
};
// the bias travels as a kernel parameter of its own: growing AttnTcArgs changes the unbiased kernels' code
struct TcBias {
  const float* bias; int64_t nmax;   // read by the BIAS kernels only
};

__device__ __forceinline__ int find_graph_tc(const int* __restrict__ gptr, int B, int node) {
  int lo = 0, hi = B;   // largest g with gptr[g] <= node (graphs may be empty)
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (gptr[mid] <= node) lo = mid; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// one query row as seen by one lane: graph key range, running max / partial sum, cached dropout draw
struct RowState {
  int i, gs, ge;
  float m, l;
  int rq_quad;
  Philox4 rq;
};

// NKB: 64-column blocks of the padded head dim (1: hd_pad <= 64, 2: <= 128) = the P V instruction width / 64
template <int NKB, bool SPLIT, bool BIAS>
__global__ void __launch_bounds__(kThreadsA, 1)
k_attn_tc_fwd(const __grid_constant__ CUtensorMap tmQK, const __grid_constant__ CUtensorMap tmV, const AttnTcArgs a,
              const TcBias tb) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int planes = SPLIT ? 2 : 1;
  constexpr int q_bytes = NKB * 16384, k_bytes = NKB * 16384, v_bytes = 2 * NKB * 8192;   // per plane
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + planes * q_bytes;
  uint8_t* sV = sK + planes * k_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + planes * v_bytes);   // q_full, k_full, v_full, k_empty, v_empty
  int* range = reinterpret_cast<int*>(bars + 8);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int q0 = blockIdx.x * kTile, h = blockIdx.y;
  const uint32_t b_q = smem_u32(&bars[0]), b_kf = smem_u32(&bars[1]), b_vf = smem_u32(&bars[2]),
                 b_ke = smem_u32(&bars[3]), b_ve = smem_u32(&bars[4]);

  if (tid == 0) {
    mbar_init(b_q, 1); mbar_init(b_kf, 1); mbar_init(b_vf, 1); mbar_init(b_ke, kSoftWarps); mbar_init(b_ve, kSoftWarps);
    fence_barrier_init();
    const int last = min(q0 + kTile, a.N) - 1;
    const int g0 = find_graph_tc(a.gptr, a.B, q0), g1 = find_graph_tc(a.gptr, a.B, last);
    range[0] = a.gptr[g0];
    range[1] = a.gptr[g1 + 1];
  }
  __syncthreads();
  const int kmin = range[0], kmax = range[1];
  const int ntiles = max(1, (kmax - kmin + kTile - 1) / kTile);

  auto load_k = [&](int t) {   // thread 0: K tile t (its slot was released by both warpgroups' S of tile t - 1)
    if (t > 0) mbar_wait(b_ke, (uint32_t)(t - 1) & 1u);
    mbar_arrive_expect_tx(b_kf, (uint32_t)(planes * k_bytes));
    for (int pl = 0; pl < planes; ++pl)
      for (int kb = 0; kb < NKB; ++kb)
        tma_tile_3d(smem_u32(sK + pl * k_bytes + kb * 16384), &tmQK, (a.H + h) * a.hd_pad + 64 * kb, kmin + t * kTile, pl,
                    b_kf);
  };
  auto load_v = [&](int t) {   // thread 0: V tile t (after both warpgroups' P V of tile t - 1)
    if (t > 0) mbar_wait(b_ve, (uint32_t)(t - 1) & 1u);
    mbar_arrive_expect_tx(b_vf, (uint32_t)(planes * v_bytes));
    for (int pl = 0; pl < planes; ++pl)
      for (int kk = 0; kk < 2; ++kk)
        for (int nb = 0; nb < NKB; ++nb)
          tma_tile_3d(smem_u32(sV + pl * v_bytes + (kk * NKB + nb) * 8192), &tmV, (2 * a.H + h) * a.hd_pad + 64 * nb,
                      kmin + t * kTile + 64 * kk, pl, b_vf);
  };
  if (tid == 0) {
    tma_prefetch_desc(&tmQK);
    tma_prefetch_desc(&tmV);
    mbar_arrive_expect_tx(b_q, (uint32_t)(planes * q_bytes));
    for (int pl = 0; pl < planes; ++pl)
      for (int kb = 0; kb < NKB; ++kb)
        tma_tile_3d(smem_u32(sQ + pl * q_bytes + kb * 16384), &tmQK, h * a.hd_pad + 64 * kb, q0, pl, b_q);
    load_k(0);
    load_v(0);
  }

  // =========================================================== MMA / softmax warpgroups
  // fragment of a 64 x N accumulator: lane of warp w holds rows 16 (w & 3) + lane / 4 (+ 8) of the warpgroup's 64 rows
  // and columns 8 j + 2 (lane % 4) (+ 1), at acc[4 j + {0, 1}] (row) and acc[4 j + {2, 3}] (row + 8)
  const int wg = warp >> 2;
  const int rloc = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // tile row of the first of this lane's two rows
  const int cq = 2 * (lane & 3);
  RowState rs[2];
  const float* brow[2] = {nullptr, nullptr};   // BIAS: bias rows of the lane's two queries
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    RowState& R = rs[u];
    R.i = q0 + rloc + 8 * u;
    R.gs = 0; R.ge = 0;
    if (R.i < a.N) {
      const int g = find_graph_tc(a.gptr, a.B, R.i);
      R.gs = a.gptr[g];
      R.ge = a.gptr[g + 1];
      if constexpr (BIAS) brow[u] = tb.bias + (((int64_t)g * a.H + h) * tb.nmax + (R.i - R.gs)) * tb.nmax;
    }
    R.m = -INFINITY; R.l = 0.f; R.rq_quad = -1;
  }
  const uint64_t offs = a.offset + ((a.p_drop > 0.f && a.offset_dev) ? *a.offset_dev : 0ull);
  const bool use_drop = a.p_drop > 0.f;
  const uint32_t drop_thr = (uint32_t)fminf(a.p_drop * 4294967296.f, 4294967295.f);
  const float keep_scale = use_drop ? 1.f / (1.f - a.p_drop) : 1.f;
  const bool dump = a.dbg && blockIdx.x == 0 && blockIdx.y == 0;
  const float sc = BIAS ? 1.f : a.scale;   // BIAS: S is scaled (and biased) in place before the softmax

  float o[NKB * 32];
#pragma unroll
  for (int e = 0; e < NKB * 32; ++e) o[e] = 0.f;
  const uint32_t aQ = smem_u32(sQ) + (uint32_t)wg * 8192u, aK = smem_u32(sK), aV = smem_u32(sV);
  const int qk_steps = a.hd_pad >> 4;
  if (lane == 0) mbar_wait(b_q, 0u);
  __syncwarp();
  for (int t = 0; t < ntiles; ++t) {
    const int key0 = kmin + t * kTile;
    // ---- S = Q K^T
    float sacc[64];
#pragma unroll
    for (int e = 0; e < 64; ++e) sacc[e] = 0.f;
    if (lane == 0) mbar_wait(b_kf, (uint32_t)t & 1u);
    __syncwarp();
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < NKB * 4; ++ks) {
      if (ks < qk_steps) {
        const uint32_t off = (ks >> 2) * 16384 + (ks & 3) * 32;
        const uint64_t dq_hi = make_desc(aQ + off, 16, 1024);
        const uint64_t dk_hi = make_desc(aK + off, 16, 1024);
        if (SPLIT) {
          const uint64_t dq_lo = make_desc(aQ + q_bytes + off, 16, 1024);
          const uint64_t dk_lo = make_desc(aK + k_bytes + off, 16, 1024);
          wgmma_ss<128, 0, 0>(sacc, dq_lo, dk_hi, 1u);
          wgmma_ss<128, 0, 0>(sacc, dq_hi, dk_lo, 1u);
        }
        wgmma_ss<128, 0, 0>(sacc, dq_hi, dk_hi, 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<64>(sacc);
    __syncwarp();
    if (lane == 0) mbar_arrive(b_ke);
    if (tid == 0 && t + 1 < ntiles) load_k(t + 1);
    if constexpr (BIAS) {
#pragma unroll
      for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int key = key0 + 8 * j + cq + e;
            float& v = sacc[4 * j + 2 * u + e];
            if (key >= rs[u].gs && key < rs[u].ge) v = v * a.scale + brow[u][key - rs[u].gs];
          }
    }
    // ---- online softmax on the registers: row maximum over the valid (same-graph) logits, quad-reduced
    float corr[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      RowState& R = rs[u];
      float mnew = R.m;
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = key0 + 8 * j + cq + e;
          if (key >= R.gs && key < R.ge) mnew = fmaxf(mnew, sacc[4 * j + 2 * u + e] * sc);
        }
      mnew = fmaxf(mnew, __shfl_xor_sync(0xffffffffu, mnew, 1));
      mnew = fmaxf(mnew, __shfl_xor_sync(0xffffffffu, mnew, 2));
      corr[u] = (R.m == -INFINITY) ? 1.f : __expf(R.m - mnew);
      R.l *= corr[u];
      R.m = mnew;
    }
#pragma unroll
    for (int j = 0; j < NKB * 8; ++j) {
      o[4 * j] *= corr[0]; o[4 * j + 1] *= corr[0];
      o[4 * j + 2] *= corr[1]; o[4 * j + 3] *= corr[1];
    }
    // ---- P = exp(S - m) (dropout applied, denominators from the undropped values), in place of S
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      RowState& R = rs[u];
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = key0 + 8 * j + cq + e;
          float& v = sacc[4 * j + 2 * u + e];
          const float sraw = v;
          float pr = 0.f;
          if (key >= R.gs && key < R.ge) {
            pr = __expf(v * sc - R.m);
            R.l += pr;
            if (use_drop) {
              const int jl = key - R.gs;
              if ((jl >> 2) != R.rq_quad) {
                R.rq_quad = jl >> 2;
                R.rq = philox4x32(a.seed, offs + (uint64_t)(GPS_SITE_ATTN_P + h), ((uint64_t)R.i << 20) | (uint64_t)R.rq_quad);
              }
              const int k4 = jl & 3;
              const uint32_t bits = k4 == 0 ? R.rq.v[0] : k4 == 1 ? R.rq.v[1] : k4 == 2 ? R.rq.v[2] : R.rq.v[3];
              pr = bits >= drop_thr ? pr * keep_scale : 0.f;
            }
          }
          v = pr;
          if (dump && t == 0) {
            const int r = rloc + 8 * u, c = 8 * j + cq + e;
            a.dbg[r * 128 + c] = sraw;
            a.dbg[16384 + r * 128 + c] = pr;
          }
        }
    }
    // ---- O += P V: the S fragment of keys [16 ks, 16 ks + 16) is the register A fragment of k-step ks
    uint32_t ph[32], pl[SPLIT ? 32 : 1];
#pragma unroll
    for (int x = 0; x < 32; ++x) {
      const float p0 = sacc[2 * x], p1 = sacc[2 * x + 1];
      __nv_bfloat162 hb = __floats2bfloat162_rn(p0, p1);
      ph[x] = *reinterpret_cast<uint32_t*>(&hb);
      if (SPLIT) pl[x] = pack_bf16x2(p0 - __low2float(hb), p1 - __high2float(hb));
    }
    if (lane == 0) mbar_wait(b_vf, (uint32_t)t & 1u);
    __syncwarp();
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint32_t voff = ((ks >> 2) * NKB) * 8192 + (ks & 3) * 2048;
      const uint64_t dv_hi = make_desc(aV + voff, 8192, 1024);
      if (SPLIT) {
        const uint64_t dv_lo = make_desc(aV + v_bytes + voff, 8192, 1024);
        wgmma_rs<NKB * 64, 1>(o, pl + 4 * ks, dv_hi, 1u);
        wgmma_rs<NKB * 64, 1>(o, ph + 4 * ks, dv_lo, 1u);
      }
      wgmma_rs<NKB * 64, 1>(o, ph + 4 * ks, dv_hi, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<NKB * 32>(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(b_ve);
    if (tid == 0 && t + 1 < ntiles) load_v(t + 1);
  }
  // ---- epilogue: O / l -> fp32 rows (+ operand planes for the output projection), log-sum-exp for the backward pass
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    RowState& R = rs[u];
    R.l += __shfl_xor_sync(0xffffffffu, R.l, 1);
    R.l += __shfl_xor_sync(0xffffffffu, R.l, 2);
    const float inv = R.l > 0.f ? 1.f / R.l : 0.f;
    const bool row_ok = R.i < a.N;
#pragma unroll
    for (int j = 0; j < NKB * 8; ++j) {
      const int col = 8 * j + cq;
      const float v0 = o[4 * j + 2 * u], v1 = o[4 * j + 2 * u + 1];
      if (dump) {
        a.dbg[32768 + (rloc + 8 * u) * 128 + col] = v0;
        a.dbg[32768 + (rloc + 8 * u) * 128 + col + 1] = v1;
      }
      if (!row_ok || col >= a.hd) continue;
      const float w0 = v0 * inv, w1 = v1 * inv;
      float* dst = a.O + (int64_t)R.i * a.ldo + (int64_t)h * a.hd + col;
      dst[0] = w0;
      dst[1] = w1;
      if (a.Op.hi) {
        const int64_t off = (int64_t)R.i * a.Op.ld + (int64_t)h * a.hd + col;
        __nv_bfloat162 hb = __floats2bfloat162_rn(w0, w1);
        *reinterpret_cast<__nv_bfloat162*>(a.Op.hi + off) = hb;
        if (a.Op.lo) *reinterpret_cast<uint32_t*>(a.Op.lo + off) = pack_bf16x2(w0 - __low2float(hb), w1 - __high2float(hb));
      }
    }
    if (row_ok && (lane & 3) == 0) a.lse[(int64_t)R.i * a.H + h] = R.m + __logf(R.l);
  }
}

template <int NKB, bool SPLIT, bool BIAS>
int launch_attn(const CUtensorMap& tQK, const CUtensorMap& tV, const AttnTcArgs& a, const TcBias& tb, dim3 grid,
                size_t smem, cudaStream_t stream) {
  static bool attr_done = false;
  if (!attr_done) {
    GPS_CUDA(cudaFuncSetAttribute(k_attn_tc_fwd<NKB, SPLIT, BIAS>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_done = true;
  }
  k_attn_tc_fwd<NKB, SPLIT, BIAS><<<grid, kThreadsA, smem, stream>>>(tQK, tV, a, tb);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

float* g_attn_dbg = nullptr;
}  // namespace

void attention_tc_set_debug(float* buf) { g_attn_dbg = buf; }
bool attention_tc_supported(int64_t hd) { return hd > 0 && hd % 4 == 0 && hd <= 128; }
int64_t attention_tc_hd_pad(int64_t hd) { return round_up(hd, 16); }

// qkv: bf16 hi/lo planes [N, 3 * H * hd_pad] in the per-head padded layout (which * H + h) * hd_pad + k, pads zero.
int attention_tc_fwd(const GpsGraph& g, int64_t heads, int64_t hd, Planes qkv, float* O, int64_t ldo, Planes Op, float* lse,
                     float p_drop, uint64_t seed, uint64_t offset, const unsigned long long* offset_dev, int precision,
                     cudaStream_t stream, const GpsAttnBias* bias) {
  if (g.N == 0) return GPS_OK;
  GPS_REQUIRE(attention_tc_supported(hd) && qkv.hi && (precision != GPS_PREC_FP32 || qkv.lo) && qkv.ld % 8 == 0, GPS_ERR_UNSUPPORTED,
              "attention_tc: head dim %lld / planes not supported", (long long)hd);
  AttnTcArgs a{};
  a.gptr = g.graph_ptr; a.B = (int)g.B; a.N = (int)g.N; a.H = (int)heads; a.hd = (int)hd;
  a.hd_pad = (int)attention_tc_hd_pad(hd);
  a.planes = precision == GPS_PREC_FP32 ? 2 : 1;
  a.O = O; a.ldo = ldo; a.Op = Op; a.lse = lse;
  a.scale = 1.f / sqrtf((float)hd); a.p_drop = p_drop; a.seed = seed; a.offset = offset; a.offset_dev = offset_dev;
  a.dbg = g_attn_dbg;
  TcBias tb{};
  if (bias) tb = TcBias{bias->bias, bias->nmax};
  const int64_t cols = 3 * heads * a.hd_pad;
  CUtensorMap tQK, tV;
  GPS_TRY(make_tensor_map(qkv.hi, qkv.lo, a.planes, g.N, cols, qkv.ld, 128, &tQK));
  GPS_TRY(make_tensor_map(qkv.hi, qkv.lo, a.planes, g.N, cols, qkv.ld, 64, &tV));
  const int nkb = (a.hd_pad + 63) >> 6;
  const size_t smem = (size_t)a.planes * nkb * (16384 + 16384 + 16384) + 1024 + 256;
  dim3 grid((unsigned)ceil_div(g.N, kTile), (unsigned)heads);
  if (bias) {
    if (nkb == 1) return a.planes == 2 ? launch_attn<1, true, true>(tQK, tV, a, tb, grid, smem, stream)
                                       : launch_attn<1, false, true>(tQK, tV, a, tb, grid, smem, stream);
    return a.planes == 2 ? launch_attn<2, true, true>(tQK, tV, a, tb, grid, smem, stream)
                         : launch_attn<2, false, true>(tQK, tV, a, tb, grid, smem, stream);
  }
  if (nkb == 1) return a.planes == 2 ? launch_attn<1, true, false>(tQK, tV, a, tb, grid, smem, stream)
                                     : launch_attn<1, false, false>(tQK, tV, a, tb, grid, smem, stream);
  return a.planes == 2 ? launch_attn<2, true, false>(tQK, tV, a, tb, grid, smem, stream)
                       : launch_attn<2, false, false>(tQK, tV, a, tb, grid, smem, stream);
}

}  // namespace gps
