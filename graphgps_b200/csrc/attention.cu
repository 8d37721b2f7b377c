// attention.cu — exact softmax attention over each graph's own node set, without densification.
//
// Replaces to_dense_batch -> nn.MultiheadAttention core -> [mask] of the reference
// (graphgps/layer/gps_layer.py:199-201, 234-241): the padded [B,Nmax,d] tensor, the key-padding
// mask and the boolean-mask gather (two host syncs per layer) disappear; every query row attends to
// the rows [graph_ptr[g], graph_ptr[g+1]) of its own graph directly in the packed [N, *] layout.
//
// Mapping (CUDA-core version; the flop share of this stage is <1% of the layer at the PCQM/ZINC
// shapes, 4*d*sum n_g^2 vs 24*N*d^2 — SURVEY.md 8d): query rows are packed densely into warps
// regardless of graph boundaries; LPR lanes cooperate on one row, each holding CH float4 chunks
// of the head dimension (single floats when the head dim is not a multiple of 4, VW = 1), so q/o (fwd)
// and k/v/dk/dv (bwd) live in registers and a dot product is an LPR-lane shuffle reduction.
// Online softmax in fp32; dropout on the probabilities uses the Philox stream (site GPS_SITE_ATTN_P + head).
// Backward = two passes (query-major for dQ and delta, key-major for dK, dV): no atomics.
// BIAS (BiasedTransformer, gps_layer.py:202-204): S = (q . k) / sqrt(hd) + bias[g, h, i - gs, j - gs] with the caller's
// dense [B*H, nmax, nmax] bias.  The query-major backward visits every (query, key, head) once and writes the score
// gradient there, so grad_bias needs no atomics either.
#include "kernels.cuh"

namespace gps {

namespace {

constexpr int kWarpsPerBlock = 4;

__device__ __forceinline__ int find_graph(const int* __restrict__ gptr, int B, int node) {
  // largest g with gptr[g] <= node  (graphs may be empty)
  int lo = 0, hi = B;  // invariant: gptr[lo] <= node < gptr[hi]
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (gptr[mid] <= node) lo = mid; else hi = mid;
  }
  return lo;
}

template <int LPR>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ int warp_max_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Dropout on the attention probabilities: one Philox call yields the keep decisions of 4 consecutive keys
// (query i, keys 4*(jl>>2) .. +3) of one head; callers cache it across those 4 loop iterations.
struct DropQuad {
  Philox4 r;
  uint32_t thr;
  float keep_scale;
};
__device__ __forceinline__ void drop_quad_refresh(DropQuad& q, float p, uint64_t seed, uint64_t offset, int head, int i, int jl) {
  q.r = philox4x32(seed, offset + (uint64_t)(GPS_SITE_ATTN_P + head), ((uint64_t)i << 20) | (uint64_t)(jl >> 2));
}
__device__ __forceinline__ float drop_quad_scale(const DropQuad& q, int jl) {
  const int k = jl & 3;
  const uint32_t bits = k == 0 ? q.r.v[0] : k == 1 ? q.r.v[1] : k == 2 ? q.r.v[2] : q.r.v[3];
  return bits >= q.thr ? q.keep_scale : 0.f;
}
__device__ __forceinline__ void drop_quad_init(DropQuad& q, float p) {
  q.thr = (uint32_t)fminf(p * 4294967296.f, 4294967295.f);
  q.keep_scale = 1.f / (1.f - p);
}

// Chunks of the head dimension.  VW = 4: float4 chunks, for head dims that are a multiple of 4 with 16-byte aligned rows.
// VW = 1: one float per chunk, for any other head dim (Graphormer on ZINC has hd = 80 / 8 = 10; an odd hd also leaves
// each head's columns without 8-byte alignment).  The per-key updates of a float4 chunk are written out per component
// as before, so the VW = 4 kernels compile to the same instructions.
template <int VW> struct VecT;
template <> struct VecT<4> { using T = float4; };
template <> struct VecT<1> { using T = float; };

template <int VW> __device__ __forceinline__ typename VecT<VW>::T vld(const float* p);
template <> __device__ __forceinline__ float4 vld<4>(const float* p) { return ld4(p); }
template <> __device__ __forceinline__ float vld<1>(const float* p) { return *p; }
template <int VW> __device__ __forceinline__ typename VecT<VW>::T vzero();
template <> __device__ __forceinline__ float4 vzero<4>() { return f4zero(); }
template <> __device__ __forceinline__ float vzero<1>() { return 0.f; }
__device__ __forceinline__ void vst(float* p, float4 v) { st4(p, v); }
__device__ __forceinline__ void vst(float* p, float v) { *p = v; }
__device__ __forceinline__ float4 vscale(float4 a, float s) { return f4scale(a, s); }
__device__ __forceinline__ float vscale(float a, float s) { return a * s; }
__device__ __forceinline__ float vdot(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
__device__ __forceinline__ float vdot(float a, float b) { return a * b; }
__device__ __forceinline__ void vplanes_store(const Planes& p, int64_t r, int64_t c, float4 v) { planes_store4(p, r, c, v); }
__device__ __forceinline__ void vplanes_store(const Planes& p, int64_t r, int64_t c, float v) {
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  p.hi[r * p.ld + c] = h;
  if (p.lo) p.lo[r * p.ld + c] = __float2bfloat16_rn(v - __bfloat162float(h));
}

// lane-slice helpers: lane `sub` of a row group owns chunks sub, sub+LPR, ... (< nch) of VW floats each
template <int CH, int LPR, int VW>
__device__ __forceinline__ void load_slice(typename VecT<VW>::T* dst, const float* row, int sub, int nch, bool ok) {
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    int ch = sub + c * LPR;
    dst[c] = (ok && ch < nch) ? vld<VW>(row + ch * VW) : vzero<VW>();
  }
}
template <int CH, int LPR, int VW>
__device__ __forceinline__ void store_slice(const typename VecT<VW>::T* src, float* row, int sub, int nch) {
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    int ch = sub + c * LPR;
    if (ch < nch) vst(row + ch * VW, src[c]);
  }
}
// the same slice into the bf16 hi/lo planes of the tensor (operand image of the next GEMM), columns col0 ...
template <int CH, int LPR, int VW>
__device__ __forceinline__ void store_slice_planes(const typename VecT<VW>::T* src, const Planes& p, int64_t r, int64_t col0,
                                                   int sub, int nch) {
  if (!p.hi) return;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    int ch = sub + c * LPR;
    if (ch < nch) vplanes_store(p, r, col0 + ch * VW, src[c]);
  }
}
template <int CH, typename V>
__device__ __forceinline__ float dot_slice(const V* a, const V* b) {
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c) s += vdot(a[c], b[c]);
  return s;
}

struct AttnArgs {
  const int* gptr; int B; int N; int H; int hd;
  const float* Q; const float* K; const float* V; int64_t ld;
  float* O; const float* Oc; const float* dO; int64_t ldo;
  float* lse; const float* lsec; float* delta; const float* deltac;
  float* dQ; float* dK; float* dV; int64_t ldg;
  float scale; float p_drop; uint64_t seed, offset;
  const unsigned long long* offset_dev;
  Planes Op, dQp, dKp, dVp;   // optional bf16 hi/lo plane copies of O (forward) / dQ, dK, dV (backward)
  const float* bias; int64_t nmax; float* gbias;   // BIAS kernels only: [B*H, nmax, nmax], grad_bias (may be NULL)
};
__device__ __forceinline__ uint64_t eff_offset(const AttnArgs& a) {
  return a.offset + ((a.p_drop > 0.f && a.offset_dev) ? *a.offset_dev : 0ull);
}

template <int CH, int LPR, bool BIAS, int VW>
__global__ void __launch_bounds__(kWarpsPerBlock * 32) k_attn_fwd(AttnArgs a) {
  using V = typename VecT<VW>::T;
  constexpr int RPW = 32 / LPR;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sub = lane % LPR, rloc = lane / LPR;
  const int h = blockIdx.y;
  const int i = (blockIdx.x * kWarpsPerBlock + warp) * RPW + rloc;
  const bool row_ok = i < a.N;
  const int nch = a.hd / VW;
  const uint64_t offs = eff_offset(a);
  int gs = 0, n = 0;
  const float* brow = nullptr;   // BIAS: bias row of (graph, head, query)
  if (row_ok) {
    int g = find_graph(a.gptr, a.B, i);
    gs = a.gptr[g];
    n = a.gptr[g + 1] - gs;
    if constexpr (BIAS) brow = a.bias + (((int64_t)g * a.H + h) * a.nmax + (i - gs)) * a.nmax;
  }
  const int nloop = warp_max_i(n);
  const int64_t hoff = (int64_t)h * a.hd;
  V q[CH], o[CH];
  load_slice<CH, LPR, VW>(q, a.Q + (int64_t)(row_ok ? i : 0) * a.ld + hoff, sub, nch, row_ok);
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    q[c] = vscale(q[c], a.scale);
    o[c] = vzero<VW>();
  }
  float m = -INFINITY, l = 0.f;
  const bool use_drop = a.p_drop > 0.f;
  DropQuad dq;
  drop_quad_init(dq, a.p_drop);
  // software pipeline: the K/V rows of key jl+1 are in flight while key jl is processed (the loop is a chain of
  // load -> dot -> shuffle -> exp -> fma, i.e. latency bound at these tiny graph sizes)
  V kc[CH], vc[CH];
  load_slice<CH, LPR, VW>(kc, a.K + (int64_t)gs * a.ld + hoff, sub, nch, n > 0);
  load_slice<CH, LPR, VW>(vc, a.V + (int64_t)gs * a.ld + hoff, sub, nch, n > 0);
  float bc = 0.f;
  if constexpr (BIAS) bc = n > 0 ? brow[0] : 0.f;
  for (int jl = 0; jl < nloop; ++jl) {
    if (use_drop && (jl & 3) == 0) drop_quad_refresh(dq, a.p_drop, a.seed, offs, h, i, jl);
    const bool valid = jl < n;
    const bool nvalid = jl + 1 < n;
    const int jn = gs + (nvalid ? jl + 1 : 0);
    V kn[CH], vn[CH];
    load_slice<CH, LPR, VW>(kn, a.K + (int64_t)jn * a.ld + hoff, sub, nch, nvalid);
    load_slice<CH, LPR, VW>(vn, a.V + (int64_t)jn * a.ld + hoff, sub, nch, nvalid);
    float bn = 0.f;
    if constexpr (BIAS) bn = nvalid ? brow[jl + 1] : 0.f;
    float s = group_sum<LPR>(dot_slice<CH>(q, kc));
    if constexpr (BIAS) s += bc;
    s = valid ? s : -INFINITY;
    const float m_new = fmaxf(m, s);
    const float corr = (m_new == -INFINITY) ? 1.f : __expf(m - m_new);
    const float p = valid ? __expf(s - m_new) : 0.f;
    l = l * corr + p;
    const float pd = use_drop ? p * drop_quad_scale(dq, jl) : p;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      if constexpr (VW == 4) {
        o[c].x = o[c].x * corr + pd * vc[c].x;
        o[c].y = o[c].y * corr + pd * vc[c].y;
        o[c].z = o[c].z * corr + pd * vc[c].z;
        o[c].w = o[c].w * corr + pd * vc[c].w;
      } else {
        o[c] = o[c] * corr + pd * vc[c];
      }
      kc[c] = kn[c];
      vc[c] = vn[c];
    }
    if constexpr (BIAS) bc = bn;
    m = m_new;
  }
  if (row_ok) {
    const float inv = 1.f / l;
#pragma unroll
    for (int c = 0; c < CH; ++c) o[c] = vscale(o[c], inv);
    store_slice<CH, LPR, VW>(o, a.O + (int64_t)i * a.ldo + hoff, sub, nch);
    store_slice_planes<CH, LPR, VW>(o, a.Op, i, hoff, sub, nch);
    if (sub == 0) a.lse[(int64_t)i * a.H + h] = m + __logf(l);
  }
}

// delta_i = dO_i . O_i per (row, head): 8 lanes per pair read consecutive chunks (float4: 128 B per group)
template <int VW>
__global__ void k_attn_delta(AttnArgs a) {
  using V = typename VecT<VW>::T;
  const int64_t t = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  const int sub = threadIdx.x & 7;
  const bool ok = t < (int64_t)a.N * a.H;
  const int64_t i = ok ? t / a.H : 0;
  const int h = ok ? (int)(t - i * a.H) : 0;
  const V* go = reinterpret_cast<const V*>(a.dO + i * a.ldo + (int64_t)h * a.hd);
  const V* oo = reinterpret_cast<const V*>(a.Oc + i * a.ldo + (int64_t)h * a.hd);
  float acc = 0.f;
  if (ok)
    for (int c = sub; c < a.hd / VW; c += 8) {
      const V x = __ldg(go + c), y = __ldg(oo + c);
      acc += vdot(x, y);
    }
  acc += __shfl_xor_sync(0xffffffffu, acc, 4);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  if (ok && sub == 0) a.delta[t] = acc;
}

// query-major backward: dQ_i (delta precomputed by k_attn_delta); BIAS: grad_bias[g, h, i - gs, jl] = ds
template <int CH, int LPR, bool BIAS, int VW>
__device__ __forceinline__ void attn_bwd_q_body(const AttnArgs& a) {
  using V = typename VecT<VW>::T;
  constexpr int RPW = 32 / LPR;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sub = lane % LPR, rloc = lane / LPR;
  const int h = blockIdx.y;
  const int i = (blockIdx.x * kWarpsPerBlock + warp) * RPW + rloc;
  const bool row_ok = i < a.N;
  const int nch = a.hd / VW;
  const uint64_t offs = eff_offset(a);
  int gs = 0, n = 0;
  int64_t brow = 0;   // BIAS: offset of the (graph, head, query) row in bias / grad_bias
  if (row_ok) {
    int g = find_graph(a.gptr, a.B, i);
    gs = a.gptr[g];
    n = a.gptr[g + 1] - gs;
    if constexpr (BIAS) brow = (((int64_t)g * a.H + h) * a.nmax + (i - gs)) * a.nmax;
  }
  const int nloop = warp_max_i(n);
  const int64_t hoff = (int64_t)h * a.hd;
  const int ir = row_ok ? i : 0;
  V q[CH], go[CH], gq[CH];
  load_slice<CH, LPR, VW>(q, a.Q + (int64_t)ir * a.ld + hoff, sub, nch, row_ok);
  load_slice<CH, LPR, VW>(go, a.dO + (int64_t)ir * a.ldo + hoff, sub, nch, row_ok);
  {
    const float dl = row_ok ? a.deltac[(int64_t)i * a.H + h] : 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) gq[c] = vzero<VW>();
    const float lse = row_ok ? a.lsec[(int64_t)i * a.H + h] : 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) q[c] = vscale(q[c], a.scale);
    const bool use_drop = a.p_drop > 0.f;
    DropQuad dq;
    drop_quad_init(dq, a.p_drop);
    V kk[CH], vv[CH];
    load_slice<CH, LPR, VW>(kk, a.K + (int64_t)gs * a.ld + hoff, sub, nch, n > 0);
    load_slice<CH, LPR, VW>(vv, a.V + (int64_t)gs * a.ld + hoff, sub, nch, n > 0);
    float bc = 0.f;
    if constexpr (BIAS) bc = n > 0 ? a.bias[brow] : 0.f;
    for (int jl = 0; jl < nloop; ++jl) {
      if (use_drop && (jl & 3) == 0) drop_quad_refresh(dq, a.p_drop, a.seed, offs, h, i, jl);
      const bool valid = jl < n;
      const bool nvalid = jl + 1 < n;
      const int jn = gs + (nvalid ? jl + 1 : 0);
      V kn[CH], vn[CH];
      load_slice<CH, LPR, VW>(kn, a.K + (int64_t)jn * a.ld + hoff, sub, nch, nvalid);
      load_slice<CH, LPR, VW>(vn, a.V + (int64_t)jn * a.ld + hoff, sub, nch, nvalid);
      float bn = 0.f;
      if constexpr (BIAS) bn = nvalid ? a.bias[brow + jl + 1] : 0.f;
      float s = dot_slice<CH>(q, kk), dp = dot_slice<CH>(go, vv);
#pragma unroll
      for (int ofs = LPR / 2; ofs > 0; ofs >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, ofs);
        dp += __shfl_xor_sync(0xffffffffu, dp, ofs);
      }
      if constexpr (BIAS) s += bc;
      const float p = valid ? __expf(s - lse) : 0.f;
      const float ds = p * (dp * (use_drop ? drop_quad_scale(dq, jl) : 1.f) - dl);
      if constexpr (BIAS) {
        if (a.gbias && valid && sub == 0) a.gbias[brow + jl] = ds;
        bc = bn;
      }
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        if constexpr (VW == 4) {
          gq[c].x += ds * kk[c].x;
          gq[c].y += ds * kk[c].y;
          gq[c].z += ds * kk[c].z;
          gq[c].w += ds * kk[c].w;
        } else {
          gq[c] += ds * kk[c];
        }
        kk[c] = kn[c];
        vv[c] = vn[c];
      }
    }
  }
  if (row_ok) {
#pragma unroll
    for (int c = 0; c < CH; ++c) gq[c] = vscale(gq[c], a.scale);
    store_slice<CH, LPR, VW>(gq, a.dQ + (int64_t)i * a.ldg + hoff, sub, nch);
    store_slice_planes<CH, LPR, VW>(gq, a.dQp, i, hoff, sub, nch);
  }
}

// key-major backward: dK_j, dV_j (BIAS: p recomputed with the bias column of key j)
template <int CH, int LPR, bool BIAS, int VW>
__device__ __forceinline__ void attn_bwd_kv_body(const AttnArgs& a) {
  using V = typename VecT<VW>::T;
  constexpr int RPW = 32 / LPR;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sub = lane % LPR, rloc = lane / LPR;
  const int h = blockIdx.y;
  const int j = (blockIdx.x * kWarpsPerBlock + warp) * RPW + rloc;
  const bool row_ok = j < a.N;
  const int nch = a.hd / VW;
  const uint64_t offs = eff_offset(a);
  int gs = 0, n = 0;
  const float* bcol = nullptr;   // BIAS: bias column of (graph, head, key); query il at bcol[il * nmax]
  if (row_ok) {
    int g = find_graph(a.gptr, a.B, j);
    gs = a.gptr[g];
    n = a.gptr[g + 1] - gs;
    if constexpr (BIAS) bcol = a.bias + ((int64_t)g * a.H + h) * a.nmax * a.nmax + (j - gs);
  }
  const int nloop = warp_max_i(n);
  const int jl = j - gs;
  const int64_t hoff = (int64_t)h * a.hd;
  const int jr = row_ok ? j : 0;
  V kk[CH], vv[CH], gk[CH], gv[CH];
  load_slice<CH, LPR, VW>(kk, a.K + (int64_t)jr * a.ld + hoff, sub, nch, row_ok);
  load_slice<CH, LPR, VW>(vv, a.V + (int64_t)jr * a.ld + hoff, sub, nch, row_ok);
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    gk[c] = vzero<VW>();
    gv[c] = vzero<VW>();
  }
  V q[CH], go[CH];
  load_slice<CH, LPR, VW>(q, a.Q + (int64_t)gs * a.ld + hoff, sub, nch, n > 0);
  load_slice<CH, LPR, VW>(go, a.dO + (int64_t)gs * a.ldo + hoff, sub, nch, n > 0);
  for (int il = 0; il < nloop; ++il) {
    const bool valid = il < n;
    const int i = gs + (valid ? il : 0);
    const bool nvalid = il + 1 < n;
    const int in_ = gs + (nvalid ? il + 1 : 0);
    V qn[CH], gon[CH];
    load_slice<CH, LPR, VW>(qn, a.Q + (int64_t)in_ * a.ld + hoff, sub, nch, nvalid);
    load_slice<CH, LPR, VW>(gon, a.dO + (int64_t)in_ * a.ldo + hoff, sub, nch, nvalid);
    float s = dot_slice<CH>(q, kk), dp = dot_slice<CH>(go, vv);
#pragma unroll
    for (int ofs = LPR / 2; ofs > 0; ofs >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, ofs);
      dp += __shfl_xor_sync(0xffffffffu, dp, ofs);
    }
    const float lse = valid ? a.lsec[(int64_t)i * a.H + h] : 0.f;
    const float dl = valid ? a.deltac[(int64_t)i * a.H + h] : 0.f;
    float p;
    if constexpr (BIAS) p = valid ? __expf(s * a.scale + bcol[(int64_t)il * a.nmax] - lse) : 0.f;
    else p = valid ? __expf(s * a.scale - lse) : 0.f;
    float dsc = 1.f;
    if (a.p_drop > 0.f) {
      DropQuad dq;
      drop_quad_init(dq, a.p_drop);
      drop_quad_refresh(dq, a.p_drop, a.seed, offs, h, i, jl);
      dsc = drop_quad_scale(dq, jl);
    }
    const float pd = p * dsc;
    const float ds = p * (dp * dsc - dl) * a.scale;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      if constexpr (VW == 4) {
        gk[c].x += ds * q[c].x; gk[c].y += ds * q[c].y; gk[c].z += ds * q[c].z; gk[c].w += ds * q[c].w;
        gv[c].x += pd * go[c].x; gv[c].y += pd * go[c].y; gv[c].z += pd * go[c].z; gv[c].w += pd * go[c].w;
      } else {
        gk[c] += ds * q[c];
        gv[c] += pd * go[c];
      }
      q[c] = qn[c];
      go[c] = gon[c];
    }
  }
  if (row_ok) {
    store_slice<CH, LPR, VW>(gk, a.dK + (int64_t)j * a.ldg + hoff, sub, nch);
    store_slice<CH, LPR, VW>(gv, a.dV + (int64_t)j * a.ldg + hoff, sub, nch);
    store_slice_planes<CH, LPR, VW>(gk, a.dKp, j, hoff, sub, nch);
    store_slice_planes<CH, LPR, VW>(gv, a.dVp, j, hoff, sub, nch);
  }
}

// both backward passes in one grid (blockIdx.z picks the pass) so they share the SMs instead of queueing
template <int CH, int LPR, bool BIAS, int VW>
__global__ void __launch_bounds__(kWarpsPerBlock * 32) k_attn_bwd(AttnArgs a) {
  if (blockIdx.z == 0) attn_bwd_kv_body<CH, LPR, BIAS, VW>(a);
  else attn_bwd_q_body<CH, LPR, BIAS, VW>(a);
}

enum { KFWD = 0, KBWD = 1 };

// whether the float4 kernels take these head dim and leading dimensions (else the VW = 1 kernels run)
static bool attn_vec4(const AttnArgs& a, int which) {
  return a.hd % 4 == 0 && a.ld % 4 == 0 && a.ldo % 4 == 0 && (which == KFWD || a.ldg % 4 == 0);
}

template <int CH, int LPR, bool BIAS, int VW>
static void launch_one(int which, const AttnArgs& a, cudaStream_t stream) {
  constexpr int RPW = 32 / LPR;
  dim3 grid((unsigned)ceil_div(a.N, (int64_t)RPW * kWarpsPerBlock), (unsigned)a.H, which == KFWD ? 1 : 2);
  dim3 block(kWarpsPerBlock * 32);
  if (which == KFWD) k_attn_fwd<CH, LPR, BIAS, VW><<<grid, block, 0, stream>>>(a);
  else k_attn_bwd<CH, LPR, BIAS, VW><<<grid, block, 0, stream>>>(a);
}

static int dispatch(int which, const AttnArgs& a, cudaStream_t stream) {
  GPS_REQUIRE(a.hd > 0 && a.hd <= 192, GPS_ERR_UNSUPPORTED, "attention: head dim %d must be in 1..192", a.hd);
  if (a.N == 0) return GPS_OK;
  const int vw = attn_vec4(a, which) ? 4 : 1;
  const int nch = a.hd / vw;
  // smallest power-of-two lane group with <= 6 chunks per lane
  int lpr = 1;
  while ((nch + lpr - 1) / lpr > 6) lpr *= 2;
  const int ch = (nch + lpr - 1) / lpr;
#define GPS_ATTN_CASE(VWV, CHV, LPRV)                                  \
  if (vw == VWV && ch == CHV && lpr == LPRV) {                         \
    if (a.bias) launch_one<CHV, LPRV, true, VWV>(which, a, stream);    \
    else launch_one<CHV, LPRV, false, VWV>(which, a, stream);          \
    GPS_LAUNCH_CHECK();                                                \
    return GPS_OK;                                                     \
  }
  GPS_ATTN_CASE(4, 1, 1) GPS_ATTN_CASE(4, 2, 1) GPS_ATTN_CASE(4, 3, 1) GPS_ATTN_CASE(4, 4, 1) GPS_ATTN_CASE(4, 5, 1)
  GPS_ATTN_CASE(4, 6, 1) GPS_ATTN_CASE(4, 4, 2) GPS_ATTN_CASE(4, 5, 2) GPS_ATTN_CASE(4, 6, 2) GPS_ATTN_CASE(4, 4, 4)
  GPS_ATTN_CASE(4, 5, 4) GPS_ATTN_CASE(4, 6, 4) GPS_ATTN_CASE(4, 4, 8) GPS_ATTN_CASE(4, 5, 8) GPS_ATTN_CASE(4, 6, 8)
  GPS_ATTN_CASE(1, 1, 1) GPS_ATTN_CASE(1, 2, 1) GPS_ATTN_CASE(1, 3, 1) GPS_ATTN_CASE(1, 4, 1) GPS_ATTN_CASE(1, 5, 1)
  GPS_ATTN_CASE(1, 6, 1) GPS_ATTN_CASE(1, 4, 2) GPS_ATTN_CASE(1, 5, 2) GPS_ATTN_CASE(1, 6, 2) GPS_ATTN_CASE(1, 4, 4)
  GPS_ATTN_CASE(1, 5, 4) GPS_ATTN_CASE(1, 6, 4) GPS_ATTN_CASE(1, 4, 8) GPS_ATTN_CASE(1, 5, 8) GPS_ATTN_CASE(1, 6, 8)
  GPS_ATTN_CASE(1, 4, 16) GPS_ATTN_CASE(1, 5, 16) GPS_ATTN_CASE(1, 6, 16) GPS_ATTN_CASE(1, 4, 32)
  GPS_ATTN_CASE(1, 5, 32) GPS_ATTN_CASE(1, 6, 32)
#undef GPS_ATTN_CASE
  set_error("attention: no kernel for head dim %d", a.hd);
  return GPS_ERR_UNSUPPORTED;
}

}  // namespace

int attention_fwd(const GpsGraph& g, int64_t heads, int64_t hd, const float* Q, const float* K, const float* V,
                  int64_t ld, float* O, int64_t ldo, float* lse, float p_drop, uint64_t seed, uint64_t offset,
                  cudaStream_t stream, const unsigned long long* offset_dev, Planes Op, const GpsAttnBias* bias) {
  AttnArgs a{};
  a.offset_dev = offset_dev;
  a.Op = Op;
  if (bias) { a.bias = bias->bias; a.nmax = bias->nmax; }
  a.gptr = g.graph_ptr; a.B = (int)g.B; a.N = (int)g.N; a.H = (int)heads; a.hd = (int)hd;
  a.Q = Q; a.K = K; a.V = V; a.ld = ld; a.O = O; a.ldo = ldo; a.lse = lse;
  a.scale = 1.f / sqrtf((float)hd); a.p_drop = p_drop; a.seed = seed; a.offset = offset;
  return dispatch(KFWD, a, stream);
}

int attention_bwd(const GpsGraph& g, int64_t heads, int64_t hd, const float* Q, const float* K, const float* V,
                  int64_t ld, const float* O, const float* dO, int64_t ldo, const float* lse, float* delta,
                  float* dQ, float* dK, float* dV, int64_t ldg, float p_drop, uint64_t seed, uint64_t offset,
                  cudaStream_t stream, const unsigned long long* offset_dev, Planes dQp, Planes dKp, Planes dVp,
                  const GpsAttnBias* bias) {
  AttnArgs a{};
  a.offset_dev = offset_dev;
  if (bias) { a.bias = bias->bias; a.nmax = bias->nmax; a.gbias = bias->grad_bias; }
  a.dQp = dQp; a.dKp = dKp; a.dVp = dVp;
  a.gptr = g.graph_ptr; a.B = (int)g.B; a.N = (int)g.N; a.H = (int)heads; a.hd = (int)hd;
  a.Q = Q; a.K = K; a.V = V; a.ld = ld; a.Oc = O; a.dO = dO; a.ldo = ldo; a.lsec = lse;
  a.delta = delta; a.deltac = delta; a.dQ = dQ; a.dK = dK; a.dV = dV; a.ldg = ldg;
  a.scale = 1.f / sqrtf((float)hd); a.p_drop = p_drop; a.seed = seed; a.offset = offset;
  GPS_REQUIRE(a.hd > 0 && a.hd <= 192, GPS_ERR_UNSUPPORTED, "attention: head dim %d must be in 1..192", a.hd);
  if (a.gbias)   // entries of padded rows / columns stay 0; the kernel writes every in-graph (query, key) pair
    GPS_CUDA(cudaMemsetAsync(a.gbias, 0, (size_t)(g.B * heads * a.nmax * a.nmax) * sizeof(float), stream));
  if (a.N == 0) return GPS_OK;
  const int64_t nt = (int64_t)a.N * a.H * 8;
  if (attn_vec4(a, KBWD)) k_attn_delta<4><<<(unsigned)ceil_div(nt, (int64_t)256), 256, 0, stream>>>(a);
  else k_attn_delta<1><<<(unsigned)ceil_div(nt, (int64_t)256), 256, 0, stream>>>(a);
  GPS_LAUNCH_CHECK();
  return dispatch(KBWD, a, stream);
}

}  // namespace gps
