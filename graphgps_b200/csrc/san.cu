// san.cu — the SAN layer (graphgps/layer/san_layer.py:10-210 with full_graph=True, batch_norm=True, layer_norm=False,
// residual=True, use_bias=False), its attention kernels and its C ABI.
//
// Attention, for destination (query) node i and head h, with the clamp bounding every exponent (no running max):
//   real edge k: j -> i   t = sum_c K[j,c] Q[i,c] E[k,c] / sqrt(hd)     s = exp(clamp(t, -5, 5)) / (gamma + 1)
//   fake pair j -> i      t = sum_c K2[j,c] Q2'[i,c] / sqrt(hd)         s = gamma exp(clamp(t, -5, 5)) / (gamma + 1)
//   attn[i] = sum s V[j] / (sum s + 1e-6)
// with Q2' = Q2 (.) E2 (E2 = W_E2 fake_edge_emb, one d-vector) and the fake pairs the complement of the real edges
// within each graph, without self pairs.  A row bitmap [N, ceil(nmax / 32)] (bit jl of row i: a real edge from the
// jl-th node of i's graph into i) is built once per call from the CSR, one thread per row, so no atomics and no memset;
// the kernels test it per pair, so the fake terms are never formed for real pairs (no cancelling subtraction).  Real
// edges are counted per edge (duplicates twice, self loops included); a pair with a real edge is excluded once.
//
// Kernels: one warp per (node row, head) over the node's graph range (the packed-row layout of attention.cu); the lanes
// take 32 keys at a time, each lane owns channels lane, lane + 32, ... of the accumulators.  Backward: a query-major
// pass (g_Q, g_Q2 and each real edge's g_E row, one writer per row) and a key-major pass (g_K, g_V, g_K2; real part over
// the CSC, fake part over the graph's queries, scores recomputed), then the fixed-order column sum
// g_E2 = sum_i g_Q2'[i] (.) Q2[i] and the fold's backward.  No float atomics: two runs give the same bits.
//
// SAN2Layer (GpsSanArgs.variant = 1) shares the layer and swaps the attention stage: k_san2_fwd / k_san2_bwd_q /
// k_san2_bwd_k / k_san2_gamma below (softmax per set with a running max, the learned float64 gamma read on the
// device); only the attention's saved buffers differ (R, F, lse in place of rz).
//
// Layer (one C call per direction; dense products on the TMA GEMM through layer_ops.cuh, BatchNorms through the bn_*
// stages of kernels.cuh):
//   forward:  planes -> bitmap + E2 -> [Q|K|V|Q2|K2] = x Wcat^T  (and E = edge_attr W_E^T on the side stream)
//             -> attention (+ drop_13) -> z1 = x + O_h(.) (+ BN1 sums) -> h1 = BN1(z1) (+ planes)
//             -> hid = drop_14(relu(FFN1(h1))) -> z2 = h1 + FFN2(hid) (+ BN2 sums) -> out = BN2(z2)
//   backward: the mirror image; the weight products run on the side stream.
#include <string.h>

#include "layer_ops.cuh"

namespace gps {

namespace {

constexpr int kSanWarps = 4;       // warps per CTA of the attention kernels
constexpr int kSanMaxHd = 192;
constexpr int kSanCh = kSanMaxHd / 32;   // accumulator channels per lane
constexpr int kSanRowChunk = 256;  // rows per partial of the g_E2 column sum
constexpr float kSanEps = 1e-6f;   // h_out = wV / (Z + 1e-6), san_layer.py:118

struct SanAttn {
  GpsGraph g;
  int H, hd;
  int64_t d;
  const float *Q, *K, *V, *Q2, *K2;   // [N, ld] column blocks
  int64_t ld;
  const float* E;                      // [E, d] edge projection, edge-id order
  const float* E2;                     // [d]
  const uint32_t* bits;                // [N, W]
  int W;
  float cr, cf, scale;                 // 1 / (gamma + 1), gamma / (gamma + 1), 1 / sqrt(hd)
};

__device__ __forceinline__ void plane_store1(const Planes& p, int64_t r, int64_t c, float v) {
  if (!p.hi) return;
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  p.hi[r * p.ld + c] = h;
  if (p.lo) p.lo[r * p.ld + c] = __float2bfloat16_rn(v - __bfloat162float(h));
}

__device__ __forceinline__ int graph_of_node(const int32_t* gp, int64_t B, int i) {   // last g with gp[g] <= i
  int lo = 0, hi = (int)B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(gp + mid) <= i) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ bool is_real(const SanAttn& a, int i, int jl) {
  return (__ldg(a.bits + (int64_t)i * a.W + (jl >> 5)) >> (jl & 31)) & 1u;
}

__device__ __forceinline__ float san_exp(float t) { return expf(fminf(fmaxf(t, -5.f), 5.f)); }
// torch.clamp passes the gradient where -5 <= t <= 5, bounds included
__device__ __forceinline__ float san_pass(float t) { return (t >= -5.f && t <= 5.f) ? 1.f : 0.f; }

__device__ __forceinline__ float drop_scale1(const DropCfg& c, int64_t flat) {
  const uint64_t off = c.offset + (c.offset_dev ? *c.offset_dev : 0ull);
  const float4 s = dropout_scale4(c.p, c.seed, off, c.site, (uint64_t)flat >> 2);
  const int k = (int)(flat & 3);
  return k == 0 ? s.x : k == 1 ? s.y : k == 2 ? s.z : s.w;
}

// ------------------------------------------------------------------------------- bitmap and E2 fold
// threads [0, N): row i of the bitmap, zeroed, then bit jl set for every in-edge j -> i (jl = j - first node of i's
// graph; an edge from outside i's graph is not a pair of the graph and sets nothing).  Threads [N, N + d), when E2 is
// set: E2[r] = sum_c W_E2[r, c] emb[c].
__global__ void k_san_prep(GpsGraph g, uint32_t* __restrict__ bits, int W, const float* __restrict__ We2,
                           const float* __restrict__ emb, float* __restrict__ E2, int64_t d) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < g.N) {
    const int i = (int)t;
    uint32_t* row = bits + (int64_t)i * W;
    for (int w = 0; w < W; ++w) row[w] = 0u;
    const int gi = graph_of_node(g.graph_ptr, g.B, i);
    const int g0 = g.graph_ptr[gi], g1 = g.graph_ptr[gi + 1];
    for (int e = g.dst_ptr[i]; e < g.dst_ptr[i + 1]; ++e) {
      const int j = g.dst_src[e];
      if (j < g0 || j >= g1) continue;
      const int jl = j - g0;
      row[jl >> 5] |= 1u << (jl & 31);
    }
    return;
  }
  const int64_t r = t - g.N;
  if (!E2 || r >= d) return;
  float acc = 0.f;
  for (int64_t c = 0; c < d; ++c) acc = fmaf(__ldg(We2 + r * d + c), __ldg(emb + c), acc);
  E2[r] = acc;
}

// ------------------------------------------------------------------------------- forward
// one warp per (i, h): attn = wV / (Z + eps) (and attn times the dropout scales in Od when drop.p > 0, with Od's planes),
// rz[i, h] = 1 / (Z + eps)
__global__ void __launch_bounds__(32 * kSanWarps) k_san_fwd(SanAttn a, float* __restrict__ O, float* __restrict__ Od,
                                                            int64_t ldo, Planes Odp, float* __restrict__ rz,
                                                            DropCfg drop) {
  __shared__ float s_q[kSanWarps][kSanMaxHd], s_q2[kSanWarps][kSanMaxHd];
  __shared__ float s_s[kSanWarps][32];
  __shared__ int s_j[kSanWarps][32];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t item = (int64_t)blockIdx.x * kSanWarps + w;
  if (item >= a.g.N * a.H) return;
  const int i = (int)(item / a.H), h = (int)(item % a.H), hd = a.hd;
  const int64_t col = (int64_t)h * hd;
  float* q = s_q[w];
  float* q2 = s_q2[w];
  for (int c = lane; c < hd; c += 32) {
    q[c] = a.Q[(int64_t)i * a.ld + col + c];
    q2[c] = a.Q2[(int64_t)i * a.ld + col + c] * __ldg(a.E2 + col + c);
  }
  __syncwarp();
  const int gi = graph_of_node(a.g.graph_ptr, a.g.B, i);
  const int g0 = a.g.graph_ptr[gi], g1 = a.g.graph_ptr[gi + 1];
  float acc[kSanCh];
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) acc[m] = 0.f;
  float z = 0.f;
  // fake pairs: every key of the graph but i itself and the real sources of i
  for (int j0 = g0; j0 < g1; j0 += 32) {
    const int j = j0 + lane;
    float s = 0.f;
    if (j < g1 && j != i && !is_real(a, i, j - g0)) {
      const float* k2 = a.K2 + (int64_t)j * a.ld + col;
      float t = 0.f;
      for (int c = 0; c < hd; ++c) t = fmaf(k2[c], q2[c], t);
      s = a.cf * san_exp(t * a.scale);
    }
    z += s;
    s_s[w][lane] = s;
    __syncwarp();
    const int nk = min(32, g1 - j0);
    for (int kk = 0; kk < nk; ++kk) {
      const float sk = s_s[w][kk];
      if (sk == 0.f) continue;
      const float* v = a.V + (int64_t)(j0 + kk) * a.ld + col;
#pragma unroll
      for (int m = 0; m < kSanCh; ++m) {
        const int c = lane + 32 * m;
        if (c < hd) acc[m] = fmaf(sk, v[c], acc[m]);
      }
    }
    __syncwarp();
  }
  // real edges into i, in CSR order
  const int e0 = a.g.dst_ptr[i], e1 = a.g.dst_ptr[i + 1];
  for (int eb = e0; eb < e1; eb += 32) {
    const int e = eb + lane;
    float s = 0.f;
    int j = 0;
    if (e < e1) {
      j = a.g.dst_src[e];
      const int64_t k = a.g.dst_eid[e];
      const float* kr = a.K + (int64_t)j * a.ld + col;
      const float* er = a.E + k * a.d + col;
      float t = 0.f;
      for (int c = 0; c < hd; ++c) t = fmaf(kr[c] * q[c], er[c], t);
      s = a.cr * san_exp(t * a.scale);
    }
    z += s;
    s_s[w][lane] = s;
    s_j[w][lane] = j;
    __syncwarp();
    const int nk = min(32, e1 - eb);
    for (int kk = 0; kk < nk; ++kk) {
      const float sk = s_s[w][kk];
      const float* v = a.V + (int64_t)s_j[w][kk] * a.ld + col;
#pragma unroll
      for (int m = 0; m < kSanCh; ++m) {
        const int c = lane + 32 * m;
        if (c < hd) acc[m] = fmaf(sk, v[c], acc[m]);
      }
    }
    __syncwarp();
  }
  z = warp_sum(z);
  const float r = 1.f / (z + kSanEps);
  if (lane == 0) rz[item] = r;
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) {
    const int c = lane + 32 * m;
    if (c >= hd) continue;
    const float o = acc[m] * r;
    const int64_t cc = col + c;
    O[(int64_t)i * ldo + cc] = o;
    float od = o;
    if (drop.p > 0.f) {
      od = o * drop_scale1(drop, (int64_t)i * a.d + cc);
      Od[(int64_t)i * ldo + cc] = od;
    }
    plane_store1(Odp, i, cc, od);
  }
}

// ------------------------------------------------------------------------------- backward
// Per (i, h): g_wV = gO[i] r, D = -(gO[i] . O[i]) r; for each term with score s (pre-clamp t) and value V[j]:
// g_t = s (g_wV . V[j] + D) [|t| <= 5].
// Query-major pass: g_Q, g_Q2 = g_Q2' (.) E2 into gY (+ planes), each real edge's g_E row (+ planes),
// pq[i] = g_Q2'[i] (.) Q2[i] (the terms of g_E2), Dq[i, h] = D.
struct SanGrad {
  float *gQ, *gK, *gV, *gQ2, *gK2;   // [N, ldg] column blocks
  int64_t ldg;
  Planes gQp, gKp, gVp, gQ2p, gK2p;
  float* gE;                          // [E, d]
  Planes gEp;
};

__global__ void __launch_bounds__(32 * kSanWarps) k_san_bwd_q(SanAttn a, const float* __restrict__ O,
                                                              const float* __restrict__ gO, int64_t ldo,
                                                              const float* __restrict__ rz, float* __restrict__ Dq,
                                                              SanGrad G, float* __restrict__ pq) {
  __shared__ float s_q[kSanWarps][kSanMaxHd], s_q2[kSanWarps][kSanMaxHd], s_g[kSanWarps][kSanMaxHd];
  __shared__ float s_t[kSanWarps][32];
  __shared__ int s_j[kSanWarps][32], s_k[kSanWarps][32];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t item = (int64_t)blockIdx.x * kSanWarps + w;
  if (item >= a.g.N * a.H) return;
  const int i = (int)(item / a.H), h = (int)(item % a.H), hd = a.hd;
  const int64_t col = (int64_t)h * hd;
  const float r = rz[item];
  float* q = s_q[w];
  float* q2 = s_q2[w];
  float* gw = s_g[w];
  float dd = 0.f;
  for (int c = lane; c < hd; c += 32) {
    q[c] = a.Q[(int64_t)i * a.ld + col + c];
    q2[c] = a.Q2[(int64_t)i * a.ld + col + c] * __ldg(a.E2 + col + c);
    const float go = gO[(int64_t)i * ldo + col + c];
    gw[c] = go * r;
    dd = fmaf(go, O[(int64_t)i * ldo + col + c], dd);
  }
  const float D = -warp_sum(dd) * r;
  if (lane == 0) Dq[item] = D;
  __syncwarp();
  const int gi = graph_of_node(a.g.graph_ptr, a.g.B, i);
  const int g0 = a.g.graph_ptr[gi], g1 = a.g.graph_ptr[gi + 1];
  float acc[kSanCh];
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) acc[m] = 0.f;
  for (int j0 = g0; j0 < g1; j0 += 32) {
    const int j = j0 + lane;
    float gt = 0.f;
    if (j < g1 && j != i && !is_real(a, i, j - g0)) {
      const float* k2 = a.K2 + (int64_t)j * a.ld + col;
      const float* v = a.V + (int64_t)j * a.ld + col;
      float t = 0.f, gv = 0.f;
      for (int c = 0; c < hd; ++c) {
        t = fmaf(k2[c], q2[c], t);
        gv = fmaf(gw[c], v[c], gv);
      }
      t *= a.scale;
      gt = a.cf * san_exp(t) * (gv + D) * san_pass(t) * a.scale;
    }
    s_t[w][lane] = gt;
    __syncwarp();
    const int nk = min(32, g1 - j0);
    for (int kk = 0; kk < nk; ++kk) {
      const float g = s_t[w][kk];
      if (g == 0.f) continue;
      const float* k2 = a.K2 + (int64_t)(j0 + kk) * a.ld + col;
#pragma unroll
      for (int m = 0; m < kSanCh; ++m) {
        const int c = lane + 32 * m;
        if (c < hd) acc[m] = fmaf(g, k2[c], acc[m]);
      }
    }
    __syncwarp();
  }
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) {   // acc = g_Q2'
    const int c = lane + 32 * m;
    if (c >= hd) continue;
    const int64_t cc = col + c;
    const float gq2 = acc[m] * __ldg(a.E2 + cc);
    G.gQ2[(int64_t)i * G.ldg + cc] = gq2;
    plane_store1(G.gQ2p, i, cc, gq2);
    pq[(int64_t)i * a.d + cc] = acc[m] * a.Q2[(int64_t)i * a.ld + cc];
    acc[m] = 0.f;
  }
  const int e0 = a.g.dst_ptr[i], e1 = a.g.dst_ptr[i + 1];
  for (int eb = e0; eb < e1; eb += 32) {
    const int e = eb + lane;
    float gt = 0.f;
    int j = 0, k = 0;
    if (e < e1) {
      j = a.g.dst_src[e];
      k = a.g.dst_eid[e];
      const float* kr = a.K + (int64_t)j * a.ld + col;
      const float* er = a.E + (int64_t)k * a.d + col;
      const float* v = a.V + (int64_t)j * a.ld + col;
      float t = 0.f, gv = 0.f;
      for (int c = 0; c < hd; ++c) {
        t = fmaf(kr[c] * q[c], er[c], t);
        gv = fmaf(gw[c], v[c], gv);
      }
      t *= a.scale;
      gt = a.cr * san_exp(t) * (gv + D) * san_pass(t) * a.scale;
    }
    s_t[w][lane] = gt;
    s_j[w][lane] = j;
    s_k[w][lane] = k;
    __syncwarp();
    const int nk = min(32, e1 - eb);
    for (int kk = 0; kk < nk; ++kk) {
      const float g = s_t[w][kk];
      const int jj = s_j[w][kk], ke = s_k[w][kk];
      const float* kr = a.K + (int64_t)jj * a.ld + col;
      const float* er = a.E + (int64_t)ke * a.d + col;
#pragma unroll
      for (int m = 0; m < kSanCh; ++m) {
        const int c = lane + 32 * m;
        if (c >= hd) continue;
        const float kc = kr[c];
        acc[m] = fmaf(g * kc, er[c], acc[m]);
        const float ge = g * kc * q[c];
        G.gE[(int64_t)ke * a.d + col + c] = ge;
        plane_store1(G.gEp, ke, col + c, ge);
      }
    }
    __syncwarp();
  }
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) {
    const int c = lane + 32 * m;
    if (c >= hd) continue;
    G.gQ[(int64_t)i * G.ldg + col + c] = acc[m];
    plane_store1(G.gQp, i, col + c, acc[m]);
  }
}

// Key-major pass, one warp per (j, h): g_K (real edges out of j, over the CSC), g_K2 (fake pairs: the graph's queries
// i != j without a real edge j -> i) and g_V (both), scores recomputed.
__global__ void __launch_bounds__(32 * kSanWarps) k_san_bwd_k(SanAttn a, const float* __restrict__ gO, int64_t ldo,
                                                              const float* __restrict__ rz,
                                                              const float* __restrict__ Dq, SanGrad G) {
  __shared__ float s_k[kSanWarps][kSanMaxHd], s_k2[kSanWarps][kSanMaxHd], s_v[kSanWarps][kSanMaxHd];
  __shared__ float s_t[kSanWarps][32], s_s[kSanWarps][32];
  __shared__ int s_i[kSanWarps][32], s_e[kSanWarps][32];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t item = (int64_t)blockIdx.x * kSanWarps + w;
  if (item >= a.g.N * a.H) return;
  const int j = (int)(item / a.H), h = (int)(item % a.H), hd = a.hd;
  const int64_t col = (int64_t)h * hd;
  float* kk_ = s_k[w];
  float* k2 = s_k2[w];
  float* vj = s_v[w];
  for (int c = lane; c < hd; c += 32) {
    kk_[c] = a.K[(int64_t)j * a.ld + col + c];
    k2[c] = a.K2[(int64_t)j * a.ld + col + c];
    vj[c] = a.V[(int64_t)j * a.ld + col + c];
  }
  __syncwarp();
  const int gi = graph_of_node(a.g.graph_ptr, a.g.B, j);
  const int g0 = a.g.graph_ptr[gi], g1 = a.g.graph_ptr[gi + 1];
  float gk[kSanCh], gv[kSanCh];
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) gk[m] = gv[m] = 0.f;
  // fake pairs j -> i
  for (int i0 = g0; i0 < g1; i0 += 32) {
    const int i = i0 + lane;
    float gt = 0.f, s = 0.f, r = 0.f;
    if (i < g1 && i != j && !is_real(a, i, j - g0)) {
      const float* q2 = a.Q2 + (int64_t)i * a.ld + col;
      const float* go = gO + (int64_t)i * ldo + col;
      float t = 0.f, gvv = 0.f;
      for (int c = 0; c < hd; ++c) {
        t = fmaf(k2[c], q2[c] * __ldg(a.E2 + col + c), t);
        gvv = fmaf(go[c], vj[c], gvv);
      }
      t *= a.scale;
      r = rz[(int64_t)i * a.H + h];
      s = a.cf * san_exp(t);
      gt = s * (gvv * r + Dq[(int64_t)i * a.H + h]) * san_pass(t) * a.scale;
    }
    s_t[w][lane] = gt;
    s_s[w][lane] = s * r;
    __syncwarp();
    const int nq = min(32, g1 - i0);
    for (int qq = 0; qq < nq; ++qq) {
      const float sr = s_s[w][qq];
      if (sr == 0.f) continue;
      const float g = s_t[w][qq];
      const float* q2 = a.Q2 + (int64_t)(i0 + qq) * a.ld + col;
      const float* go = gO + (int64_t)(i0 + qq) * ldo + col;
#pragma unroll
      for (int m = 0; m < kSanCh; ++m) {
        const int c = lane + 32 * m;
        if (c >= hd) continue;
        gk[m] = fmaf(g, q2[c] * __ldg(a.E2 + col + c), gk[m]);   // g_K2
        gv[m] = fmaf(sr, go[c], gv[m]);
      }
    }
    __syncwarp();
  }
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) {
    const int c = lane + 32 * m;
    if (c >= hd) continue;
    G.gK2[(int64_t)j * G.ldg + col + c] = gk[m];
    plane_store1(G.gK2p, j, col + c, gk[m]);
    gk[m] = 0.f;
  }
  // real edges j -> i, in CSC order
  const int e0 = a.g.src_ptr[j], e1 = a.g.src_ptr[j + 1];
  for (int eb = e0; eb < e1; eb += 32) {
    const int e = eb + lane;
    float gt = 0.f, sr = 0.f;
    int i = 0, k = 0;
    if (e < e1) {
      i = a.g.src_dst[e];
      k = a.g.src_eid[e];
      const float* q = a.Q + (int64_t)i * a.ld + col;
      const float* er = a.E + (int64_t)k * a.d + col;
      const float* go = gO + (int64_t)i * ldo + col;
      float t = 0.f, gvv = 0.f;
      for (int c = 0; c < hd; ++c) {
        t = fmaf(kk_[c] * q[c], er[c], t);
        gvv = fmaf(go[c], vj[c], gvv);
      }
      t *= a.scale;
      const float r = rz[(int64_t)i * a.H + h];
      const float s = a.cr * san_exp(t);
      gt = s * (gvv * r + Dq[(int64_t)i * a.H + h]) * san_pass(t) * a.scale;
      sr = s * r;
    }
    s_t[w][lane] = gt;
    s_s[w][lane] = sr;
    s_i[w][lane] = i;
    s_e[w][lane] = k;
    __syncwarp();
    const int nq = min(32, e1 - eb);
    for (int qq = 0; qq < nq; ++qq) {
      const float g = s_t[w][qq], s = s_s[w][qq];
      const int ii = s_i[w][qq], ke = s_e[w][qq];
      const float* q = a.Q + (int64_t)ii * a.ld + col;
      const float* er = a.E + (int64_t)ke * a.d + col;
      const float* go = gO + (int64_t)ii * ldo + col;
#pragma unroll
      for (int m = 0; m < kSanCh; ++m) {
        const int c = lane + 32 * m;
        if (c >= hd) continue;
        gk[m] = fmaf(g * q[c], er[c], gk[m]);
        gv[m] = fmaf(s, go[c], gv[m]);
      }
    }
    __syncwarp();
  }
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) {
    const int c = lane + 32 * m;
    if (c >= hd) continue;
    G.gK[(int64_t)j * G.ldg + col + c] = gk[m];
    plane_store1(G.gKp, j, col + c, gk[m]);
    G.gV[(int64_t)j * G.ldg + col + c] = gv[m];
    plane_store1(G.gVp, j, col + c, gv[m]);
  }
}

// part[b, c] = sum of pq[r, c] over the rows r of chunk b, in row order
__global__ void k_san_colsum_part(const float* __restrict__ pq, int64_t N, int64_t d, float* __restrict__ part) {
  const int64_t c = (int64_t)blockIdx.y * blockDim.x + threadIdx.x;
  if (c >= d) return;
  const int64_t r0 = (int64_t)blockIdx.x * kSanRowChunk, r1 = min(N, r0 + kSanRowChunk);
  float s = 0.f;
  for (int64_t r = r0; r < r1; ++r) s += pq[r * d + c];
  part[(int64_t)blockIdx.x * d + c] = s;
}

// g_E2 = sum of the partials in chunk order (written to gE2 when set); g_W_E2[r, c] = g_E2[r] emb[c] and
// g_emb[c] = sum_r g_E2[r] W_E2[r, c], written or added.  Block b takes rows / columns [32 b, 32 b + 32).
__global__ void k_san_fold_bwd(const float* __restrict__ part, int nparts, int64_t d, const float* __restrict__ We2,
                               const float* __restrict__ emb, float* __restrict__ gE2, float* __restrict__ gW,
                               float* __restrict__ gemb, int accumulate) {
  extern __shared__ float s_ge[];
  for (int64_t r = threadIdx.x; r < d; r += blockDim.x) {
    float s = 0.f;
    for (int b = 0; b < nparts; ++b) s += part[(int64_t)b * d + r];
    s_ge[r] = s;
    if (gE2 && blockIdx.x == 0) gE2[r] = s;
  }
  __syncthreads();
  const int64_t lo = (int64_t)blockIdx.x * 32, hi = min(d, lo + 32);
  if (gW)
    for (int64_t idx = threadIdx.x; idx < (hi - lo) * d; idx += blockDim.x) {
      const int64_t r = lo + idx / d, c = idx % d;
      const float v = s_ge[r] * emb[c];
      gW[r * d + c] = accumulate ? gW[r * d + c] + v : v;
    }
  if (gemb && threadIdx.x < 32 && lo + threadIdx.x < d) {
    const int64_t c = lo + threadIdx.x;
    float s = 0.f;
    for (int64_t r = 0; r < d; ++r) s = fmaf(s_ge[r], We2[r * d + c], s);
    gemb[c] = accumulate ? gemb[c] + s : s;
  }
}

// =================================================================================== SAN2 attention
// SAN2Layer (graphgps/layer/san2_layer.py): per (i, h) a softmax over the real in-edges and one over the fake pairs,
//   R = sum_k alpha_k V[j_k],  alpha = exp(t - max) / (sum exp(t - max) + 1e-16)     (pyg_softmax, san2_layer.py:11-33)
//   F = sum_p beta_p V[j_p],   beta likewise over the fake scores u
//   attn = (R + gamma F) / (gamma + 1)
// with gamma one float64 read on the device.  No clamp: each set keeps a running max, its accumulators are rescaled
// when the max grows, and its log-sum-exp lse = max + log(sum) is saved, so the backward recomputes alpha = exp(t -
// lse) and beta = exp(u - lse_f).  Backward, per (i, h), with g = g_attn[i]:
//   Dr = g . R, Df = g . F;  g_t = alpha (g . V[j] - Dr) / (gamma + 1),  g_u = gamma beta (g . V[j] - Df) / (gamma + 1)
//   g_gamma = sum_{i,h} (Df - Dr) / (gamma + 1)^2
constexpr float kSan2Eps = 1e-16f;   // pyg_softmax's denominator term (san2_layer.py:31)

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

struct San2Mix {
  float cr, cf;   // 1 / (gamma + 1), gamma / (gamma + 1), formed in float64 as the SAN path forms them on the host
};

__device__ __forceinline__ San2Mix san2_mix(const double* gamma) {
  const double gm = *gamma;
  return {(float)(1.0 / (gm + 1.0)), (float)(gm / (gm + 1.0))};
}

// One set's online softmax over chunks of 32 keys: the lane's score t (-inf when the lane has no key), value row v.
struct San2Acc {
  float acc[kSanCh];
  float m, z;   // running max (warp-uniform) and this lane's share of the sum
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int c = 0; c < kSanCh; ++c) acc[c] = 0.f;
    m = -INFINITY;
    z = 0.f;
  }
  // s_s / s_v: the warp's staging rows.  Returns after the chunk's values are accumulated.
  __device__ __forceinline__ void chunk(float t, const float* vrow, float* s_s, const float** s_v, int nk, int lane,
                                        int hd) {
    const float cm = warp_max(t);
    if (cm == -INFINITY) return;   // no key in this chunk (warp-uniform)
    const float mn = fmaxf(m, cm);
    const float corr = expf(m - mn);   // 0 on the first chunk (m = -inf), when acc and z are 0
    const float s = t == -INFINITY ? 0.f : expf(t - mn);
    z = z * corr + s;
#pragma unroll
    for (int c = 0; c < kSanCh; ++c) acc[c] *= corr;
    m = mn;
    s_s[lane] = s;
    s_v[lane] = vrow;
    __syncwarp();
    for (int kk = 0; kk < nk; ++kk) {
      const float sk = s_s[kk];
      if (sk == 0.f) continue;
      const float* v = s_v[kk];
#pragma unroll
      for (int c = 0; c < kSanCh; ++c) {
        const int cc = lane + 32 * c;
        if (cc < hd) acc[c] = fmaf(sk, v[cc], acc[c]);
      }
    }
    __syncwarp();
  }
};

// one warp per (i, h): R, F (pitch d), lse [2, N, H]; attn = cr R + cf F into O (and times the dropout scales into Od
// when drop.p > 0, with Od's planes)
__global__ void __launch_bounds__(32 * kSanWarps) k_san2_fwd(SanAttn a, const double* __restrict__ gamma,
                                                             float* __restrict__ O, float* __restrict__ Od, int64_t ldo,
                                                             Planes Odp, float* __restrict__ R, float* __restrict__ F,
                                                             float* __restrict__ lse, DropCfg drop) {
  __shared__ float s_q[kSanWarps][kSanMaxHd], s_q2[kSanWarps][kSanMaxHd];
  __shared__ float s_s[kSanWarps][32];
  __shared__ const float* s_v[kSanWarps][32];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t item = (int64_t)blockIdx.x * kSanWarps + w;
  if (item >= a.g.N * a.H) return;
  const int i = (int)(item / a.H), h = (int)(item % a.H), hd = a.hd;
  const int64_t col = (int64_t)h * hd, NH = a.g.N * a.H;
  const San2Mix mx = san2_mix(gamma);
  float* q = s_q[w];
  float* q2 = s_q2[w];
  for (int c = lane; c < hd; c += 32) {
    q[c] = a.Q[(int64_t)i * a.ld + col + c];
    q2[c] = a.Q2[(int64_t)i * a.ld + col + c] * __ldg(a.E2 + col + c);
  }
  __syncwarp();
  const int gi = graph_of_node(a.g.graph_ptr, a.g.B, i);
  const int g0 = a.g.graph_ptr[gi], g1 = a.g.graph_ptr[gi + 1];
  float o[kSanCh];
  // fake pairs: every key of the graph but i itself and the real sources of i
  San2Acc st;
  st.init();
  for (int j0 = g0; j0 < g1; j0 += 32) {
    const int j = j0 + lane;
    float t = -INFINITY;
    const float* vrow = nullptr;
    if (j < g1 && j != i && !is_real(a, i, j - g0)) {
      const float* k2 = a.K2 + (int64_t)j * a.ld + col;
      float u = 0.f;
      for (int c = 0; c < hd; ++c) u = fmaf(k2[c], q2[c], u);
      t = u * a.scale;
      vrow = a.V + (int64_t)j * a.ld + col;
    }
    st.chunk(t, vrow, s_s[w], s_v[w], min(32, g1 - j0), lane, hd);
  }
  float z = warp_sum(st.z);
  float r = 1.f / (z + kSan2Eps);
  if (lane == 0) lse[NH + item] = z > 0.f ? st.m + logf(z) : 0.f;
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) {
    const int c = lane + 32 * m;
    const float f = st.acc[m] * r;
    o[m] = mx.cf * f;
    if (c < hd) F[(int64_t)i * a.d + col + c] = f;
  }
  // real edges into i, in CSR order
  st.init();
  const int e0 = a.g.dst_ptr[i], e1 = a.g.dst_ptr[i + 1];
  for (int eb = e0; eb < e1; eb += 32) {
    const int e = eb + lane;
    float t = -INFINITY;
    const float* vrow = nullptr;
    if (e < e1) {
      const int j = a.g.dst_src[e];
      const int64_t k = a.g.dst_eid[e];
      const float* kr = a.K + (int64_t)j * a.ld + col;
      const float* er = a.E + k * a.d + col;
      float u = 0.f;
      for (int c = 0; c < hd; ++c) u = fmaf(kr[c] * q[c], er[c], u);
      t = u * a.scale;
      vrow = a.V + (int64_t)j * a.ld + col;
    }
    st.chunk(t, vrow, s_s[w], s_v[w], min(32, e1 - eb), lane, hd);
  }
  z = warp_sum(st.z);
  r = 1.f / (z + kSan2Eps);
  if (lane == 0) lse[item] = z > 0.f ? st.m + logf(z) : 0.f;
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) {
    const int c = lane + 32 * m;
    if (c >= hd) continue;
    const float rr = st.acc[m] * r;
    const int64_t cc = col + c;
    R[(int64_t)i * a.d + cc] = rr;
    const float ov = fmaf(mx.cr, rr, o[m]);
    O[(int64_t)i * ldo + cc] = ov;
    float od = ov;
    if (drop.p > 0.f) {
      od = ov * drop_scale1(drop, (int64_t)i * a.d + cc);
      Od[(int64_t)i * ldo + cc] = od;
    }
    plane_store1(Odp, i, cc, od);
  }
}

// Query-major pass, one warp per (i, h): Dr, Df [N, H]; g_Q2' -> g_Q2 = g_Q2' (.) E2 and pq = g_Q2' (.) Q2; g_Q and
// each real edge's g_E row.
__global__ void __launch_bounds__(32 * kSanWarps) k_san2_bwd_q(SanAttn a, const double* __restrict__ gamma,
                                                               const float* __restrict__ R,
                                                               const float* __restrict__ F,
                                                               const float* __restrict__ lse,
                                                               const float* __restrict__ gO, int64_t ldo,
                                                               float* __restrict__ Dr, float* __restrict__ Df,
                                                               SanGrad G, float* __restrict__ pq) {
  __shared__ float s_q[kSanWarps][kSanMaxHd], s_q2[kSanWarps][kSanMaxHd], s_g[kSanWarps][kSanMaxHd];
  __shared__ float s_t[kSanWarps][32];
  __shared__ int s_j[kSanWarps][32], s_k[kSanWarps][32];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t item = (int64_t)blockIdx.x * kSanWarps + w;
  if (item >= a.g.N * a.H) return;
  const int i = (int)(item / a.H), h = (int)(item % a.H), hd = a.hd;
  const int64_t col = (int64_t)h * hd, NH = a.g.N * a.H;
  const San2Mix mx = san2_mix(gamma);
  float* q = s_q[w];
  float* q2 = s_q2[w];
  float* gw = s_g[w];
  float dr = 0.f, df = 0.f;
  for (int c = lane; c < hd; c += 32) {
    q[c] = a.Q[(int64_t)i * a.ld + col + c];
    q2[c] = a.Q2[(int64_t)i * a.ld + col + c] * __ldg(a.E2 + col + c);
    const float go = gO[(int64_t)i * ldo + col + c];
    gw[c] = go;
    dr = fmaf(go, R[(int64_t)i * a.d + col + c], dr);
    df = fmaf(go, F[(int64_t)i * a.d + col + c], df);
  }
  dr = warp_sum(dr);
  df = warp_sum(df);
  if (lane == 0) {
    Dr[item] = dr;
    Df[item] = df;
  }
  const float lr = lse[item], lf = lse[NH + item];
  __syncwarp();
  const int gi = graph_of_node(a.g.graph_ptr, a.g.B, i);
  const int g0 = a.g.graph_ptr[gi], g1 = a.g.graph_ptr[gi + 1];
  float acc[kSanCh];
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) acc[m] = 0.f;
  for (int j0 = g0; j0 < g1; j0 += 32) {
    const int j = j0 + lane;
    float gt = 0.f;
    if (j < g1 && j != i && !is_real(a, i, j - g0)) {
      const float* k2 = a.K2 + (int64_t)j * a.ld + col;
      const float* v = a.V + (int64_t)j * a.ld + col;
      float t = 0.f, gv = 0.f;
      for (int c = 0; c < hd; ++c) {
        t = fmaf(k2[c], q2[c], t);
        gv = fmaf(gw[c], v[c], gv);
      }
      gt = mx.cf * expf(t * a.scale - lf) * (gv - df) * a.scale;
    }
    s_t[w][lane] = gt;
    __syncwarp();
    const int nk = min(32, g1 - j0);
    for (int kk = 0; kk < nk; ++kk) {
      const float g = s_t[w][kk];
      if (g == 0.f) continue;
      const float* k2 = a.K2 + (int64_t)(j0 + kk) * a.ld + col;
#pragma unroll
      for (int m = 0; m < kSanCh; ++m) {
        const int c = lane + 32 * m;
        if (c < hd) acc[m] = fmaf(g, k2[c], acc[m]);
      }
    }
    __syncwarp();
  }
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) {   // acc = g_Q2'
    const int c = lane + 32 * m;
    if (c >= hd) continue;
    const int64_t cc = col + c;
    const float gq2 = acc[m] * __ldg(a.E2 + cc);
    G.gQ2[(int64_t)i * G.ldg + cc] = gq2;
    plane_store1(G.gQ2p, i, cc, gq2);
    pq[(int64_t)i * a.d + cc] = acc[m] * a.Q2[(int64_t)i * a.ld + cc];
    acc[m] = 0.f;
  }
  const int e0 = a.g.dst_ptr[i], e1 = a.g.dst_ptr[i + 1];
  for (int eb = e0; eb < e1; eb += 32) {
    const int e = eb + lane;
    float gt = 0.f;
    int j = 0, k = 0;
    if (e < e1) {
      j = a.g.dst_src[e];
      k = a.g.dst_eid[e];
      const float* kr = a.K + (int64_t)j * a.ld + col;
      const float* er = a.E + (int64_t)k * a.d + col;
      const float* v = a.V + (int64_t)j * a.ld + col;
      float t = 0.f, gv = 0.f;
      for (int c = 0; c < hd; ++c) {
        t = fmaf(kr[c] * q[c], er[c], t);
        gv = fmaf(gw[c], v[c], gv);
      }
      gt = mx.cr * expf(t * a.scale - lr) * (gv - dr) * a.scale;
    }
    s_t[w][lane] = gt;
    s_j[w][lane] = j;
    s_k[w][lane] = k;
    __syncwarp();
    const int nk = min(32, e1 - eb);
    for (int kk = 0; kk < nk; ++kk) {
      const float g = s_t[w][kk];
      const int jj = s_j[w][kk], ke = s_k[w][kk];
      const float* kr = a.K + (int64_t)jj * a.ld + col;
      const float* er = a.E + (int64_t)ke * a.d + col;
#pragma unroll
      for (int m = 0; m < kSanCh; ++m) {
        const int c = lane + 32 * m;
        if (c >= hd) continue;
        const float kc = kr[c];
        acc[m] = fmaf(g * kc, er[c], acc[m]);
        const float ge = g * kc * q[c];
        G.gE[(int64_t)ke * a.d + col + c] = ge;
        plane_store1(G.gEp, ke, col + c, ge);
      }
    }
    __syncwarp();
  }
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) {
    const int c = lane + 32 * m;
    if (c >= hd) continue;
    G.gQ[(int64_t)i * G.ldg + col + c] = acc[m];
    plane_store1(G.gQp, i, col + c, acc[m]);
  }
}

// Key-major pass, one warp per (j, h): g_K (real edges out of j, over the CSC), g_K2 (fake pairs: the graph's queries
// i != j without a real edge j -> i) and g_V (both), the weights recomputed from the saved log-sum-exps.
__global__ void __launch_bounds__(32 * kSanWarps) k_san2_bwd_k(SanAttn a, const double* __restrict__ gamma,
                                                               const float* __restrict__ lse,
                                                               const float* __restrict__ gO, int64_t ldo,
                                                               const float* __restrict__ Dr,
                                                               const float* __restrict__ Df, SanGrad G) {
  __shared__ float s_k[kSanWarps][kSanMaxHd], s_k2[kSanWarps][kSanMaxHd], s_v[kSanWarps][kSanMaxHd];
  __shared__ float s_t[kSanWarps][32], s_s[kSanWarps][32];
  __shared__ int s_i[kSanWarps][32], s_e[kSanWarps][32];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t item = (int64_t)blockIdx.x * kSanWarps + w;
  if (item >= a.g.N * a.H) return;
  const int j = (int)(item / a.H), h = (int)(item % a.H), hd = a.hd;
  const int64_t col = (int64_t)h * hd, NH = a.g.N * a.H;
  const San2Mix mx = san2_mix(gamma);
  float* kk_ = s_k[w];
  float* k2 = s_k2[w];
  float* vj = s_v[w];
  for (int c = lane; c < hd; c += 32) {
    kk_[c] = a.K[(int64_t)j * a.ld + col + c];
    k2[c] = a.K2[(int64_t)j * a.ld + col + c];
    vj[c] = a.V[(int64_t)j * a.ld + col + c];
  }
  __syncwarp();
  const int gi = graph_of_node(a.g.graph_ptr, a.g.B, j);
  const int g0 = a.g.graph_ptr[gi], g1 = a.g.graph_ptr[gi + 1];
  float gk[kSanCh], gv[kSanCh];
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) gk[m] = gv[m] = 0.f;
  // fake pairs j -> i
  for (int i0 = g0; i0 < g1; i0 += 32) {
    const int i = i0 + lane;
    float gt = 0.f, sr = 0.f;
    if (i < g1 && i != j && !is_real(a, i, j - g0)) {
      const float* q2 = a.Q2 + (int64_t)i * a.ld + col;
      const float* go = gO + (int64_t)i * ldo + col;
      float t = 0.f, gvv = 0.f;
      for (int c = 0; c < hd; ++c) {
        t = fmaf(k2[c], q2[c] * __ldg(a.E2 + col + c), t);
        gvv = fmaf(go[c], vj[c], gvv);
      }
      const int64_t ih = (int64_t)i * a.H + h;
      sr = mx.cf * expf(t * a.scale - lse[NH + ih]);
      gt = sr * (gvv - Df[ih]) * a.scale;
    }
    s_t[w][lane] = gt;
    s_s[w][lane] = sr;
    __syncwarp();
    const int nq = min(32, g1 - i0);
    for (int qq = 0; qq < nq; ++qq) {
      const float s = s_s[w][qq];
      if (s == 0.f) continue;
      const float g = s_t[w][qq];
      const float* q2 = a.Q2 + (int64_t)(i0 + qq) * a.ld + col;
      const float* go = gO + (int64_t)(i0 + qq) * ldo + col;
#pragma unroll
      for (int m = 0; m < kSanCh; ++m) {
        const int c = lane + 32 * m;
        if (c >= hd) continue;
        gk[m] = fmaf(g, q2[c] * __ldg(a.E2 + col + c), gk[m]);   // g_K2
        gv[m] = fmaf(s, go[c], gv[m]);
      }
    }
    __syncwarp();
  }
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) {
    const int c = lane + 32 * m;
    if (c >= hd) continue;
    G.gK2[(int64_t)j * G.ldg + col + c] = gk[m];
    plane_store1(G.gK2p, j, col + c, gk[m]);
    gk[m] = 0.f;
  }
  // real edges j -> i, in CSC order
  const int e0 = a.g.src_ptr[j], e1 = a.g.src_ptr[j + 1];
  for (int eb = e0; eb < e1; eb += 32) {
    const int e = eb + lane;
    float gt = 0.f, sr = 0.f;
    int i = 0, k = 0;
    if (e < e1) {
      i = a.g.src_dst[e];
      k = a.g.src_eid[e];
      const float* q = a.Q + (int64_t)i * a.ld + col;
      const float* er = a.E + (int64_t)k * a.d + col;
      const float* go = gO + (int64_t)i * ldo + col;
      float t = 0.f, gvv = 0.f;
      for (int c = 0; c < hd; ++c) {
        t = fmaf(kk_[c] * q[c], er[c], t);
        gvv = fmaf(go[c], vj[c], gvv);
      }
      const int64_t ih = (int64_t)i * a.H + h;
      sr = mx.cr * expf(t * a.scale - lse[ih]);
      gt = sr * (gvv - Dr[ih]) * a.scale;
    }
    s_t[w][lane] = gt;
    s_s[w][lane] = sr;
    s_i[w][lane] = i;
    s_e[w][lane] = k;
    __syncwarp();
    const int nq = min(32, e1 - eb);
    for (int qq = 0; qq < nq; ++qq) {
      const float g = s_t[w][qq], s = s_s[w][qq];
      const int ii = s_i[w][qq], ke = s_e[w][qq];
      const float* q = a.Q + (int64_t)ii * a.ld + col;
      const float* er = a.E + (int64_t)ke * a.d + col;
      const float* go = gO + (int64_t)ii * ldo + col;
#pragma unroll
      for (int m = 0; m < kSanCh; ++m) {
        const int c = lane + 32 * m;
        if (c >= hd) continue;
        gk[m] = fmaf(g * q[c], er[c], gk[m]);
        gv[m] = fmaf(s, go[c], gv[m]);
      }
    }
    __syncwarp();
  }
#pragma unroll
  for (int m = 0; m < kSanCh; ++m) {
    const int c = lane + 32 * m;
    if (c >= hd) continue;
    G.gK[(int64_t)j * G.ldg + col + c] = gk[m];
    plane_store1(G.gKp, j, col + c, gk[m]);
    G.gV[(int64_t)j * G.ldg + col + c] = gv[m];
    plane_store1(G.gVp, j, col + c, gv[m]);
  }
}

// g_gamma = sum over (i, h) of (Df - Dr) / (gamma + 1)^2, one CTA: each thread sums a fixed stride of items in float64,
// then a fixed tree; written, or added when accumulate
constexpr int kSan2GammaThreads = 256;
__global__ void __launch_bounds__(kSan2GammaThreads) k_san2_gamma(const float* __restrict__ Dr,
                                                                  const float* __restrict__ Df, int64_t n,
                                                                  const double* __restrict__ gamma,
                                                                  double* __restrict__ gg, int accumulate) {
  __shared__ double s[kSan2GammaThreads];
  double acc = 0.0;
  for (int64_t t = threadIdx.x; t < n; t += kSan2GammaThreads) acc += (double)Df[t] - (double)Dr[t];
  s[threadIdx.x] = acc;
  __syncthreads();
  for (int o = kSan2GammaThreads / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double gp1 = *gamma + 1.0;
    const double v = s[0] / (gp1 * gp1);
    *gg = accumulate ? *gg + v : v;
  }
}

// ------------------------------------------------------------------------------- launchers
int san_check(int64_t d, int64_t H) {
  GPS_REQUIRE(H > 0 && d > 0 && d % H == 0, GPS_ERR_ARG, "san: d %lld must be a positive multiple of heads %lld",
              (long long)d, (long long)H);
  GPS_REQUIRE(d % 4 == 0 && d <= 4096, GPS_ERR_UNSUPPORTED, "san: d must be a multiple of 4 and <= 4096 (got %lld)",
              (long long)d);
  GPS_REQUIRE(d / H <= kSanMaxHd, GPS_ERR_UNSUPPORTED, "san: head dim %lld > %d is not built", (long long)(d / H),
              kSanMaxHd);
  return GPS_OK;
}

int san_words(int64_t nmax) { return (int)ceil_div(nmax > 0 ? nmax : 1, 32); }

SanAttn san_attn(const GpsGraph& g, int64_t H, int64_t hd, const float* Y, int64_t ld, const float* E, const float* E2,
                 const uint32_t* bits, int64_t nmax, float gamma) {
  SanAttn a;
  a.g = g; a.H = (int)H; a.hd = (int)hd; a.d = H * hd;
  const int64_t d = a.d;
  a.Q = Y; a.K = Y + d; a.V = Y + 2 * d; a.Q2 = Y + 3 * d; a.K2 = Y + 4 * d;
  a.ld = ld; a.E = E; a.E2 = E2; a.bits = bits; a.W = san_words(nmax);
  a.cr = (float)(1.0 / ((double)gamma + 1.0));
  a.cf = (float)((double)gamma / ((double)gamma + 1.0));
  a.scale = (float)(1.0 / sqrt((double)hd));
  return a;
}

int san_prep(const GpsGraph& g, uint32_t* bits, int64_t nmax, const float* We2, const float* emb, float* E2, int64_t d,
             cudaStream_t st) {
  const int64_t n = g.N + (E2 ? d : 0);
  if (n == 0) return GPS_OK;
  k_san_prep<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(g, bits, san_words(nmax), We2, emb, E2, d);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int san_attn_fwd(const SanAttn& a, float* O, float* Od, int64_t ldo, Planes Odp, float* rz, const DropCfg& drop,
                 cudaStream_t st) {
  const int64_t items = a.g.N * a.H;
  if (items == 0) return GPS_OK;
  k_san_fwd<<<(unsigned)ceil_div(items, kSanWarps), 32 * kSanWarps, 0, st>>>(a, O, Od, ldo, Odp, rz, drop);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int64_t san_parts(int64_t N) { return ceil_div(N > 0 ? N : 1, kSanRowChunk); }

// the fixed-order column sum g_E2 = sum_i pq[i] and the fold's backward (gW / gemb NULL: not wanted)
int san_e2_bwd(const float* pq, int64_t N, int64_t d, float* part, const float* We2, const float* emb, float* gE2,
               float* gW, float* gemb, bool accumulate, cudaStream_t st) {
  const int64_t nparts = san_parts(N);
  if (N > 0) {
    k_san_colsum_part<<<dim3((unsigned)nparts, (unsigned)ceil_div(d, 128)), 128, 0, st>>>(pq, N, d, part);
    GPS_LAUNCH_CHECK();
  } else {
    GPS_CUDA(cudaMemsetAsync(part, 0, (size_t)d * sizeof(float), st));
  }
  k_san_fold_bwd<<<(unsigned)ceil_div(d, 32), 256, (size_t)d * sizeof(float), st>>>(part, (int)nparts, d, We2, emb, gE2,
                                                                                  gW, gemb, accumulate ? 1 : 0);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

// both passes, then the g_E2 column sum and the fold's backward (gW / gemb NULL: not wanted)
int san_attn_bwd(const SanAttn& a, const float* O, const float* gO, int64_t ldo, const float* rz, float* Dq,
                 const SanGrad& G, float* pq, float* part, const float* We2, const float* emb, float* gE2, float* gW,
                 float* gemb, bool accumulate, cudaStream_t st) {
  const int64_t items = a.g.N * a.H, d = a.d;
  if (items > 0) {
    k_san_bwd_q<<<(unsigned)ceil_div(items, kSanWarps), 32 * kSanWarps, 0, st>>>(a, O, gO, ldo, rz, Dq, G, pq);
    GPS_LAUNCH_CHECK();
    k_san_bwd_k<<<(unsigned)ceil_div(items, kSanWarps), 32 * kSanWarps, 0, st>>>(a, gO, ldo, rz, Dq, G);
    GPS_LAUNCH_CHECK();
  }
  return san_e2_bwd(pq, a.g.N, d, part, We2, emb, gE2, gW, gemb, accumulate, st);
}

// SAN2's saved attention state: R, F [N, d] and lse [2, N, H]
struct San2Saved {
  float *R, *F, *lse;
};

int san2_attn_fwd(const SanAttn& a, const double* gamma, float* O, float* Od, int64_t ldo, Planes Odp,
                  const San2Saved& S, const DropCfg& drop, cudaStream_t st) {
  const int64_t items = a.g.N * a.H;
  if (items == 0) return GPS_OK;
  k_san2_fwd<<<(unsigned)ceil_div(items, kSanWarps), 32 * kSanWarps, 0, st>>>(a, gamma, O, Od, ldo, Odp, S.R, S.F,
                                                                               S.lse, drop);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

// both passes, the g_gamma reduction (gg NULL: not wanted), then the g_E2 column sum and the fold's backward as SAN's.
// D: [2, N, H] scratch (Dr, Df)
int san2_attn_bwd(const SanAttn& a, const double* gamma, const float* R, const float* F, const float* lse,
                  const float* gO, int64_t ldo, float* D,
                  const SanGrad& G, double* gg, float* pq, float* part, const float* We2, const float* emb, float* gE2,
                  float* gW, float* gemb, bool accumulate, cudaStream_t st) {
  const int64_t items = a.g.N * a.H, d = a.d;
  float *Dr = D, *Df = D + items;
  if (items > 0) {
    k_san2_bwd_q<<<(unsigned)ceil_div(items, kSanWarps), 32 * kSanWarps, 0, st>>>(a, gamma, R, F, lse, gO, ldo, Dr,
                                                                                   Df, G, pq);
    GPS_LAUNCH_CHECK();
    k_san2_bwd_k<<<(unsigned)ceil_div(items, kSanWarps), 32 * kSanWarps, 0, st>>>(a, gamma, lse, gO, ldo, Dr, Df, G);
    GPS_LAUNCH_CHECK();
  }
  if (gg) {
    k_san2_gamma<<<1, kSan2GammaThreads, 0, st>>>(Dr, Df, items, gamma, gg, accumulate ? 1 : 0);
    GPS_LAUNCH_CHECK();
  }
  return san_e2_bwd(pq, a.g.N, d, part, We2, emb, gE2, gW, gemb, accumulate, st);
}

// =================================================================================== layer
struct SanPlan {
  int64_t N, E, d, H, hd, nmax;
  int prec;
  bool train, grads_prezeroed, grads_accumulate, use_planes;
  int variant;                   // 0: SANLayer, 1: SAN2Layer
  float gamma;                   // variant 0
  const double* gamma_dev;       // variant 1: the learned gamma on the device
  DropCfg drop_attn, drop_ffn;   // sites 13, 14 (p = 0 in eval mode)
  // saved
  float *Wcat, *Y, *Ee, *E2, *rz, *attn, *attn_d, *z1, *h1, *hid, *z2, *bnbuf;
  San2Saved s2;                  // variant 1, in place of rz
  uint32_t* bits;
  Planes Wcat_p, WE_p, WO_p, W1_p, W2_p, x_p, e_p, attnd_p, h1_p, hid_p;
  int64_t saved_bytes;
  // forward workspace: the column sums of BN1 and BN2 [2][2][d]
  double* fstats;
  int64_t fwd_bytes;
  // backward workspace
  double* bsums;
  float *g_z2, *g_hid, *g_h1, *g_z1, *g_attn, *gY, *gE, *Dq, *pq, *part;   // Dq: [N, H], variant 1 [2, N, H]
  Planes gz2_p, ghid_p, gz1_p, gY_p, gE_p;
  int64_t bwd_bytes;
};

int make_plan(const GpsSanArgs* a, SanPlan* P, bool bind) {
  memset(P, 0, sizeof(*P));
  GPS_REQUIRE(a, GPS_ERR_ARG, "san: null args");
  GPS_TRY(san_check(a->d, a->heads));
  GPS_REQUIRE(a->precision == GPS_PREC_FP32 || a->precision == GPS_PREC_BF16, GPS_ERR_ARG,
              "san: unknown precision %d", a->precision);
  GPS_REQUIRE(a->graph.N >= 0 && a->graph.E >= 0 && a->graph.B >= 0, GPS_ERR_ARG, "san: negative graph sizes");
  GPS_REQUIRE(a->graph.N == 0 || a->graph.B > 0, GPS_ERR_ARG, "san: a batch with nodes needs at least one graph");
  GPS_REQUIRE(a->nmax >= 0 && (a->graph.N == 0 || a->nmax >= 1) && a->nmax <= a->graph.N, GPS_ERR_ARG,
              "san: nmax %lld must be the size of the largest graph (N = %lld)", (long long)a->nmax,
              (long long)a->graph.N);
  GPS_REQUIRE(a->dropout >= 0.f && a->dropout < 1.f, GPS_ERR_ARG, "san: dropout must be in [0,1)");
  GPS_REQUIRE(a->variant == 0 || a->variant == 1, GPS_ERR_UNSUPPORTED, "san: unknown variant %d (0: SANLayer, "
              "1: SAN2Layer)", a->variant);
  GPS_REQUIRE(a->variant == 1 || a->gamma >= 0.f, GPS_ERR_ARG, "san: gamma must be >= 0");
  const int64_t N = a->graph.N, E = a->graph.E, d = a->d;
  P->N = N; P->E = E; P->d = d; P->H = a->heads; P->hd = d / a->heads; P->nmax = a->nmax;
  P->prec = a->precision;
  P->variant = a->variant;
  P->gamma = a->gamma;
  P->gamma_dev = a->gamma_param;
  P->train = a->training != 0;
  set_grad_flags(P, a->flags);
  P->drop_attn = drop_cfg(a->dropout, P->train, a->seed, a->offset, a->offset_dev, GPS_SITE_SAN_ATTN);
  P->drop_ffn = drop_cfg(a->dropout, P->train, a->seed, a->offset, a->offset_dev, GPS_SITE_SAN_FFN);
  P->use_planes = d % 8 == 0;
  const bool lo = a->precision == GPS_PREC_FP32;

  Arena S(bind ? a->saved : nullptr, a->saved_bytes);
  if (!P->use_planes) P->Wcat = S.alloc<float>(5 * d * d);
  P->Y = S.alloc<float>(N * 5 * d);
  P->Ee = S.alloc<float>(E * d);
  P->E2 = S.alloc<float>(d);
  P->bits = S.alloc<uint32_t>(N * san_words(a->nmax));
  if (P->variant == 0) {
    P->rz = S.alloc<float>(N * P->H);
  } else {
    P->s2.lse = S.alloc<float>(2 * N * P->H);
    P->s2.R = S.alloc<float>(N * d);
    P->s2.F = S.alloc<float>(N * d);
  }
  P->attn = S.alloc<float>(N * d);
  P->attn_d = P->drop_attn.p > 0.f ? S.alloc<float>(N * d) : P->attn;
  P->z1 = S.alloc<float>(N * d);
  P->h1 = S.alloc<float>(N * d);
  P->hid = S.alloc<float>(N * 2 * d);
  P->z2 = S.alloc<float>(N * d);
  P->bnbuf = S.alloc<float>(2 * 2 * d);
  if (P->use_planes) {
    P->Wcat_p = arena_planes(S, 5 * d, d, lo);
    P->WE_p = arena_planes(S, d, d, lo);
    P->WO_p = arena_planes(S, d, d, lo);
    P->W1_p = arena_planes(S, 2 * d, d, lo);
    P->W2_p = arena_planes(S, d, 2 * d, lo);
    P->x_p = arena_planes(S, N, d, lo);
    P->e_p = arena_planes(S, E, d, lo);
    P->attnd_p = arena_planes(S, N, d, lo);
    P->h1_p = arena_planes(S, N, d, lo);
    P->hid_p = arena_planes(S, N, 2 * d, lo);
  }
  P->saved_bytes = S.used;
  GPS_REQUIRE(!S.overflow, GPS_ERR_ARG, "san: saved buffer too small (%lld < %lld)", (long long)a->saved_bytes,
              (long long)S.used);

  Arena F(bind ? a->workspace : nullptr, a->workspace_bytes);
  P->fstats = F.alloc<double>(2 * 2 * d);
  P->fwd_bytes = F.used;

  Arena Bk(bind ? a->workspace : nullptr, a->workspace_bytes);
  P->bsums = Bk.alloc<double>(2 * 2 * d);
  P->g_z2 = Bk.alloc<float>(N * d);
  P->g_hid = Bk.alloc<float>(N * 2 * d);
  P->g_h1 = Bk.alloc<float>(N * d);
  P->g_z1 = Bk.alloc<float>(N * d);
  P->g_attn = Bk.alloc<float>(N * d);
  P->gY = Bk.alloc<float>(N * 5 * d);
  P->gE = Bk.alloc<float>(E * d);
  P->Dq = Bk.alloc<float>((P->variant == 0 ? 1 : 2) * N * P->H);
  P->pq = Bk.alloc<float>(N * d);
  P->part = Bk.alloc<float>(san_parts(N) * d);
  if (P->use_planes) {
    P->gz2_p = arena_planes(Bk, N, d, lo);
    P->ghid_p = arena_planes(Bk, N, 2 * d, lo);
    P->gz1_p = arena_planes(Bk, N, d, lo);
    P->gY_p = arena_planes(Bk, N, 5 * d, lo);
    P->gE_p = arena_planes(Bk, E, d, lo);
  }
  P->bwd_bytes = Bk.used;
  return GPS_OK;
}

const GpsLinear* node_linears(const GpsSanArgs* a, int i) {
  const GpsLinear* ls[5] = {&a->Q, &a->K, &a->V, &a->Q2, &a->K2};
  return ls[i];
}

int check_params(const GpsSanArgs* a) {
  const struct { const GpsLinear* l; const char* name; bool bias; } ps[] = {
      {&a->Q, "attention.Q", false},    {&a->K, "attention.K", false},     {&a->V, "attention.V", false},
      {&a->Q2, "attention.Q_2", false}, {&a->K2, "attention.K_2", false},  {&a->E, "attention.E", false},
      {&a->E2, "attention.E_2", false}, {&a->O_h, "O_h", true},            {&a->ffn1, "FFN_h_layer1", true},
      {&a->ffn2, "FFN_h_layer2", true}};
  for (const auto& p : ps) {
    GPS_REQUIRE(p.l->weight, GPS_ERR_ARG, "san: missing parameter %s.weight", p.name);
    GPS_REQUIRE(!p.bias || p.l->bias, GPS_ERR_ARG, "san: missing parameter %s.bias", p.name);
  }
  GPS_REQUIRE(a->fake_edge_emb, GPS_ERR_ARG, "san: missing parameter attention.fake_edge_emb.weight");
  GPS_REQUIRE(a->bn1.weight && a->bn1.bias && a->bn1.running_mean && a->bn1.running_var, GPS_ERR_ARG,
              "san: missing parameter or buffer of batch_norm1_h");
  GPS_REQUIRE(a->bn2.weight && a->bn2.bias && a->bn2.running_mean && a->bn2.running_var, GPS_ERR_ARG,
              "san: missing parameter or buffer of batch_norm2_h");
  GPS_REQUIRE(a->variant == 0 || a->gamma_param, GPS_ERR_ARG, "san: missing parameter attention.gamma (SAN2Layer)");
  return GPS_OK;
}

// plan, buffers and parameters of one call, all before any CUDA call
int prepare(const GpsSanArgs* a, bool fwd, SanPlan* P) {
  GPS_TRY(make_plan(a, P, true));
  GPS_TRY(check_params(a));
  GPS_REQUIRE(a->x && a->saved && a->workspace, GPS_ERR_ARG, "san: x, saved and workspace are required");
  GPS_REQUIRE(P->E == 0 || a->edge_attr, GPS_ERR_ARG, "san: edge_attr is required");
  const int64_t ws = fwd ? P->fwd_bytes : P->bwd_bytes;
  GPS_REQUIRE(a->workspace_bytes >= ws, GPS_ERR_ARG, "san: workspace too small (%lld < %lld)",
              (long long)a->workspace_bytes, (long long)ws);
  if (fwd) GPS_REQUIRE(a->x_out, GPS_ERR_ARG, "san: x_out is required");
  else GPS_REQUIRE(a->grad_x_out && a->grad_x, GPS_ERR_ARG, "san: grad_x_out and grad_x are required");
  return GPS_OK;
}

BnView bn_slot(const SanPlan& P, int which, const GpsBatchNorm& bn, int64_t fwd_rows = -1) {
  return bn_view_at(P, P.bnbuf + (int64_t)which * 2 * P.d, P.fstats + (int64_t)which * 2 * P.d, P.d, bn, fwd_rows);
}

// =================================================================================== forward
int san_forward(const GpsSanArgs* a, cudaStream_t st) {
  SanPlan P;
  GPS_TRY(prepare(a, true, &P));
  const int64_t N = P.N, E = P.E, d = P.d;
  if (N == 0) return GPS_OK;
  if (P.train) GPS_CUDA(cudaMemsetAsync(P.fstats, 0, (size_t)2 * 2 * d * sizeof(double), st));
  // the weights (and x, edge_attr) -> bf16 planes, one launch; without planes the fp32 node weights are packed
  if (P.use_planes) {
    ToPlanesItem it[16];
    int n = 0;
    for (int i = 0; i < 5; ++i) it[n++] = {node_linears(a, i)->weight, d, (int)d, (int)d, P.Wcat_p.rows(i * d)};
    it[n++] = {a->E.weight, d, (int)d, (int)d, P.WE_p};
    it[n++] = {a->O_h.weight, d, (int)d, (int)d, P.WO_p};
    it[n++] = {a->ffn1.weight, d, (int)(2 * d), (int)d, P.W1_p};
    it[n++] = {a->ffn2.weight, 2 * d, (int)d, (int)(2 * d), P.W2_p};
    it[n++] = {a->x, d, (int)N, (int)d, P.x_p};
    if (E > 0) it[n++] = {a->edge_attr, d, (int)E, (int)d, P.e_p};
    GPS_TRY(to_planes(it, n, st));
  } else {
    for (int i = 0; i < 5; ++i)
      GPS_CUDA(cudaMemcpyAsync(P.Wcat + i * d * d, node_linears(a, i)->weight, (size_t)(d * d) * sizeof(float),
                               cudaMemcpyDeviceToDevice, st));
  }
  // the exclusion bitmap and E2 = W_E2 emb
  GPS_TRY(san_prep(a->graph, P.bits, P.nmax, a->E2.weight, a->fake_edge_emb, P.E2, d, st));
  // E = edge_attr W_E^T on the side stream, next to the node projection
  Side* sd;
  GPS_TRY(side_stream(&sd));
  if (E > 0) {
    GPS_TRY(sd->fork(st));
    GPS_TRY(gemm(linear_fwd(P, E, d, d, {a->edge_attr, d, P.e_p}, {a->E.weight, d, P.WE_p}, P.Ee, d), sd->s));
  }
  // [Q | K | V | Q2 | K2] = x Wcat^T
  const float* Wcat = P.use_planes ? nullptr : P.Wcat;   // with planes the product reads the planes only
  GPS_TRY(gemm(linear_fwd(P, N, 5 * d, d, {a->x, d, P.x_p}, {Wcat, d, P.Wcat_p}, P.Y, 5 * d), st));
  if (E > 0) GPS_TRY(sd->join(st));
  const SanAttn at = san_attn(a->graph, P.H, P.hd, P.Y, 5 * d, P.Ee, P.E2, P.bits, P.nmax, P.gamma);
  if (P.variant == 0) GPS_TRY(san_attn_fwd(at, P.attn, P.attn_d, d, P.attnd_p, P.rz, P.drop_attn, st));
  else GPS_TRY(san2_attn_fwd(at, P.gamma_dev, P.attn, P.attn_d, d, P.attnd_p, P.s2, P.drop_attn, st));
  // z1 = x + O_h(drop(attn)), BN1's column sums
  GemmParams g = linear_fwd(P, N, d, d, {P.attn_d, d, P.attnd_p}, {a->O_h.weight, d, P.WO_p}, P.z1, d, a->O_h.bias);
  g.R1 = a->x; g.ldr1 = (int)d;
  g.stats = P.train ? P.fstats : nullptr;
  GPS_TRY(gemm(g, st));
  // h1 = BN1(z1)
  GPS_TRY(bn_combine(P.z1, bn_slot(P, 0, a->bn1, N), nullptr, BnView(), P.h1, N, d, st, P.h1_p));
  // hid = drop(relu(h1 W1^T + b1))
  GemmParams g1 = linear_fwd(P, N, 2 * d, d, {P.h1, d, P.h1_p}, {a->ffn1.weight, d, P.W1_p}, P.hid, 2 * d,
                             a->ffn1.bias);
  g1.act = GPS_ACT_RELU; g1.Cp = P.hid_p;
  set_dropout(g1, P.drop_ffn);
  GPS_TRY(gemm(g1, st));
  // z2 = h1 + hid W2^T + b2, BN2's column sums; out = BN2(z2)
  GemmParams g2 = linear_fwd(P, N, d, 2 * d, {P.hid, 2 * d, P.hid_p}, {a->ffn2.weight, 2 * d, P.W2_p}, P.z2, d,
                             a->ffn2.bias);
  g2.R1 = P.h1; g2.ldr1 = (int)d;
  g2.stats = P.train ? P.fstats + 2 * d : nullptr;
  GPS_TRY(gemm(g2, st));
  return bn_combine(P.z2, bn_slot(P, 1, a->bn2, N), nullptr, BnView(), a->x_out, N, d, st);
}

// =================================================================================== backward
int zero_grads(const GpsSanArgs* a, const SanPlan& P, cudaStream_t st) {
  if (P.grads_prezeroed) return GPS_OK;
  const int64_t d = P.d;
  const GpsLinear* ls[10] = {&a->Q, &a->K, &a->V, &a->Q2, &a->K2, &a->E, &a->E2, &a->O_h, &a->ffn1, &a->ffn2};
  const int64_t rows[10] = {d, d, d, d, d, d, d, d, 2 * d, d}, cols[10] = {d, d, d, d, d, d, d, d, d, 2 * d};
  GPS_TRY(zero_linear_grads(ls, rows, cols, 10, st));
  for (const GpsBatchNorm* b : {&a->bn1, &a->bn2}) {
    if (b->grad_weight) GPS_CUDA(cudaMemsetAsync(b->grad_weight, 0, (size_t)d * sizeof(float), st));
    if (b->grad_bias) GPS_CUDA(cudaMemsetAsync(b->grad_bias, 0, (size_t)d * sizeof(float), st));
  }
  if (a->grad_fake_edge_emb) GPS_CUDA(cudaMemsetAsync(a->grad_fake_edge_emb, 0, (size_t)d * sizeof(float), st));
  if (P.variant == 1 && a->grad_gamma) GPS_CUDA(cudaMemsetAsync(a->grad_gamma, 0, sizeof(double), st));
  return GPS_OK;
}

int san_backward(const GpsSanArgs* a, cudaStream_t st) {
  SanPlan P;
  GPS_TRY(prepare(a, false, &P));
  const int64_t N = P.N, E = P.E, d = P.d;
  if (N == 0) return zero_grads(a, P, st);
  const DropCfg nodrop;
  Side* sd;
  GPS_TRY(side_stream(&sd));
  cudaStream_t s2 = sd->s;
  GPS_CUDA(cudaMemsetAsync(P.bsums, 0, (size_t)2 * 2 * d * sizeof(double), st));
  // BN2: g_z2
  const BnView v2 = bn_slot(P, 1, a->bn2);
  GPS_TRY(bn_bwd_reduce(a->grad_x_out, d, P.z2, d, N, d, v2, -1, nodrop, P.bsums + 2 * d, st));
  GPS_TRY(bn_bwd_apply(a->grad_x_out, d, P.z2, d, N, d, v2, -1, nodrop, P.bsums + 2 * d, P.g_z2, d, a->bn2.grad_weight,
                       a->bn2.grad_bias, st, P.grads_accumulate, P.gz2_p));
  const Operand g_z2{P.g_z2, d, P.gz2_p};
  // g_hid = (g_z2 W2) * relu'(hid) * drop_14
  GemmParams g = linear_dgrad(P, N, 2 * d, d, g_z2, {a->ffn2.weight, 2 * d, P.W2_p}, P.g_hid, 2 * d);
  set_act_mask(g, GPS_ACT_RELU, P.hid, nullptr, 2 * d);
  set_dropout(g, P.drop_ffn);
  g.Cp = P.ghid_p;
  GPS_TRY(gemm(g, st));
  const Operand g_hid{P.g_hid, 2 * d, P.ghid_p};
  GPS_TRY(sd->fork(st));
  GPS_TRY(linear_wgrad(P, g_z2, {P.hid, 2 * d, P.hid_p}, N, d, 2 * d, a->ffn2.grad_weight, a->ffn2.grad_bias, s2));
  GPS_TRY(linear_wgrad(P, g_hid, {P.h1, d, P.h1_p}, N, 2 * d, d, a->ffn1.grad_weight, a->ffn1.grad_bias, s2));
  // g_h1 = g_z2 + g_hid W1
  GemmParams gh = linear_dgrad(P, N, d, 2 * d, g_hid, {a->ffn1.weight, d, P.W1_p}, P.g_h1, d);
  gh.R1 = P.g_z2; gh.ldr1 = (int)d;
  GPS_TRY(gemm(gh, st));
  // BN1: g_z1
  const BnView v1 = bn_slot(P, 0, a->bn1);
  GPS_TRY(bn_bwd_reduce(P.g_h1, d, P.z1, d, N, d, v1, -1, nodrop, P.bsums, st));
  GPS_TRY(bn_bwd_apply(P.g_h1, d, P.z1, d, N, d, v1, -1, nodrop, P.bsums, P.g_z1, d, a->bn1.grad_weight,
                       a->bn1.grad_bias, st, P.grads_accumulate, P.gz1_p));
  const Operand g_z1{P.g_z1, d, P.gz1_p};
  // z1 = x + O_h(drop_13(attn)): g_attn = (g_z1 W_O) * drop_13
  GemmParams go = linear_dgrad(P, N, d, d, g_z1, {a->O_h.weight, d, P.WO_p}, P.g_attn, d);
  set_dropout(go, P.drop_attn);
  GPS_TRY(gemm(go, st));
  GPS_TRY(sd->fork(st));
  GPS_TRY(linear_wgrad(P, g_z1, {P.attn_d, d, P.attnd_p}, N, d, d, a->O_h.grad_weight, a->O_h.grad_bias, s2));
  // attention: g_Q | g_K | g_V | g_Q2 | g_K2 into gY (+ planes), g_E, and the fold's gradients
  const SanAttn at = san_attn(a->graph, P.H, P.hd, P.Y, 5 * d, P.Ee, P.E2, P.bits, P.nmax, P.gamma);
  SanGrad G;
  G.gQ = P.gY; G.gK = P.gY + d; G.gV = P.gY + 2 * d; G.gQ2 = P.gY + 3 * d; G.gK2 = P.gY + 4 * d;
  G.ldg = 5 * d;
  G.gQp = P.gY_p.cols(0); G.gKp = P.gY_p.cols(d); G.gVp = P.gY_p.cols(2 * d); G.gQ2p = P.gY_p.cols(3 * d);
  G.gK2p = P.gY_p.cols(4 * d);
  G.gE = P.gE; G.gEp = P.gE_p;
  if (P.variant == 0)
    GPS_TRY(san_attn_bwd(at, P.attn, P.g_attn, d, P.rz, P.Dq, G, P.pq, P.part, a->E2.weight, a->fake_edge_emb, nullptr,
                         a->E2.grad_weight, a->grad_fake_edge_emb, P.grads_accumulate, st));
  else
    GPS_TRY(san2_attn_bwd(at, P.gamma_dev, P.s2.R, P.s2.F, P.s2.lse, P.g_attn, d, P.Dq, G, a->grad_gamma, P.pq, P.part, a->E2.weight,
                          a->fake_edge_emb, nullptr, a->E2.grad_weight, a->grad_fake_edge_emb, P.grads_accumulate, st));
  // weight gradients of the five node projections (one product when the caller's buffers are consecutive) and of E
  GPS_TRY(sd->fork(st));
  const Operand gY{P.gY, 5 * d, P.gY_p};
  const Operand xo{a->x, d, P.x_p};
  bool packed = a->Q.grad_weight != nullptr;
  for (int i = 1; i < 5; ++i) packed = packed && node_linears(a, i)->grad_weight == a->Q.grad_weight + i * d * d;
  if (packed) {
    GPS_TRY(linear_wgrad(P, gY, xo, N, 5 * d, d, a->Q.grad_weight, nullptr, s2));
  } else {
    for (int i = 0; i < 5; ++i)
      GPS_TRY(linear_wgrad(P, {P.gY + i * d, 5 * d, P.gY_p.cols(i * d)}, xo, N, d, d, node_linears(a, i)->grad_weight,
                           nullptr, s2));
  }
  GPS_TRY(linear_wgrad(P, {P.gE, d, P.gE_p}, {a->edge_attr, d, P.e_p}, E, d, d, a->E.grad_weight, nullptr, s2));
  // grad_x = g_z1 + gY Wcat; grad_edge_attr = g_E W_E
  const float* Wcat = P.use_planes ? nullptr : P.Wcat;
  GemmParams gx = linear_dgrad(P, N, d, 5 * d, gY, {Wcat, d, P.Wcat_p}, a->grad_x, d);
  gx.R1 = P.g_z1; gx.ldr1 = (int)d;
  GPS_TRY(gemm(gx, st));
  if (a->grad_edge_attr && E > 0)
    GPS_TRY(gemm(linear_dgrad(P, E, d, d, {P.gE, d, P.gE_p}, {a->E.weight, d, P.WE_p}, a->grad_edge_attr, d), st));
  return sd->join(st);
}

}  // namespace

}  // namespace gps

// =================================================================================== C ABI
using namespace gps;

extern "C" int gps_san_plan(const GpsSanArgs* args, GpsSanPlan* plan) {
  GPS_REQUIRE(args && plan, GPS_ERR_ARG, "gps_san_plan: null argument");
  SanPlan P;
  GPS_TRY(make_plan(args, &P, false));
  plan->saved_bytes = P.saved_bytes;
  plan->fwd_workspace_bytes = P.fwd_bytes;
  plan->bwd_workspace_bytes = P.bwd_bytes;
  return GPS_OK;
}

extern "C" int gps_san_forward(const GpsSanArgs* args, void* stream) {
  return san_forward(args, (cudaStream_t)stream);
}

extern "C" int gps_san_backward(const GpsSanArgs* args, void* stream) {
  return san_backward(args, (cudaStream_t)stream);
}

extern "C" int64_t gps_san_attention_workspace_bytes(int64_t N, int64_t d, int64_t heads, int64_t nmax) {
  Arena A(nullptr, 0);
  A.alloc<uint32_t>(N * san_words(nmax));
  A.alloc<float>(N * (heads > 0 ? heads : 1));
  A.alloc<float>(N * d);
  A.alloc<float>(san_parts(N) * d);
  return A.used;
}

namespace {
// the stage calls' common checks and the workspace carve-up (bitmap | D | pq | part)
int san_stage_setup(const GpsGraph* g, int64_t heads, int64_t hd, int64_t nmax, int64_t ld, void* ws, int64_t ws_bytes,
                    uint32_t** bits, float** Dq, float** pq, float** part) {
  GPS_REQUIRE(g, GPS_ERR_ARG, "san attention: null graph");
  GPS_REQUIRE(heads > 0 && hd > 0, GPS_ERR_ARG, "san attention: heads and hd must be positive");
  GPS_TRY(san_check(heads * hd, heads));
  const int64_t d = heads * hd;
  GPS_REQUIRE(ld >= 5 * d, GPS_ERR_ARG, "san attention: ld %lld < 5 d", (long long)ld);
  GPS_REQUIRE(nmax >= 0 && (g->N == 0 || nmax >= 1) && nmax <= g->N, GPS_ERR_ARG, "san attention: bad nmax %lld",
              (long long)nmax);
  GPS_REQUIRE(ws && ws_bytes >= gps_san_attention_workspace_bytes(g->N, d, heads, nmax), GPS_ERR_ARG,
              "san attention: workspace too small");
  Arena A(ws, ws_bytes);
  *bits = A.alloc<uint32_t>(g->N * san_words(nmax));
  *Dq = A.alloc<float>(g->N * heads);
  *pq = A.alloc<float>(g->N * d);
  *part = A.alloc<float>(san_parts(g->N) * d);
  return GPS_OK;
}
}  // namespace

extern "C" int gps_san_attention_forward(const GpsGraph* g, int64_t heads, int64_t hd, const float* Y, int64_t ld,
                                         const float* E, const float* E2, float gamma, int64_t nmax, void* workspace,
                                         int64_t workspace_bytes, float* O, int64_t ldo, float* rz, void* stream) {
  uint32_t* bits;
  float *Dq, *pq, *part;
  GPS_TRY(san_stage_setup(g, heads, hd, nmax, ld, workspace, workspace_bytes, &bits, &Dq, &pq, &part));
  GPS_REQUIRE(Y && E2 && O && rz && (g->E == 0 || E), GPS_ERR_ARG, "san attention: null pointer");
  GPS_REQUIRE(ldo >= heads * hd, GPS_ERR_ARG, "san attention: ldo too small");
  cudaStream_t st = (cudaStream_t)stream;
  GPS_TRY(san_prep(*g, bits, nmax, nullptr, nullptr, nullptr, heads * hd, st));
  const SanAttn a = san_attn(*g, heads, hd, Y, ld, E, E2, bits, nmax, gamma);
  return san_attn_fwd(a, O, O, ldo, Planes(), rz, DropCfg(), st);
}

extern "C" int gps_san_attention_backward(const GpsGraph* g, int64_t heads, int64_t hd, const float* Y, int64_t ld,
                                          const float* E, const float* E2, float gamma, int64_t nmax, void* workspace,
                                          int64_t workspace_bytes, const float* O, const float* dO, int64_t ldo,
                                          const float* rz, float* dY, int64_t ldg, float* dE, float* dE2,
                                          void* stream) {
  uint32_t* bits;
  float *Dq, *pq, *part;
  GPS_TRY(san_stage_setup(g, heads, hd, nmax, ld, workspace, workspace_bytes, &bits, &Dq, &pq, &part));
  GPS_REQUIRE(Y && E2 && O && dO && rz && dY && dE2 && (g->E == 0 || (E && dE)), GPS_ERR_ARG,
              "san attention: null pointer");
  GPS_REQUIRE(ldo >= heads * hd && ldg >= 5 * heads * hd, GPS_ERR_ARG, "san attention: ldo / ldg too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t d = heads * hd;
  GPS_TRY(san_prep(*g, bits, nmax, nullptr, nullptr, nullptr, d, st));
  const SanAttn a = san_attn(*g, heads, hd, Y, ld, E, E2, bits, nmax, gamma);
  SanGrad G;
  G.gQ = dY; G.gK = dY + d; G.gV = dY + 2 * d; G.gQ2 = dY + 3 * d; G.gK2 = dY + 4 * d;
  G.ldg = ldg;
  G.gE = dE;
  return san_attn_bwd(a, O, dO, ldo, rz, Dq, G, pq, part, nullptr, nullptr, dE2, nullptr, nullptr, false, st);
}

extern "C" int64_t gps_san2_attention_workspace_bytes(int64_t N, int64_t d, int64_t heads, int64_t nmax) {
  Arena A(nullptr, 0);
  A.alloc<uint32_t>(N * san_words(nmax));
  A.alloc<float>(2 * N * (heads > 0 ? heads : 1));
  A.alloc<float>(N * d);
  A.alloc<float>(san_parts(N) * d);
  return A.used;
}

namespace {
// SAN2's stage calls: the SAN stage's checks with the workspace carve-up (bitmap | Dr, Df | pq | part)
int san2_stage_setup(const GpsGraph* g, int64_t heads, int64_t hd, int64_t nmax, int64_t ld, const double* gamma,
                     void* ws, int64_t ws_bytes, uint32_t** bits, float** D, float** pq, float** part) {
  GPS_REQUIRE(g, GPS_ERR_ARG, "san2 attention: null graph");
  GPS_REQUIRE(heads > 0 && hd > 0, GPS_ERR_ARG, "san2 attention: heads and hd must be positive");
  GPS_TRY(san_check(heads * hd, heads));
  const int64_t d = heads * hd;
  GPS_REQUIRE(ld >= 5 * d, GPS_ERR_ARG, "san2 attention: ld %lld < 5 d", (long long)ld);
  GPS_REQUIRE(nmax >= 0 && (g->N == 0 || nmax >= 1) && nmax <= g->N, GPS_ERR_ARG, "san2 attention: bad nmax %lld",
              (long long)nmax);
  GPS_REQUIRE(gamma, GPS_ERR_ARG, "san2 attention: null gamma");
  GPS_REQUIRE(ws && ws_bytes >= gps_san2_attention_workspace_bytes(g->N, d, heads, nmax), GPS_ERR_ARG,
              "san2 attention: workspace too small");
  Arena A(ws, ws_bytes);
  *bits = A.alloc<uint32_t>(g->N * san_words(nmax));
  *D = A.alloc<float>(2 * g->N * heads);
  *pq = A.alloc<float>(g->N * d);
  *part = A.alloc<float>(san_parts(g->N) * d);
  return GPS_OK;
}
}  // namespace

extern "C" int gps_san2_attention_forward(const GpsGraph* g, int64_t heads, int64_t hd, const float* Y, int64_t ld,
                                          const float* E, const float* E2, const double* gamma, int64_t nmax,
                                          void* workspace, int64_t workspace_bytes, float* O, int64_t ldo, float* R,
                                          float* F, float* lse, void* stream) {
  uint32_t* bits;
  float *D, *pq, *part;
  GPS_TRY(san2_stage_setup(g, heads, hd, nmax, ld, gamma, workspace, workspace_bytes, &bits, &D, &pq, &part));
  GPS_REQUIRE(Y && E2 && O && R && F && lse && (g->E == 0 || E), GPS_ERR_ARG, "san2 attention: null pointer");
  GPS_REQUIRE(ldo >= heads * hd, GPS_ERR_ARG, "san2 attention: ldo too small");
  cudaStream_t st = (cudaStream_t)stream;
  GPS_TRY(san_prep(*g, bits, nmax, nullptr, nullptr, nullptr, heads * hd, st));
  const SanAttn a = san_attn(*g, heads, hd, Y, ld, E, E2, bits, nmax, 0.f);
  San2Saved S;
  S.R = R; S.F = F; S.lse = lse;
  return san2_attn_fwd(a, gamma, O, O, ldo, Planes(), S, DropCfg(), st);
}

extern "C" int gps_san2_attention_backward(const GpsGraph* g, int64_t heads, int64_t hd, const float* Y, int64_t ld,
                                           const float* E, const float* E2, const double* gamma, int64_t nmax,
                                           void* workspace, int64_t workspace_bytes, const float* R, const float* F,
                                           const float* lse, const float* dO, int64_t ldo, float* dY, int64_t ldg,
                                           float* dE, float* dE2, double* dgamma, void* stream) {
  uint32_t* bits;
  float *D, *pq, *part;
  GPS_TRY(san2_stage_setup(g, heads, hd, nmax, ld, gamma, workspace, workspace_bytes, &bits, &D, &pq, &part));
  GPS_REQUIRE(Y && E2 && R && F && lse && dO && dY && dE2 && dgamma && (g->E == 0 || (E && dE)), GPS_ERR_ARG,
              "san2 attention: null pointer");
  GPS_REQUIRE(ldo >= heads * hd && ldg >= 5 * heads * hd, GPS_ERR_ARG, "san2 attention: ldo / ldg too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t d = heads * hd;
  GPS_TRY(san_prep(*g, bits, nmax, nullptr, nullptr, nullptr, d, st));
  const SanAttn a = san_attn(*g, heads, hd, Y, ld, E, E2, bits, nmax, 0.f);
  SanGrad G;
  G.gQ = dY; G.gK = dY + d; G.gV = dY + 2 * d; G.gQ2 = dY + 3 * d; G.gK2 = dY + 4 * d;
  G.ldg = ldg;
  G.gE = dE;
  return san2_attn_bwd(a, gamma, R, F, lse, dO, ldo, D, G, dgamma, pq, part, nullptr, nullptr, dE2, nullptr, nullptr, false, st);
}
