// performer_quad.cu — FAVOR+ linear attention evaluated in its pairwise form for batches of small graphs.
//
//   out_i = ( q'_i . (sum_j k'_j^T v_j) ) / ( q'_i . sum_j k'_j )  ==  sum_j (q'_i.k'_j) v_j / sum_j (q'_i.k'_j)
//
// (graphgps/layer/performer_layer.py:200-205 computes the left form; both are the same sums of positive terms).
// With n_g ~ 14 nodes per graph and m = 266 features the pairwise form needs n^2 (m + 64) multiply-adds per
// (graph, head) instead of 2 n m 64 — 5x fewer — and, more importantly, it maps onto the row-packed warp layout of
// attention.cu (no per-(graph, head) CTA with a 272x64 context, whose 4096 single-resident CTAs were latency bound:
// 2.8 ms backward at the C4 shape).  The padded rows of the reference's dense batch enter exactly as in
// performer.cu: (Nmax - n) k'_pad joins the denominator.  The per-graph context kernels remain the path for large
// graphs (the dispatcher switches on the mean graph size).
#include "kernels.cuh"

namespace gps {

namespace {

constexpr int DH = 64, MP = 272;
constexpr int LPR = 8;            // lanes per row
constexpr int RPW = 32 / LPR;     // rows per warp
constexpr int CQ = 9;             // float4 chunks of the 272 features per lane (8 lanes x 9 x 4 = 288 >= 272)
constexpr int CV = 2;             // float4 chunks of the 64-wide value / output per lane
constexpr int NQ = MP / 4;        // 68 chunks
constexpr int kWarps = 4;
constexpr float kEpsF = 1e-4f;

__device__ __forceinline__ int find_graph_q(const int* __restrict__ gptr, int B, int node) {
  int lo = 0, hi = B;
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (gptr[mid] <= node) lo = mid; else hi = mid;
  }
  return lo;
}
__device__ __forceinline__ float gsum(float v) {
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int wmax(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
template <int C, int NCH>
__device__ __forceinline__ void ld_slice(float4* dst, const float* row, int sub, bool ok) {
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const int ch = sub + c * LPR;
    dst[c] = (ok && ch < NCH) ? ld4(row + ch * 4) : f4zero();
  }
}
template <int C, int NCH>
__device__ __forceinline__ void st_slice(const float4* src, float* row, int sub) {
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const int ch = sub + c * LPR;
    if (ch < NCH) st4(row + ch * 4, src[c]);
  }
}
template <int C>
__device__ __forceinline__ float dotc(const float4* a, const float4* b) {
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < C; ++c) s += a[c].x * b[c].x + a[c].y * b[c].y + a[c].z * b[c].z + a[c].w * b[c].w;
  return s;
}
template <int C>
__device__ __forceinline__ float sumc(const float4* a) {
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < C; ++c) s += a[c].x + a[c].y + a[c].z + a[c].w;
  return s;
}

struct QArgs {
  const int* gptr; const int* nmax; int B, N, H, m; float ratio;
  const float* qf; const float* kf; const float* V; const float* gmax;
  float* O; float* den;                                  // forward outputs ([N,H*64], [N*H])
  const float* gO; float* gden; float* g_qf; float* g_kf; float* gV; float* gmrow;   // backward
};

// row r = (node i, head h) lives at qf/kf + (i*H + h)*MP and V/O + (i*H + h)*64
__global__ void __launch_bounds__(kWarps * 32) k_perf_quad_fwd(QArgs a) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, sub = lane % LPR, rloc = lane / LPR;
  const int h = blockIdx.y;
  const int i = (blockIdx.x * kWarps + warp) * RPW + rloc;
  const bool ok = i < a.N;
  int gs = 0, n = 0, g = 0;
  if (ok) {
    g = find_graph_q(a.gptr, a.B, i);
    gs = a.gptr[g];
    n = a.gptr[g + 1] - gs;
  }
  const int nloop = wmax(n);
  const int64_t r = (int64_t)(ok ? i : 0) * a.H + h;
  float4 q[CQ], o[CV];
  ld_slice<CQ, NQ>(q, a.qf + r * MP, sub, ok);
#pragma unroll
  for (int c = 0; c < CV; ++c) o[c] = f4zero();
  float den = 0.f;
  for (int jl = 0; jl < nloop; ++jl) {
    const bool valid = jl < n;
    const int64_t rj = (int64_t)(gs + (valid ? jl : 0)) * a.H + h;
    float4 k[CQ], v[CV];
    ld_slice<CQ, NQ>(k, a.kf + rj * MP, sub, valid);
    ld_slice<CV, DH / 4>(v, a.V + rj * DH, sub, valid);
    const float s = gsum(dotc<CQ>(q, k));   // 0 for invalid keys (k = 0)
    den += s;
#pragma unroll
    for (int c = 0; c < CV; ++c) o[c] = make_float4(fmaf(s, v[c].x, o[c].x), fmaf(s, v[c].y, o[c].y),
                                                   fmaf(s, v[c].z, o[c].z), fmaf(s, v[c].w, o[c].w));
  }
  const float qsum = gsum(sumc<CQ>(q));     // every lane takes part in the shuffle (q = 0 on idle rows)
  if (ok) {
    // padded rows of the reference's dense batch: (Nmax - n) k'_pad on the m real features
    const float kpad = a.ratio * (__expf(-a.gmax[g * a.H + h]) + kEpsF) * (float)(*a.nmax - n);
    den += kpad * qsum;                      // feature-padding entries of q' are 0
    const float inv = 1.f / den;
#pragma unroll
    for (int c = 0; c < CV; ++c) o[c] = f4scale(o[c], inv);
    st_slice<CV, DH / 4>(o, a.O + r * DH, sub);
    if (sub == 0) a.den[r] = den;
  }
}

// query-major backward: g_q'_i, g_den_i, and row i's pad-term stabiliser gradient into its own slot gmrow[i*H + h]
__global__ void __launch_bounds__(kWarps * 32) k_perf_quad_bwd_q(QArgs a) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, sub = lane % LPR, rloc = lane / LPR;
  const int h = blockIdx.y;
  const int i = (blockIdx.x * kWarps + warp) * RPW + rloc;
  const bool ok = i < a.N;
  int gs = 0, n = 0, g = 0;
  if (ok) {
    g = find_graph_q(a.gptr, a.B, i);
    gs = a.gptr[g];
    n = a.gptr[g + 1] - gs;
  }
  const int nloop = wmax(n);
  const int64_t r = (int64_t)(ok ? i : 0) * a.H + h;
  float4 q[CQ], gq[CQ], gu[CV], oo[CV];
  ld_slice<CQ, NQ>(q, a.qf + r * MP, sub, ok);
  ld_slice<CV, DH / 4>(gu, a.gO + r * DH, sub, ok);
  ld_slice<CV, DH / 4>(oo, a.O + r * DH, sub, ok);
  const float den = ok ? a.den[r] : 1.f;
  const float inv = 1.f / den;
  const float gden = -gsum(dotc<CV>(gu, oo)) * inv;       // d out / d den = -out / den
#pragma unroll
  for (int c = 0; c < CV; ++c) gu[c] = f4scale(gu[c], inv);   // g_u = gO / den
#pragma unroll
  for (int c = 0; c < CQ; ++c) gq[c] = f4zero();
  for (int jl = 0; jl < nloop; ++jl) {
    const bool valid = jl < n;
    const int64_t rj = (int64_t)(gs + (valid ? jl : 0)) * a.H + h;
    float4 k[CQ], v[CV];
    ld_slice<CQ, NQ>(k, a.kf + rj * MP, sub, valid);
    ld_slice<CV, DH / 4>(v, a.V + rj * DH, sub, valid);
    const float gsij = gsum(dotc<CV>(gu, v)) + gden;       // d / d s_ij
#pragma unroll
    for (int c = 0; c < CQ; ++c) gq[c] = make_float4(fmaf(gsij, k[c].x, gq[c].x), fmaf(gsij, k[c].y, gq[c].y),
                                                     fmaf(gsij, k[c].z, gq[c].z), fmaf(gsij, k[c].w, gq[c].w));
  }
  const float rq = gsum(sumc<CQ>(q));
  if (ok) {
    const float npad = (float)(*a.nmax - n);
    const float gm = a.gmax[g * a.H + h];
    const float kpad = a.ratio * (__expf(-gm) + kEpsF) * npad;
    const float c0 = gden * kpad;                          // den += kpad * sum_{j<m} q'_j
#pragma unroll
    for (int c = 0; c < CQ; ++c) {
      const int j0 = (sub + c * LPR) * 4;
      gq[c].x += (j0 + 0 < a.m) ? c0 : 0.f;
      gq[c].y += (j0 + 1 < a.m) ? c0 : 0.f;
      gq[c].z += (j0 + 2 < a.m) ? c0 : 0.f;
      gq[c].w += (j0 + 3 < a.m) ? c0 : 0.f;
    }
    st_slice<CQ, NQ>(gq, a.g_qf + r * MP, sub);
    if (sub == 0) {
      a.gden[r] = gden;
      // k'_pad = ratio (exp(-gmax) + eps):  d den / d gmax = -npad * ratio * exp(-gmax) * sum_j q'_j
      a.gmrow[r] = npad > 0.f ? -gden * npad * a.ratio * __expf(-gm) * rq : 0.f;
    }
  }
}

// key-major backward: g_k'_j = sum_i g_s_ij q'_i ;  g_v_j = sum_i s_ij g_u_i
__global__ void __launch_bounds__(kWarps * 32) k_perf_quad_bwd_kv(QArgs a) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, sub = lane % LPR, rloc = lane / LPR;
  const int h = blockIdx.y;
  const int j = (blockIdx.x * kWarps + warp) * RPW + rloc;
  const bool ok = j < a.N;
  int gs = 0, n = 0;
  if (ok) {
    const int g = find_graph_q(a.gptr, a.B, j);
    gs = a.gptr[g];
    n = a.gptr[g + 1] - gs;
  }
  const int nloop = wmax(n);
  const int64_t rj = (int64_t)(ok ? j : 0) * a.H + h;
  float4 k[CQ], gk[CQ], v[CV], gv[CV];
  ld_slice<CQ, NQ>(k, a.kf + rj * MP, sub, ok);
  ld_slice<CV, DH / 4>(v, a.V + rj * DH, sub, ok);
#pragma unroll
  for (int c = 0; c < CQ; ++c) gk[c] = f4zero();
#pragma unroll
  for (int c = 0; c < CV; ++c) gv[c] = f4zero();
  for (int il = 0; il < nloop; ++il) {
    const bool valid = il < n;
    const int64_t ri = (int64_t)(gs + (valid ? il : 0)) * a.H + h;
    float4 q[CQ], gu[CV];
    ld_slice<CQ, NQ>(q, a.qf + ri * MP, sub, valid);
    ld_slice<CV, DH / 4>(gu, a.gO + ri * DH, sub, valid);
    const float inv = valid ? 1.f / a.den[ri] : 0.f;
    const float gden = valid ? a.gden[ri] : 0.f;
    float s = dotc<CQ>(q, k), t = dotc<CV>(gu, v);
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    const float gsij = valid ? t * inv + gden : 0.f;
    const float su = s * inv;   // s_ij / den_i
#pragma unroll
    for (int c = 0; c < CQ; ++c) gk[c] = make_float4(fmaf(gsij, q[c].x, gk[c].x), fmaf(gsij, q[c].y, gk[c].y),
                                                     fmaf(gsij, q[c].z, gk[c].z), fmaf(gsij, q[c].w, gk[c].w));
#pragma unroll
    for (int c = 0; c < CV; ++c) gv[c] = make_float4(fmaf(su, gu[c].x, gv[c].x), fmaf(su, gu[c].y, gv[c].y),
                                                     fmaf(su, gu[c].z, gv[c].z), fmaf(su, gu[c].w, gv[c].w));
  }
  if (ok) {
    st_slice<CQ, NQ>(gk, a.g_kf + rj * MP, sub);
    st_slice<CV, DH / 4>(gv, a.gV + rj * DH, sub);
  }
}

}  // namespace

int perf_quad_fwd(const GpsGraph& g, int64_t H, int64_t m, const int* nmax, const float* qf, const float* kf,
                  const float* V, const float* gmax, float* O, float* den, cudaStream_t st) {
  if (g.N == 0) return GPS_OK;
  QArgs a{};
  a.gptr = g.graph_ptr; a.nmax = nmax; a.B = (int)g.B; a.N = (int)g.N; a.H = (int)H; a.m = (int)m;
  a.ratio = 1.f / sqrtf((float)m); a.qf = qf; a.kf = kf; a.V = V; a.gmax = gmax; a.O = O; a.den = den;
  dim3 grid((unsigned)ceil_div(g.N, (int64_t)RPW * kWarps), (unsigned)H);
  k_perf_quad_fwd<<<grid, kWarps * 32, 0, st>>>(a);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int perf_quad_bwd(const GpsGraph& g, int64_t H, int64_t m, const int* nmax, const float* qf, const float* kf,
                  const float* V, const float* gmax, const float* O, const float* den, const float* gO, float* gden,
                  float* g_qf, float* g_kf, float* gV, float* gmrow, cudaStream_t st) {
  if (g.N == 0) return GPS_OK;
  QArgs a{};
  a.gptr = g.graph_ptr; a.nmax = nmax; a.B = (int)g.B; a.N = (int)g.N; a.H = (int)H; a.m = (int)m;
  a.ratio = 1.f / sqrtf((float)m); a.qf = qf; a.kf = kf; a.V = V; a.gmax = gmax;
  a.O = const_cast<float*>(O); a.den = const_cast<float*>(den); a.gO = gO; a.gden = gden;
  a.g_qf = g_qf; a.g_kf = g_kf; a.gV = gV; a.gmrow = gmrow;
  dim3 grid((unsigned)ceil_div(g.N, (int64_t)RPW * kWarps), (unsigned)H);
  k_perf_quad_bwd_q<<<grid, kWarps * 32, 0, st>>>(a);
  GPS_LAUNCH_CHECK();
  k_perf_quad_bwd_kv<<<grid, kWarps * 32, 0, st>>>(a);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

}  // namespace gps
