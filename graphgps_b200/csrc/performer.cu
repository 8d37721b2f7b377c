// performer.cu — FAVOR+ (Performer) global attention of GPSLayer on packed graphs.
//
// Reference: performer_pytorch.SelfAttention as used at graphgps/layer/gps_layer.py:111-114,205-206; the code is
// the in-repo copy graphgps/layer/performer_layer.py: softmax_kernel :119-144, linear_attention :200-205,
// Attention.forward :476-503.  dim_head = 64 and nb_features = int(64 ln 64) = 266 are fixed by the reference's
// constructor defaults (:427,:261).
//
//   q' = m^-1/2 (exp(dd_q - diag_q - max_j dd_q) + 1e-4)        dd = (x 64^-1/4) P^T,  diag = |x|^2/2 * 64^-1/2
//   k' = m^-1/2 (exp(dd_k - diag_k - max_{n,j} dd_k) + 1e-4)    max over ALL rows of the padded [Nmax] graph
//   out_n = (q'_n . (sum_n k'_n^T v_n)) / (q'_n . sum_n k'_n)
//
// The reference runs this on the zero-padded dense batch [B, Nmax, .] and masks only v (:485-487), so padded
// rows (x = 0 => k = 0 => dd = 0, diag = 0) still (i) put 0 into the key stabiliser max and (ii) add
// (Nmax - n_g) * k'_pad to sum_n k'.  Both effects are reproduced analytically here on the packed layout —
// no padding is materialised (SURVEY.md section 7, hard part 6).  The stabiliser is NOT detached in the in-repo
// copy, so its gradient (to the arg-max element) is propagated as autograd does.
//
// Ties: when several elements share the maximum, the kernels give the whole stabiliser gradient to the lowest index
// (the lowest feature of a query row; the lowest flat (row, feature) index of a (graph, head), real rows before the
// padded ones), where torch.amax splits it evenly among the tied elements.  The total per max is the same, and g_Q /
// g_K differ from the reference only when the tied elements come from rows of Pn that differ.
//
// Kernels: feature maps are warp-per-row; the per-(graph, head) linear attention keeps the 272x64 context in
// registers (68 per thread) in forward and additionally in shared memory in backward.  The backward has no float
// atomics: the stabiliser gradient of each key row goes to its own slot of a [N*H] buffer, and k_perf_gmax_scatter
// sums each (graph, head)'s slots in a fixed order, so two runs give the same bits.
#include <limits.h>

#include "kernels.cuh"

namespace gps {

namespace {

constexpr int DH = 64;      // dim_head
constexpr int MP = 272;     // nb_features (266) rounded up to a multiple of 16
constexpr int JT = MP / 4;  // 68 feature rows per thread in the (b,h) kernels
constexpr float kEpsF = 1e-4f;

__device__ __forceinline__ int find_graph_p(const int* __restrict__ gptr, int B, int node) {
  int lo = 0, hi = B;
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (gptr[mid] <= node) lo = mid; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
  // valid for any mix of signs (IEEE ordering trick); -0.0 takes the first branch with its sign bit cleared
  if (v >= 0.f) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v) & 0x7fffffff);
  else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

// Pn = dn * P padded with zero rows; nmax = max graph size; gmax init (0 if the graph has padded rows, else -inf)
__global__ void k_perf_prep(const float* __restrict__ P, int m, float dn, float* __restrict__ Pn, const int* __restrict__ gptr,
                            int B, int H, int* __restrict__ nmax_out, float* __restrict__ gmax, int* __restrict__ argk) {
  __shared__ int s_max;
  if (threadIdx.x == 0) s_max = 0;
  __syncthreads();
  int loc = 0;
  for (int b = threadIdx.x; b < B; b += blockDim.x) loc = max(loc, gptr[b + 1] - gptr[b]);
  atomicMax(&s_max, loc);
  __syncthreads();
  const int nmax = s_max;
  if (threadIdx.x == 0) *nmax_out = nmax;
  for (int i = threadIdx.x; i < MP * DH; i += blockDim.x) Pn[i] = (i / DH) < m ? dn * P[i] : 0.f;
  for (int i = threadIdx.x; i < B * H; i += blockDim.x) {
    const int b = i / H;
    gmax[i] = (gptr[b + 1] - gptr[b]) < nmax ? 0.f : -INFINITY;
    argk[i] = INT_MAX;
  }
}

// warp per row of dd_k [N*H, MP]: row max over the m real features -> atomic max per (graph, head)
__global__ void k_perf_kmax(const float* __restrict__ ddk, int N, int H, int m, const int* __restrict__ gptr, int B,
                            float* __restrict__ gmax) {
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= N * H) return;
  const float* row = ddk + (int64_t)r * MP;
  float mx = -INFINITY;
  for (int j = lane; j < m; j += 32) mx = fmaxf(mx, row[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) {
    const int n = r / H, h = r % H;
    atomic_max_float(&gmax[find_graph_p(gptr, B, n) * H + h], mx);
  }
}

// warp per row; rows [0, NH) are queries, [NH, 2NH) keys.  In place: dd -> feature map.
__global__ void k_perf_features(float* __restrict__ fq, float* __restrict__ fk, const float* __restrict__ Q,
                                const float* __restrict__ K, int N, int H, int m, float dn, float ratio,
                                const int* __restrict__ gptr, int B, const float* __restrict__ gmax,
                                int* __restrict__ argq, int* __restrict__ argk) {
  const int NH = N * H;
  int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= 2 * NH) return;
  const bool is_q = r < NH;
  if (!is_q) r -= NH;
  float* row = (is_q ? fq : fk) + (int64_t)r * MP;
  const float* xrow = (is_q ? Q : K) + (int64_t)r * DH;
  float x0 = xrow[lane], x1 = xrow[lane + 32];
  float ss = x0 * x0 + x1 * x1;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float diag = 0.5f * dn * dn * ss;
  float v[9];
  float mx = -INFINITY;
  int mj = INT_MAX;
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    const int j = lane + 32 * i;
    v[i] = j < m ? row[j] : -INFINITY;
    if (v[i] > mx) { mx = v[i]; mj = j; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oj = __shfl_xor_sync(0xffffffffu, mj, o);
    if (om > mx || (om == mx && oj < mj)) { mx = om; mj = oj; }
  }
  float stab = mx;
  if (is_q) {
    if (lane == 0) argq[r] = mj;
  } else {
    const int n = r / H, h = r % H;
    const int bh = find_graph_p(gptr, B, n) * H + h;
    stab = gmax[bh];
    if (lane == 0 && mx == stab) atomicMin(&argk[bh], r * MP + mj);   // arg-max is a real element
  }
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    const int j = lane + 32 * i;
    if (j < MP) row[j] = j < m ? ratio * (__expf(v[i] - diag - stab) + kEpsF) : 0.f;
  }
}

// ---- per (graph, head) linear attention.  thread t: e = t & 63, jg = t >> 6, features j = jg + 4 i.
struct LinArgs {
  const int* gptr; const int* nmax; int H; int m; float ratio;
  const float* qf; const float* kf; const float* V; float* O;        // V/O: [N, H*64]
  const float* gmax;
  // backward
  const float* gO; float* g_qf; float* g_kf; float* gV; float* ggmax;
};

__device__ __forceinline__ void ctx_accumulate(const LinArgs& a, int gs, int n, int h, int H, float* acc, float* s_row,
                                               float* s_v, float* s_ksum) {
  const int t = threadIdx.x, e = t & 63, jg = t >> 6;
  for (int nn = 0; nn < n; ++nn) {
    const int64_t r = (int64_t)(gs + nn) * H + h;
    for (int j = t; j < MP; j += 256) s_row[j] = a.kf[r * MP + j];
    if (t < DH) s_v[t] = a.V[r * DH + t];
    __syncthreads();
    const float ve = s_v[e];
#pragma unroll
    for (int i = 0; i < JT; ++i) acc[i] = fmaf(s_row[jg + 4 * i], ve, acc[i]);
    for (int j = t; j < MP; j += 256) s_ksum[j] += s_row[j];
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) k_perf_linattn_fwd(LinArgs a) {
  __shared__ float s_row[MP], s_v[DH], s_ksum[MP], s_red[4][DH], s_den;
  const int b = blockIdx.x, h = blockIdx.y, H = a.H;
  const int gs = a.gptr[b], n = a.gptr[b + 1] - gs;
  if (n == 0) return;
  const int t = threadIdx.x, e = t & 63, jg = t >> 6, lane = t & 31;
  float acc[JT];
#pragma unroll
  for (int i = 0; i < JT; ++i) acc[i] = 0.f;
  for (int j = t; j < MP; j += 256) s_ksum[j] = 0.f;
  __syncthreads();
  ctx_accumulate(a, gs, n, h, H, acc, s_row, s_v, s_ksum);
  {  // padded rows of the dense batch: (Nmax - n) * k'_pad on the real features
    const float kpad = a.ratio * (__expf(-a.gmax[b * H + h]) + kEpsF) * (float)(*a.nmax - n);
    for (int j = t; j < a.m; j += 256) s_ksum[j] += kpad;
  }
  __syncthreads();
  for (int nn = 0; nn < n; ++nn) {
    const int64_t r = (int64_t)(gs + nn) * H + h;
    for (int j = t; j < MP; j += 256) s_row[j] = a.qf[r * MP + j];
    __syncthreads();
    if (t < 32) {
      float d = 0.f;
      for (int j = lane; j < MP; j += 32) d = fmaf(s_row[j], s_ksum[j], d);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
      if (lane == 0) s_den = d;
    }
    float u = 0.f;
#pragma unroll
    for (int i = 0; i < JT; ++i) u = fmaf(s_row[jg + 4 * i], acc[i], u);
    s_red[jg][e] = u;
    __syncthreads();
    if (jg == 0) a.O[r * DH + e] = (s_red[0][e] + s_red[1][e] + s_red[2][e] + s_red[3][e]) / s_den;
    __syncthreads();
  }
}

constexpr int CTX_LD = DH + 1;   // padded row stride of the shared-memory context (conflict-free column reads)

__global__ void __launch_bounds__(256) k_perf_linattn_bwd(LinArgs a) {
  extern __shared__ float s_ctx[];   // [MP][CTX_LD]: context, later its gradient
  __shared__ float s_row[MP], s_v[DH], s_ksum[MP], s_gks[MP], s_red[4][DH], s_u[DH], s_sc[2];
  const int b = blockIdx.x, h = blockIdx.y, H = a.H;
  const int gs = a.gptr[b], n = a.gptr[b + 1] - gs;
  const int t = threadIdx.x, e = t & 63, jg = t >> 6, lane = t & 31;
  if (n == 0) {
    if (t == 0) a.ggmax[b * H + h] = 0.f;
    return;
  }
  float acc[JT], gacc[JT];
#pragma unroll
  for (int i = 0; i < JT; ++i) { acc[i] = 0.f; gacc[i] = 0.f; }
  for (int j = t; j < MP; j += 256) { s_ksum[j] = 0.f; s_gks[j] = 0.f; }
  __syncthreads();
  ctx_accumulate(a, gs, n, h, H, acc, s_row, s_v, s_ksum);
  const float gm = a.gmax[b * H + h];
  const float npad = (float)(*a.nmax - n);
  {
    const float kpad = a.ratio * (__expf(-gm) + kEpsF) * npad;
    for (int j = t; j < a.m; j += 256) s_ksum[j] += kpad;
  }
#pragma unroll
  for (int i = 0; i < JT; ++i) s_ctx[(jg + 4 * i) * CTX_LD + e] = acc[i];
  __syncthreads();

  // ---- pass A over queries: g_q', g_ctx (registers), g_ksum (shared)
  for (int nn = 0; nn < n; ++nn) {
    const int64_t r = (int64_t)(gs + nn) * H + h;
    for (int j = t; j < MP; j += 256) s_row[j] = a.qf[r * MP + j];
    if (t < DH) s_v[t] = a.gO[r * DH + t];
    __syncthreads();
    if (t < 32) {
      float d = 0.f;
      for (int j = lane; j < MP; j += 32) d = fmaf(s_row[j], s_ksum[j], d);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
      if (lane == 0) s_sc[0] = 1.f / d;   // Dinv
    }
    float u = 0.f;
#pragma unroll
    for (int i = 0; i < JT; ++i) u = fmaf(s_row[jg + 4 * i], acc[i], u);
    s_red[jg][e] = u;
    __syncthreads();
    if (jg == 0) s_u[e] = s_red[0][e] + s_red[1][e] + s_red[2][e] + s_red[3][e];
    __syncthreads();
    if (t < 32) {
      float d = s_v[lane] * s_u[lane] + s_v[lane + 32] * s_u[lane + 32];   // gO . u
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
      if (lane == 0) s_sc[1] = -s_sc[0] * s_sc[0] * d;   // g_den
    }
    __syncthreads();
    const float dinv = s_sc[0], gden = s_sc[1];
    const float gu = dinv * s_v[e];
#pragma unroll
    for (int i = 0; i < JT; ++i) gacc[i] = fmaf(s_row[jg + 4 * i], gu, gacc[i]);
    for (int j = t; j < MP; j += 256) {
      float g = gden * s_ksum[j];
      const float* c = s_ctx + j * CTX_LD;
#pragma unroll 8
      for (int ee = 0; ee < DH; ++ee) g = fmaf(c[ee], dinv * s_v[ee], g);
      a.g_qf[r * MP + j] = g;
      s_gks[j] += gden * s_row[j];
    }
    __syncthreads();
  }
  // ---- context gradient to shared memory (context itself is no longer needed)
#pragma unroll
  for (int i = 0; i < JT; ++i) s_ctx[(jg + 4 * i) * CTX_LD + e] = gacc[i];
  __syncthreads();
  // stabiliser gradient through the padded rows' k'_pad = ratio (exp(-gmax) + eps)
  if (t < 32) {
    float d = 0.f;
    for (int j = lane; j < a.m; j += 32) d += s_gks[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    if (lane == 0) a.ggmax[b * H + h] = -npad * d * a.ratio * __expf(-gm);
  }
  // ---- pass B over keys: g_k', g_v
  for (int nn = 0; nn < n; ++nn) {
    const int64_t r = (int64_t)(gs + nn) * H + h;
    for (int j = t; j < MP; j += 256) s_row[j] = a.kf[r * MP + j];
    if (t < DH) s_v[t] = a.V[r * DH + t];
    __syncthreads();
    float gv = 0.f;
#pragma unroll
    for (int i = 0; i < JT; ++i) gv = fmaf(s_row[jg + 4 * i], gacc[i], gv);
    s_red[jg][e] = gv;
    for (int j = t; j < MP; j += 256) {
      float g = s_gks[j];
      const float* c = s_ctx + j * CTX_LD;
#pragma unroll 8
      for (int ee = 0; ee < DH; ++ee) g = fmaf(c[ee], s_v[ee], g);
      a.g_kf[r * MP + j] = g;
    }
    __syncthreads();
    if (jg == 0) a.gV[r * DH + e] = s_red[0][e] + s_red[1][e] + s_red[2][e] + s_red[3][e];
    __syncthreads();
  }
}

// warp per row: g_f -> g_dd in place, diag gradient into gQ/gK, stabiliser gradients.  Key row r's gradient of its
// (graph, head)'s max, -S, goes to gmrow[r]: added to the pairwise form's padded-row term there (add_rows), else stored.
__global__ void k_perf_features_bwd(float* __restrict__ gq, float* __restrict__ gk, const float* __restrict__ fq,
                                    const float* __restrict__ fk, const float* __restrict__ Q, const float* __restrict__ K,
                                    float* __restrict__ gQ, float* __restrict__ gK, int N, int H, int m, float dn,
                                    float ratio, const int* __restrict__ argq, float* __restrict__ gmrow, bool add_rows) {
  const int NH = N * H;
  int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= 2 * NH) return;
  const bool is_q = r < NH;
  if (!is_q) r -= NH;
  float* grow = (is_q ? gq : gk) + (int64_t)r * MP;
  const float* frow = (is_q ? fq : fk) + (int64_t)r * MP;
  float tv[9];
  float S = 0.f;
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    const int j = lane + 32 * i;
    tv[i] = 0.f;
    if (j < m) {
      const float E = frow[j] / ratio - kEpsF;
      tv[i] = grow[j] * ratio * E;
      S += tv[i];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) S += __shfl_xor_sync(0xffffffffu, S, o);
  const int aj = is_q ? argq[r] : -1;
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    const int j = lane + 32 * i;
    if (j < MP) grow[j] = tv[i] - (j == aj ? S : 0.f);   // row-max stabiliser of the queries
  }
  if (!is_q && lane == 0) gmrow[r] = (add_rows ? gmrow[r] : 0.f) - S;
  // diag = |x|^2 / 2 * dn^2  ->  g_x = -S * dn^2 * x
  const float* xrow = (is_q ? Q : K) + (int64_t)r * DH;
  float* gx = (is_q ? gQ : gK) + (int64_t)r * DH;
  const float c = -S * dn * dn;
  gx[lane] = c * xrow[lane];
  gx[lane + 32] = c * xrow[lane + 32];
}

// warp per (graph, head): the gradient of its key max is the sum of its rows' gmrow slots (lane-strided, then a fixed
// shuffle tree) plus the context form's ggmax; it goes to the arg-max element, unless the max is a padded row's 0
__global__ void k_perf_gmax_scatter(float* __restrict__ g_ddk, const int* __restrict__ argk, const float* __restrict__ ggmax,
                                    const float* __restrict__ gmrow, const int* __restrict__ gptr, int B, int H) {
  const int bh = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (bh >= B * H) return;
  const int a = argk[bh];
  if (a == INT_MAX) return;
  const int b = bh / H, h = bh % H, gs = gptr[b], n = gptr[b + 1] - gs;
  float s = 0.f;
  for (int nn = lane; nn < n; nn += 32) s += gmrow[(int64_t)(gs + nn) * H + h];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) g_ddk[a] += (ggmax ? ggmax[bh] : 0.f) + s;
}

}  // namespace

int perf_supported(int64_t dim_head, int64_t features) {
  GPS_REQUIRE(dim_head == DH && features > MP - 16 && features <= MP, GPS_ERR_UNSUPPORTED,
              "Performer kernels are built for dim_head=64, nb_features=266 (got %lld, %lld)", (long long)dim_head,
              (long long)features);
  return GPS_OK;
}
int64_t perf_mp() { return MP; }
// argk holds the flat int index r * MP + j of the [N*H, MP] key feature map
int perf_index_range(int64_t N, int64_t H) {
  GPS_REQUIRE(H > 0 && N >= 0 && N <= INT_MAX / MP / H, GPS_ERR_UNSUPPORTED,
              "Performer kernels index the [N*H, %d] feature maps with int32: N*H = %lld*%lld exceeds %d", MP,
              (long long)N, (long long)H, INT_MAX / MP);
  return GPS_OK;
}

int perf_prep(const float* P, int64_t m, float* Pn, const GpsGraph& g, int64_t H, int* nmax, float* gmax, int* argk,
              cudaStream_t st) {
  const float dn = powf((float)DH, -0.25f);
  k_perf_prep<<<1, 256, 0, st>>>(P, (int)m, dn, Pn, g.graph_ptr, (int)g.B, (int)H, nmax, gmax, argk);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int perf_features_fwd(float* fq, float* fk, const float* Q, const float* K, const GpsGraph& g, int64_t H, int64_t m,
                      float* gmax, int* argq, int* argk, cudaStream_t st) {
  const int64_t NH = g.N * H;
  if (NH == 0) return GPS_OK;
  const float dn = powf((float)DH, -0.25f), ratio = 1.f / sqrtf((float)m);
  k_perf_kmax<<<(unsigned)ceil_div(NH, 8), 256, 0, st>>>(fk, (int)g.N, (int)H, (int)m, g.graph_ptr, (int)g.B, gmax);
  GPS_LAUNCH_CHECK();
  k_perf_features<<<(unsigned)ceil_div(2 * NH, 8), 256, 0, st>>>(fq, fk, Q, K, (int)g.N, (int)H, (int)m, dn, ratio,
                                                                  g.graph_ptr, (int)g.B, gmax, argq, argk);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int perf_linattn_fwd(const GpsGraph& g, int64_t H, int64_t m, const int* nmax, const float* qf, const float* kf,
                     const float* V, const float* gmax, float* O, cudaStream_t st) {
  if (g.B == 0 || g.N == 0) return GPS_OK;
  LinArgs a{};
  a.gptr = g.graph_ptr; a.nmax = nmax; a.H = (int)H; a.m = (int)m; a.ratio = 1.f / sqrtf((float)m);
  a.qf = qf; a.kf = kf; a.V = V; a.O = O; a.gmax = gmax;
  k_perf_linattn_fwd<<<dim3((unsigned)g.B, (unsigned)H), 256, 0, st>>>(a);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int perf_linattn_bwd(const GpsGraph& g, int64_t H, int64_t m, const int* nmax, const float* qf, const float* kf,
                     const float* V, const float* gmax, const float* gO, float* g_qf, float* g_kf, float* gV,
                     float* ggmax, cudaStream_t st) {
  if (g.B == 0 || g.N == 0) return GPS_OK;
  LinArgs a{};
  a.gptr = g.graph_ptr; a.nmax = nmax; a.H = (int)H; a.m = (int)m; a.ratio = 1.f / sqrtf((float)m);
  a.qf = qf; a.kf = kf; a.V = V; a.gmax = gmax; a.gO = gO; a.g_qf = g_qf; a.g_kf = g_kf; a.gV = gV; a.ggmax = ggmax;
  const size_t smem = (size_t)MP * CTX_LD * sizeof(float);
  static bool attr = false;
  if (!attr) {
    GPS_CUDA(cudaFuncSetAttribute(k_perf_linattn_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  k_perf_linattn_bwd<<<dim3((unsigned)g.B, (unsigned)H), 256, smem, st>>>(a);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int perf_features_bwd(float* g_fq, float* g_fk, const float* fq, const float* fk, const float* Q, const float* K,
                      float* gQ, float* gK, const GpsGraph& g, int64_t H, int64_t m, const int* argq, const int* argk,
                      const float* ggmax, float* gmrow, bool pairwise, cudaStream_t st) {
  const int64_t NH = g.N * H;
  if (NH == 0) return GPS_OK;
  const float dn = powf((float)DH, -0.25f), ratio = 1.f / sqrtf((float)m);
  k_perf_features_bwd<<<(unsigned)ceil_div(2 * NH, 8), 256, 0, st>>>(g_fq, g_fk, fq, fk, Q, K, gQ, gK, (int)g.N, (int)H,
                                                                      (int)m, dn, ratio, argq, gmrow, pairwise);
  GPS_LAUNCH_CHECK();
  const int64_t BH = g.B * H;
  k_perf_gmax_scatter<<<(unsigned)ceil_div(BH, 8), 256, 0, st>>>(g_fk, argk, pairwise ? nullptr : ggmax, gmrow,
                                                                  g.graph_ptr, (int)g.B, (int)H);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

}  // namespace gps
