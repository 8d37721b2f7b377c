// graph_head.cu — the graph-prediction heads of the graph-level configs, forward and backward, one C call per direction,
// and their C ABI: SANGraphHead (graphgps/head/san_graph.py) and GraphormerHead (graphgps/head/graphormer_graph.py).
//
//   SAN        forward   pad weights (+ planes) -> h_0 = pool(x) at pitch p_0 (+ planes)
//                        -> h_{l+1} = act(h_l W_l^T + b_l) (+ planes) -> pred = h_L W_L^T + b_L -> unpad pred
//              backward  g_L = pad(grad_pred) (+ planes) -> for l = L..0: dW_l, db_l (split-K) and
//                        g_{l-1} = (g_l W_l) act'(.) (+ planes), g_h0 = g_0 W_0 -> grad_x = pool'(g_h0) -> unpad grads
//   Graphormer forward   pad weight -> z = token rows of x -> h = LayerNorm(z) (+ planes) -> pred = h W^T + b -> unpad
//              backward  pad grad_pred -> dW, db -> g_h = g W -> g_z = LayerNorm'(g_h) -> grad_x = pool'(g_z) -> unpad
//
// Every width w runs at p = round_up(w, 8) with zero pad columns (as custom_gnn.cu and link_head.cu do), so the dense
// products are the TMA GEMM with its fused bias / activation epilogues; the pad columns of every activation and every
// gradient stay zero.
//
// Pooling (mean / add): the rows are cut into chunks of kPoolRows; one CTA per (chunk, column block) walks its rows in
// order.  A graph that lies inside one chunk is finished there; a graph that crosses a chunk boundary leaves its
// in-chunk sum as the chunk's `first` (it began before the chunk) and / or `last` (it goes on after it) partial, and a
// second launch adds them in chunk order: last[c0] + first[c0 + 1] + ... + first[c1].  So one large graph spreads over
// many SMs, and the order of every sum is fixed.
#include <string.h>

#include "layer_ops.cuh"

namespace gps {

namespace {

constexpr int kPoolRows = 64;     // rows per chunk of the pooling forward
constexpr float kLnEps = 1e-5f;   // nn.LayerNorm's default, as GraphormerHead builds `ln`

// the graph that holds row r: the last g with ptr[g] <= r (for r < ptr[B] it is non-empty)
__device__ __forceinline__ int graph_of_row(const int* __restrict__ ptr, int B, int64_t r) {
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (ptr[mid] <= r) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

struct PoolOut {
  float* f; int64_t ld;   // [B, cols] at pitch ld
  Planes p;               // optional planes (then cols % 4 == 0)
  int cols;               // columns written: d real ones, zeros beyond
};

__device__ __forceinline__ void store_row(const PoolOut& o, int64_t g, int c, const float v[4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (c + j < o.cols) o.f[g * o.ld + c + j] = v[j];
  if (o.p.hi) planes_store4(o.p, g, c, make_float4(v[0], v[1], v[2], v[3]));
}

__device__ __forceinline__ void load4(const float* row, int c, int d, float v[4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = c + j < d ? row[c + j] : 0.f;
}

// mean / add, first pass: see the comment at the top.  first / last: [chunks][pc], pc = round_up(cols, 4)
__global__ void k_pool_chunk(const int* __restrict__ ptr, int B, int64_t N, const float* __restrict__ x, int d,
                             PoolOut o, int pc, int mean, float* __restrict__ first, float* __restrict__ last) {
  const int c = (blockIdx.y * blockDim.x + threadIdx.x) * 4;
  if (c >= o.cols) return;
  const int64_t chunk = blockIdx.x;
  const int64_t r0 = chunk * kPoolRows, r1 = min(N, r0 + kPoolRows);
  int g = graph_of_row(ptr, B, r0);
  int64_t s = r0;
  while (s < r1) {
    const int64_t gs = ptr[g], ge = ptr[g + 1];
    const int64_t e = min(ge, r1);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int64_t r = s; r < e; ++r) {
      float v[4];
      load4(x + r * d, c, d, v);
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] += v[j];
    }
    if (gs >= r0 && ge <= r1) {   // the whole graph lies in this chunk
      if (mean) {
        const float n = (float)(ge - gs);
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] /= n;
      }
      store_row(o, g, c, acc);
    } else {
      if (gs < r0) st4(first + chunk * pc + c, make_float4(acc[0], acc[1], acc[2], acc[3]));
      if (ge > r1) st4(last + chunk * pc + c, make_float4(acc[0], acc[1], acc[2], acc[3]));
    }
    s = e;
    if (s < r1)
      while (ptr[g + 1] <= s) ++g;   // the next non-empty graph
  }
}

// per graph: graph_token = its first row; mean / add: the graphs k_pool_chunk left open (crossing a chunk boundary)
// from their partials in chunk order, and empty graphs as zero rows
__global__ void k_pool_finish(const int* __restrict__ ptr, const float* __restrict__ x, int d, PoolOut o, int pc,
                              int pooling, const float* __restrict__ first, const float* __restrict__ last) {
  const int g = blockIdx.x;
  const int64_t gs = ptr[g], ge = ptr[g + 1];
  const int64_t c0 = gs / kPoolRows, c1 = (ge - 1) / kPoolRows;
  if (pooling != GPS_POOL_GRAPH_TOKEN && ge > gs && c0 == c1) return;   // finished by k_pool_chunk
  for (int c = threadIdx.x * 4; c < o.cols; c += blockDim.x * 4) {
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (ge > gs && pooling == GPS_POOL_GRAPH_TOKEN) {
      load4(x + gs * d, c, d, v);
    } else if (ge > gs) {
      float4 a = ld4(last + c0 * pc + c);
      for (int64_t k = c0 + 1; k <= c1; ++k) a = f4add(a, ld4(first + k * pc + c));
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
      if (pooling == GPS_POOL_MEAN) {
        const float n = (float)(ge - gs);
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] /= n;
      }
    }
    store_row(o, g, c, v);
  }
}

// grad_x [N, d] whole: mean g[b] / count, add g[b], graph_token g[b] on each token row and 0 elsewhere.  One warp per row.
__global__ void k_pool_bwd(const int* __restrict__ ptr, int B, int64_t N, int pooling, const float* __restrict__ gh,
                           int64_t ldg, int d, float* __restrict__ gx) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < N; r += warps) {
    const int g = graph_of_row(ptr, B, r);
    const int64_t gs = ptr[g];
    float scale = 1.f;
    if (pooling == GPS_POOL_MEAN) scale = 1.f / (float)(ptr[g + 1] - gs);
    const bool zero = pooling == GPS_POOL_GRAPH_TOKEN && r != gs;
    const float* src = gh + (int64_t)g * ldg;
    for (int c = lane; c < d; c += 32) {
      float v = zero ? 0.f : src[c];
      if (pooling == GPS_POOL_MEAN) v = v * scale;
      gx[r * d + c] = v;
    }
  }
}

// row g of f [B, cols] (pitch ld) and of its planes (columns up to p_cols) = 0 for every empty graph g.  GraphormerHead:
// LayerNorm maps the zero row an empty graph pools to onto beta, where the reference pools after the LayerNorm and so
// keeps the row at zero; in the backward the same rows of g_h are zeroed, so they add nothing to ln's gradients.
__global__ void k_zero_empty_rows(const int* __restrict__ ptr, float* __restrict__ f, int64_t ld, int cols, Planes p,
                                  int p_cols) {
  const int g = blockIdx.x;
  if (ptr[g + 1] > ptr[g]) return;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) f[(int64_t)g * ld + c] = 0.f;
  if (p.hi)
    for (int c = threadIdx.x * 4; c < p_cols; c += blockDim.x * 4) planes_store4(p, g, c, f4zero());
}

int zero_empty_rows(const GpsGraph& g, float* f, int64_t ld, int64_t cols, Planes p, int64_t p_cols, cudaStream_t st) {
  if (g.B == 0) return GPS_OK;
  k_zero_empty_rows<<<(unsigned)g.B, 128, 0, st>>>(g.graph_ptr, f, ld, (int)cols, p, (int)p_cols);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int64_t pool_chunks(int64_t N) { return ceil_div(N, kPoolRows); }

int pool_check(const GpsGraph* g, int pooling, const char* what) {
  GPS_REQUIRE(g, GPS_ERR_ARG, "%s: null graph", what);
  GPS_REQUIRE(g->N >= 0 && g->B >= 0 && g->N < (1ll << 31) && g->B < (1ll << 31), GPS_ERR_ARG,
              "%s: graph sizes out of range", what);
  GPS_REQUIRE(g->B == 0 || g->graph_ptr, GPS_ERR_ARG, "%s: graph without graph_ptr", what);
  GPS_REQUIRE(g->N == 0 || g->B > 0, GPS_ERR_ARG, "%s: %lld rows in no graph", what, (long long)g->N);
  GPS_REQUIRE(pooling == GPS_POOL_MEAN || pooling == GPS_POOL_ADD || pooling == GPS_POOL_GRAPH_TOKEN,
              GPS_ERR_UNSUPPORTED, "%s: pooling %d is not built (mean, add and graph_token are)", what, pooling);
  return GPS_OK;
}

int64_t pool_part_floats(int64_t N, int64_t cols) { return 2 * pool_chunks(N) * round_up(cols, 4); }

// out rows [B, o.cols] from x [N, d]; part: pool_part_floats(N, o.cols) floats (mean / add)
int pool_fwd(const GpsGraph& g, int pooling, const float* x, int64_t d, PoolOut o, float* part, cudaStream_t st) {
  if (g.B == 0) return GPS_OK;
  const int c4 = (int)ceil_div(o.cols, 4), pc = 4 * c4;
  float* first = part;
  float* last = part ? part + pool_chunks(g.N) * pc : nullptr;
  if (pooling != GPS_POOL_GRAPH_TOKEN && g.N > 0) {
    const int threads = (int)std::min<int64_t>(128, round_up(c4, 32));
    const dim3 grid((unsigned)pool_chunks(g.N), (unsigned)ceil_div(c4, threads));
    k_pool_chunk<<<grid, threads, 0, st>>>(g.graph_ptr, (int)g.B, g.N, x, (int)d, o, pc, pooling == GPS_POOL_MEAN,
                                           first, last);
    GPS_LAUNCH_CHECK();
  }
  const int threads = (int)std::min<int64_t>(256, round_up(c4, 32));
  k_pool_finish<<<(unsigned)g.B, threads, 0, st>>>(g.graph_ptr, x, (int)d, o, pc, pooling, first, last);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int pool_bwd(const GpsGraph& g, int pooling, const float* gh, int64_t ldg, int64_t d, float* gx, cudaStream_t st) {
  if (g.N == 0) return GPS_OK;
  const int64_t blocks = std::min<int64_t>(ceil_div(g.N, 8), (int64_t)kNumSMs * 16);
  k_pool_bwd<<<(unsigned)blocks, 256, 0, st>>>(g.graph_ptr, (int)g.B, g.N, pooling, gh, ldg, (int)d, gx);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

// =================================================================================== plan
constexpr int kMaxLin = GPS_GRAPH_HEAD_MAX_L + 1;

struct GhPlan {
  int64_t N, B, L, d, dout;
  int kind, pooling, act, prec;
  bool grads_prezeroed = true;   // linear_wgrad: the gradient region is zeroed once per backward call
  int64_t win[kMaxLin], wout[kMaxLin], pin[kMaxLin], pout[kMaxLin];   // real and padded widths of fc[l]
  // saved: padded fc weights (+ planes) and biases; h_l [B, pin[l]] (+ planes), with h_0 = the pooled rows (SAN) or
  // LayerNorm(z) (Graphormer, pitch d); pre_l (GELU) [B, pin[l]]; Graphormer: z [B, d] and the row statistics [2][B]
  float *W[kMaxLin], *b[kMaxLin], *h[kMaxLin], *pre[kMaxLin], *z, *stat;
  Planes W_p[kMaxLin], h_p[kMaxLin];
  int64_t saved_bytes;
  // forward workspace: pooling partials, padded pred
  float *part, *pred;
  int64_t fwd_bytes;
  // backward workspace: dW_l | db_l zeroed as one region, g_l [B, pout[l]] (+ planes), g_h0, LayerNorm partials, g_z
  float *gW[kMaxLin], *gb[kMaxLin], *g[kMaxLin], *gh0, *lnpart, *gz;
  Planes g_p[kMaxLin];
  int64_t grads_bytes, bwd_bytes;
};

int make_plan(const GpsGraphHeadArgs* a, GhPlan* P, bool bind) {
  memset(P, 0, sizeof(*P));
  P->grads_prezeroed = true;
  GPS_REQUIRE(a, GPS_ERR_ARG, "graph_head: null args");
  GPS_REQUIRE(a->kind == GPS_GRAPH_HEAD_SAN || a->kind == GPS_GRAPH_HEAD_GRAPHORMER, GPS_ERR_ARG,
              "graph_head: unknown head kind %d", a->kind);
  GPS_REQUIRE(a->dim_in >= 1 && a->dim_out >= 1, GPS_ERR_ARG, "graph_head: dim_in and dim_out must be positive");
  GPS_REQUIRE(a->dim_in <= 4096 && a->dim_out <= 4096, GPS_ERR_UNSUPPORTED,
              "graph_head: dim_in and dim_out <= 4096 (got %lld, %lld)", (long long)a->dim_in, (long long)a->dim_out);
  GPS_REQUIRE(a->precision == GPS_PREC_FP32 || a->precision == GPS_PREC_BF16, GPS_ERR_ARG,
              "graph_head: unknown precision %d", a->precision);
  GPS_REQUIRE(a->flags == 0, GPS_ERR_ARG, "graph_head: flags are reserved (got %d)", a->flags);
  GPS_REQUIRE(a->graph.N >= 0 && a->graph.B >= 0, GPS_ERR_ARG, "graph_head: negative graph sizes");
  GPS_REQUIRE(a->L >= 0, GPS_ERR_ARG, "graph_head: L must be >= 0 (got %d)", a->L);
  GPS_REQUIRE(a->pooling == GPS_POOL_MEAN || a->pooling == GPS_POOL_ADD || a->pooling == GPS_POOL_GRAPH_TOKEN,
              GPS_ERR_UNSUPPORTED, "graph_head: pooling %d is not built (mean, add and graph_token are)", a->pooling);
  if (a->kind == GPS_GRAPH_HEAD_SAN) {
    GPS_REQUIRE(a->L <= GPS_GRAPH_HEAD_MAX_L && (a->dim_in >> a->L) >= 1, GPS_ERR_UNSUPPORTED,
                "graph_head: dim_in %lld >> L %d leaves a zero width", (long long)a->dim_in, a->L);
    GPS_REQUIRE(a->act == GPS_ACT_RELU || a->act == GPS_ACT_GELU, GPS_ERR_UNSUPPORTED,
                "graph_head: activation %d is not built (relu and gelu are)", a->act);
  } else {
    GPS_REQUIRE(a->L == 0, GPS_ERR_ARG, "graph_head: the Graphormer head has no hidden layers (L = %d)", a->L);
    GPS_REQUIRE(a->pooling == GPS_POOL_GRAPH_TOKEN, GPS_ERR_UNSUPPORTED,
                "graph_head: the Graphormer head is built for graph_token pooling only");
    GPS_REQUIRE(a->dim_in % 4 == 0, GPS_ERR_UNSUPPORTED, "graph_head: the Graphormer head needs dim_in %% 4 == 0");
  }
  const int64_t N = a->graph.N, B = a->graph.B, L = a->L, d = a->dim_in;
  P->N = N; P->B = B; P->L = L; P->d = d; P->dout = a->dim_out;
  P->kind = a->kind; P->pooling = a->pooling; P->act = a->act; P->prec = a->precision;
  for (int64_t l = 0; l <= L; ++l) {
    P->win[l] = d >> l;
    P->wout[l] = l < L ? d >> (l + 1) : a->dim_out;
    P->pin[l] = round_up(P->win[l], 8);
    P->pout[l] = round_up(P->wout[l], 8);
  }
  const bool lo = a->precision == GPS_PREC_FP32;
  const bool gr = a->kind == GPS_GRAPH_HEAD_GRAPHORMER;

  Arena S(bind ? a->saved : nullptr, a->saved_bytes);
  for (int64_t l = 0; l <= L; ++l) {
    P->W[l] = S.alloc<float>(P->pout[l] * P->pin[l]);
    P->W_p[l] = arena_planes(S, P->pout[l], P->pin[l], lo);
    P->b[l] = S.alloc<float>(P->pout[l]);
    P->h[l] = S.alloc<float>(B * P->pin[l]);
    P->h_p[l] = arena_planes(S, B, P->pin[l], lo);
    if (l > 0 && a->act == GPS_ACT_GELU) P->pre[l] = S.alloc<float>(B * P->pin[l]);
  }
  if (gr) {
    P->z = S.alloc<float>(B * d);
    P->stat = S.alloc<float>(2 * B);
  }
  P->saved_bytes = S.used;
  GPS_REQUIRE(!bind || !S.overflow, GPS_ERR_ARG, "graph_head: saved buffer too small (%lld < %lld)",
              (long long)a->saved_bytes, (long long)S.used);

  Arena F(bind ? a->workspace : nullptr, a->workspace_bytes);
  if (a->pooling != GPS_POOL_GRAPH_TOKEN) P->part = F.alloc<float>(pool_part_floats(N, P->pin[0]));
  P->pred = F.alloc<float>(B * P->pout[L]);
  P->fwd_bytes = F.used;

  Arena Bk(bind ? a->workspace : nullptr, a->workspace_bytes);
  const int64_t g0 = Bk.used;
  for (int64_t l = 0; l <= L; ++l) {
    P->gW[l] = Bk.alloc<float>(P->pout[l] * P->pin[l]);
    P->gb[l] = Bk.alloc<float>(P->pout[l]);
  }
  P->grads_bytes = Bk.used - g0;
  for (int64_t l = 0; l <= L; ++l) {
    P->g[l] = Bk.alloc<float>(B * P->pout[l]);
    P->g_p[l] = arena_planes(Bk, B, P->pout[l], lo);
  }
  P->gh0 = Bk.alloc<float>(B * P->pin[0]);
  if (gr) {
    P->lnpart = Bk.alloc<float>(layernorm_part_floats(d));
    P->gz = Bk.alloc<float>(B * d);
  }
  P->bwd_bytes = Bk.used;
  return GPS_OK;
}

// plan, buffers and pointers of one call, all before any CUDA call
int prepare(const GpsGraphHeadArgs* a, bool fwd, GhPlan* P) {
  GPS_REQUIRE(a, GPS_ERR_ARG, "graph_head: null args");
  GPS_REQUIRE(a->saved && a->workspace, GPS_ERR_ARG, "graph_head: saved and workspace are required");
  GPS_TRY(make_plan(a, P, true));
  GPS_TRY(pool_check(&a->graph, a->pooling, "graph_head"));
  const int64_t ws = fwd ? P->fwd_bytes : P->bwd_bytes;
  GPS_REQUIRE(a->workspace_bytes >= ws, GPS_ERR_ARG, "graph_head: workspace too small (%lld < %lld)",
              (long long)a->workspace_bytes, (long long)ws);
  for (int64_t l = 0; l <= P->L; ++l)
    GPS_REQUIRE(a->fc[l].weight && a->fc[l].bias, GPS_ERR_ARG, "graph_head: missing fc[%lld] weight / bias",
                (long long)l);
  if (P->kind == GPS_GRAPH_HEAD_GRAPHORMER)
    GPS_REQUIRE(a->ln.weight && a->ln.bias, GPS_ERR_ARG, "graph_head: missing ln weight / bias");
  if (fwd) {
    GPS_REQUIRE(P->N == 0 || a->x, GPS_ERR_ARG, "graph_head: x is required");
    GPS_REQUIRE(P->B == 0 || a->pred, GPS_ERR_ARG, "graph_head: pred is required");
  } else {
    GPS_REQUIRE(P->B == 0 || a->grad_pred, GPS_ERR_ARG, "graph_head: grad_pred is required");
    GPS_REQUIRE(P->N == 0 || a->grad_x, GPS_ERR_ARG, "graph_head: grad_x is required");
  }
  return GPS_OK;
}

int gh_forward(const GpsGraphHeadArgs* a, cudaStream_t st) {
  GhPlan P;
  GPS_TRY(prepare(a, true, &P));
  const int64_t B = P.B, L = P.L, d = P.d;
  if (B == 0) return GPS_OK;
  {
    PadList W;
    for (int64_t l = 0; l <= L; ++l) {
      if (W.n + 2 > kPadItems) {
        GPS_TRY(W.run(st));
        W.n = 0;
      }
      W.add(a->fc[l].weight, P.win[l], P.wout[l], P.win[l], P.W[l], P.pin[l], P.pout[l], P.pin[l], P.W_p[l]);
      W.add(a->fc[l].bias, P.wout[l], 1, P.wout[l], P.b[l], P.pout[l], 1, P.pout[l]);
    }
    GPS_TRY(W.run(st));
  }
  if (P.kind == GPS_GRAPH_HEAD_SAN) {
    GPS_TRY(pool_fwd(a->graph, P.pooling, a->x, d, PoolOut{P.h[0], P.pin[0], P.h_p[0], (int)P.pin[0]}, P.part, st));
  } else {
    GPS_TRY(pool_fwd(a->graph, P.pooling, a->x, d, PoolOut{P.z, d, Planes(), (int)d}, nullptr, st));
    if (d != P.pin[0]) {   // LayerNorm writes the d real columns of the planes; the pad columns are K of the product
      GPS_CUDA(cudaMemsetAsync(P.h_p[0].hi, 0, (size_t)(B * P.pin[0] + 8) * sizeof(__nv_bfloat16), st));
      if (P.h_p[0].lo)
        GPS_CUDA(cudaMemsetAsync(P.h_p[0].lo, 0, (size_t)(B * P.pin[0] + 8) * sizeof(__nv_bfloat16), st));
    }
    GPS_TRY(layernorm_fwd(P.z, B, d, a->ln.weight, a->ln.bias, kLnEps, P.stat, P.stat + B, P.h[0], P.h_p[0], nullptr,
                          nullptr, DropCfg(), nullptr, st));
    GPS_TRY(zero_empty_rows(a->graph, P.h[0], d, d, P.h_p[0], P.pin[0], st));
  }
  const int64_t ld0 = P.kind == GPS_GRAPH_HEAD_SAN ? P.pin[0] : d;
  for (int64_t l = 0; l <= L; ++l) {
    const Operand h{P.h[l], l == 0 ? ld0 : P.pin[l], P.h_p[l]};
    const bool last = l == L;
    GemmParams g = linear_fwd(P, B, P.pout[l], P.pin[l], h, {P.W[l], P.pin[l], P.W_p[l]}, last ? P.pred : P.h[l + 1],
                              P.pout[l], P.b[l]);
    if (!last) {
      g.act = P.act;
      g.Cp = P.h_p[l + 1];
      if (P.pre[l + 1]) {
        g.C_pre = P.pre[l + 1];
        g.ldpre = (int)P.pout[l];
      }
    }
    GPS_TRY(gemm(g, st));
  }
  PadList U;
  U.add(P.pred, P.pout[L], B, P.dout, a->pred, P.dout, B, P.dout);
  return U.run(st);
}

int gh_backward(const GpsGraphHeadArgs* a, cudaStream_t st) {
  GhPlan P;
  GPS_TRY(prepare(a, false, &P));
  const int64_t B = P.B, L = P.L, d = P.d;
  GPS_CUDA(cudaMemsetAsync(P.gW[0], 0, (size_t)P.grads_bytes, st));
  if (B > 0) {
    PadList G;
    G.add(a->grad_pred, P.dout, B, P.dout, P.g[L], P.pout[L], B, P.pout[L], P.g_p[L]);
    GPS_TRY(G.run(st));
    const int64_t ld0 = P.kind == GPS_GRAPH_HEAD_SAN ? P.pin[0] : d;
    for (int64_t l = L; l >= 0; --l) {
      const Operand gl{P.g[l], P.pout[l], P.g_p[l]};
      const Operand h{P.h[l], l == 0 ? ld0 : P.pin[l], P.h_p[l]};
      GPS_TRY(linear_wgrad(P, gl, h, B, P.pout[l], P.pin[l], P.gW[l], P.gb[l], st));
      const Operand W{P.W[l], P.pin[l], P.W_p[l]};
      if (l > 0) {   // g_{l-1} = (g_l W_l) act'(pre), the gradient of h_l's pre-activation
        GemmParams g = linear_dgrad(P, B, P.pin[l], P.pout[l], gl, W, P.g[l - 1], P.pin[l]);
        set_act_mask(g, P.act, P.h[l], P.pre[l], P.pin[l]);
        g.Cp = P.g_p[l - 1];
        GPS_TRY(gemm(g, st));
      } else if (P.kind == GPS_GRAPH_HEAD_SAN) {
        GPS_TRY(gemm(linear_dgrad(P, B, P.pin[0], P.pout[0], gl, W, P.gh0, P.pin[0]), st));
      } else {   // the d real columns of g_h, at LayerNorm's pitch d
        GPS_TRY(gemm(linear_dgrad(P, B, d, P.pout[0], gl, W, P.gh0, d), st));
      }
    }
  }
  if (P.kind == GPS_GRAPH_HEAD_SAN) {
    GPS_TRY(pool_bwd(a->graph, P.pooling, P.gh0, P.pin[0], d, a->grad_x, st));
  } else {
    GPS_TRY(zero_empty_rows(a->graph, P.gh0, d, d, Planes(), 0, st));
    GPS_TRY(layernorm_bwd(P.gh0, DropCfg(), P.z, B, d, a->ln.weight, P.stat, P.stat + B, nullptr, Planes(), DropCfg(),
                          P.gz, nullptr, P.lnpart, a->ln.grad_weight, a->ln.grad_bias, false, st));
    GPS_TRY(pool_bwd(a->graph, P.pooling, P.gz, d, d, a->grad_x, st));
  }
  PadList U;
  for (int64_t l = 0; l <= L; ++l) {
    if (U.n + 2 > kPadItems) {
      GPS_TRY(U.run(st));
      U.n = 0;
    }
    U.add(P.gW[l], P.pin[l], P.wout[l], P.win[l], a->fc[l].grad_weight, P.win[l], P.wout[l], P.win[l]);
    U.add(P.gb[l], P.pout[l], 1, P.wout[l], a->fc[l].grad_bias, P.wout[l], 1, P.wout[l]);
  }
  return U.run(st);
}

}  // namespace

}  // namespace gps

// =================================================================================== C ABI
using namespace gps;

extern "C" int gps_graph_head_plan(const GpsGraphHeadArgs* args, GpsGraphHeadPlan* plan) {
  GPS_REQUIRE(args && plan, GPS_ERR_ARG, "gps_graph_head_plan: null argument");
  GhPlan P;
  GPS_TRY(make_plan(args, &P, false));
  plan->saved_bytes = P.saved_bytes;
  plan->fwd_workspace_bytes = P.fwd_bytes;
  plan->bwd_workspace_bytes = P.bwd_bytes;
  return GPS_OK;
}

extern "C" int gps_graph_head_forward(const GpsGraphHeadArgs* args, void* stream) {
  return gh_forward(args, (cudaStream_t)stream);
}

extern "C" int gps_graph_head_backward(const GpsGraphHeadArgs* args, void* stream) {
  return gh_backward(args, (cudaStream_t)stream);
}

extern "C" int gps_graph_pool_forward(const GpsGraph* graph, int32_t pooling, const float* x, int64_t d, float* out,
                                      int64_t ldo, void* workspace, int64_t workspace_bytes, void* stream) {
  GPS_TRY(pool_check(graph, pooling, "gps_graph_pool_forward"));
  GPS_REQUIRE(d >= 1 && d <= 4096 && ldo >= d, GPS_ERR_ARG, "gps_graph_pool_forward: needs 1 <= d <= 4096 and ldo >= d");
  GPS_REQUIRE(graph->N == 0 || x, GPS_ERR_ARG, "gps_graph_pool_forward: x is required");
  GPS_REQUIRE(graph->B == 0 || out, GPS_ERR_ARG, "gps_graph_pool_forward: out is required");
  GPS_REQUIRE(((uintptr_t)workspace & 15) == 0, GPS_ERR_ARG,
              "gps_graph_pool_forward: workspace must be 16-byte aligned (the partials move as float4)");
  const bool token = pooling == GPS_POOL_GRAPH_TOKEN;
  const int64_t need = token ? 0 : 4 * pool_part_floats(graph->N, d);
  GPS_REQUIRE(need == 0 || (workspace && workspace_bytes >= need), GPS_ERR_ARG,
              "gps_graph_pool_forward: workspace too small (%lld < %lld)", (long long)workspace_bytes, (long long)need);
  return pool_fwd(*graph, pooling, x, d, PoolOut{out, ldo, Planes(), (int)d}, token ? nullptr : (float*)workspace,
                  (cudaStream_t)stream);
}

extern "C" int gps_graph_pool_backward(const GpsGraph* graph, int32_t pooling, const float* grad_out, int64_t ldg,
                                       int64_t d, float* grad_x, void* stream) {
  GPS_TRY(pool_check(graph, pooling, "gps_graph_pool_backward"));
  GPS_REQUIRE(d >= 1 && d <= 4096 && ldg >= d, GPS_ERR_ARG, "gps_graph_pool_backward: needs 1 <= d <= 4096 and ldg >= d");
  GPS_REQUIRE(graph->N == 0 || (grad_out && grad_x), GPS_ERR_ARG, "gps_graph_pool_backward: grad_out and grad_x are required");
  return pool_bwd(*graph, pooling, grad_out, ldg, d, grad_x, (cudaStream_t)stream);
}
