// link_head.cu — the inductive link-prediction head of the PCQM-Contact configs (graphgps/head/inductive_edge.py,
// GNNInductiveEdgeHead with edge_decoding "dot" and layers_post_mp 1), forward and backward, one C call per direction,
// and its C ABI.
//
//   forward   pack x, W, b at pitch dp = round_up(d, 8) (+ planes) -> y = x W^T + b -> pred[k] = <y[s_k], y[t_k]>
//             -> (eval) ranking statistics -> unpack y
//   backward  dy = grad_y + segmented pair sums (+ planes) -> dW = dy^T x, db = sum dy (split-K) -> grad_x = dy W -> unpack
//
// The dense products run the TMA GEMM on zero-padded operands exactly as custom_gnn.cu runs widths that are not a
// multiple of 8; the pad columns of y and dy are zero, so every dot product over dp equals the one over d.
//
// Ranking (eval): one CTA per graph.  For each source node with positives, its row y_i is staged in shared memory and
// the graph's candidate rows pass through shared memory in tiles, one candidate per thread, so any graph size works.
// The positive's own score and every candidate's score come from the same fused multiply-add chain, so bitwise-equal
// rows give bitwise-equal scores and ties resolve by the rule in gps_b200.h.  Per-positive counts are integer, the
// per-graph means are summed in pair order in fp64 and a second launch averages the graphs in a fixed order.
#include <string.h>

#include "layer_ops.cuh"

namespace gps {

namespace {

constexpr int kRankThreads = 64;     // candidates per tile (one per thread)
constexpr int kRankChunk = 64;       // positives of one source node counted per pass over the candidates
constexpr int kRankSmemCap = 100 * 1024;

// pred[k] = <y[s_k], y[t_k]> over dp columns (pad columns are zero): one warp per pair, fixed reduction order
__global__ void k_pair_score(const float* __restrict__ y, int64_t dp, int64_t N, const int64_t* __restrict__ eli,
                             int64_t K, float* __restrict__ pred) {
  const int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (k >= K) return;
  const int64_t s = eli[k], t = eli[K + k];
  float acc = 0.f;
  if (s >= 0 && s < N && t >= 0 && t < N) {
    const float* ys = y + s * dp;
    const float* yt = y + t * dp;
    for (int64_t c = (int64_t)lane * 4; c < dp; c += 128) {
      const float4 a = ld4(ys + c), b = ld4(yt + c);
      acc = fmaf(a.x, b.x, acc);
      acc = fmaf(a.y, b.y, acc);
      acc = fmaf(a.z, b.z, acc);
      acc = fmaf(a.w, b.w, acc);
    }
  }
  acc = warp_sum(acc);
  if (lane == 0) pred[k] = acc;
}

// dy[n] = grad_y[n] + sum_{k: s_k = n} g_k y[t_k] + sum_{k: t_k = n} g_k y[s_k], at pitch dp with zero pad columns and
// its planes: one warp per node, both segments walked in pair-id order (gps_graph_build), no atomics
__global__ void k_pair_grad(const GpsGraph g, const float* __restrict__ y, int64_t dp, const float* __restrict__ gy,
                            int64_t d, const float* __restrict__ gpred, float* __restrict__ dy, Planes dyp) {
  const int64_t n = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (n >= g.N) return;
  const int sb = g.src_ptr[n], se = g.src_ptr[n + 1];
  const int db = g.dst_ptr[n], de = g.dst_ptr[n + 1];
  for (int64_t c = (int64_t)lane * 4; c < dp; c += 128) {
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = gy && c + j < d ? gy[n * d + c + j] : 0.f;
    float4 acc = make_float4(v[0], v[1], v[2], v[3]);
    if (gpred) {
      for (int e = sb; e < se; ++e) {
        const int t = g.src_dst[e];
        if ((unsigned)t < (unsigned)g.N) {
          const float w = gpred[g.src_eid[e]];
          acc = f4fma(make_float4(w, w, w, w), ld4(y + (int64_t)t * dp + c), acc);
        }
      }
      for (int e = db; e < de; ++e) {
        const int s = g.dst_src[e];
        if ((unsigned)s < (unsigned)g.N) {
          const float w = gpred[g.dst_eid[e]];
          acc = f4fma(make_float4(w, w, w, w), ld4(y + (int64_t)s * dp + c), acc);
        }
      }
    }
    st4(dy + n * dp + c, acc);
    if (dyp.hi) planes_store4(dyp, n, c, acc);
  }
}

// <a, b> over d columns as one chain of fused multiply-adds in column order: the score of the positive and of every
// candidate, so equal rows give equal bits wherever it is inlined (no reassociation without fast-math)
__device__ __forceinline__ float rank_dot(const float* a, const float* b, int d) {
  float acc = 0.f;
  for (int c = 0; c < d; ++c) acc = fmaf(a[c], b[c], acc);
  return acc;
}

__device__ __forceinline__ bool is_positive(const void* lab, int bytes, int64_t k) {
  return bytes == 8 ? reinterpret_cast<const long long*>(lab)[k] == 1 : reinterpret_cast<const int*>(lab)[k] == 1;
}

// per_graph[g] = {hits@1, hits@3, hits@10, mrr} of graph g (0 without positives); see the comment at the top
__global__ void __launch_bounds__(kRankThreads) k_rank(const GpsGraph g, const float* __restrict__ y, int64_t ld, int d,
                                                       int pitch, int tile_rows, const void* __restrict__ lab,
                                                       int label_bytes, double* __restrict__ per_graph) {
  extern __shared__ float sm[];
  float* yi = sm;                                   // [d]
  float* tile = sm + pitch;                         // [tile_rows][pitch]
  __shared__ int pos_t[kRankChunk], pos_cnt[kRankChunk];
  __shared__ float pos_s[kRankChunk];
  __shared__ int s_m, s_next;
  const int tid = threadIdx.x, lane = tid & 31;
  const int gi = blockIdx.x;
  const int n0 = g.graph_ptr[gi], n1 = g.graph_ptr[gi + 1];
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  long long npos = 0;
  for (int i = n0; i < n1; ++i) {
    const int se = g.src_ptr[i + 1];
    int e = g.src_ptr[i];
    while (e < se) {
      __syncthreads();   // the previous chunk's readers are done with the shared state
      if (tid == 0) {    // the next positives of i in pair order
        int m = 0;
        for (; e < se && m < kRankChunk; ++e) {
          const int t = g.src_dst[e];
          if (t >= n0 && t < n1 && is_positive(lab, label_bytes, g.src_eid[e])) pos_t[m++] = t;
        }
        s_m = m;
        s_next = e;
      }
      for (int c = tid; c < d; c += kRankThreads) yi[c] = y[(int64_t)i * ld + c];
      __syncthreads();
      const int m = s_m;
      e = s_next;
      if (m == 0) continue;
      for (int p = tid; p < m; p += kRankThreads) {
        pos_s[p] = rank_dot(yi, y + (int64_t)pos_t[p] * ld, d);
        pos_cnt[p] = 0;
      }
      for (int k0 = n0; k0 < n1; k0 += tile_rows) {
        const int rows = min(tile_rows, n1 - k0);
        __syncthreads();   // pos_s / pos_cnt initialised, the previous tile consumed
        for (int r = tid >> 5; r < rows; r += kRankThreads / 32)
          for (int c = lane; c < d; c += 32) tile[r * pitch + c] = y[(int64_t)(k0 + r) * ld + c];
        __syncthreads();
        const bool live = tid < rows;
        const float s = live ? rank_dot(yi, tile + tid * pitch, d) : 0.f;
        for (int p = 0; p < m; ++p) {
          const unsigned above = __ballot_sync(0xffffffffu, live && k0 + tid != pos_t[p] && s > pos_s[p]);
          if (lane == 0 && above) atomicAdd(&pos_cnt[p], __popc(above));
        }
      }
      __syncthreads();
      if (tid == 0)
        for (int p = 0; p < m; ++p) {
          const int rank = 1 + pos_cnt[p];
          acc[0] += rank <= 1 ? 1.0 : 0.0;
          acc[1] += rank <= 3 ? 1.0 : 0.0;
          acc[2] += rank <= 10 ? 1.0 : 0.0;
          acc[3] += 1.0 / (double)rank;
          ++npos;
        }
    }
  }
  if (tid == 0)
    for (int q = 0; q < 4; ++q) per_graph[(int64_t)gi * 4 + q] = npos ? acc[q] / (double)npos : 0.0;
}

// stats[q] = mean over graphs of per_graph[:, q] in a fixed order (0 for no graphs)
__global__ void __launch_bounds__(256) k_rank_mean(const double* __restrict__ per_graph, int64_t B,
                                                   double* __restrict__ stats) {
  __shared__ double part[4][256];
  const int tid = threadIdx.x;
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (int64_t b = tid; b < B; b += 256)
    for (int q = 0; q < 4; ++q) s[q] += per_graph[b * 4 + q];
  for (int q = 0; q < 4; ++q) part[q][tid] = s[q];
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (tid < w)
      for (int q = 0; q < 4; ++q) part[q][tid] += part[q][tid + w];
    __syncthreads();
  }
  if (tid < 4) stats[tid] = B > 0 ? part[tid][0] / (double)B : 0.0;
}

int check_pairs(const GpsGraph* g, bool ranking, const char* what) {
  GPS_REQUIRE(g->N >= 0 && g->E >= 0 && g->B >= 0 && g->N < (1ll << 31) && g->E < (1ll << 31), GPS_ERR_ARG,
              "%s: pair graph sizes out of range", what);
  GPS_REQUIRE(g->N == 0 || (g->src_ptr && g->dst_ptr), GPS_ERR_ARG, "%s: pair graph without src_ptr / dst_ptr", what);
  GPS_REQUIRE(g->E == 0 || (g->src_dst && g->src_eid && g->dst_src && g->dst_eid), GPS_ERR_ARG,
              "%s: pair graph without its segments", what);
  GPS_REQUIRE(!ranking || g->graph_ptr, GPS_ERR_ARG, "%s: pair graph without graph_ptr", what);
  return GPS_OK;
}

int rank_metrics(const GpsGraph& g, const float* y, int64_t ld, int64_t d, const void* lab, int label_bytes,
                 double* stats, double* per_graph, cudaStream_t st) {
  if (g.B > 0) {
    const int pitch = (int)(d | 1);   // odd: consecutive threads read one column of consecutive rows conflict-free
    const int64_t per_row = (int64_t)pitch * sizeof(float);
    const int tile_rows = (int)std::min<int64_t>(kRankThreads, (kRankSmemCap - per_row) / per_row);
    const size_t smem = (size_t)(1 + tile_rows) * per_row;
    if (smem > 48 * 1024)
      GPS_CUDA(cudaFuncSetAttribute(k_rank, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_rank<<<(unsigned)g.B, kRankThreads, smem, st>>>(g, y, ld, (int)d, pitch, tile_rows, lab, label_bytes, per_graph);
    GPS_LAUNCH_CHECK();
  }
  k_rank_mean<<<1, 256, 0, st>>>(per_graph, g.B, stats);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

// =================================================================================== plan
struct LhPlan {
  int64_t N, K, B, d, dp;
  int prec;
  bool train;
  bool grads_prezeroed = true;   // linear_wgrad: the gradient region is zeroed once per backward call
  // saved: padded x, W, b (+ planes of x and W) and y
  float *x, *W, *b, *y;
  Planes x_p, W_p;
  int64_t saved_bytes;
  // forward workspace: per-graph ranking values (eval)
  double* per_graph;
  int64_t fwd_bytes;
  // backward workspace: dy (+ planes), dW | db zeroed as one region, padded grad_x
  float *dy, *gW, *gb, *gx;
  Planes dy_p;
  int64_t grads_bytes, bwd_bytes;
};

int make_plan(const GpsLinkHeadArgs* a, LhPlan* P, bool bind) {
  memset(P, 0, sizeof(*P));
  P->grads_prezeroed = true;
  GPS_REQUIRE(a, GPS_ERR_ARG, "link_head: null args");
  GPS_REQUIRE(a->d > 0, GPS_ERR_ARG, "link_head: d must be positive (got %lld)", (long long)a->d);
  GPS_REQUIRE(a->d <= 4096, GPS_ERR_UNSUPPORTED, "link_head: d <= 4096 (got %lld)", (long long)a->d);
  GPS_REQUIRE(a->precision == GPS_PREC_FP32 || a->precision == GPS_PREC_BF16, GPS_ERR_ARG,
              "link_head: unknown precision %d", a->precision);
  GPS_REQUIRE(a->flags == 0, GPS_ERR_ARG, "link_head: flags are reserved (got %d)", a->flags);
  GPS_REQUIRE(a->pairs.N >= 0 && a->pairs.E >= 0 && a->pairs.B >= 0, GPS_ERR_ARG, "link_head: negative sizes");
  const int64_t N = a->pairs.N, K = a->pairs.E, B = a->pairs.B, d = a->d, dp = round_up(d, 8);
  P->N = N; P->K = K; P->B = B; P->d = d; P->dp = dp;
  P->prec = a->precision;
  P->train = a->training != 0;
  const bool lo = a->precision == GPS_PREC_FP32;

  Arena S(bind ? a->saved : nullptr, a->saved_bytes);
  P->x = S.alloc<float>(N * dp);
  P->x_p = arena_planes(S, N, dp, lo);
  P->W = S.alloc<float>(dp * dp);
  P->W_p = arena_planes(S, dp, dp, lo);
  P->b = S.alloc<float>(dp);
  P->y = S.alloc<float>(N * dp);
  P->saved_bytes = S.used;
  GPS_REQUIRE(!bind || !S.overflow, GPS_ERR_ARG, "link_head: saved buffer too small (%lld < %lld)",
              (long long)a->saved_bytes, (long long)S.used);

  Arena F(bind ? a->workspace : nullptr, a->workspace_bytes);
  if (!P->train) P->per_graph = F.alloc<double>(4 * B);
  P->fwd_bytes = F.used;

  Arena Bk(bind ? a->workspace : nullptr, a->workspace_bytes);
  const int64_t g0 = Bk.used;
  P->gW = Bk.alloc<float>(dp * dp);
  P->gb = Bk.alloc<float>(dp);
  P->grads_bytes = Bk.used - g0;
  P->dy = Bk.alloc<float>(N * dp);
  P->dy_p = arena_planes(Bk, N, dp, lo);
  P->gx = Bk.alloc<float>(N * dp);
  P->bwd_bytes = Bk.used;
  return GPS_OK;
}

// plan, buffers and pointers of one call, all before any CUDA call
int prepare(const GpsLinkHeadArgs* a, bool fwd, LhPlan* P) {
  GPS_REQUIRE(a, GPS_ERR_ARG, "link_head: null args");
  GPS_REQUIRE(a->saved && a->workspace, GPS_ERR_ARG, "link_head: saved and workspace are required");
  GPS_TRY(make_plan(a, P, true));
  const bool stats = fwd && !P->train;
  GPS_TRY(check_pairs(&a->pairs, stats, "link_head"));
  const int64_t ws = fwd ? P->fwd_bytes : P->bwd_bytes;
  GPS_REQUIRE(a->workspace_bytes >= ws, GPS_ERR_ARG, "link_head: workspace too small (%lld < %lld)",
              (long long)a->workspace_bytes, (long long)ws);
  GPS_REQUIRE(a->lin.weight && a->lin.bias, GPS_ERR_ARG, "link_head: missing layer_post_mp weight / bias");
  GPS_REQUIRE(P->K == 0 || a->edge_index_labeled, GPS_ERR_ARG, "link_head: edge_index_labeled is required");
  if (fwd) {
    GPS_REQUIRE(P->N == 0 || (a->x && a->y), GPS_ERR_ARG, "link_head: x and y are required");
    GPS_REQUIRE(P->K == 0 || a->pred, GPS_ERR_ARG, "link_head: pred is required");
    if (stats) {
      GPS_REQUIRE(a->stats, GPS_ERR_ARG, "link_head: stats is required in eval mode");
      GPS_REQUIRE(a->label_bytes == 4 || a->label_bytes == 8, GPS_ERR_ARG, "link_head: label_bytes must be 4 or 8");
      GPS_REQUIRE(P->K == 0 || a->edge_label, GPS_ERR_ARG, "link_head: edge_label is required in eval mode");
    }
  } else {
    GPS_REQUIRE(P->N == 0 || a->grad_x, GPS_ERR_ARG, "link_head: grad_x is required");
  }
  return GPS_OK;
}

int lh_forward(const GpsLinkHeadArgs* a, cudaStream_t st) {
  LhPlan P;
  GPS_TRY(prepare(a, true, &P));
  const int64_t N = P.N, K = P.K, d = P.d, dp = P.dp;
  if (N > 0) {
    PadList L;
    L.add(a->x, d, N, d, P.x, dp, N, dp, P.x_p);
    L.add(a->lin.weight, d, d, d, P.W, dp, dp, dp, P.W_p);
    L.add(a->lin.bias, d, 1, d, P.b, dp, 1, dp);
    GPS_TRY(L.run(st));
    GPS_TRY(gemm(linear_fwd(P, N, dp, dp, {P.x, dp, P.x_p}, {P.W, dp, P.W_p}, P.y, dp, P.b), st));
  }
  if (K > 0) {
    k_pair_score<<<(unsigned)ceil_div(K * 32, 256), 256, 0, st>>>(P.y, dp, N, a->edge_index_labeled, K, a->pred);
    GPS_LAUNCH_CHECK();
  }
  if (!P.train)
    GPS_TRY(rank_metrics(a->pairs, P.y, dp, d, a->edge_label, a->label_bytes, a->stats, P.per_graph, st));
  if (N == 0) return GPS_OK;
  PadList U;
  U.add(P.y, dp, N, d, a->y, d, N, d);
  return U.run(st);
}

int lh_backward(const GpsLinkHeadArgs* a, cudaStream_t st) {
  LhPlan P;
  GPS_TRY(prepare(a, false, &P));
  const int64_t N = P.N, d = P.d, dp = P.dp;
  GPS_CUDA(cudaMemsetAsync(P.gW, 0, (size_t)P.grads_bytes, st));
  if (N > 0) {
    k_pair_grad<<<(unsigned)ceil_div(N * 32, 256), 256, 0, st>>>(a->pairs, P.y, dp, a->grad_y, d,
                                                                 P.K > 0 ? a->grad_pred : nullptr, P.dy, P.dy_p);
    GPS_LAUNCH_CHECK();
    const Operand dy{P.dy, dp, P.dy_p};
    GPS_TRY(linear_wgrad(P, dy, {P.x, dp, P.x_p}, N, dp, dp, P.gW, P.gb, st));
    GPS_TRY(gemm(linear_dgrad(P, N, dp, dp, dy, {P.W, dp, P.W_p}, P.gx, dp), st));
  }
  PadList U;
  U.add(P.gW, dp, d, d, a->lin.grad_weight, d, d, d);
  U.add(P.gb, dp, 1, d, a->lin.grad_bias, d, 1, d);
  U.add(P.gx, dp, N, d, a->grad_x, d, N, d);
  return U.run(st);
}

}  // namespace

}  // namespace gps

// =================================================================================== C ABI
using namespace gps;

extern "C" int gps_link_head_plan(const GpsLinkHeadArgs* args, GpsLinkHeadPlan* plan) {
  GPS_REQUIRE(args && plan, GPS_ERR_ARG, "gps_link_head_plan: null argument");
  LhPlan P;
  GPS_TRY(make_plan(args, &P, false));
  plan->saved_bytes = P.saved_bytes;
  plan->fwd_workspace_bytes = P.fwd_bytes;
  plan->bwd_workspace_bytes = P.bwd_bytes;
  return GPS_OK;
}

extern "C" int gps_link_head_forward(const GpsLinkHeadArgs* args, void* stream) {
  return lh_forward(args, (cudaStream_t)stream);
}

extern "C" int gps_link_head_backward(const GpsLinkHeadArgs* args, void* stream) {
  return lh_backward(args, (cudaStream_t)stream);
}

extern "C" int gps_link_rank_metrics(const GpsGraph* pairs, const float* y, int64_t ld, int64_t d,
                                     const void* edge_label, int32_t label_bytes, double* stats, void* workspace,
                                     int64_t workspace_bytes, void* stream) {
  GPS_REQUIRE(pairs && stats && workspace, GPS_ERR_ARG, "gps_link_rank_metrics: null argument");
  GPS_TRY(check_pairs(pairs, true, "gps_link_rank_metrics"));
  GPS_REQUIRE(d >= 1 && d <= 4096 && ld >= d, GPS_ERR_ARG, "gps_link_rank_metrics: needs 1 <= d <= 4096 and ld >= d");
  GPS_REQUIRE(pairs->N == 0 || y, GPS_ERR_ARG, "gps_link_rank_metrics: y is required");
  GPS_REQUIRE(label_bytes == 4 || label_bytes == 8, GPS_ERR_ARG, "gps_link_rank_metrics: label_bytes must be 4 or 8");
  GPS_REQUIRE(pairs->E == 0 || edge_label, GPS_ERR_ARG, "gps_link_rank_metrics: edge_label is required");
  GPS_REQUIRE(workspace_bytes >= 32 * pairs->B, GPS_ERR_ARG, "gps_link_rank_metrics: workspace too small (%lld < %lld)",
              (long long)workspace_bytes, (long long)(32 * pairs->B));
  return rank_metrics(*pairs, y, ld, d, edge_label, label_bytes, stats, (double*)workspace, (cudaStream_t)stream);
}
