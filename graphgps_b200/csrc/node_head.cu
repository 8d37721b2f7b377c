// node_head.cu — the node-prediction heads of the node-level configs and their losses, forward and backward, one C
// call per direction, and their C ABI: GraphGym's MLP under graphgps/head/inductive_node.py (GNNInductiveNodeHead)
// and GraphGym's GNNNodeHead (`node`, a row selection by the split's mask), then weighted_cross_entropy
// (graphgps/loss/weighted_cross_entropy.py) or GraphGym's cross_entropy.
//
//   head forward   pad weights and x (+ planes) -> for l < L-1: h_{l+1} = relu(h_l W_l^T + b_l) (GEMM epilogue),
//                  then normalised in place (+ planes, row norms saved) -> y = h_{L-1} W^T + b -> unpad y, pred = y[rows]
//   head backward  g_{L-1} = pad(grad_y) (+ planes), + grad_pred on rows -> for l = L-1..0: dW_l, db_l (split-K) and
//                  G = g_l W_l; l > 0: g_{l-1} = normalize'(G) relu'(.) (+ planes) -> unpad grads and grad_x
//   loss forward   per row: log_softmax (sigmoid for C = 1), the row's loss term, the class counts (integer atomics)
//                  -> per-CTA fp64 partials of sum w_{y_i} term_i and sum w_{y_i} -> one CTA adds them in order
//   loss backward  per row: grad_pred from the loss's scalar gradient and the gradient of pred_score
//
// Every width w runs at p = round_up(w, 8) with zero pad columns (as graph_head.cu does), so the dense products are the
// TMA GEMM with its fused bias / ReLU epilogues and the pad columns of every activation and gradient stay zero.
#include <string.h>

#include "layer_ops.cuh"

namespace gps {

namespace {

constexpr float kNormEps = 1e-12f;   // F.normalize's default eps
constexpr int kLossParts = 264;      // CTAs of the loss's partial sums (two per SM)

// ------------------------------------------------------------------------------- row normalisation
// One warp per row of d columns (d % 4 == 0) at pitch ld: the sum of squares in lane order, then the butterfly.
// out may alias r and gin may alias g (in place): those pointers carry no __restrict__
__global__ void k_l2norm_fwd(const float* r, int64_t rows, int d, int64_t ld, float* out,
                             float* __restrict__ norm, Planes p) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < rows; i += warps) {
    const float* src = r + i * ld;
    float s = 0.f;
    for (int c = lane * 4; c < d; c += 128) {
      const float4 v = ld4(src + c);
      s = fmaf(v.x, v.x, s); s = fmaf(v.y, v.y, s); s = fmaf(v.z, v.z, s); s = fmaf(v.w, v.w, s);
    }
    s = warp_sum(s);
    const float n = sqrtf(s), den = fmaxf(n, kNormEps);
    for (int c = lane * 4; c < d; c += 128) {
      const float4 v = ld4(src + c);
      const float4 o = make_float4(v.x / den, v.y / den, v.z / den, v.w / den);
      st4(out + i * ld + c, o);
      if (p.hi) planes_store4(p, i, c, o);
    }
    if (lane == 0) norm[i] = n;
  }
}

// grad_in = (g - h (h.g)) / n for n >= eps, g / eps below, times relu'(.) = [h > 0]; h = the forward's output
__global__ void k_l2norm_bwd(const float* g, const float* __restrict__ h, const float* __restrict__ norm,
                             int64_t rows, int d, int64_t ld, float* gin, Planes p) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < rows; i += warps) {
    const float* gr = g + i * ld;
    const float* hr = h + i * ld;
    const float n = norm[i];
    const bool big = n >= kNormEps;
    float dot = 0.f;
    if (big) {
      for (int c = lane * 4; c < d; c += 128) {
        const float4 a = ld4(gr + c), b = ld4(hr + c);
        dot = fmaf(a.x, b.x, dot); dot = fmaf(a.y, b.y, dot); dot = fmaf(a.z, b.z, dot); dot = fmaf(a.w, b.w, dot);
      }
      dot = warp_sum(dot);
    }
    const float den = big ? n : kNormEps;
    for (int c = lane * 4; c < d; c += 128) {
      const float4 a = ld4(gr + c), b = ld4(hr + c);
      float4 o;
      o.x = b.x > 0.f ? (a.x - b.x * dot) / den : 0.f;
      o.y = b.y > 0.f ? (a.y - b.y * dot) / den : 0.f;
      o.z = b.z > 0.f ? (a.z - b.z * dot) / den : 0.f;
      o.w = b.w > 0.f ? (a.w - b.w * dot) / den : 0.f;
      st4(gin + i * ld + c, o);
      if (p.hi) planes_store4(p, i, c, o);
    }
  }
}

// blocks of 8 warps for one warp per row
unsigned warp_blocks(int64_t rows) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div(rows, 8), (int64_t)kNumSMs * 16));
}

int l2norm_fwd(const float* r, int64_t rows, int64_t d, int64_t ld, float* out, float* norm, Planes p, cudaStream_t st) {
  if (rows == 0) return GPS_OK;
  k_l2norm_fwd<<<warp_blocks(rows), 256, 0, st>>>(r, rows, (int)d, ld, out, norm, p);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int l2norm_bwd(const float* g, const float* h, const float* norm, int64_t rows, int64_t d, int64_t ld, float* gin,
               Planes p, cudaStream_t st) {
  if (rows == 0) return GPS_OK;
  k_l2norm_bwd<<<warp_blocks(rows), 256, 0, st>>>(g, h, norm, rows, (int)d, ld, gin, p);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

// ------------------------------------------------------------------------------- head output / gradient seed
// y [N, dout] = ypad[:, :dout]; pred [M, dout] = ypad[rows] (rows outside [0, N) are skipped)
__global__ void k_head_out(const float* __restrict__ ypad, int64_t ld, int64_t N, int dout, float* __restrict__ y,
                           const int64_t* __restrict__ rows, int64_t M, float* __restrict__ pred) {
  const int64_t total = (N + M) * dout;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = k / dout;
    const int c = (int)(k - i * dout);
    if (i < N) {
      y[i * dout + c] = ypad[i * ld + c];
    } else {
      const int64_t r = rows[i - N];
      if (r >= 0 && r < N) pred[(i - N) * dout + c] = ypad[r * ld + c];
    }
  }
}

// g [N, ld] = grad_y (or 0) with zero pad columns, + planes; one thread per 4 columns
__global__ void k_grad_seed(const float* __restrict__ gy, int64_t N, int dout, int64_t ld, float* __restrict__ g,
                            Planes p) {
  const int64_t q = ld / 4, total = N * q;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = k / q;
    const int c = (int)(k - i * q) * 4;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = gy && c + j < dout ? gy[i * dout + c + j] : 0.f;
    const float4 o = make_float4(v[0], v[1], v[2], v[3]);
    st4(g + i * ld + c, o);
    if (p.hi) planes_store4(p, i, c, o);
  }
}

// g[rows[m]] += grad_pred[m] (+ planes of those rows); rows are distinct, so no two threads share an element
__global__ void k_grad_rows(const float* __restrict__ gp, const int64_t* __restrict__ rows, int64_t M, int64_t N,
                            int dout, int64_t ld, float* __restrict__ g, Planes p) {
  const int64_t q = ld / 4, total = M * q;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = k / q;
    const int c = (int)(k - m * q) * 4;
    const int64_t r = rows[m];
    if (r < 0 || r >= N) continue;
    float4 o = ld4(g + r * ld + c);
    float v[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (c + j < dout) v[j] += gp[m * dout + c + j];
    o = make_float4(v[0], v[1], v[2], v[3]);
    st4(g + r * ld + c, o);
    if (p.hi) planes_store4(p, r, c, o);
  }
}

unsigned grid_for(int64_t total, int threads) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div(total, threads), (int64_t)kNumSMs * 32));
}

// =================================================================================== head plan
constexpr int kMaxL = GPS_NODE_HEAD_MAX_L;

struct NhPlan {
  int64_t N, M, L, din, dinner, dout;
  int prec;
  bool grads_prezeroed = true;   // linear_wgrad: the gradient region is zeroed once per backward call
  int64_t win[kMaxL], wout[kMaxL], pin[kMaxL], pout[kMaxL];   // real and padded widths of fc[l]
  // saved: padded weights (+ planes) and biases, h_l [N, pin[l]] (+ planes; h_0 = padded x, h_l the normalised rows)
  // and the row norms of h_l (l >= 1)
  float *W[kMaxL], *b[kMaxL], *h[kMaxL], *norm[kMaxL];
  Planes W_p[kMaxL], h_p[kMaxL];
  int64_t saved_bytes;
  float* ypad;   // forward workspace [N, pout[L-1]]
  int64_t fwd_bytes;
  // backward workspace: dW_l | db_l zeroed as one region, g_l [N, pout[l]] (+ planes), G [N, max pin] (dgrad output)
  float *gW[kMaxL], *gb[kMaxL], *g[kMaxL], *G;
  Planes g_p[kMaxL];
  int64_t grads_bytes, bwd_bytes;
};

int make_head_plan(const GpsNodeHeadArgs* a, NhPlan* P, bool bind) {
  memset(P, 0, sizeof(*P));
  P->grads_prezeroed = true;
  GPS_REQUIRE(a, GPS_ERR_ARG, "node_head: null args");
  GPS_REQUIRE(a->L >= 1, GPS_ERR_ARG, "node_head: L must be >= 1 (got %d)", a->L);
  GPS_REQUIRE(a->L <= kMaxL, GPS_ERR_UNSUPPORTED, "node_head: L <= %d (got %d)", kMaxL, a->L);
  GPS_REQUIRE(a->dim_in >= 1 && a->dim_out >= 1 && (a->L == 1 || a->dim_inner >= 1), GPS_ERR_ARG,
              "node_head: dim_in, dim_inner and dim_out must be positive");
  GPS_REQUIRE(a->dim_in <= 4096 && a->dim_out <= 4096 && (a->L == 1 || a->dim_inner <= 4096), GPS_ERR_UNSUPPORTED,
              "node_head: dim_in, dim_inner and dim_out <= 4096");
  GPS_REQUIRE(a->precision == GPS_PREC_FP32 || a->precision == GPS_PREC_BF16, GPS_ERR_ARG,
              "node_head: unknown precision %d", a->precision);
  GPS_REQUIRE(a->flags == 0, GPS_ERR_ARG, "node_head: flags are reserved (got %d)", a->flags);
  GPS_REQUIRE(a->N >= 0 && a->N < (1ll << 31) && a->M >= 0 && a->M < (1ll << 31), GPS_ERR_ARG,
              "node_head: N and M out of range");
  const int64_t N = a->N, L = a->L;
  P->N = N; P->M = a->M; P->L = L; P->din = a->dim_in; P->dinner = a->dim_inner; P->dout = a->dim_out;
  P->prec = a->precision;
  for (int64_t l = 0; l < L; ++l) {
    P->win[l] = l == 0 ? a->dim_in : a->dim_inner;
    P->wout[l] = l == L - 1 ? a->dim_out : a->dim_inner;
    P->pin[l] = round_up(P->win[l], 8);
    P->pout[l] = round_up(P->wout[l], 8);
  }
  const bool lo = a->precision == GPS_PREC_FP32;
  Arena S(bind ? a->saved : nullptr, a->saved_bytes);
  for (int64_t l = 0; l < L; ++l) {
    P->W[l] = S.alloc<float>(P->pout[l] * P->pin[l]);
    P->W_p[l] = arena_planes(S, P->pout[l], P->pin[l], lo);
    P->b[l] = S.alloc<float>(P->pout[l]);
    P->h[l] = S.alloc<float>(N * P->pin[l]);
    P->h_p[l] = arena_planes(S, N, P->pin[l], lo);
    if (l > 0) P->norm[l] = S.alloc<float>(N);
  }
  P->saved_bytes = S.used;
  GPS_REQUIRE(!bind || !S.overflow, GPS_ERR_ARG, "node_head: saved buffer too small (%lld < %lld)",
              (long long)a->saved_bytes, (long long)S.used);

  Arena F(bind ? a->workspace : nullptr, a->workspace_bytes);
  P->ypad = F.alloc<float>(N * P->pout[L - 1]);
  P->fwd_bytes = F.used;

  Arena Bk(bind ? a->workspace : nullptr, a->workspace_bytes);
  for (int64_t l = 0; l < L; ++l) {
    P->gW[l] = Bk.alloc<float>(P->pout[l] * P->pin[l]);
    P->gb[l] = Bk.alloc<float>(P->pout[l]);
  }
  P->grads_bytes = Bk.used;
  int64_t pmax = 0;
  for (int64_t l = 0; l < L; ++l) {
    P->g[l] = Bk.alloc<float>(N * P->pout[l]);
    P->g_p[l] = arena_planes(Bk, N, P->pout[l], lo);
    pmax = std::max(pmax, P->pin[l]);
  }
  P->G = Bk.alloc<float>(N * pmax);
  P->bwd_bytes = Bk.used;
  return GPS_OK;
}

int prepare_head(const GpsNodeHeadArgs* a, bool fwd, NhPlan* P) {
  GPS_REQUIRE(a, GPS_ERR_ARG, "node_head: null args");
  GPS_REQUIRE(a->saved && a->workspace, GPS_ERR_ARG, "node_head: saved and workspace are required");
  GPS_TRY(make_head_plan(a, P, true));
  const int64_t ws = fwd ? P->fwd_bytes : P->bwd_bytes;
  GPS_REQUIRE(a->workspace_bytes >= ws, GPS_ERR_ARG, "node_head: workspace too small (%lld < %lld)",
              (long long)a->workspace_bytes, (long long)ws);
  for (int64_t l = 0; l < P->L; ++l)
    GPS_REQUIRE(a->fc[l].weight && a->fc[l].bias, GPS_ERR_ARG, "node_head: missing fc[%lld] weight / bias",
                (long long)l);
  GPS_REQUIRE(P->M == 0 || a->rows, GPS_ERR_ARG, "node_head: M > 0 needs rows");
  if (fwd) {
    GPS_REQUIRE(P->N == 0 || (a->x && a->y), GPS_ERR_ARG, "node_head: x and y are required");
    GPS_REQUIRE(P->M == 0 || a->pred, GPS_ERR_ARG, "node_head: pred is required with rows");
  } else {
    GPS_REQUIRE(P->N == 0 || a->grad_x, GPS_ERR_ARG, "node_head: grad_x is required");
  }
  return GPS_OK;
}

int nh_forward(const GpsNodeHeadArgs* a, cudaStream_t st) {
  NhPlan P;
  GPS_TRY(prepare_head(a, true, &P));
  const int64_t N = P.N, L = P.L;
  {
    PadList W;
    for (int64_t l = 0; l < L; ++l) {
      W.add(a->fc[l].weight, P.win[l], P.wout[l], P.win[l], P.W[l], P.pin[l], P.pout[l], P.pin[l], P.W_p[l]);
      W.add(a->fc[l].bias, P.wout[l], 1, P.wout[l], P.b[l], P.pout[l], 1, P.pout[l]);
    }
    if (N > 0) W.add(a->x, P.din, N, P.din, P.h[0], P.pin[0], N, P.pin[0], P.h_p[0]);
    GPS_TRY(W.run(st));
  }
  if (N == 0) return GPS_OK;
  for (int64_t l = 0; l < L; ++l) {
    const Operand h{P.h[l], P.pin[l], P.h_p[l]};
    const bool last = l == L - 1;
    GemmParams g = linear_fwd(P, N, P.pout[l], P.pin[l], h, {P.W[l], P.pin[l], P.W_p[l]}, last ? P.ypad : P.h[l + 1],
                              P.pout[l], P.b[l]);
    if (!last) g.act = GPS_ACT_RELU;
    GPS_TRY(gemm(g, st));
    if (!last)
      GPS_TRY(l2norm_fwd(P.h[l + 1], N, P.pin[l + 1], P.pin[l + 1], P.h[l + 1], P.norm[l + 1], P.h_p[l + 1], st));
  }
  const int64_t total = (N + P.M) * P.dout;
  k_head_out<<<grid_for(total, 256), 256, 0, st>>>(P.ypad, P.pout[L - 1], N, (int)P.dout, a->y, a->rows, P.M, a->pred);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int nh_backward(const GpsNodeHeadArgs* a, cudaStream_t st) {
  NhPlan P;
  GPS_TRY(prepare_head(a, false, &P));
  const int64_t N = P.N, L = P.L;
  GPS_CUDA(cudaMemsetAsync(P.gW[0], 0, (size_t)P.grads_bytes, st));
  if (N > 0) {
    const int64_t ldl = P.pout[L - 1];
    k_grad_seed<<<grid_for(N * ldl / 4, 256), 256, 0, st>>>(a->grad_y, N, (int)P.dout, ldl, P.g[L - 1], P.g_p[L - 1]);
    GPS_LAUNCH_CHECK();
    if (P.M > 0 && a->grad_pred) {
      k_grad_rows<<<grid_for(P.M * ldl / 4, 256), 256, 0, st>>>(a->grad_pred, a->rows, P.M, N, (int)P.dout, ldl,
                                                                P.g[L - 1], P.g_p[L - 1]);
      GPS_LAUNCH_CHECK();
    }
    for (int64_t l = L - 1; l >= 0; --l) {
      const Operand gl{P.g[l], P.pout[l], P.g_p[l]};
      const Operand h{P.h[l], P.pin[l], P.h_p[l]};
      GPS_TRY(linear_wgrad(P, gl, h, N, P.pout[l], P.pin[l], P.gW[l], P.gb[l], st));
      GPS_TRY(gemm(linear_dgrad(P, N, P.pin[l], P.pout[l], gl, {P.W[l], P.pin[l], P.W_p[l]}, P.G, P.pin[l]), st));
      if (l > 0)   // the gradient of layer l-1's pre-activation, through the normalisation and the ReLU
        GPS_TRY(l2norm_bwd(P.G, P.h[l], P.norm[l], N, P.pin[l], P.pin[l], P.g[l - 1], P.g_p[l - 1], st));
    }
  }
  PadList U;
  for (int64_t l = 0; l < L; ++l) {
    U.add(P.gW[l], P.pin[l], P.wout[l], P.win[l], a->fc[l].grad_weight, P.win[l], P.wout[l], P.win[l]);
    U.add(P.gb[l], P.pout[l], 1, P.wout[l], a->fc[l].grad_bias, P.wout[l], 1, P.wout[l]);
  }
  if (N > 0) U.add(P.G, P.pin[0], N, P.din, a->grad_x, P.din, N, P.din);
  return U.run(st);
}

// =================================================================================== loss
struct NlPlan {
  int64_t M, C, K;   // K = classes counted: max(C, 2)
  int weighted;
  int* counts;       // saved [K]
  float* den;        // saved [1]: the loss's denominator
  int64_t saved_bytes;
  float* term;       // workspace [M]: each row's loss term
  double* part;      // workspace [kLossParts][2]
  int64_t fwd_bytes, bwd_bytes;
};

int make_loss_plan(const GpsNodeLossArgs* a, NlPlan* P, bool bind) {
  memset(P, 0, sizeof(*P));
  GPS_REQUIRE(a, GPS_ERR_ARG, "node_loss: null args");
  GPS_REQUIRE(a->M >= 0 && a->M < (1ll << 31), GPS_ERR_ARG, "node_loss: M out of range (%lld)", (long long)a->M);
  GPS_REQUIRE(a->C >= 1, GPS_ERR_ARG, "node_loss: C must be positive (got %lld)", (long long)a->C);
  GPS_REQUIRE(a->C <= GPS_NODE_LOSS_MAX_C, GPS_ERR_UNSUPPORTED, "node_loss: C <= %d (got %lld)", GPS_NODE_LOSS_MAX_C,
              (long long)a->C);
  GPS_REQUIRE(a->weighted == 0 || a->weighted == 1, GPS_ERR_ARG, "node_loss: weighted is 0 or 1 (got %d)",
              a->weighted);
  GPS_REQUIRE(a->C > 1 || a->weighted, GPS_ERR_UNSUPPORTED,
              "node_loss: C = 1 (binary) is built for the weighted loss only");
  GPS_REQUIRE(a->flags == 0, GPS_ERR_ARG, "node_loss: flags are reserved (got %d)", a->flags);
  P->M = a->M; P->C = a->C; P->K = std::max<int64_t>(a->C, 2); P->weighted = a->weighted;
  Arena S(bind ? a->saved : nullptr, a->saved_bytes);
  P->counts = S.alloc<int>(P->K);
  P->den = S.alloc<float>(1);
  P->saved_bytes = S.used;
  GPS_REQUIRE(!bind || !S.overflow, GPS_ERR_ARG, "node_loss: saved buffer too small (%lld < %lld)",
              (long long)a->saved_bytes, (long long)S.used);
  Arena F(bind ? a->workspace : nullptr, a->workspace_bytes);
  P->term = F.alloc<float>(std::max<int64_t>(P->M, 1));
  P->part = F.alloc<double>(2 * kLossParts);
  P->fwd_bytes = F.used;
  P->bwd_bytes = 0;
  return GPS_OK;
}

// the class weight w_c as the reference computes it: float32 (V - count) / V, times [count > 0]
__device__ __forceinline__ float class_weight(const int* counts, int64_t K, int64_t t, int64_t V) {
  if (t < 0 || t >= K) return __int_as_float(0x7fc00000);   // never reached through the Python module
  const int n = counts[t];
  return n > 0 ? (float)(V - n) / (float)V : 0.f;
}

// one warp per row: pred_score, the row's term (-log p[y] or bce) and, weighted, the class count
__global__ void k_loss_rows(const float* __restrict__ pred, const int64_t* __restrict__ label, int64_t M, int C,
                            int64_t K, int weighted, float* __restrict__ score, float* __restrict__ term,
                            int* __restrict__ counts) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < M; i += warps) {
    const int64_t t = label[i];
    const bool ok = t >= 0 && t < K;
    if (weighted && ok && lane == 0) atomicAdd(counts + t, 1);
    const float* x = pred + i * C;
    if (C == 1) {
      if (lane == 0) {
        const float v = x[0], y = (float)t;
        score[i] = 1.f / (1.f + expf(-v));
        term[i] = ok ? fmaxf(v, 0.f) - v * y + log1pf(expf(-fabsf(v))) : __int_as_float(0x7fc00000);
      }
      continue;
    }
    float m = -INFINITY;
    for (int c = lane; c < C; c += 32) m = fmaxf(m, x[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += expf(x[c] - m);
    s = warp_sum(s);
    const float ls = logf(s);
    for (int c = lane; c < C; c += 32) score[i * C + c] = (x[c] - m) - ls;
    if (lane == 0) term[i] = ok ? -((x[t] - m) - ls) : __int_as_float(0x7fc00000);
  }
}

// CTA b sums rows [b * chunk, (b + 1) * chunk): each thread in row order, then a fixed tree; part[b] = (num, den)
__global__ void k_loss_part(const float* __restrict__ term, const int64_t* __restrict__ label, int64_t M, int64_t K,
                            int weighted, const int* __restrict__ counts, int64_t chunk, double* __restrict__ part) {
  __shared__ double sn[256], sd[256];
  const int64_t r0 = (int64_t)blockIdx.x * chunk, r1 = min(M, r0 + chunk);
  double num = 0.0, den = 0.0;
  for (int64_t i = r0 + threadIdx.x; i < r1; i += blockDim.x) {
    const float w = weighted ? class_weight(counts, K, label[i], M) : 1.f;
    num += (double)w * (double)term[i];
    den += (double)w;
  }
  sn[threadIdx.x] = num;
  sd[threadIdx.x] = den;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) {
      sn[threadIdx.x] += sn[threadIdx.x + s];
      sd[threadIdx.x] += sd[threadIdx.x + s];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    part[2 * blockIdx.x] = sn[0];
    part[2 * blockIdx.x + 1] = sd[0];
  }
}

// the partials in CTA order; binary divides by M (BCE's mean), multiclass by sum w_{y_i} (nll_loss's weighted mean)
__global__ void k_loss_final(const double* __restrict__ part, int parts, int64_t M, int binary, float* __restrict__ loss,
                             float* __restrict__ den_out) {
  double num = 0.0, den = 0.0;
  for (int b = 0; b < parts; ++b) {
    num += part[2 * b];
    den += part[2 * b + 1];
  }
  if (binary) den = (double)M;
  loss[0] = (float)(num / den);
  den_out[0] = (float)den;
}

// grad_pred from g = grad_loss and the gradient of pred_score (one warp per row)
__global__ void k_loss_bwd(const float* __restrict__ score, const int64_t* __restrict__ label, int64_t M, int C,
                           int64_t K, int weighted, const int* __restrict__ counts, const float* __restrict__ den,
                           const float* __restrict__ grad_loss, const float* __restrict__ gs,
                           float* __restrict__ gp) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  // no loss gradient adds nothing (a zero one would still be 0 * (0 / 0) = NaN over weights that sum to 0, as in torch)
  const bool has_loss = grad_loss != nullptr;
  const float coef = has_loss ? grad_loss[0] / den[0] : 0.f;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < M; i += warps) {
    const int64_t t = label[i];
    const float w = weighted ? class_weight(counts, K, t, M) : 1.f;
    if (C == 1) {
      if (lane == 0) {
        const float sg = score[i];
        float v = has_loss ? (sg - (float)t) * w * coef : 0.f;
        if (gs) v += gs[i] * (1.f - sg) * sg;
        gp[i] = v;
      }
      continue;
    }
    const float* sr = score + i * C;
    float sum = 0.f;
    for (int c = lane; c < C; c += 32) {
      float G = gs ? gs[i * C + c] : 0.f;
      if (has_loss && c == t) G += w * -coef;
      sum += G;
    }
    sum = warp_sum(sum);
    for (int c = lane; c < C; c += 32) {
      float G = gs ? gs[i * C + c] : 0.f;
      if (has_loss && c == t) G += w * -coef;
      gp[i * C + c] = G - expf(sr[c]) * sum;
    }
  }
}

int nl_forward(const GpsNodeLossArgs* a, cudaStream_t st) {
  NlPlan P;
  GPS_REQUIRE(a, GPS_ERR_ARG, "node_loss: null args");
  GPS_REQUIRE(a->saved && a->workspace, GPS_ERR_ARG, "node_loss: saved and workspace are required");
  GPS_TRY(make_loss_plan(a, &P, true));
  GPS_REQUIRE(a->workspace_bytes >= P.fwd_bytes, GPS_ERR_ARG, "node_loss: workspace too small (%lld < %lld)",
              (long long)a->workspace_bytes, (long long)P.fwd_bytes);
  GPS_REQUIRE(a->loss, GPS_ERR_ARG, "node_loss: loss is required");
  GPS_REQUIRE(P.M == 0 || (a->pred && a->label && a->pred_score), GPS_ERR_ARG,
              "node_loss: pred, label and pred_score are required");
  if (P.weighted) GPS_CUDA(cudaMemsetAsync(P.counts, 0, (size_t)P.K * sizeof(int), st));
  if (P.M > 0) {
    k_loss_rows<<<warp_blocks(P.M), 256, 0, st>>>(a->pred, a->label, P.M, (int)P.C, P.K, P.weighted, a->pred_score,
                                                   P.term, P.counts);
    GPS_LAUNCH_CHECK();
  }
  const int parts = (int)std::max<int64_t>(1, std::min<int64_t>(kLossParts, ceil_div(P.M, 1024)));
  const int64_t chunk = std::max<int64_t>(1, ceil_div(P.M, parts));
  k_loss_part<<<parts, 256, 0, st>>>(P.term, a->label, P.M, P.K, P.weighted, P.counts, chunk, P.part);
  GPS_LAUNCH_CHECK();
  k_loss_final<<<1, 1, 0, st>>>(P.part, parts, P.M, P.C == 1, a->loss, P.den);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int nl_backward(const GpsNodeLossArgs* a, cudaStream_t st) {
  NlPlan P;
  GPS_REQUIRE(a, GPS_ERR_ARG, "node_loss: null args");
  GPS_REQUIRE(a->saved, GPS_ERR_ARG, "node_loss: saved is required");
  GPS_TRY(make_loss_plan(a, &P, true));
  GPS_REQUIRE(P.M == 0 || (a->label && a->pred_score && a->grad_pred), GPS_ERR_ARG,
              "node_loss: label, pred_score and grad_pred are required");
  if (P.M == 0) return GPS_OK;
  k_loss_bwd<<<warp_blocks(P.M), 256, 0, st>>>(a->pred_score, a->label, P.M, (int)P.C, P.K, P.weighted, P.counts,
                                                P.den, a->grad_loss, a->grad_score, a->grad_pred);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int l2norm_check(int64_t rows, int64_t d, int64_t ld, const char* what) {
  GPS_REQUIRE(rows >= 0 && d >= 1 && ld >= d, GPS_ERR_ARG, "%s: needs rows >= 0, d >= 1 and ld >= d", what);
  GPS_REQUIRE(d % 4 == 0 && ld % 4 == 0 && d <= 4096, GPS_ERR_UNSUPPORTED,
              "%s: needs d %% 4 == 0, ld %% 4 == 0 and d <= 4096 (got d %lld, ld %lld)", what, (long long)d,
              (long long)ld);
  return GPS_OK;
}

}  // namespace

}  // namespace gps

// =================================================================================== C ABI
using namespace gps;

extern "C" int gps_node_head_plan(const GpsNodeHeadArgs* args, GpsNodeHeadPlan* plan) {
  GPS_REQUIRE(args && plan, GPS_ERR_ARG, "gps_node_head_plan: null argument");
  NhPlan P;
  GPS_TRY(make_head_plan(args, &P, false));
  plan->saved_bytes = P.saved_bytes;
  plan->fwd_workspace_bytes = P.fwd_bytes;
  plan->bwd_workspace_bytes = P.bwd_bytes;
  return GPS_OK;
}

extern "C" int gps_node_head_forward(const GpsNodeHeadArgs* args, void* stream) {
  return nh_forward(args, (cudaStream_t)stream);
}

extern "C" int gps_node_head_backward(const GpsNodeHeadArgs* args, void* stream) {
  return nh_backward(args, (cudaStream_t)stream);
}

extern "C" int gps_row_l2norm_forward(const float* r, int64_t rows, int64_t d, int64_t ld, float* out, float* norm,
                                      void* stream) {
  GPS_TRY(l2norm_check(rows, d, ld, "gps_row_l2norm_forward"));
  GPS_REQUIRE(rows == 0 || (r && out && norm), GPS_ERR_ARG, "gps_row_l2norm_forward: r, out and norm are required");
  return l2norm_fwd(r, rows, d, ld, out, norm, Planes(), (cudaStream_t)stream);
}

extern "C" int gps_row_l2norm_backward(const float* g, const float* out, const float* norm, int64_t rows, int64_t d,
                                       int64_t ld, float* grad_in, void* stream) {
  GPS_TRY(l2norm_check(rows, d, ld, "gps_row_l2norm_backward"));
  GPS_REQUIRE(rows == 0 || (g && out && norm && grad_in), GPS_ERR_ARG,
              "gps_row_l2norm_backward: g, out, norm and grad_in are required");
  return l2norm_bwd(g, out, norm, rows, d, ld, grad_in, Planes(), (cudaStream_t)stream);
}

extern "C" int gps_node_loss_plan(const GpsNodeLossArgs* args, GpsNodeLossPlan* plan) {
  GPS_REQUIRE(args && plan, GPS_ERR_ARG, "gps_node_loss_plan: null argument");
  NlPlan P;
  GPS_TRY(make_loss_plan(args, &P, false));
  plan->saved_bytes = P.saved_bytes;
  plan->fwd_workspace_bytes = P.fwd_bytes;
  plan->bwd_workspace_bytes = P.bwd_bytes;
  return GPS_OK;
}

extern "C" int gps_node_loss_forward(const GpsNodeLossArgs* args, void* stream) {
  return nl_forward(args, (cudaStream_t)stream);
}

extern "C" int gps_node_loss_backward(const GpsNodeLossArgs* args, void* stream) {
  return nl_backward(args, (cudaStream_t)stream);
}
