// layer_ops.cuh — host-side building blocks of the layer orchestrations (layer.cu: GPSLayer, graphormer.cu, san.cu,
// custom_gnn.cu): side streams, the plan prologue, the dense products of a Linear and its gradients, and the
// dropout-only pass.
// The plan-typed helpers read P.prec (GPS_PREC_*), and linear_wgrad also P.grads_prezeroed.
#pragma once
#include <algorithm>

#include "gemm.cuh"
#include "kernels.cuh"

namespace gps {

// ------------------------------------------------------------------------------- side stream (fork / join)
// Independent stages run concurrently with the main chain: the edge projection next to the node projections, the
// attention branch next to the message-passing branch (gps_layer.py:161-218 computes both from the same h_in1),
// and every weight-gradient GEMM next to the data-gradient chain.  Fork = event on the caller's stream that the
// side stream waits on; join = the reverse.  All of it is capturable into a CUDA graph.
struct Side {
  cudaStream_t s = nullptr;    // weight gradients / edge projection / forward attention branch
  cudaStream_t s3 = nullptr;   // backward attention branch (next to the message-passing backward)
  cudaStream_t s4 = nullptr;   // edge-side BatchNorm backward (depends on grad_edge_out only, so it starts at once)
  cudaEvent_t ev[32];
  int next = 0;
  bool ok = false;
  int init() {
    if (ok) return GPS_OK;
    GPS_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    GPS_CUDA(cudaStreamCreateWithFlags(&s3, cudaStreamNonBlocking));
    GPS_CUDA(cudaStreamCreateWithFlags(&s4, cudaStreamNonBlocking));
    for (int i = 0; i < 32; ++i) GPS_CUDA(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
    ok = true;
    return GPS_OK;
  }
  int order(cudaStream_t from, cudaStream_t to) {   // `to` waits for everything enqueued on `from` so far
    cudaEvent_t e = ev[next++ & 31];
    GPS_CUDA(cudaEventRecord(e, from));
    GPS_CUDA(cudaStreamWaitEvent(to, e, 0));
    return GPS_OK;
  }
  int fork(cudaStream_t main) { return order(main, s); }
  int join(cudaStream_t main) { return order(s, main); }
};

// the side streams of the current device, created on its first use (layer.cu)
int side_stream(Side** out);

// ------------------------------------------------------------------------------- plan prologue
// The bf16 planes of a [rows, cols] operand, carved from A: ld = cols rounded up to 8, rows * ld + 8 elements per
// plane, and the lo plane only in fp32 mode (lo = true).
inline Planes arena_planes(Arena& A, int64_t rows, int64_t cols, bool lo) {
  Planes q;
  q.ld = round_up(cols, 8);
  q.hi = A.alloc<__nv_bfloat16>(rows * q.ld + 8);
  q.lo = lo ? A.alloc<__nv_bfloat16>(rows * q.ld + 8) : nullptr;
  return q;
}

// ------------------------------------------------------------------------------- pad / unpad
// dst [rows_p, cols_p] (pitch ldd) = src [rows, cols] (pitch lds) with zeros beyond rows x cols, and / or the bf16 planes
// of that block (p.hi set; then cols_p % 4 == 0).  Unpadding is the same copy with rows_p = rows and cols_p = cols.
// Up to kPadItems blocks per launch (run: custom_gnn.cu).
struct PadItem {
  const float* src; int64_t lds; int rows, cols;
  float* dst; int64_t ldd; int rows_p, cols_p;
  Planes p;
};
constexpr int kPadItems = 24;
struct PadList {
  PadItem it[kPadItems];
  int n = 0;
  bool overflow = false;
  void add(const float* src, int64_t lds, int64_t rows, int64_t cols, float* dst, int64_t ldd, int64_t rows_p,
           int64_t cols_p, Planes p = Planes()) {
    if (!src || rows_p <= 0 || cols_p <= 0 || (!dst && !p.hi)) return;
    if (n == kPadItems) {
      overflow = true;
      return;
    }
    it[n++] = PadItem{src, lds, (int)rows, (int)cols, dst, ldd, (int)rows_p, (int)cols_p, p};
  }
  int run(cudaStream_t st) const;
};

// One dropout site of a call; p = 0 in eval mode
inline DropCfg drop_cfg(float p, bool train, uint64_t seed, uint64_t offset, const uint64_t* offset_dev, int site) {
  DropCfg c;
  c.p = train ? p : 0.f;
  c.seed = seed; c.offset = offset; c.site = site;
  c.offset_dev = (const unsigned long long*)offset_dev;
  return c;
}

// P->grads_accumulate / P->grads_prezeroed from GPS_FLAG_GRADS_*: accumulating buffers are never zeroed either
template <class PlanT>
inline void set_grad_flags(PlanT* P, int flags) {
  P->grads_accumulate = (flags & GPS_FLAG_GRADS_ACCUMULATE) != 0;
  P->grads_prezeroed = (flags & GPS_FLAG_GRADS_ZEROED) != 0 || P->grads_accumulate;
}

// zero the gradients of n Linears, weight [rows[i], cols[i]] and bias [rows[i]]: a backward over no rows writes none
inline int zero_linear_grads(const GpsLinear* const* ls, const int64_t* rows, const int64_t* cols, int n,
                             cudaStream_t st) {
  for (int i = 0; i < n; ++i) {
    if (ls[i]->grad_weight)
      GPS_CUDA(cudaMemsetAsync(ls[i]->grad_weight, 0, (size_t)(rows[i] * cols[i]) * sizeof(float), st));
    if (ls[i]->grad_bias) GPS_CUDA(cudaMemsetAsync(ls[i]->grad_bias, 0, (size_t)rows[i] * sizeof(float), st));
  }
  return GPS_OK;
}

// ------------------------------------------------------------------------------- dense products
// An operand: fp32 values with leading dimension ld and, where the layer keeps them, their bf16 planes.
struct Operand {
  const float* f;
  int64_t ld;
  Planes p;
};

// y[M,N] = x[M,K] W[N,K]^T (+ bias[N]); the caller adds the rest of the epilogue
template <class PlanT>
inline GemmParams linear_fwd(const PlanT& P, int64_t M, int64_t N, int64_t K, Operand x, Operand W, float* y,
                             int64_t ldy, const float* bias = nullptr) {
  GemmParams g;
  g.M = (int)M; g.N = (int)N; g.K = (int)K;
  g.A = x.f; g.lda = (int)x.ld; g.Ap = x.p;
  g.B = W.f; g.ldb = (int)W.ld; g.Bp = W.p;
  g.C = y; g.ldc = (int)ldy;
  g.bias = bias;
  g.precision = P.prec;
  return g;
}

// g_x[M,N] = g[M,K] W[K,N]: the input gradient of linear_fwd
template <class PlanT>
inline GemmParams linear_dgrad(const PlanT& P, int64_t M, int64_t N, int64_t K, Operand g, Operand W, float* gx,
                               int64_t ldgx) {
  GemmParams p = linear_fwd(P, M, N, K, g, W, gx, ldgx);
  p.tb = 1;
  return p;
}

inline void set_dropout(GemmParams& g, const DropCfg& c) {
  g.p_drop = c.p; g.seed = c.seed; g.offset = c.offset; g.site = c.site; g.offset_dev = c.offset_dev;
}

// multiply by act'(pre-activation); ReLU reads the mask off the stored post-activation value instead
inline void set_act_mask(GemmParams& g, int act, const float* post, const float* pre, int64_t ld) {
  if (act == GPS_ACT_RELU) {
    g.mask_src = post; g.mask_is_post = 1;
  } else {
    g.mask_src = pre; g.mask_act = act;
  }
  g.ldmask = (int)ld;
}

inline int splitk_for(int64_t rows, int64_t out, int64_t in) {
  // Weight gradients reduce over `rows` (nodes/edges) into a small [out, in] tile grid: split the reduction so
  // that tiles x splits ~ 300 CTAs (two per SM), at least 4 k-blocks of 64 rows per CTA (tools/gemm_tune.py).
  const int64_t tiles = ceil_div(out, 128) * ceil_div(in, in >= 160 ? 160 : 64);
  int64_t s = ceil_div(300, tiles > 0 ? tiles : 1);
  const int64_t max_s = rows / 256;
  if (s > max_s) s = max_s;
  if (s < 1) s = 1;
  if (s > 64) s = 64;
  return (int)s;
}

// dW[out,in] += G[rows,out]^T X[rows,in], db[out] += colsum(G), into zeroed dW / db
template <class PlanT>
inline int wgrad_add(const PlanT& P, Operand G, Operand X, int64_t rows, int64_t out, int64_t in, float* dW, float* db,
                     cudaStream_t st) {
  if (rows == 0) return GPS_OK;
  GemmParams p;
  p.M = (int)out; p.N = (int)in; p.K = (int)rows;
  p.A = G.f; p.lda = (int)G.ld; p.ta = 1; p.Ap = G.p;
  p.B = X.f; p.ldb = (int)X.ld; p.tb = 1; p.Bp = X.p;
  p.C = dW; p.ldc = (int)in;
  p.splitk = std::max(2, splitk_for(rows, out, in));   // the accumulating split-K path also for tiny inputs
  p.colsum_a = db;
  p.precision = P.prec;
  if (P.prec == GPS_PREC_BF16 && G.p.hi && db) {
    // bf16 mode stores no lo plane: summing ~N bf16-rounded rows would put ~sqrt(N) 2^-9 of noise on a bias gradient
    // that is often a near-cancelling sum (every Linear here feeds a BatchNorm) -> exact fp32 column sum instead
    p.colsum_a = nullptr;
    GPS_TRY(colsum(G.f, G.ld, rows, out, db, st));
  }
  return gemm(p, st);
}

// weight gradient of a Linear into the caller's buffers: dW[out,in] = G[rows,out]^T X[rows,in], db[out] = colsum(G)
template <class PlanT>
inline int linear_wgrad(const PlanT& P, Operand G, Operand X, int64_t rows, int64_t out, int64_t in, float* dW,
                        float* db, cudaStream_t st) {
  if (!dW) return GPS_OK;
  if (!P.grads_prezeroed) {
    GPS_CUDA(cudaMemsetAsync(dW, 0, (size_t)(out * in) * sizeof(float), st));
    if (db) GPS_CUDA(cudaMemsetAsync(db, 0, (size_t)out * sizeof(float), st));
  }
  return wgrad_add(P, G, X, rows, out, in, dW, db, st);
}

// A BatchNorm as its consumer kernels see it.  Eval: the running statistics (mode 2); BatchNorm is then a per-column
// affine map and its backward has no batch terms.  Training backward: the batch statistics the forward pass saved (mode
// 0).  Training forward, over fwd_rows rows: the consumer kernel finalises the statistics from the producer's column
// sums, saves them for the backward and updates the running statistics (mode 1).  The statistics slot of a BatchNorm
// over w columns: saved [mean | invstd] (2w floats) and the forward's column sums (2w doubles).  Reads P.train.
template <class PlanT>
inline BnView bn_view_at(const PlanT& P, float* saved, double* fsums, int64_t w, const GpsBatchNorm& bn,
                         int64_t fwd_rows) {
  const bool fwd = fwd_rows >= 0;
  BnView v;
  v.mean = saved;
  v.invstd = v.mean + w;
  v.gamma = bn.weight;
  v.beta = bn.bias;
  if (fwd) v.d = w;
  if (fwd || !P.train) {
    v.running_mean = bn.running_mean;
    v.running_var = bn.running_var;
  }
  if (!P.train) {
    v.mode = 2;
  } else if (fwd) {
    const int64_t n = fwd_rows;
    v.mode = 1;
    v.sums = fsums;
    v.inv_n = 1.0 / (double)(n > 0 ? n : 1);
    v.unbias = n > 1 ? (double)n / (double)(n - 1) : 1.0;
    v.save_mean = saved;
    v.save_invstd = v.save_mean + w;
    v.nbt = (long long*)bn.num_batches_tracked;
  }
  return v;
}

// dst [rows, d] = src times the dropout scales of c (and, p2 > 0, of the site site2 as well), with dst's planes when
// dstp.hi is set (layer.cu)
int dropmul_rows(const float* src, float* dst, int64_t rows, int64_t d, const DropCfg& c, float p2, int site2,
                 Planes dstp, cudaStream_t st);

}  // namespace gps
