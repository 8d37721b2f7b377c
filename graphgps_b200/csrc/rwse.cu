// rwse.cu — RWSE, the random-walk structural encoding: the landing probabilities diag(P^k) of every node on the device
// (graphgps/transform/posenc_stats.py:get_rw_landing_probs) and the kernel-PE node encoder, forward and backward
// (graphgps/encoder/kernel_pos_encoder.py:KernelPENodeEncoder, model "linear").  C ABI at the bottom.
//
// Landing probabilities: P = D_out^-1 A is block-diagonal over the graphs, so one CTA takes one graph and a block of R
// of its source nodes i and keeps their walk vectors v_i = e_i P^t, an R x n_g block, double-buffered in shared memory.
// A step is a gather over in-edges, v'[d] = sum_{s -> d} v[s] dinv[s], in CSR order with an fp64 accumulator; the
// column whose step matches reads v_i[i].  Every term is non-negative, so each entry has a relative error of at most
// one fp32 rounding per step.  R is the whole graph at molecule sizes and follows from shared memory at large ones
// (about 5 rows at 5 000 nodes).
//
// Encoder, w = dim_emb - dim_pe, Kp = round_up(K, 4):
//   forward   [training] per-CTA double column sums of pestat -> their fixed-order total
//             -> zhat = (pestat - mean) invstd [N, Kp] (BnRegs: mode 1 derives the statistics from the sums and applies
//                the running update, mode 2 reads the running statistics)
//             -> out[r, c] = c < w ? h[r, c] : bp + sum_k (gamma zhat + beta)[r, k] Wp[c - w, k]
//   backward  grad_x and gz = g[:, w:] Wp [N, Kp] -> per-CTA partials of every weight-gradient entry (and of the
//             BatchNorm's sum gz zhat, sum gz) over 32-row chunks -> their fixed-order totals into the gradients
// The widths are small (K <= 64, dim_pe <= 28 and dim_in 5 in the shipped configs), so every product is CUDA-core fp32
// with the weights read through L1, not the TMA GEMM.
#include <string.h>

#include "layer_ops.cuh"

namespace gps {

namespace {

// ================================================================================ landing probabilities
constexpr int kRwSmemMax = 227 * 1024;   // opt-in shared memory per CTA on sm_90

struct Ksteps {
  int k[GPS_RWSE_MAX_COLS];
  int n, kmax;
};

__global__ void k_rw_dinv(const int* __restrict__ src_ptr, int64_t N, double* __restrict__ dinv) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x) {
    const int deg = src_ptr[i + 1] - src_ptr[i];
    dinv[i] = deg > 0 ? 1.0 / (double)deg : 0.0;   // pow(-1) with inf -> 0, as the reference masks it
  }
}

// CTA (graph blockIdx.x, source rows blockIdx.y * R ..): see the comment at the top.  Shared memory: 2 x R x nmax floats.
__global__ void __launch_bounds__(512) k_rw_landing(const int* __restrict__ graph_ptr, const int* __restrict__ dst_ptr,
                                                    const int* __restrict__ dst_src, const double* __restrict__ dinv,
                                                    Ksteps ks, int R, float* __restrict__ out) {
  extern __shared__ float sm[];
  const int g0 = graph_ptr[blockIdx.x], n = graph_ptr[blockIdx.x + 1] - g0;
  const int i0 = blockIdx.y * R;
  if (i0 >= n) return;
  const int rows = min(R, n - i0), cells = rows * n;
  float* v = sm;
  float* w = sm + (size_t)R * n;
  for (int idx = threadIdx.x; idx < cells; idx += blockDim.x) {
    const int r = idx / n;
    v[idx] = idx - r * n == i0 + r ? 1.f : 0.f;
  }
  for (int idx = threadIdx.x; idx < rows * ks.n; idx += blockDim.x) {
    const int r = idx / ks.n, j = idx - r * ks.n;
    if (ks.k[j] == 0) out[(int64_t)(g0 + i0 + r) * ks.n + j] = 1.f;
  }
  __syncthreads();
  for (int t = 1; t <= ks.kmax; ++t) {
    // consecutive threads take the rows of one destination, so they share its in-edge list
    for (int idx = threadIdx.x; idx < cells; idx += blockDim.x) {
      const int d = idx / rows, r = idx - d * rows;
      const float* vr = v + r * n;
      double acc = 0.0;
      for (int e = dst_ptr[g0 + d], e1 = dst_ptr[g0 + d + 1]; e < e1; ++e) {
        const int s = dst_src[e] - g0;
        if ((unsigned)s < (unsigned)n) acc += (double)vr[s] * dinv[g0 + s];   // PyG batches have no cross-graph edges
      }
      w[r * n + d] = (float)acc;
    }
    __syncthreads();   // w complete; v is not read again before the next step overwrites it
    for (int idx = threadIdx.x; idx < rows * ks.n; idx += blockDim.x) {
      const int r = idx / ks.n, j = idx - r * ks.n;
      if (ks.k[j] == t) out[(int64_t)(g0 + i0 + r) * ks.n + j] = w[r * n + i0 + r];
    }
    float* tmp = v;
    v = w;
    w = tmp;
  }
}

struct RwGeom {
  int R, threads;
  size_t smem;
};

int rw_geom(int64_t N, int64_t nmax, RwGeom* G) {
  const int64_t fit = kRwSmemMax / (2 * (int64_t)sizeof(float) * std::max<int64_t>(nmax, 1));
  GPS_REQUIRE(fit >= 1, GPS_ERR_UNSUPPORTED,
              "rwse_landing: a graph of %lld nodes does not fit on chip (one walk row of at most %lld nodes)",
              (long long)nmax, (long long)(kRwSmemMax / (2 * sizeof(float))));
  // whole graphs per CTA at molecule sizes; at least ~2 CTAs per SM when the batch has the rows for it
  int64_t R = std::min<int64_t>({fit, std::max<int64_t>(nmax, 1), std::max<int64_t>(32, ceil_div(N, 2 * kNumSMs))});
  G->R = (int)R;
  G->threads = (int)std::min<int64_t>(512, std::max<int64_t>(64, round_up(R * nmax, 32)));
  G->smem = (size_t)(2 * R * std::max<int64_t>(nmax, 1)) * sizeof(float);
  return GPS_OK;
}

int rw_check(const GpsGraph* g, const int32_t* ksteps, int32_t nk, int32_t nmax, float* out, void* ws,
             int64_t ws_bytes, Ksteps* ks) {
  GPS_REQUIRE(g, GPS_ERR_ARG, "rwse_landing: null graph");
  GPS_REQUIRE(g->N >= 0 && g->E >= 0 && g->B >= 0 && g->N < (1ll << 31) && g->E < (1ll << 31) && g->B < (1ll << 31),
              GPS_ERR_ARG, "rwse_landing: graph sizes out of range");
  GPS_REQUIRE(g->N == 0 || g->B > 0, GPS_ERR_ARG, "rwse_landing: %lld rows in no graph", (long long)g->N);
  GPS_REQUIRE(g->B == 0 || g->graph_ptr, GPS_ERR_ARG, "rwse_landing: graph without graph_ptr");
  GPS_REQUIRE(g->N == 0 || (g->dst_ptr && g->src_ptr && (g->E == 0 || g->dst_src)), GPS_ERR_ARG,
              "rwse_landing: graph without its CSR (dst_ptr, dst_src, src_ptr)");
  GPS_REQUIRE(ksteps && nk >= 1, GPS_ERR_ARG, "rwse_landing: needs ksteps and nk >= 1");
  GPS_REQUIRE(nk <= GPS_RWSE_MAX_COLS, GPS_ERR_UNSUPPORTED, "rwse_landing: %d columns (at most %d are built)", nk,
              GPS_RWSE_MAX_COLS);
  ks->n = nk;
  ks->kmax = 0;
  for (int j = 0; j < nk; ++j) {
    GPS_REQUIRE(ksteps[j] >= 0, GPS_ERR_ARG, "rwse_landing: ksteps[%d] = %d is negative", j, ksteps[j]);
    GPS_REQUIRE(ksteps[j] <= GPS_RWSE_MAX_STEPS, GPS_ERR_UNSUPPORTED, "rwse_landing: ksteps[%d] = %d (at most %d)", j,
                ksteps[j], GPS_RWSE_MAX_STEPS);
    ks->k[j] = ksteps[j];
    ks->kmax = std::max(ks->kmax, (int)ksteps[j]);
  }
  GPS_REQUIRE(nmax >= 0 && nmax <= g->N, GPS_ERR_ARG, "rwse_landing: nmax %d outside [0, N = %lld]", nmax,
              (long long)g->N);
  GPS_REQUIRE(g->N == 0 || nmax >= 1, GPS_ERR_ARG, "rwse_landing: nmax must be >= 1 for %lld rows", (long long)g->N);
  GPS_REQUIRE(g->N == 0 || out, GPS_ERR_ARG, "rwse_landing: out is required");
  GPS_REQUIRE(((uintptr_t)ws & 7) == 0, GPS_ERR_ARG, "rwse_landing: workspace must be 8-byte aligned");
  GPS_REQUIRE(g->N == 0 || (ws && ws_bytes >= 8 * g->N), GPS_ERR_ARG, "rwse_landing: workspace too small (%lld < %lld)",
              (long long)ws_bytes, (long long)(8 * g->N));
  RwGeom G;
  return rw_geom(g->N, nmax, &G);
}

int rw_landing(const GpsGraph& g, const Ksteps& ks, int64_t nmax, float* out, double* dinv, cudaStream_t st) {
  if (g.N == 0) return GPS_OK;
  RwGeom G;
  GPS_TRY(rw_geom(g.N, nmax, &G));
  k_rw_dinv<<<(unsigned)std::min<int64_t>(ceil_div(g.N, 256), kNumSMs * 8), 256, 0, st>>>(g.src_ptr, g.N, dinv);
  GPS_LAUNCH_CHECK();
  GPS_CUDA(cudaFuncSetAttribute(k_rw_landing, cudaFuncAttributeMaxDynamicSharedMemorySize, kRwSmemMax));
  const dim3 grid((unsigned)g.B, (unsigned)ceil_div(nmax, G.R));
  k_rw_landing<<<grid, G.threads, G.smem, st>>>(g.graph_ptr, g.dst_ptr, g.dst_src, dinv, ks, G.R, out);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

// ================================================================================ kernel-PE encoder
constexpr int kStatRows = 64;    // rows per CTA of the forward column sums
constexpr int kGradRows = 32;    // rows per CTA of the weight-gradient partials
constexpr int64_t kMaxPartials = 1ll << 24;

struct PePlan {
  int64_t N, K, Kp, din, demb, dpe, w;
  bool expand, bn, train, pad;
  int64_t fchunks, bchunks, brows, npairs;
  // saved: zhat [N, Kp], save_mean / save_invstd [Kp], padded gamma | beta | running_mean | running_var [4][Kp]
  float *zhat, *mean, *invstd, *prm;
  int64_t saved_bytes;
  // forward workspace: column-sum partials [fchunks][2][Kp] and their total [2][Kp]
  double *fpart, *sums;
  int64_t fwd_bytes;
  // backward workspace: gz [N, Kp], weight-gradient partials [bchunks][npairs]
  float* gz;
  double* bpart;
  int64_t bwd_bytes;
};

int make_plan(const GpsKernelPeArgs* a, PePlan* P, bool bind) {
  memset(P, 0, sizeof(*P));
  GPS_REQUIRE(a, GPS_ERR_ARG, "kernel_pe: null args");
  GPS_REQUIRE(a->N >= 0 && a->N < (1ll << 31), GPS_ERR_ARG, "kernel_pe: N out of range");
  GPS_REQUIRE(a->K >= 1 && a->dim_in >= 1 && a->dim_pe >= 1 && a->dim_emb >= a->dim_pe, GPS_ERR_ARG,
              "kernel_pe: needs K, dim_in, dim_pe >= 1 and dim_emb >= dim_pe (got K %lld, dim_in %lld, dim_pe %lld, "
              "dim_emb %lld)", (long long)a->K, (long long)a->dim_in, (long long)a->dim_pe, (long long)a->dim_emb);
  GPS_REQUIRE(a->K <= GPS_RWSE_MAX_COLS && a->dim_in <= 4096 && a->dim_emb <= 4096, GPS_ERR_UNSUPPORTED,
              "kernel_pe: needs K <= %d and dim_in, dim_emb <= 4096", GPS_RWSE_MAX_COLS);
  GPS_REQUIRE(a->expand_x == 0 || a->expand_x == 1, GPS_ERR_ARG, "kernel_pe: expand_x must be 0 or 1");
  GPS_REQUIRE(a->batch_norm == 0 || a->batch_norm == 1, GPS_ERR_ARG, "kernel_pe: batch_norm must be 0 or 1");
  GPS_REQUIRE(a->flags == 0, GPS_ERR_ARG, "kernel_pe: flags are reserved (got %d)", a->flags);
  P->N = a->N; P->K = a->K; P->Kp = round_up(a->K, 4);
  P->din = a->dim_in; P->demb = a->dim_emb; P->dpe = a->dim_pe; P->w = a->dim_emb - a->dim_pe;
  P->expand = a->expand_x && P->w > 0;
  GPS_REQUIRE(P->expand || P->din == P->w || (P->w == 0 && !a->expand_x), GPS_ERR_ARG,
              "kernel_pe: without expand_x x must have dim_emb - dim_pe = %lld columns (got dim_in %lld)",
              (long long)P->w, (long long)P->din);
  P->bn = a->batch_norm;
  P->train = a->training != 0;
  P->pad = P->bn && P->K % 4 != 0;
  GPS_REQUIRE(!(P->bn && P->train) || P->N >= 2, GPS_ERR_ARG,
              "kernel_pe: BatchNorm in training needs more than one row (got %lld)", (long long)P->N);
  const int64_t N = P->N, Kp = P->Kp;
  P->fchunks = ceil_div(N, kStatRows);
  P->npairs = P->dpe * (P->K + 1) + (P->expand ? P->w * (P->din + 1) : 0) + (P->bn ? 2 * P->K : 0);
  P->bchunks = std::min<int64_t>(ceil_div(N, kGradRows), std::max<int64_t>(1, kMaxPartials / P->npairs));
  P->brows = P->bchunks ? ceil_div(N, P->bchunks) : 0;

  Arena S(bind ? a->saved : nullptr, a->saved_bytes);
  if (P->bn) {
    P->zhat = S.alloc<float>(N * Kp);
    P->mean = S.alloc<float>(Kp);
    P->invstd = S.alloc<float>(Kp);
    if (P->pad) P->prm = S.alloc<float>(4 * Kp);
  }
  P->saved_bytes = S.used;
  GPS_REQUIRE(!bind || !S.overflow, GPS_ERR_ARG, "kernel_pe: saved buffer too small (%lld < %lld)",
              (long long)a->saved_bytes, (long long)S.used);
  Arena F(bind ? a->workspace : nullptr, a->workspace_bytes);
  if (P->bn && P->train) {
    P->fpart = F.alloc<double>(P->fchunks * 2 * Kp);
    P->sums = F.alloc<double>(2 * Kp);
  }
  P->fwd_bytes = F.used;
  Arena Bk(bind ? a->workspace : nullptr, a->workspace_bytes);
  if (P->bn) P->gz = Bk.alloc<float>(N * Kp);
  P->bpart = Bk.alloc<double>(P->bchunks * P->npairs);
  P->bwd_bytes = Bk.used;
  return GPS_OK;
}

int prepare(const GpsKernelPeArgs* a, bool fwd, PePlan* P) {
  GPS_REQUIRE(a, GPS_ERR_ARG, "kernel_pe: null args");
  GPS_TRY(make_plan(a, P, true));
  GPS_REQUIRE(a->saved && a->workspace, GPS_ERR_ARG, "kernel_pe: saved and workspace are required");
  GPS_REQUIRE(((uintptr_t)a->saved & 15) == 0 && ((uintptr_t)a->workspace & 15) == 0, GPS_ERR_ARG,
              "kernel_pe: saved and workspace must be 16-byte aligned");
  const int64_t ws = fwd ? P->fwd_bytes : P->bwd_bytes;
  GPS_REQUIRE(a->workspace_bytes >= ws, GPS_ERR_ARG, "kernel_pe: workspace too small (%lld < %lld)",
              (long long)a->workspace_bytes, (long long)ws);
  GPS_REQUIRE(a->pe_encoder.weight && a->pe_encoder.bias, GPS_ERR_ARG, "kernel_pe: missing pe_encoder weight / bias");
  GPS_REQUIRE(!P->expand || (a->linear_x.weight && a->linear_x.bias), GPS_ERR_ARG,
              "kernel_pe: missing linear_x weight / bias");
  if (P->bn) {
    const GpsBatchNorm& b = a->raw_norm;
    GPS_REQUIRE(b.weight && b.bias && b.running_mean && b.running_var, GPS_ERR_ARG,
                "kernel_pe: missing raw_norm weight, bias or running statistics");
    // BnRegs reads them as float4: unpadded ones must be 16-byte aligned
    const uintptr_t al = (uintptr_t)b.weight | (uintptr_t)b.bias | (uintptr_t)b.running_mean | (uintptr_t)b.running_var;
    GPS_REQUIRE(P->pad || (al & 15) == 0, GPS_ERR_ARG, "kernel_pe: raw_norm parameters must be 16-byte aligned");
  }
  if (fwd) {
    GPS_REQUIRE(P->N == 0 || (a->pestat && a->out && (P->w == 0 || a->x)), GPS_ERR_ARG,
                "kernel_pe: pestat, x and out are required");
  } else {
    GPS_REQUIRE(P->N == 0 || (a->pestat && a->grad_out && (P->w == 0 || (a->x && a->grad_x))), GPS_ERR_ARG,
                "kernel_pe: pestat, x, grad_out and grad_x are required");
  }
  return GPS_OK;
}

// per-CTA column sums of pestat over kStatRows rows: part[chunk][0 | 1][Kp] = sum v | sum v^2 (zero pad columns)
__global__ void k_pe_stat_part(const float* __restrict__ pe, int64_t N, int K, int Kp, double* __restrict__ part) {
  const int k = threadIdx.x;
  if (k >= Kp) return;
  const int64_t r0 = (int64_t)blockIdx.x * kStatRows, r1 = min(N, r0 + kStatRows);
  double s = 0.0, s2 = 0.0;
  if (k < K)
    for (int64_t r = r0; r < r1; ++r) {
      const double v = pe[r * K + k];
      s += v;
      s2 += v * v;
    }
  part[(int64_t)blockIdx.x * 2 * Kp + k] = s;
  part[(int64_t)blockIdx.x * 2 * Kp + Kp + k] = s2;
}

// sums[i] = sum over chunks, in chunk order
__global__ void k_pe_stat_sum(const double* __restrict__ part, int64_t chunks, int n, double* __restrict__ sums) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double s = 0.0;
    for (int64_t c = 0; c < chunks; ++c) s += part[c * n + i];
    sums[i] = s;
  }
}

// zhat [N, Kp] = (pestat - mean) invstd, one thread per float4 column group and row lane (BnRegs' layout: CTA 0 row lane
// 0 publishes the statistics and the running update in training)
__global__ void k_pe_norm(const float* __restrict__ pe, int64_t N, int K, BnView bn, float* __restrict__ zhat) {
  const int c4 = threadIdx.x, C4 = blockDim.x;
  BnRegs reg;
  reg.load(bn, c4);
  for (int64_t r = (int64_t)blockIdx.x * blockDim.y + threadIdx.y; r < N; r += (int64_t)gridDim.x * blockDim.y) {
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = c4 * 4 + j < K ? pe[r * K + c4 * 4 + j] : 0.f;
    st4(zhat + r * (4 * C4) + c4 * 4, reg.zhat(make_float4(v[0], v[1], v[2], v[3])));
  }
}

struct PeDev {
  int64_t N;
  int K, Kp, din, demb, dpe, w, expand, bn;
  const float *pe, *zhat, *gamma, *beta, *x, *Wx, *bx, *Wp, *bp;
};

// the encoder's input to pe_encoder, column k of row r: BN(pestat) = gamma zhat + beta, or pestat
__device__ __forceinline__ float pe_in(const PeDev& p, int64_t r, int k) {
  return p.bn ? fmaf(p.zhat[r * p.Kp + k], p.gamma[k], p.beta[k]) : p.pe[r * p.K + k];
}

__global__ void k_pe_out(PeDev p, float* __restrict__ out) {
  const int64_t total = p.N * p.demb;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / p.demb;
    const int c = (int)(i - r * p.demb);
    float v;
    if (c < p.w) {
      if (p.expand) {
        v = p.bx[c];
        for (int j = 0; j < p.din; ++j) v = fmaf(p.x[r * p.din + j], p.Wx[(int64_t)c * p.din + j], v);
      } else {
        v = p.x[r * p.din + c];
      }
    } else {
      const int cp = c - p.w;
      v = p.bp[cp];
      for (int k = 0; k < p.K; ++k) v = fmaf(pe_in(p, r, k), p.Wp[(int64_t)cp * p.K + k], v);
    }
    out[i] = v;
  }
}

// grad_x [N, din] = g[:, :w] Wx (expand) or g[:, :w]; gz [N, Kp] = g[:, w:] Wp (BatchNorm; pad columns 0)
__global__ void k_pe_bwd_rows(PeDev p, const float* __restrict__ g, float* __restrict__ gx, float* __restrict__ gz) {
  const int cols = (p.w > 0 ? p.din : 0) + (p.bn ? p.Kp : 0);
  const int64_t total = p.N * cols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / cols;
    int c = (int)(i - r * cols);
    const float* gr = g + r * p.demb;
    if (p.w > 0 && c < p.din) {
      float v;
      if (p.expand) {
        v = 0.f;
        for (int o = 0; o < p.w; ++o) v = fmaf(gr[o], p.Wx[(int64_t)o * p.din + c], v);
      } else {
        v = gr[c];
      }
      gx[r * p.din + c] = v;
      continue;
    }
    if (p.w > 0) c -= p.din;
    float v = 0.f;
    if (c < p.K)
      for (int o = 0; o < p.dpe; ++o) v = fmaf(gr[p.w + o], p.Wp[(int64_t)o * p.K + c], v);
    gz[r * p.Kp + c] = v;
  }
}

// pair q of the weight gradients (see PePlan::npairs): [0, dpe (K+1)) pe_encoder (c, k), k == K its bias;
// then w (din+1) linear_x (c, j), j == din its bias (expand); then 2K BatchNorm (sum gz zhat | sum gz)
__device__ __forceinline__ double pe_pair_term(const PeDev& p, const float* g, const float* gz, int64_t r, int64_t q) {
  const float* gr = g + r * p.demb;
  const int64_t npe = (int64_t)p.dpe * (p.K + 1);
  if (q < npe) {
    const int c = (int)(q / (p.K + 1)), k = (int)(q - (int64_t)c * (p.K + 1));
    const double gv = gr[p.w + c];
    return k < p.K ? gv * (double)pe_in(p, r, k) : gv;
  }
  q -= npe;
  if (p.expand) {
    const int64_t nx = (int64_t)p.w * (p.din + 1);
    if (q < nx) {
      const int c = (int)(q / (p.din + 1)), j = (int)(q - (int64_t)c * (p.din + 1));
      const double gv = gr[c];
      return j < p.din ? gv * (double)p.x[r * p.din + j] : gv;
    }
    q -= nx;
  }
  const int k = (int)(q % p.K);
  const double gv = gz[r * p.Kp + k];
  return q < p.K ? gv * (double)p.zhat[r * p.Kp + k] : gv;
}

__global__ void k_pe_wgrad_part(PeDev p, const float* __restrict__ g, const float* __restrict__ gz, int64_t rows,
                                int64_t npairs, double* __restrict__ part) {
  const int64_t r0 = (int64_t)blockIdx.x * rows, r1 = min(p.N, r0 + rows);
  for (int64_t q = threadIdx.x; q < npairs; q += blockDim.x) {
    double s = 0.0;
    for (int64_t r = r0; r < r1; ++r) s += pe_pair_term(p, g, gz, r, q);
    part[(int64_t)blockIdx.x * npairs + q] = s;
  }
}

struct PeGrads {
  float *gWp, *gbp, *gWx, *gbx, *ggamma, *gbeta;
};

__global__ void k_pe_wgrad_sum(PeDev p, const double* __restrict__ part, int64_t chunks, int64_t npairs, PeGrads o) {
  for (int64_t q0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q0 < npairs; q0 += (int64_t)gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int64_t c = 0; c < chunks; ++c) s += part[c * npairs + q0];
    const float v = (float)s;
    int64_t q = q0;
    const int64_t npe = (int64_t)p.dpe * (p.K + 1);
    if (q < npe) {
      const int c = (int)(q / (p.K + 1)), k = (int)(q - (int64_t)c * (p.K + 1));
      if (k < p.K) {
        if (o.gWp) o.gWp[(int64_t)c * p.K + k] = v;
      } else if (o.gbp) {
        o.gbp[c] = v;
      }
      continue;
    }
    q -= npe;
    if (p.expand) {
      const int64_t nx = (int64_t)p.w * (p.din + 1);
      if (q < nx) {
        const int c = (int)(q / (p.din + 1)), j = (int)(q - (int64_t)c * (p.din + 1));
        if (j < p.din) {
          if (o.gWx) o.gWx[(int64_t)c * p.din + j] = v;
        } else if (o.gbx) {
          o.gbx[c] = v;
        }
        continue;
      }
      q -= nx;
    }
    float* dst = q < p.K ? o.ggamma : o.gbeta;
    if (dst) dst[q % p.K] = v;
  }
}

PeDev pe_dev(const GpsKernelPeArgs* a, const PePlan& P) {
  PeDev p;
  p.N = P.N; p.K = (int)P.K; p.Kp = (int)P.Kp; p.din = (int)P.din; p.demb = (int)P.demb; p.dpe = (int)P.dpe;
  p.w = (int)P.w; p.expand = P.expand; p.bn = P.bn;
  p.pe = a->pestat; p.zhat = P.zhat; p.gamma = a->raw_norm.weight; p.beta = a->raw_norm.bias;
  p.x = a->x; p.Wx = a->linear_x.weight; p.bx = a->linear_x.bias; p.Wp = a->pe_encoder.weight; p.bp = a->pe_encoder.bias;
  return p;
}

unsigned flat_grid(int64_t total, int threads) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div(total, threads), (int64_t)kNumSMs * 16));
}

int pe_forward(const GpsKernelPeArgs* a, cudaStream_t st) {
  PePlan P;
  GPS_TRY(prepare(a, true, &P));
  const int64_t N = P.N, K = P.K, Kp = P.Kp;
  if (N == 0) return GPS_OK;
  if (P.bn) {
    const GpsBatchNorm& b = a->raw_norm;
    BnView v;
    v.gamma = b.weight; v.beta = b.bias; v.running_mean = b.running_mean; v.running_var = b.running_var;
    if (P.pad) {   // BnRegs reads float4 column groups: padded copies, and the running statistics copied back after
      float* g = P.prm;
      PadList L;
      L.add(b.weight, K, 1, K, g, Kp, 1, Kp);
      L.add(b.bias, K, 1, K, g + Kp, Kp, 1, Kp);
      L.add(b.running_mean, K, 1, K, g + 2 * Kp, Kp, 1, Kp);
      L.add(b.running_var, K, 1, K, g + 3 * Kp, Kp, 1, Kp);
      GPS_TRY(L.run(st));
      v.gamma = g; v.beta = g + Kp; v.running_mean = g + 2 * Kp; v.running_var = g + 3 * Kp;
    }
    v.d = Kp;
    if (P.train) {
      k_pe_stat_part<<<(unsigned)P.fchunks, (unsigned)round_up(Kp, 32), 0, st>>>(a->pestat, N, (int)K, (int)Kp, P.fpart);
      GPS_LAUNCH_CHECK();
      k_pe_stat_sum<<<1, (unsigned)round_up(2 * Kp, 32), 0, st>>>(P.fpart, P.fchunks, (int)(2 * Kp), P.sums);
      GPS_LAUNCH_CHECK();
      v.mode = 1;
      v.sums = P.sums;
      v.inv_n = 1.0 / (double)N;
      v.unbias = (double)N / (double)(N - 1);
      v.save_mean = P.mean;
      v.save_invstd = P.invstd;
      v.nbt = (long long*)b.num_batches_tracked;
    } else {
      v.mode = 2;
    }
    const int C4 = (int)(Kp / 4), RY = std::max(1, 256 / C4);
    k_pe_norm<<<(unsigned)std::min<int64_t>(ceil_div(N, RY), kNumSMs * 4), dim3(C4, RY), 0, st>>>(a->pestat, N, (int)K,
                                                                                                  v, P.zhat);
    GPS_LAUNCH_CHECK();
    if (P.pad && P.train) {
      PadList U;
      U.add(P.prm + 2 * Kp, Kp, 1, K, b.running_mean, K, 1, K);
      U.add(P.prm + 3 * Kp, Kp, 1, K, b.running_var, K, 1, K);
      GPS_TRY(U.run(st));
    }
  }
  k_pe_out<<<flat_grid(N * P.demb, 256), 256, 0, st>>>(pe_dev(a, P), a->out);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int pe_backward(const GpsKernelPeArgs* a, cudaStream_t st) {
  PePlan P;
  GPS_TRY(prepare(a, false, &P));
  const PeDev p = pe_dev(a, P);
  const int64_t N = P.N;
  const int64_t cols = (P.w > 0 ? P.din : 0) + (P.bn ? P.Kp : 0);
  if (N > 0 && cols > 0) {
    k_pe_bwd_rows<<<flat_grid(N * cols, 256), 256, 0, st>>>(p, a->grad_out, a->grad_x, P.gz);
    GPS_LAUNCH_CHECK();
  }
  const int64_t chunks = N > 0 ? P.bchunks : 0;
  if (chunks > 0) {
    k_pe_wgrad_part<<<(unsigned)chunks, 256, 0, st>>>(p, a->grad_out, P.gz, P.brows, P.npairs, P.bpart);
    GPS_LAUNCH_CHECK();
  }
  PeGrads o{a->pe_encoder.grad_weight, a->pe_encoder.grad_bias, P.expand ? a->linear_x.grad_weight : nullptr,
            P.expand ? a->linear_x.grad_bias : nullptr, P.bn ? a->raw_norm.grad_weight : nullptr,
            P.bn ? a->raw_norm.grad_bias : nullptr};
  k_pe_wgrad_sum<<<flat_grid(P.npairs, 256), 256, 0, st>>>(p, P.bpart, chunks, P.npairs, o);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

}  // namespace

}  // namespace gps

// =================================================================================== C ABI
using namespace gps;

extern "C" int gps_rwse_landing(const GpsGraph* graph, const int32_t* ksteps, int32_t nk, int32_t nmax, float* out,
                                void* workspace, int64_t workspace_bytes, void* stream) {
  Ksteps ks;
  GPS_TRY(rw_check(graph, ksteps, nk, nmax, out, workspace, workspace_bytes, &ks));
  return rw_landing(*graph, ks, nmax, out, (double*)workspace, (cudaStream_t)stream);
}

extern "C" int gps_kernel_pe_plan(const GpsKernelPeArgs* args, GpsKernelPePlan* plan) {
  GPS_REQUIRE(args && plan, GPS_ERR_ARG, "gps_kernel_pe_plan: null argument");
  PePlan P;
  GPS_TRY(make_plan(args, &P, false));
  plan->saved_bytes = P.saved_bytes;
  plan->fwd_workspace_bytes = P.fwd_bytes;
  plan->bwd_workspace_bytes = P.bwd_bytes;
  return GPS_OK;
}

extern "C" int gps_kernel_pe_forward(const GpsKernelPeArgs* args, void* stream) {
  return pe_forward(args, (cudaStream_t)stream);
}

extern "C" int gps_kernel_pe_backward(const GpsKernelPeArgs* args, void* stream) {
  return pe_backward(args, (cudaStream_t)stream);
}
