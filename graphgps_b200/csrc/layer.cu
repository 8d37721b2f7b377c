// layer.cu — host-side orchestration of one GPSLayer forward / backward and the C ABI.
//
// Follows graphgps/layer/gps_layer.py:155-232 (composition), :234-257 (attention / FFN blocks) and
// graphgps/layer/gatedgcn_layer.py:45-88 (GatedGCN with residual=True as built at gps_layer.py:92-96).
// Stage list (training mode, CustomGatedGCN+Transformer):
//   pack W -> [Ax|Bx|Dx|Ex|Q|K|V] = x Wcat^T -> Ce = e C^T -> segmented gather-reduce (+BN stats)
//   -> x_loc = x + act(BN(x~)) (+stats), e_out = e + act(BN(e^)) -> attention -> hA = x + O Wo^T (+stats)
//   -> s = BN(x_loc) + BN(hA) -> FFN (+stats) -> BN.
// Without normalisation (GPS_NORM_NONE, batch_norm=False): the local branch joins the attention branch before the output
// projection, whose epilogue writes s = x + hA' + x_loc; the FF2 epilogue writes x_out = s + FFN(s).
// Training-mode BatchNorm: the producer accumulates column sums, and the consumer kernel finalises the statistics from
// them and normalises (BnView mode 1), so no launch sits between the two.
#include <stdarg.h>
#include <string.h>

#include <algorithm>
#include <atomic>

#include "layer_ops.cuh"

namespace gps {

// performer.cu
int perf_supported(int64_t dim_head, int64_t features);
int64_t perf_mp();
int perf_index_range(int64_t N, int64_t H);
int perf_prep(const float* P, int64_t m, float* Pn, const GpsGraph& g, int64_t H, int* nmax, float* gmax, int* argk,
              cudaStream_t st);
int perf_features_fwd(float* fq, float* fk, const float* Q, const float* K, const GpsGraph& g, int64_t H, int64_t m,
                      float* gmax, int* argq, int* argk, cudaStream_t st);
int perf_linattn_fwd(const GpsGraph& g, int64_t H, int64_t m, const int* nmax, const float* qf, const float* kf,
                     const float* V, const float* gmax, float* O, cudaStream_t st);
int perf_linattn_bwd(const GpsGraph& g, int64_t H, int64_t m, const int* nmax, const float* qf, const float* kf,
                     const float* V, const float* gmax, const float* gO, float* g_qf, float* g_kf, float* gV,
                     float* ggmax, cudaStream_t st);
int perf_features_bwd(float* g_fq, float* g_fk, const float* fq, const float* fk, const float* Q, const float* K,
                      float* gQ, float* gK, const GpsGraph& g, int64_t H, int64_t m, const int* argq, const int* argk,
                      const float* ggmax, float* gmrow, bool pairwise, cudaStream_t st);

// performer_quad.cu (pairwise form for batches of small graphs)
int perf_quad_fwd(const GpsGraph& g, int64_t H, int64_t m, const int* nmax, const float* qf, const float* kf,
                  const float* V, const float* gmax, float* O, float* den, cudaStream_t st);
int perf_quad_bwd(const GpsGraph& g, int64_t H, int64_t m, const int* nmax, const float* qf, const float* kf,
                  const float* V, const float* gmax, const float* O, const float* den, const float* gO, float* gden,
                  float* g_qf, float* g_kf, float* gV, float* gmrow, cudaStream_t st);

// ------------------------------------------------------------------------------- error plumbing
static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  set_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
  return GPS_ERR_CUDA;
}
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

static std::atomic<unsigned long long> g_fallbacks{0};

// Dispatcher: TMA-fed wgmma kernel when the caller supplies operand planes, else the register-staged wgmma kernel
// on the fp32 operands, else (odd shapes / alignment) the exact CUDA-core kernel - counted, and an error under
// GPS_B200_STRICT=1 so that a 10x slower path can never be taken silently.
int gemm(const GemmParams& p, cudaStream_t stream) {
  static const bool strict = [] {
    const char* e = getenv("GPS_B200_STRICT");
    return e && e[0] == '1';
  }();
  if (p.Ap.hi && p.Bp.hi) {
    int rc = gemm_tma(p, stream);
    if (rc != GPS_ERR_UNSUPPORTED) return rc;
  }
  GPS_REQUIRE(p.A && p.B && p.C, GPS_ERR_UNSUPPORTED, "gemm: plane operands rejected and no fp32 operands to fall back to");
  // the conversion below writes the identity layout only: per-head padded planes (the wgmma attention's Q | K | V)
  // would land at the wrong columns with their pad columns unwritten
  GPS_REQUIRE(!(p.Cp.hi && p.cp_hd > 0), GPS_ERR_UNSUPPORTED,
              "gemm: dense product M=%d N=%d K=%d (ta=%d tb=%d) with per-head padded output planes (hd %d, padded to %d) "
              "was rejected by the TMA kernel, and the fp32 fallback cannot write that layout",
              p.M, p.N, p.K, p.ta, p.tb, p.cp_hd, p.cp_hd_pad);
  GemmParams q = p;
  if (q.Cp.hi) {   // the fp32 kernels do not write planes: convert afterwards
    q.Cp = Planes();
  }
  int rc = gemm_tc(q, stream);
  if (rc == GPS_ERR_UNSUPPORTED) {
    g_fallbacks.fetch_add(1, std::memory_order_relaxed);
    GPS_REQUIRE(!strict, GPS_ERR_UNSUPPORTED,
                "GPS_B200_STRICT: dense product M=%d N=%d K=%d (ta=%d tb=%d) would fall back to the CUDA-core kernel",
                p.M, p.N, p.K, p.ta, p.tb);
    rc = gemm_simt(q, stream);
  }
  if (rc == GPS_OK && p.Cp.hi) {
    ToPlanesItem it{p.C, p.ldc, p.M, p.N, p.Cp};
    rc = to_planes(&it, 1, stream);
  }
  return rc;
}

namespace {

// ------------------------------------------------------------------------------- weight packing
// A weight [rows, d] whose rows lie ld floats apart in the caller's tensor (ld > d: a column block of a wider weight,
// as PNA's pre_nns.0.0 [d, 3d]); its gradient gw has the same pitch.
struct PackSeg {
  const float* w; const float* b; float* gw; float* gb; int rows; int ld;
};
struct PackDesc {
  PackSeg seg[8];
  int nseg; int d; int total_rows;
};

// cat[r, :] = seg.w[r - row0, :], bcat[r] = seg.b[...] (0 when the Linear has no bias).  One row per blockIdx.x.
__global__ void k_pack(PackDesc pd, float* __restrict__ Wcat, float* __restrict__ bcat) {
  const int r = blockIdx.x;
  int row0 = 0, s = 0;
  while (s < pd.nseg - 1 && r >= row0 + pd.seg[s].rows) row0 += pd.seg[s++].rows;
  const float* src = pd.seg[s].w + (int64_t)(r - row0) * pd.seg[s].ld;
  float* dst = Wcat + (int64_t)r * pd.d;
  for (int c = threadIdx.x * 4; c < pd.d; c += blockDim.x * 4) st4(dst + c, ld4(src + c));
  if (threadIdx.x == 0) bcat[r] = pd.seg[s].b ? pd.seg[s].b[r - row0] : 0.f;
}
__global__ void k_unpack(PackDesc pd, const float* __restrict__ gWcat, const float* __restrict__ gbcat, int accumulate) {
  const int r = blockIdx.x;
  int row0 = 0, s = 0;
  while (s < pd.nseg - 1 && r >= row0 + pd.seg[s].rows) row0 += pd.seg[s++].rows;
  if (pd.seg[s].gw) {
    float* dst = pd.seg[s].gw + (int64_t)(r - row0) * pd.seg[s].ld;
    const float* src = gWcat + (int64_t)r * pd.d;
    for (int c = threadIdx.x * 4; c < pd.d; c += blockDim.x * 4)
      st4(dst + c, accumulate ? f4add(ld4(dst + c), ld4(src + c)) : ld4(src + c));
  }
  if (threadIdx.x == 0 && pd.seg[s].gb) pd.seg[s].gb[r - row0] = (accumulate ? pd.seg[s].gb[r - row0] : 0.f) + gbcat[r];
}

// ---- dropout-only pass: reuse the BN-apply skeleton with an identity BatchNorm is overkill; a
// dedicated tiny kernel keeps it explicit.
__global__ void k_dropmul(const float* __restrict__ src, float* __restrict__ dst, int64_t n4, int64_t c4n, float p,
                          uint64_t seed, uint64_t offset, int site, const unsigned long long* offset_dev, float p2,
                          int site2, Planes dstp) {
  if (offset_dev) offset += *offset_dev;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 v = ld4(src + i * 4);
    if (p > 0.f) v = f4mul(v, dropout_scale4(p, seed, offset, site, (uint64_t)i));
    if (p2 > 0.f) v = f4mul(v, dropout_scale4(p2, seed, offset, site2, (uint64_t)i));
    st4(dst + i * 4, v);
    if (dstp.hi) planes_store4(dstp, i / c4n, (i % c4n) * 4, v);
  }
}
__global__ void k_dropmask(float* __restrict__ dst, int64_t n4, float p, uint64_t seed, uint64_t offset, int site) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 s = dropout_scale4(p, seed, offset, site, (uint64_t)i);
    st4(dst + i * 4, make_float4(s.x > 0.f ? 1.f : 0.f, s.y > 0.f ? 1.f : 0.f, s.z > 0.f ? 1.f : 0.f,
                                 s.w > 0.f ? 1.f : 0.f));
  }
}

enum { BN_X = 0, BN_E = 1, BN_L = 2, BN_A = 3, BN_2 = 4, BN_COUNT = 5 };

struct Plan;
// A weight that the dense products read as bf16 operand planes.  The segments of Wcat (planes == &Plan::Wcat_p) are the
// Linears k_pack concatenates; row0 is a segment's first row in Wcat.
struct LayerWeight {
  PackSeg lin;   // weight [rows, cols] with the bias and gradients k_pack / k_unpack use for a Wcat segment
  int64_t cols, row0;
  Planes Plan::*planes;
};

struct Plan {
  int64_t N, E, d, H, hd, Wy, qkv_off;
  bool gated, gine, gcn, attn, perf;
  bool loc, glob;   // the layer has a local model / a global model
  const GpsAttnBias* bias;   // the BiasedTransformer's GpsLayerArgs.attn_bias; NULL when unbiased or only sizing
  // GAT (gat.cu): saved v = fold(W_edge, att_edge) [H, d] and the scores (GatScores); backward scratch g_v [H, d] then
  // gat_bwd's workspace
  bool gat;
  float *gat_v, *gat_sc, *gat_ws;
  // GENConv (genconv.cu).  Saved: agg (in `agg`), lse, u [N,d], h1 = u W0^T and r = relu(mlp.1(h1)) [N,2d], and mlp.1's
  // batch statistics in a 2d-wide slot of their own (gen_bn: mean | invstd; the BN_* slots are d wide).  Workspace:
  // mlp.1's column sums (gen_fstats / gen_bsums, [2][2d] doubles), backward g_r, g_h1 [N,2d] and g_u [N,d].
  bool gen;
  float *gen_lse, *gen_u, *gen_h1, *gen_r, *gen_bn, *gen_gr, *gen_gh1, *gen_gu;
  double *gen_fstats, *gen_bsums;
  // PNA (pna.cu): de = edge_dim (d, the bound, when only sizes are wanted).  Saved: the fold F [d, de] with its planes
  // and c [d]; Z = [x | mean | max | sum] [N, 4d] (planes; fp32 without planes); the argmax [N, d]; h = post(Z) [N, d]
  // with planes.  Forward workspace: q = e F^T + c [E, d].  Backward:
  // g_h [N, d], g_Z [N, 4d], g_q [E, d] (+ planes), g_F [d, de] | g_c [d], g_xl.
  bool pna;
  int64_t de;
  float *pna_F, *pna_c, *pna_Z, *pna_h, *pna_q, *pna_gh, *pna_gZ, *pna_gq, *pna_gF;
  int* pna_arg;
  Planes pna_F_p, pna_Z_p, pna_h_p, pna_gh_p, pna_gq_p, post_p, lin_p;
  // GPS_NORM_NONE: no norm1_local / norm1_attn / norm2.  Only the local model's own BatchNorms (BN_X, BN_E) remain, so
  // nbn = 2 statistics slots instead of BN_COUNT; s = x_loc + hA is written by the GEMM that closes the second branch
  // and x_out by the FF2 GEMM.
  bool nonorm;
  int nbn;
  int64_t inner, mp, m;   // Performer: H*64, padded / real feature count
  float *pQ, *pK, *pV, *pfq, *pfk, *pPn, *pgmax;   // saved (Performer)
  int *pargq, *pargk, *pnmax;
  float *pden, *g_pden;   // pairwise form: denominators (saved) and their gradients
  bool perf_pairwise;     // mean graph size <= 48: n^2 (m+64) < 2 n m 64
  float *g_pfq, *g_pfk, *g_pQ, *g_pK, *g_pV, *g_pgmax, *g_xp;   // backward workspace (Performer)
  float* g_pgrow;         // [N*H] per-row stabiliser gradients, summed per (graph, head) in a fixed order
  // BigBird (bigbird.cu): the attention output and lse are O / lse.  Saved: z1 = drop(ctx Wso^T + bso) + x,
  // a = LN1(z1) (+ planes), u = act(a Wi^T + bi) (+ planes), z2 = drop(u Wo^T + bo) + a, and the row statistics
  // mean1 | rstd1 | mean2 | rstd2 [4][N].  Backward: g_od (gradient of output.dense, + planes), dz2, g_u (+ planes), g_a,
  // g_so (gradient of attention.output.dense, + planes), g_x part dz1 + g_hA, and the LayerNorm partials.
  bool bb;
  float *bb_z1, *bb_a, *bb_u, *bb_z2, *bb_stat, *bb_god, *bb_dz2, *bb_gu, *bb_ga, *bb_gso, *bb_gx, *bb_part;
  Planes bb_a_p, bb_u_p, bb_so_p, bb_in_p, bb_out_p, bb_god_p, bb_gu_p, bb_gso_p;
  // saved
  float *Wcat, *bcat, *Y1, *ehat, *xt, *xloc, *O, *lse, *hA, *s, *hid, *hid_pre, *t, *bnbuf;
  float *agg, *h1, *h1_pre;
  float* dinv;   // GCN: deg^-1/2 per node
  // EquivStableLapPE edge gate (eslap.cu): saved r_e, rho_e; backward g_den [N,d], g_z / g_r [E], column-sum parts
  bool eslap;
  float *pe_r, *pe_rho, *g_den, *pe_gz, *pe_gr, *pe_part;
  // bf16 hi/lo operand planes of the TMA-fed GEMM (gemm_tma.cu).  Saved: layer inputs, weights and the forward
  // activations the weight gradients re-read; workspace: the backward gradients that feed GEMMs.
  bool use_planes;
  Planes x_p, e_p, O_p, s_p, hid_p, agg_p, h1_p, Wcat_p, C_p, out_p, ff1_p, ff2_p, g0_p, g1_p, pq_p, pk_p, pv_p;
  Planes gt_p, ghid_p, ghA_p, ge_p, gY1_p, gtmp_p, gtmp2_p, gtmp3_p, gl1_p, gh1_p;
  Planes gs_p;         // GPS_NORM_NONE: planes of g_s, the upstream gradient of both branches
  Planes gen_u_p, gen_r_p, gen_gh1_p, mlp0_p, mlp4_p;   // GENConv: u, r, g_h1 and the weights of mlp.0 / mlp.4
  Planes qkv_p;        // Q | K | V per head, padded to hd_pad columns: operands of the wgmma attention
  bool attn_tc;        // softmax attention on the tensor cores (attention_tc.cu)
  // the weights with operand planes, in the order their planes are allocated and converted (list_weights)
  LayerWeight weights[16];
  int nweights;
  int64_t saved_bytes;
  int64_t wplanes_bytes;
  // forward workspace
  double* fstats;
  int64_t fwd_bytes;
  // backward workspace
  double* bsums;
  float *g_t, *g_hid, *g_s, *g_xloc, *g_hA, *g_O, *gY1, *g_e, *g_num, *delta, *g_tmp, *g_tmp2, *g_tmp3, *g_h1, *g_agg, *gWcat,
      *gbcat, *g_xl;
  int64_t bwd_bytes;
  // per call
  bool train;
  int prec;                // GPS_PREC_*
  DropCfg dropout;         // GPSLayer.dropout: p = 0 in eval mode; the site is set per use (drop())
  float pa;                // attn_dropout, 0 in eval mode
  bool grads_prezeroed;    // GPS_FLAG_GRADS_ZEROED: the caller already zeroed every parameter-gradient buffer
                           // (one multi-tensor fill instead of a memset per weight and bias)
  bool grads_accumulate;   // GPS_FLAG_GRADS_ACCUMULATE: parameter gradients are ADDED to the caller's buffers (torch's
                           // .grad accumulation semantics on a static gradient bucket: graphgps_b200/dp.py); implies
                           // grads_prezeroed
  DropCfg drop(int site) const {
    DropCfg c = dropout;
    c.site = site;
    return c;
  }
};

// The weights with operand planes.  Wcat = [A;B;D;E | conv | in_proj] holds the node projections, so that one GEMM
// computes [Ax|Bx|Dx|Ex|Q|K|V]; this list is the one statement of that layout and sets Wy and qkv_off.
static void list_weights(const GpsLayerArgs* a, Plan* P) {
  const int64_t d = P->d, kout = P->perf ? P->inner : d;
  auto add_seg = [&](const PackSeg& seg, int64_t cols, Planes Plan::*planes) {
    const bool wcat = planes == &Plan::Wcat_p;
    P->weights[P->nweights++] = LayerWeight{seg, cols, wcat ? P->Wy : 0, planes};
    if (wcat) P->Wy += seg.rows;
  };
  auto add = [&](const GpsLinear& l, int64_t rows, int64_t cols, Planes Plan::*planes, bool bias = true) {
    add_seg(PackSeg{l.weight, bias ? l.bias : nullptr, l.grad_weight, bias ? l.grad_bias : nullptr, (int)rows, (int)cols},
            cols, planes);
  };
  if (P->gated) {
    add(a->gcn_A, d, d, &Plan::Wcat_p);
    add(a->gcn_B, d, d, &Plan::Wcat_p);
    add(a->gcn_D, d, d, &Plan::Wcat_p);
    add(a->gcn_E, d, d, &Plan::Wcat_p);
    add(a->gcn_C, d, d, &Plan::C_p);
  }
  // GCNConv.lin has no bias; GCNConv.bias is added after the aggregation (scatter.cu)
  if (P->gcn) add(a->gcn_conv, d, d, &Plan::Wcat_p, false);
  // GATConv.lin_src (= lin_dst) has no bias; GATConv.bias is added after the aggregation (gat.cu)
  if (P->gat) add(a->gat.lin_src, d, d, &Plan::Wcat_p, false);
  // PNA: the destination and source column blocks of pre_nns.0.0.weight [d, 3d] give P_dst | P_src; pre's bias enters
  // through the edge term (pna.cu)
  if (P->pna) {
    const GpsLinear& pre = a->pna.pre;
    for (int64_t blk = 0; blk < 2; ++blk)
      add_seg(PackSeg{pre.weight ? pre.weight + blk * d : nullptr, nullptr,
                      pre.grad_weight ? pre.grad_weight + blk * d : nullptr, nullptr, (int)d, (int)(3 * d)},
              d, &Plan::Wcat_p);
  }
  P->qkv_off = P->Wy;
  if (P->attn) add(a->attn_in, 3 * d, d, &Plan::Wcat_p);
  if (P->attn || P->perf) add(a->attn_out, d, kout, &Plan::out_p);
  if (P->bb) {   // attention.self.{query,key,value} (bias only with use_bias) fill the in_proj rows of Wcat
    const GpsBigBird& b = a->bigbird;
    add(b.query, d, d, &Plan::Wcat_p);
    add(b.key, d, d, &Plan::Wcat_p);
    add(b.value, d, d, &Plan::Wcat_p);
    add(b.self_out, d, d, &Plan::bb_so_p);
    add(b.intermediate, d, d, &Plan::bb_in_p);
    add(b.output, d, d, &Plan::bb_out_p);
  }
  add(a->ff1, 2 * d, d, &Plan::ff1_p);
  add(a->ff2, d, 2 * d, &Plan::ff2_p);
  if (P->gine) {
    add(a->gine_lin0, d, d, &Plan::g0_p);
    add(a->gine_lin1, d, d, &Plan::g1_p);
  }
  if (P->gen) {   // GENConv's MLP Linears have no bias
    add(a->genconv.lin0, 2 * d, d, &Plan::mlp0_p, false);
    add(a->genconv.lin1, d, 2 * d, &Plan::mlp4_p, false);
  }
  if (P->pna) {
    add(a->pna.post, d, 4 * d, &Plan::post_p);
    add(a->pna.lin, d, d, &Plan::lin_p);
  }
  if (P->perf) {
    add(a->perf_q, P->inner, d, &Plan::pq_p);
    add(a->perf_k, P->inner, d, &Plan::pk_p);
    add(a->perf_v, P->inner, d, &Plan::pv_p);
  }
}

// Planes the caller hands over: a previous layer's output planes, or buffers for this layer's output planes.  Taken
// when they hold what the precision needs (lo in fp32 mode) with a TMA-aligned pitch, else empty.
static Planes caller_planes(const GpsPlanes& g, int64_t d, int precision) {
  const bool lo = precision == GPS_PREC_FP32;
  if (!g.hi || (lo && !g.lo) || g.ld < d || g.ld % 8 != 0) return Planes();
  return Planes{(__nv_bfloat16*)g.hi, lo ? (__nv_bfloat16*)g.lo : nullptr, g.ld};
}

static int make_plan(const GpsLayerArgs* a, Plan* P, bool bind) {
  memset(P, 0, sizeof(*P));
  GPS_REQUIRE(a, GPS_ERR_ARG, "null args");
  P->N = a->graph.N;
  P->E = a->graph.E;
  P->d = a->d;
  P->H = a->heads;
  GPS_REQUIRE(a->d > 0 && a->d % 4 == 0, GPS_ERR_UNSUPPORTED, "dim_h must be a positive multiple of 4 (got %lld)",
              (long long)a->d);
  P->gated = a->local_type == GPS_LOCAL_GATEDGCN;
  P->gine = a->local_type == GPS_LOCAL_GINE;
  P->gcn = a->local_type == GPS_LOCAL_GCN;
  P->gat = a->local_type == GPS_LOCAL_GAT;
  P->gen = a->local_type == GPS_LOCAL_GENCONV;
  P->pna = a->local_type == GPS_LOCAL_PNA;
  P->loc = P->gated || P->gine || P->gcn || P->gat || P->gen || P->pna;
  P->de = bind ? a->pna.edge_dim : a->d;   // sizes alone: edge_dim <= d is the bound
  GPS_REQUIRE(a->local_type == GPS_LOCAL_NONE || P->loc, GPS_ERR_ARG, "unknown local_type %d", a->local_type);
  if (P->pna) GPS_TRY(pna_check(a->d, P->de));
  if (P->gat) GPS_TRY(gat_check(a->d, a->heads));
  GPS_REQUIRE(!P->gen || a->d <= 2048, GPS_ERR_UNSUPPORTED,
              "GENConv needs dim_h <= 2048: its 2 dim_h-wide BatchNorm runs on the row-wise stages (got %lld)",
              (long long)a->d);
  P->eslap = a->pe != nullptr;
  GPS_REQUIRE(!P->eslap || P->gated, GPS_ERR_ARG, "pe (EquivStableLapPE) is read by the GatedGCN local model only");
  GPS_REQUIRE(!P->eslap || a->pe_dim >= 1, GPS_ERR_ARG, "pe_dim must be >= 1 (got %lld)", (long long)a->pe_dim);
  GPS_REQUIRE(a->global_type == GPS_GLOBAL_NONE || a->global_type == GPS_GLOBAL_TRANSFORMER ||
                  a->global_type == GPS_GLOBAL_PERFORMER || a->global_type == GPS_GLOBAL_BIGBIRD,
              GPS_ERR_ARG, "unknown global_type %d", a->global_type);
  P->attn = a->global_type == GPS_GLOBAL_TRANSFORMER;
  P->perf = a->global_type == GPS_GLOBAL_PERFORMER;
  P->bb = a->global_type == GPS_GLOBAL_BIGBIRD;
  P->glob = P->attn || P->perf || P->bb;
  if (bind) {   // attention bias of the BiasedTransformer; NULL bias = none
    const GpsAttnBias& ab = a->attn_bias;
    GPS_REQUIRE(ab.bias || (ab.nmax == 0 && !ab.grad_bias), GPS_ERR_ARG,
                "attention bias: null bias pointer with nmax %lld / grad_bias set", (long long)ab.nmax);
    GPS_REQUIRE(!ab.bias || P->attn, GPS_ERR_ARG, "an attention bias needs global_type GPS_GLOBAL_TRANSFORMER (got %d)",
                a->global_type);
    GPS_REQUIRE(!ab.bias || ab.nmax >= 1, GPS_ERR_ARG, "attention bias: nmax must be >= 1 (got %lld)",
                (long long)ab.nmax);
    P->bias = ab.bias ? &ab : nullptr;
  }
  if (P->bb) {   // any head dim (the shipped BigBird config has hd = 7)
    GPS_REQUIRE(a->heads > 0 && a->d % a->heads == 0, GPS_ERR_ARG, "dim_h %% num_heads != 0");
    P->hd = a->d / a->heads;
    if (bind) GPS_TRY(bb_check(a->d, a->heads, &a->bigbird));
  }
  if (P->perf) {
    GPS_TRY(perf_supported(a->perf_dim_head, a->perf_features));
    GPS_REQUIRE(a->heads > 0, GPS_ERR_ARG, "num_heads must be positive");
    GPS_TRY(perf_index_range(a->graph.N, a->heads));
    P->inner = a->heads * a->perf_dim_head;
    P->mp = perf_mp();
    P->m = a->perf_features;
  }
  GPS_REQUIRE(a->local_type != GPS_LOCAL_NONE || P->glob, GPS_ERR_ARG,
              "GPSLayer needs a local model or a global model");
  GPS_REQUIRE(a->norm_type == GPS_NORM_BATCH || a->norm_type == GPS_NORM_NONE, GPS_ERR_UNSUPPORTED,
              "norm_type %d is not built (GPS_NORM_BATCH = 0, GPS_NORM_NONE = 1)", a->norm_type);
  P->nonorm = a->norm_type == GPS_NORM_NONE;
  P->nbn = P->nonorm ? BN_L : BN_COUNT;   // BN_X, BN_E come first
  if (P->attn) {
    GPS_REQUIRE(a->heads > 0 && a->d % a->heads == 0, GPS_ERR_ARG, "dim_h %% num_heads != 0");
    P->hd = a->d / a->heads;
    GPS_REQUIRE(P->hd % 4 == 0, GPS_ERR_UNSUPPORTED, "head dim %lld must be a multiple of 4", (long long)P->hd);
  }
  GPS_REQUIRE(a->act == GPS_ACT_RELU || a->act == GPS_ACT_GELU, GPS_ERR_ARG, "unknown activation %d", a->act);
  GPS_REQUIRE(a->dropout >= 0.f && a->dropout < 1.f && a->attn_dropout >= 0.f && a->attn_dropout < 1.f,
              GPS_ERR_ARG, "dropout probabilities must be in [0,1)");
  P->train = a->training != 0;
  P->prec = a->precision;
  P->dropout = drop_cfg(a->dropout, P->train, a->seed, a->offset, a->offset_dev, 0);
  P->pa = P->train ? a->attn_dropout : 0.f;
  set_grad_flags(P, a->flags);
  list_weights(a, P);
  const int64_t N = P->N, E = P->E, d = P->d;
  const bool gelu = a->act == GPS_ACT_GELU;

  Arena S(bind ? a->saved : nullptr, a->saved_bytes);
  P->bnbuf = S.alloc<float>(P->nbn * 2 * d);
  if (P->Wy) {
    P->Wcat = S.alloc<float>(P->Wy * d);
    P->bcat = S.alloc<float>(P->Wy);
    P->Y1 = S.alloc<float>(N * P->Wy);
  }
  if (P->gated) {
    P->ehat = S.alloc<float>(E * d);
    P->xt = S.alloc<float>(N * d);
    if (P->eslap) {
      P->pe_r = S.alloc<float>(E);
      P->pe_rho = S.alloc<float>(E);
    }
  }
  if (P->gine) {
    P->agg = S.alloc<float>(N * d);
    P->h1 = S.alloc<float>(N * d);
    if (gelu) P->h1_pre = S.alloc<float>(N * d);
  }
  if (P->gcn) P->dinv = S.alloc<float>(N);
  if (P->gat) {
    P->gat_v = S.alloc<float>(P->H * d);
    P->gat_sc = S.alloc<float>((4 * N + E) * P->H);
  }
  if (P->gen) {
    P->agg = S.alloc<float>(N * d);
    P->gen_lse = S.alloc<float>(N * d);
    P->gen_u = S.alloc<float>(N * d);
    P->gen_h1 = S.alloc<float>(N * 2 * d);
    P->gen_r = S.alloc<float>(N * 2 * d);
    P->gen_bn = S.alloc<float>(2 * 2 * d);
  }
  if (P->pna) {
    P->pna_F = S.alloc<float>(d * P->de);
    P->pna_c = S.alloc<float>(d);
    P->pna_arg = S.alloc<int>(N * d);
    P->pna_h = S.alloc<float>(N * d);
  }
  if (P->loc && !P->nonorm) P->xloc = S.alloc<float>(N * d);   // read by norm1_local's backward
  if (P->attn) {
    P->O = S.alloc<float>(N * d);
    P->lse = S.alloc<float>(N * P->H);
    if (!P->nonorm) P->hA = S.alloc<float>(N * d);
  }
  if (P->perf) {
    const int64_t NH = N * P->H, BH = a->graph.B * P->H;
    P->pQ = S.alloc<float>(N * P->inner);
    P->pK = S.alloc<float>(N * P->inner);
    P->pV = S.alloc<float>(N * P->inner);
    P->pfq = S.alloc<float>(NH * P->mp);
    P->pfk = S.alloc<float>(NH * P->mp);
    P->pPn = S.alloc<float>(P->mp * a->perf_dim_head);
    P->pgmax = S.alloc<float>(BH);
    P->pargq = S.alloc<int>(NH);
    P->pargk = S.alloc<int>(BH);
    P->pnmax = S.alloc<int>(1);
    P->pden = S.alloc<float>(NH);
    P->perf_pairwise = a->graph.B > 0 && N <= 48 * a->graph.B;
    P->O = S.alloc<float>(N * P->inner);
    if (!P->nonorm) P->hA = S.alloc<float>(N * d);
  }
  if (P->bb) {
    P->O = S.alloc<float>(N * d);
    P->lse = S.alloc<float>(N * P->H);
    if (!P->nonorm) P->hA = S.alloc<float>(N * d);
    P->bb_z1 = S.alloc<float>(N * d);
    P->bb_a = S.alloc<float>(N * d);
    P->bb_u = S.alloc<float>(N * d);
    P->bb_z2 = S.alloc<float>(N * d);
    P->bb_stat = S.alloc<float>(4 * N);
  }
  P->s = S.alloc<float>(N * d);
  P->hid = S.alloc<float>(N * 2 * d);
  if (gelu) P->hid_pre = S.alloc<float>(N * 2 * d);
  if (!P->nonorm) P->t = S.alloc<float>(N * d);   // norm2's input
  P->use_planes = (d % 8 == 0) && (!P->perf || P->inner % 8 == 0);
  const bool lo = a->precision == GPS_PREC_FP32;
  if (P->use_planes) {
    const int64_t kout = P->perf ? P->inner : d;
    // inputs: the planes written by the previous layer of the stack when it hands them over
    P->x_p = caller_planes(a->x_planes_in, d, a->precision);
    if (!P->x_p.hi) P->x_p = arena_planes(S, N, d, lo);
    if (P->gated || P->gine) {
      P->e_p = caller_planes(a->e_planes_in, d, a->precision);
      if (!P->e_p.hi) P->e_p = arena_planes(S, E, d, lo);
    }
    if (P->glob) P->O_p = arena_planes(S, N, kout, lo);
    if (P->bb) {
      P->bb_a_p = arena_planes(S, N, d, lo);
      P->bb_u_p = arena_planes(S, N, d, lo);
    }
    // Forward softmax attention on the tensor cores (attention_tc.cu) when the batch's graphs are large enough for
    // 128 x 128 tiles to pay: at the PCQM4M shape (mean 14 nodes per graph) a 128-row tile sees ~45 useful keys of 256
    // in one latency-bound wave and the CUDA-core kernel is faster; the tensor-core kernel wins once a graph fills a
    // tile (ogbg-code2 shape, mean 125 / max ~1000 nodes).
    P->attn_tc = P->attn && attention_tc_supported(P->hd) && a->graph.B > 0 && N >= 64 * a->graph.B;
    if (P->attn_tc) P->qkv_p = arena_planes(S, N, 3 * P->H * attention_tc_hd_pad(P->hd), lo);
    P->s_p = arena_planes(S, N, d, lo);
    P->hid_p = arena_planes(S, N, 2 * d, lo);
    if (P->gine) {
      P->agg_p = arena_planes(S, N, d, lo);
      P->h1_p = arena_planes(S, N, d, lo);
    }
    if (P->gen) {
      P->gen_u_p = arena_planes(S, N, d, lo);
      P->gen_r_p = arena_planes(S, N, 2 * d, lo);
    }
    if (P->pna) {   // edge_attr is de wide: planes of its own, never the caller's d-wide ones
      P->e_p = arena_planes(S, E, P->de, lo);
      P->pna_F_p = arena_planes(S, d, P->de, lo);
      P->pna_Z_p = arena_planes(S, N, 4 * d, lo);
      P->pna_h_p = arena_planes(S, N, d, lo);
    }
    // weight planes: in the caller's persistent buffer when one is given (packed once per optimiser step), else in `saved`
    Arena Wa(bind ? a->wplanes : nullptr, a->wplanes_bytes);
    Arena& WA = bind && a->wplanes != nullptr ? Wa : S;
    const int64_t w0 = WA.used;
    for (int i = 0; i < P->nweights; ++i) {
      const LayerWeight& w = P->weights[i];
      if (w.row0 == 0) P->*w.planes = arena_planes(WA, w.planes == &Plan::Wcat_p ? P->Wy : w.lin.rows, w.cols, lo);
    }
    P->wplanes_bytes = WA.used - w0;
    GPS_REQUIRE(!Wa.overflow, GPS_ERR_ARG, "wplanes buffer too small (%lld < %lld)", (long long)a->wplanes_bytes,
                (long long)P->wplanes_bytes);
  }
  if (P->pna && !P->use_planes) P->pna_Z = S.alloc<float>(N * 4 * d);
  P->saved_bytes = S.used;
  GPS_REQUIRE(!S.overflow, GPS_ERR_ARG, "saved buffer too small (%lld < %lld)", (long long)a->saved_bytes,
              (long long)S.used);

  // forward and backward share the caller's workspace (never live at the same time)
  Arena F(bind ? a->workspace : nullptr, a->workspace_bytes);
  P->fstats = F.alloc<double>(P->nbn * 2 * d);
  if (P->gen) P->gen_fstats = F.alloc<double>(2 * 2 * d);
  if (P->pna) P->pna_q = F.alloc<float>(E * d);
  if (P->nonorm && P->loc) {
    // x_loc is an operand of the GEMM that writes s (and of nothing in the backward pass); a lone local model writes s
    P->xloc = P->glob ? F.alloc<float>(N * d) : P->s;
  }
  P->fwd_bytes = F.used;

  Arena Bk(bind ? a->workspace : nullptr, a->workspace_bytes);
  P->bsums = Bk.alloc<double>(P->nbn * 2 * d);
  if (!P->nonorm) P->g_t = Bk.alloc<float>(N * d);   // GPS_NORM_NONE: g_t is grad_x_out itself
  P->g_hid = Bk.alloc<float>(N * 2 * d);
  P->g_s = Bk.alloc<float>(N * d);
  P->g_tmp = Bk.alloc<float>(N * d);
  if (a->dropout > 0.f || (P->perf && a->attn_dropout > 0.f)) {   // separate dropout temporaries: side-stream weight
    P->g_tmp2 = Bk.alloc<float>(N * d);                            // gradients still read the earlier ones
    P->g_tmp3 = Bk.alloc<float>(N * d);
  }
  // GPS_NORM_NONE: the upstream gradients of x_loc and hA are both g_s
  if (P->loc && !P->nonorm) P->g_xloc = Bk.alloc<float>(N * d);
  if (P->attn) {
    if (!P->nonorm) P->g_hA = Bk.alloc<float>(N * d);
    P->g_O = Bk.alloc<float>(N * d);
    P->delta = Bk.alloc<float>(N * P->H);
  }
  if (P->perf) {
    const int64_t NH = N * P->H, BH = a->graph.B * P->H;
    if (!P->nonorm) P->g_hA = Bk.alloc<float>(N * d);
    P->g_O = Bk.alloc<float>(N * P->inner);
    P->g_pfq = Bk.alloc<float>(NH * P->mp);
    P->g_pfk = Bk.alloc<float>(NH * P->mp);
    P->g_pQ = Bk.alloc<float>(N * P->inner);
    P->g_pK = Bk.alloc<float>(N * P->inner);
    P->g_pV = Bk.alloc<float>(N * P->inner);
    P->g_pgmax = Bk.alloc<float>(BH);
    P->g_pgrow = Bk.alloc<float>(NH);
    P->g_pden = Bk.alloc<float>(NH);
    P->g_xp = Bk.alloc<float>(N * d);
  }
  if (P->bb) {
    if (!P->nonorm) P->g_hA = Bk.alloc<float>(N * d);
    P->g_O = Bk.alloc<float>(N * d);
    P->delta = Bk.alloc<float>(N * P->H);
    P->bb_god = Bk.alloc<float>(N * d);
    P->bb_dz2 = Bk.alloc<float>(N * d);
    P->bb_gu = Bk.alloc<float>(N * d);
    P->bb_ga = Bk.alloc<float>(N * d);
    P->bb_gso = Bk.alloc<float>(N * d);
    P->bb_gx = Bk.alloc<float>(N * d);
    P->bb_part = Bk.alloc<float>(layernorm_part_floats(d));
  }
  if (P->Wy) {
    P->gY1 = Bk.alloc<float>(N * P->Wy);
    P->gWcat = Bk.alloc<float>(P->Wy * d + P->Wy);   // [gWcat | gbcat] contiguous: one memset
    P->gbcat = P->gWcat ? P->gWcat + P->Wy * d : nullptr;
  }
  if (P->gated) {
    P->g_e = Bk.alloc<float>(E * d);
    P->g_num = Bk.alloc<float>(N * d);
    if (P->eslap) {
      P->g_den = Bk.alloc<float>(N * d);
      P->pe_gz = Bk.alloc<float>(E);
      P->pe_gr = Bk.alloc<float>(E);
      P->pe_part = Bk.alloc<float>(ceil_div(E, eslap_wgrad_chunk(E)) * (3 * d + 1));
    }
  }
  if (P->gine) {
    P->g_h1 = Bk.alloc<float>(N * d);
    P->g_agg = Bk.alloc<float>(N * d);
    P->g_xl = Bk.alloc<float>(N * d);
  }
  if (P->gat) P->gat_ws = Bk.alloc<float>(P->H * d + gat_bwd_workspace_floats(N, E, P->H, d));
  if (P->gen) {
    P->gen_bsums = Bk.alloc<double>(2 * 2 * d);
    P->gen_gr = Bk.alloc<float>(N * 2 * d);
    P->gen_gh1 = Bk.alloc<float>(N * 2 * d);
    P->gen_gu = Bk.alloc<float>(N * d);
    P->g_xl = Bk.alloc<float>(N * d);
  }
  if (P->pna) {
    P->pna_gh = Bk.alloc<float>(N * d);
    P->pna_gZ = Bk.alloc<float>(N * 4 * d);
    P->pna_gq = Bk.alloc<float>(E * d);
    P->pna_gF = Bk.alloc<float>(d * P->de + d);   // [g_F | g_c] contiguous: one memset
    P->g_xl = Bk.alloc<float>(N * d);
  }
  if (P->use_planes) {
    P->gt_p = arena_planes(Bk, N, d, lo);
    P->ghid_p = arena_planes(Bk, N, 2 * d, lo);
    if (P->glob && !P->nonorm) P->ghA_p = arena_planes(Bk, N, d, lo);
    if (P->bb) {
      P->bb_god_p = arena_planes(Bk, N, d, lo);
      P->bb_gu_p = arena_planes(Bk, N, d, lo);
      P->bb_gso_p = arena_planes(Bk, N, d, lo);
    }
    if (P->nonorm) P->gs_p = arena_planes(Bk, N, d, lo);
    if (P->gated) P->ge_p = arena_planes(Bk, E, d, lo);
    if (P->Wy) P->gY1_p = arena_planes(Bk, N, P->Wy, lo);
    if (a->dropout > 0.f || (P->perf && a->attn_dropout > 0.f)) {
      P->gtmp_p = arena_planes(Bk, N, d, lo);
      P->gtmp2_p = arena_planes(Bk, N, d, lo);
      P->gtmp3_p = arena_planes(Bk, N, d, lo);
    }
    if (P->gine) {
      if (!P->nonorm) P->gl1_p = arena_planes(Bk, N, d, lo);
      P->gh1_p = arena_planes(Bk, N, d, lo);
    }
    if (P->gen) {
      if (!P->nonorm) P->gl1_p = arena_planes(Bk, N, d, lo);
      P->gen_gh1_p = arena_planes(Bk, N, 2 * d, lo);
    }
    if (P->pna) {
      if (!P->nonorm) P->gl1_p = arena_planes(Bk, N, d, lo);
      P->pna_gh_p = arena_planes(Bk, N, d, lo);
      P->pna_gq_p = arena_planes(Bk, E, d, lo);
    }
  }
  P->bwd_bytes = Bk.used;
  return GPS_OK;
}

// BatchNorm `which` as its consumer kernels see it (bn_view_at, layer_ops.cuh)
static BnView bn_view(const Plan& P, int which, const GpsBatchNorm& bn, int64_t fwd_rows = -1) {
  return bn_view_at(P, P.bnbuf + (int64_t)which * 2 * P.d, P.fstats + (int64_t)which * 2 * P.d, P.d, bn, fwd_rows);
}
// GENConv's mlp.1, a BatchNorm over 2d columns with its own slot
static BnView gen_bn_view(const Plan& P, const GpsBatchNorm& bn, int64_t fwd_rows = -1) {
  return bn_view_at(P, P.gen_bn, P.gen_fstats, 2 * P.d, bn, fwd_rows);
}

static PackDesc pack_desc(const Plan& P) {
  PackDesc pd;
  memset(&pd, 0, sizeof(pd));
  pd.d = (int)P.d;
  for (int i = 0; i < P.nweights; ++i) {
    if (P.weights[i].planes != &Plan::Wcat_p) continue;
    pd.seg[pd.nseg++] = P.weights[i].lin;
    pd.total_rows += P.weights[i].lin.rows;
  }
  return pd;
}

static int check_linear(const GpsLinear& l, const char* name, bool need_bias) {
  GPS_REQUIRE(l.weight, GPS_ERR_ARG, "missing parameter %s.weight", name);
  GPS_REQUIRE(!need_bias || l.bias, GPS_ERR_ARG, "missing parameter %s.bias", name);
  return GPS_OK;
}
static int check_bn(const GpsBatchNorm& b, const char* name) {
  GPS_REQUIRE(b.weight && b.bias, GPS_ERR_ARG, "missing parameter %s.{weight,bias}", name);
  return GPS_OK;
}

static int check_params(const GpsLayerArgs* a, const Plan& P) {
  GPS_REQUIRE(a->x && (P.E == 0 || a->edge_attr || !(P.gated || P.gine || P.gat || P.gen || P.pna)), GPS_ERR_ARG,
              "missing x / edge_attr");
  if (P.gated) {
    GPS_TRY(check_linear(a->gcn_A, "local_model.A", true));
    GPS_TRY(check_linear(a->gcn_B, "local_model.B", true));
    GPS_TRY(check_linear(a->gcn_C, "local_model.C", true));
    GPS_TRY(check_linear(a->gcn_D, "local_model.D", true));
    GPS_TRY(check_linear(a->gcn_E, "local_model.E", true));
    GPS_TRY(check_bn(a->bn_node_x, "local_model.bn_node_x"));
    GPS_TRY(check_bn(a->bn_edge_e, "local_model.bn_edge_e"));
    if (P.eslap) {
      GPS_TRY(check_linear(a->pe_mlp0, "local_model.mlp_r_ij.0", true));
      GPS_TRY(check_linear(a->pe_mlp1, "local_model.mlp_r_ij.2", true));
    }
  }
  if (P.gine) {
    GPS_TRY(check_linear(a->gine_lin0, "local_model.nn.0", true));
    GPS_TRY(check_linear(a->gine_lin1, "local_model.nn.2", true));
  }
  if (P.gcn) GPS_TRY(check_linear(a->gcn_conv, "local_model.lin / local_model.bias", true));
  if (P.gat) {
    GPS_TRY(check_linear(a->gat.lin_src, "local_model.lin_src / local_model.bias", true));
    GPS_TRY(check_linear(a->gat.lin_edge, "local_model.lin_edge", false));
    GPS_REQUIRE(a->gat.att_src && a->gat.att_dst && a->gat.att_edge, GPS_ERR_ARG,
                "missing parameter local_model.att_{src,dst,edge}");
  }
  if (P.gen) {
    GPS_TRY(check_linear(a->genconv.lin0, "local_model.mlp.0", false));
    GPS_TRY(check_bn(a->genconv.bn, "local_model.mlp.1"));
    GPS_REQUIRE(a->genconv.bn.running_mean && a->genconv.bn.running_var, GPS_ERR_ARG,
                "missing buffer local_model.mlp.1.running_{mean,var}");
    GPS_TRY(check_linear(a->genconv.lin1, "local_model.mlp.4", false));
  }
  if (P.pna) {
    GPS_TRY(check_linear(a->pna.edge_encoder, "local_model.edge_encoder", true));
    GPS_TRY(check_linear(a->pna.pre, "local_model.pre_nns.0.0", true));
    GPS_TRY(check_linear(a->pna.post, "local_model.post_nns.0.0", true));
    GPS_TRY(check_linear(a->pna.lin, "local_model.lin", true));
  }
  const bool bn = !P.nonorm;   // norm1_local / norm1_attn / norm2 exist in BatchNorm mode only
  if (P.loc && bn) GPS_TRY(check_bn(a->norm1_local, "norm1_local"));
  if (P.attn) {
    GPS_TRY(check_linear(a->attn_in, "self_attn.in_proj", true));
    GPS_TRY(check_linear(a->attn_out, "self_attn.out_proj", true));
    if (bn) GPS_TRY(check_bn(a->norm1_attn, "norm1_attn"));
  }
  if (P.perf) {
    GPS_TRY(check_linear(a->perf_q, "self_attn.to_q", false));
    GPS_TRY(check_linear(a->perf_k, "self_attn.to_k", false));
    GPS_TRY(check_linear(a->perf_v, "self_attn.to_v", false));
    GPS_TRY(check_linear(a->attn_out, "self_attn.to_out", true));
    GPS_REQUIRE(a->perf_proj, GPS_ERR_ARG, "missing buffer self_attn.fast_attention.projection_matrix");
    if (bn) GPS_TRY(check_bn(a->norm1_attn, "norm1_attn"));
  }
  if (P.bb) {
    const GpsBigBird& b = a->bigbird;
    GPS_TRY(check_linear(b.query, "self_attn.encoder.layers.0.attention.self.query", false));
    GPS_TRY(check_linear(b.key, "self_attn.encoder.layers.0.attention.self.key", false));
    GPS_TRY(check_linear(b.value, "self_attn.encoder.layers.0.attention.self.value", false));
    GPS_TRY(check_linear(b.self_out, "self_attn.encoder.layers.0.attention.output.dense", true));
    GPS_TRY(check_linear(b.ln1, "self_attn.encoder.layers.0.attention.output.LayerNorm", true));
    GPS_TRY(check_linear(b.intermediate, "self_attn.encoder.layers.0.intermediate.dense", true));
    GPS_TRY(check_linear(b.output, "self_attn.encoder.layers.0.output.dense", true));
    GPS_TRY(check_linear(b.ln2, "self_attn.encoder.layers.0.output.LayerNorm", true));
    if (bn) GPS_TRY(check_bn(a->norm1_attn, "norm1_attn"));
  }
  GPS_TRY(check_linear(a->ff1, "ff_linear1", true));
  GPS_TRY(check_linear(a->ff2, "ff_linear2", true));
  if (bn) GPS_TRY(check_bn(a->norm2, "norm2"));
  return GPS_OK;
}

// The [N, d] gradient g in front of the dropout at `site` (and, p2 > 0, of the inner one at site2 before it): g times
// the dropout scales, written to the temporary tmp (and its planes tmp_p), when a dropout is active, else g itself.
static int dropmul(const Plan& P, Operand g, float* tmp, Planes tmp_p, int site, cudaStream_t st, Operand* out,
                   float p2 = 0.f, int site2 = 0) {
  *out = g;
  if (!(P.dropout.p > 0.f || p2 > 0.f)) return GPS_OK;
  *out = Operand{tmp, P.d, tmp_p};
  return dropmul_rows(g.f, tmp, P.N, P.d, P.drop(site), p2, site2, tmp_p, st);
}

}  // namespace

int side_stream(Side** out) {
  static thread_local Side sides[64];
  int dev = 0;
  GPS_CUDA(cudaGetDevice(&dev));
  GPS_REQUIRE(dev >= 0 && dev < 64, GPS_ERR_ARG, "device index %d out of range: side streams exist for devices 0..63",
              dev);
  GPS_TRY(sides[dev].init());
  *out = &sides[dev];
  return GPS_OK;
}

int dropmul_rows(const float* src, float* dst, int64_t rows, int64_t d, const DropCfg& c, float p2, int site2,
                 Planes dstp, cudaStream_t st) {
  GPS_REQUIRE(d % 4 == 0, GPS_ERR_UNSUPPORTED, "dropout pass needs d %% 4 == 0 (got %lld)", (long long)d);
  const int64_t n4 = rows * d / 4;
  if (n4 == 0) return GPS_OK;
  k_dropmul<<<(unsigned)std::min<int64_t>(ceil_div(n4, 256), kNumSMs * 8), 256, 0, st>>>(
      src, dst, n4, d / 4, c.p, c.seed, c.offset, c.site, c.offset_dev, p2, site2, dstp);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

// =================================================================================== forward
static int layer_forward(const GpsLayerArgs* a, cudaStream_t st) {
  Plan P;
  const GpsGat& gat = a->gat;   // the local model's parameters: read when local_type selects it
  const GpsGenConv& gen = a->genconv;
  const GpsPna& pna = a->pna;
  GPS_TRY(make_plan(a, &P, true));
  GPS_REQUIRE(a->saved && a->workspace, GPS_ERR_ARG, "saved/workspace buffers are required");
  GPS_REQUIRE(a->workspace_bytes >= P.fwd_bytes, GPS_ERR_ARG, "workspace too small (%lld < %lld)",
              (long long)a->workspace_bytes, (long long)P.fwd_bytes);
  GPS_TRY(check_params(a, P));
  GPS_REQUIRE(a->x_out, GPS_ERR_ARG, "x_out is null");
  const int64_t N = P.N, E = P.E, d = P.d;
  const int act = a->act;
  auto stats = [&](int which) -> double* { return P.train && which < P.nbn ? P.fstats + (int64_t)which * 2 * d : nullptr; };
  auto out_planes = [&](const GpsPlanes& g) {   // planes of this layer's outputs for the next layer of the stack
    return P.use_planes ? caller_planes(g, d, P.prec) : Planes();
  };

  if (P.train) GPS_CUDA(cudaMemsetAsync(P.fstats, 0, (size_t)P.nbn * 2 * d * sizeof(double), st));
  if (P.train && P.gen) GPS_CUDA(cudaMemsetAsync(P.gen_fstats, 0, (size_t)2 * 2 * d * sizeof(double), st));
  Side* sd;
  GPS_TRY(side_stream(&sd));
  cudaStream_t s2 = sd->s;
  const bool two_branches = P.loc && P.glob;
  // GPS_NORM_NONE: the producer that closes the last branch writes s = x_loc + hA with its planes (x_loc = s when the
  // local model is alone)
  const bool local_writes_s = P.nonorm && !P.glob;
  // GPS_NORM_NONE, attention output projection on stream sg: writes s = x + drop(.) [+ x_loc] and its planes instead of
  // hA; with a local branch, sg first waits for it
  auto close_with_s = [&](GemmParams& g, cudaStream_t sg) -> int {
    g.C = P.s; g.Cp = P.s_p;
    if (two_branches) {
      g.R2 = P.xloc; g.ldr2 = (int)d;
      GPS_TRY(sd->order(st, sg));
    }
    return GPS_OK;
  };

  // weights: concatenate the node projections
  if (P.Wy) {
    PackDesc pdsc0 = pack_desc(P);
    k_pack<<<(unsigned)pdsc0.total_rows, 128, 0, st>>>(pdsc0, P.Wcat, P.bcat);
    GPS_LAUNCH_CHECK();
  }
  if (P.use_planes) {
    // layer inputs and every weight -> bf16 hi/lo planes, one launch (the producers inside the layer write the
    // planes of their outputs themselves)
    ToPlanesItem it[16];
    int ni = 0;
    auto add = [&](const float* src, int64_t ld, int64_t rows, int64_t cols, Planes dst) {
      if (src && dst.hi && rows > 0) it[ni++] = ToPlanesItem{src, ld, (int)rows, (int)cols, dst};
    };
    if (P.x_p.hi != (__nv_bfloat16*)a->x_planes_in.hi) add(a->x, d, N, d, P.x_p);
    if ((P.gated || P.gine) && P.e_p.hi != (__nv_bfloat16*)a->e_planes_in.hi) add(a->edge_attr, d, E, d, P.e_p);
    if (P.pna) add(a->edge_attr, P.de, E, P.de, P.e_p);
    if (!(a->wplanes && a->wplanes_valid)) {
      for (int i = 0; i < P.nweights; ++i) {
        const LayerWeight& w = P.weights[i];
        add(w.lin.w, w.lin.ld, w.lin.rows, w.cols, (P.*w.planes).rows(w.row0));
      }
    }
    GPS_TRY(to_planes(it, ni, st));
  }
  if (P.pna) {   // edge term of the messages, next to the node projections: q = e F^T + c, F = W_e W_enc (pna.cu)
    GPS_TRY(sd->fork(st));
    GPS_TRY(pna_fold_fwd(pna.pre.weight, pna.pre.bias, pna.edge_encoder.weight, pna.edge_encoder.bias, d, P.de,
                         P.pna_F, P.pna_c, s2));
    if (P.pna_F_p.hi) {
      ToPlanesItem it{P.pna_F, P.de, (int)d, (int)P.de, P.pna_F_p};
      GPS_TRY(to_planes(&it, 1, s2));
    }
    if (E > 0)
      GPS_TRY(gemm(linear_fwd(P, E, d, P.de, {a->edge_attr, P.de, P.e_p}, {P.pna_F, P.de, P.pna_F_p}, P.pna_q, d,
                              P.pna_c),
                   s2));
  }
  if (P.gated) {   // edge projection has no dependency on the node side: run it next to the node projections
    GPS_REQUIRE(a->edge_out, GPS_ERR_ARG, "edge_out is null");
    GPS_TRY(sd->fork(st));
    // Ce = e C^T + bC (gatedgcn_layer.py:59)
    GPS_TRY(gemm(linear_fwd(P, E, d, d, {a->edge_attr, d, P.e_p}, {a->gcn_C.weight, d, P.C_p}, P.ehat, d,
                            a->gcn_C.bias),
                 s2));
    // EquivStableLapPE gate r_e, rho_e: reads PE, the graph and mlp_r_ij only (gatedgcn_layer.py:101-104)
    if (P.eslap)
      GPS_TRY(eslap_fwd(a->graph, a->pe, a->pe_dim, d, act, a->pe_mlp0.weight, a->pe_mlp0.bias, a->pe_mlp1.weight,
                        a->pe_mlp1.bias, P.pe_r, P.pe_rho, s2));
  }

  // ---- node projections: [Ax|Bx|Dx|Ex|Q|K|V] = x Wcat^T + bcat  (gatedgcn_layer.py:57-61, MHA in_proj)
  // The two consumers of the projections get their own GEMM: [Ax|Bx|Dx|Ex] on the main stream for the
  // message-passing branch, [Q|K|V] on the attention branch's stream, so both branches start ~25 us after the
  // pack instead of after one 50 us GEMM.
  cudaStream_t sg = st;   // stream of the global-attention branch
  if (two_branches) {
    GPS_TRY(sd->order(st, sd->s3));
    sg = sd->s3;
  }
  if (P.Wy) {
    const int64_t wl = P.qkv_off, wg = P.Wy - P.qkv_off;   // local / global column blocks
    const Operand x{a->x, d, P.x_p};
    if (wg > 0) {
      GemmParams g = linear_fwd(P, N, wg, d, x, {P.Wcat + wl * d, d, P.Wcat_p.rows(wl)}, P.Y1 + wl, P.Wy, P.bcat + wl);
      if (P.attn_tc) {   // Q | K | V additionally as padded per-head operand planes for the wgmma attention
        g.Cp = P.qkv_p; g.cp_hd = (int)P.hd; g.cp_hd_pad = (int)attention_tc_hd_pad(P.hd);
      }
      GPS_TRY(gemm(g, sg));
    }
    if (wl > 0) GPS_TRY(gemm(linear_fwd(P, N, wl, d, x, {P.Wcat, d, P.Wcat_p}, P.Y1, P.Wy, P.bcat), st));
  }

  // main waits for the edge projection
  if (P.gated || P.pna) GPS_TRY(sd->join(st));

  // ---- local model
  if (P.gated) {
    GPS_TRY(gatedgcn_fwd(a->graph, d, P.Y1, P.Y1 + d, P.Y1 + 2 * d, P.Y1 + 3 * d, P.Wy, P.ehat, P.xt,
                         stats(BN_X), stats(BN_E), st, P.pe_rho));
    // x_loc = x + drop(act(BN(x~)));  e_out = e + drop(act(BN(e^)))   (gatedgcn_layer.py:72-83)
    GPS_TRY(bn_act_residual2(P.xt, a->x, P.xloc, N, bn_view(P, BN_X, a->bn_node_x, N), P.drop(GPS_SITE_GCN_X),
                             stats(BN_L), P.ehat, a->edge_attr, a->edge_out, E, bn_view(P, BN_E, a->bn_edge_e, E),
                             P.drop(GPS_SITE_GCN_E), out_planes(a->e_planes_out), d, act, st));
  } else if (P.gine) {
    GPS_TRY(gine_fwd(a->graph, d, a->x, a->edge_attr, a->gine_eps, P.agg, st, P.agg_p));
    // h1 = act(agg W0^T + b0)
    GemmParams g = linear_fwd(P, N, d, d, {P.agg, d, P.agg_p}, {a->gine_lin0.weight, d, P.g0_p}, P.h1, d,
                              a->gine_lin0.bias);
    g.act = act; g.C_pre = P.h1_pre; g.ldpre = (int)d; g.Cp = P.h1_p;
    GPS_TRY(gemm(g, st));
    // x_loc = x + drop(h1 W1^T + b1)  (gps_layer.py:188-189)
    GemmParams g2 = linear_fwd(P, N, d, d, {P.h1, d, P.h1_p}, {a->gine_lin1.weight, d, P.g1_p}, P.xloc, d,
                               a->gine_lin1.bias);
    g2.R1 = a->x; g2.ldr1 = (int)d; g2.stats = stats(BN_L);
    if (local_writes_s) g2.Cp = P.s_p;
    set_dropout(g2, P.drop(GPS_SITE_LOCAL));
    GPS_TRY(gemm(g2, st));
  } else if (P.gcn) {
    // x_loc = x + drop(GCNConv(x))  (gps_layer.py:49-51,186-189); Y = x W^T is column block 0 of Y1
    GPS_TRY(gcn_dinv(a->graph, P.dinv, st));
    GPS_TRY(gcn_fwd(a->graph, d, P.Y1, P.Wy, P.dinv, a->gcn_conv.bias, a->x, P.xloc, P.drop(GPS_SITE_LOCAL),
                    stats(BN_L), st));
  } else if (P.gat) {
    // x_loc = x + drop(GATConv(x, edge_attr))  (gps_layer.py:70-74,183-189); Y = x W_src^T is column block 0 of Y1
    GPS_TRY(gat_fold_fwd(gat.lin_edge.weight, gat.att_edge, d, P.H, P.gat_v, st));
    GPS_TRY(gat_fwd(a->graph, d, P.H, P.Y1, P.Wy, a->edge_attr, P.gat_v, gat.att_src, gat.att_dst, gat.lin_src.bias,
                    a->x, gat_scores(P.gat_sc, N, E, P.H), P.xloc, P.drop(GPS_SITE_LOCAL), stats(BN_L), st));
  } else if (P.gen) {
    // u = agg + x, agg = softmax aggregation of relu(x_j + e_ij) + 1e-7 over each node's in-edges (GENConv.forward)
    GPS_TRY(genconv_fwd(a->graph, d, a->x, a->edge_attr, P.agg, P.gen_lse, P.gen_u, st, P.gen_u_p));
    // h1 = u W0^T [N, 2d], with mlp.1's column sums in training mode
    GemmParams g = linear_fwd(P, N, 2 * d, d, {P.gen_u, d, P.gen_u_p}, {gen.lin0.weight, d, P.mlp0_p}, P.gen_h1, 2 * d);
    g.stats = P.train ? P.gen_fstats : nullptr;
    GPS_TRY(gemm(g, st));
    // r = relu(mlp.1(h1)) (mlp.2; mlp.3 is Dropout(0))
    GPS_TRY(bn_act_residual(P.gen_h1, 2 * d, nullptr, P.gen_r, N, 2 * d, gen_bn_view(P, gen.bn, N), GPS_ACT_RELU,
                            DropCfg(), nullptr, st, P.gen_r_p));
    // x_loc = x + drop(r W4^T)  (gps_layer.py:188-189)
    GemmParams g2 = linear_fwd(P, N, d, 2 * d, {P.gen_r, 2 * d, P.gen_r_p}, {gen.lin1.weight, 2 * d, P.mlp4_p}, P.xloc,
                               d);
    g2.R1 = a->x; g2.ldr1 = (int)d; g2.stats = stats(BN_L);
    if (local_writes_s) g2.Cp = P.s_p;
    set_dropout(g2, P.drop(GPS_SITE_LOCAL));
    GPS_TRY(gemm(g2, st));
  } else if (P.pna) {
    // Z = [x | mean | max | sum] of m = P_dst[i] + P_src[j] + q[k] (PNAConv.forward, DegreeScalerAggregation); P_dst |
    // P_src is column block 0 of Y1
    GPS_TRY(pna_fwd(a->graph, d, a->x, P.Y1, P.Wy, P.pna_q, P.pna_Z, P.pna_Z_p, P.pna_arg, st));
    // h = Z W_post^T + b_post
    GemmParams g = linear_fwd(P, N, d, 4 * d, {P.pna_Z, 4 * d, P.pna_Z_p}, {pna.post.weight, 4 * d, P.post_p}, P.pna_h,
                              d, pna.post.bias);
    g.Cp = P.pna_h_p;
    GPS_TRY(gemm(g, st));
    // x_loc = x + drop(h W_lin^T + b_lin)  (gps_layer.py:188-189)
    GemmParams g2 = linear_fwd(P, N, d, d, {P.pna_h, d, P.pna_h_p}, {pna.lin.weight, d, P.lin_p}, P.xloc, d,
                               pna.lin.bias);
    g2.R1 = a->x; g2.ldr1 = (int)d; g2.stats = stats(BN_L);
    if (local_writes_s) g2.Cp = P.s_p;
    set_dropout(g2, P.drop(GPS_SITE_LOCAL));
    GPS_TRY(gemm(g2, st));
  }
  // the GatedGCN / GCN / GAT kernels write fp32 only
  if (local_writes_s && !P.gine && !P.gen && !P.pna && P.s_p.hi && N > 0) {
    ToPlanesItem it{P.s, d, (int)N, (int)d, P.s_p};
    GPS_TRY(to_planes(&it, 1, st));
  }

  // ---- global attention  (gps_layer.py:198-218, 234-241)
  if (P.attn) {
    const float* Q = P.Y1 + P.qkv_off;
    if (P.attn_tc)
      GPS_TRY(attention_tc_fwd(a->graph, P.H, P.hd, P.qkv_p, P.O, d, P.O_p, P.lse, P.pa, a->seed, a->offset,
                               (const unsigned long long*)a->offset_dev, P.prec, sg, P.bias));
    else
      GPS_TRY(attention_fwd(a->graph, P.H, P.hd, Q, Q + d, Q + 2 * d, P.Wy, P.O, d, P.lse, P.pa, a->seed, a->offset,
                            sg, (const unsigned long long*)a->offset_dev, P.O_p, P.bias));
    // hA = x + drop(O Wo^T + bo)
    GemmParams g = linear_fwd(P, N, d, d, {P.O, d, P.O_p}, {a->attn_out.weight, d, P.out_p}, P.hA, d, a->attn_out.bias);
    g.R1 = a->x; g.ldr1 = (int)d; g.stats = stats(BN_A);
    set_dropout(g, P.drop(GPS_SITE_ATTN_OUT));
    if (P.nonorm) GPS_TRY(close_with_s(g, sg));
    GPS_TRY(gemm(g, sg));
  }

  // ---- Performer global attention (gps_layer.py:205-206; performer_layer.py:476-503)
  if (P.perf) {
    const int64_t inner = P.inner, NH = N * P.H, dh = a->perf_dim_head;
    const GpsLinear* lin[3] = {&a->perf_q, &a->perf_k, &a->perf_v};
    const Planes wp[3] = {P.pq_p, P.pk_p, P.pv_p};
    float* dst[3] = {P.pQ, P.pK, P.pV};
    for (int i = 0; i < 3; ++i)   // q, k, v = x W^T (no bias)
      GPS_TRY(gemm(linear_fwd(P, N, inner, d, {a->x, d, P.x_p}, {lin[i]->weight, d, wp[i]}, dst[i], inner), sg));
    GPS_TRY(perf_prep(a->perf_proj, P.m, P.pPn, a->graph, P.H, P.pnmax, P.pgmax, P.pargk, sg));
    float* ddst[2] = {P.pfq, P.pfk};
    for (int i = 0; i < 2; ++i)   // dd = (x dn) P^T for every (node, head) row
      GPS_TRY(gemm(linear_fwd(P, NH, P.mp, dh, {dst[i], dh}, {P.pPn, dh}, ddst[i], P.mp), sg));
    GPS_TRY(perf_features_fwd(P.pfq, P.pfk, P.pQ, P.pK, a->graph, P.H, P.m, P.pgmax, P.pargq, P.pargk, sg));
    if (P.perf_pairwise)
      GPS_TRY(perf_quad_fwd(a->graph, P.H, P.m, P.pnmax, P.pfq, P.pfk, P.pV, P.pgmax, P.O, P.pden, sg));
    else
      GPS_TRY(perf_linattn_fwd(a->graph, P.H, P.m, P.pnmax, P.pfq, P.pfk, P.pV, P.pgmax, P.O, sg));
    // hA = x + drop(to_out(O))
    GemmParams g = linear_fwd(P, N, d, inner, {P.O, inner}, {a->attn_out.weight, inner}, P.hA, d, a->attn_out.bias);
    g.R1 = a->x; g.ldr1 = (int)d; g.stats = stats(BN_A);
    // SelfAttention ends with dropout(p = attn_dropout) on to_out(O) (performer_layer.py:501-503, built with
    // dropout=self.attn_dropout at gps_layer.py:112-114); GPSLayer.dropout_attn (p = dropout) follows (:212)
    set_dropout(g, P.drop(GPS_SITE_ATTN_OUT));
    g.p_drop2 = P.pa; g.site2 = GPS_SITE_PERF_OUT;
    if (P.nonorm) GPS_TRY(close_with_s(g, sg));
    GPS_TRY(gemm(g, sg));
  }

  // ---- BigBird global model (gps_layer.py:207-208; bigbird_layer.py:1116-1356)
  if (P.bb) {
    const GpsBigBird& B = a->bigbird;
    const float* Q = P.Y1 + P.qkv_off;
    GPS_TRY(bb_attn_fwd(a->graph, P.H, P.hd, B, Q, Q + d, Q + 2 * d, P.Wy, P.O, d, P.lse, sg));
    if (P.O_p.hi && N > 0) {
      ToPlanesItem it{P.O, d, (int)N, (int)d, P.O_p};
      GPS_TRY(to_planes(&it, 1, sg));
    }
    // z1 = drop(ctx Wso^T + bso) + x   (BigBirdSelfOutput)
    GemmParams g = linear_fwd(P, N, d, d, {P.O, d, P.O_p}, {B.self_out.weight, d, P.bb_so_p}, P.bb_z1, d,
                              B.self_out.bias);
    g.R1 = a->x; g.ldr1 = (int)d;
    set_dropout(g, P.drop(GPS_SITE_BB_SELF_OUT));
    GPS_TRY(gemm(g, sg));
    float* stat = P.bb_stat;
    GPS_TRY(layernorm_fwd(P.bb_z1, N, d, B.ln1.weight, B.ln1.bias, B.ln_eps, stat, stat + N, P.bb_a, P.bb_a_p, nullptr,
                          nullptr, DropCfg(), nullptr, sg));
    // u = act(a Wi^T + bi)   (BigBirdIntermediate)
    const bool relu = B.hidden_act == GPS_BIGBIRD_RELU;
    GemmParams g2 = linear_fwd(P, N, d, d, {P.bb_a, d, P.bb_a_p}, {B.intermediate.weight, d, P.bb_in_p}, P.bb_u, d,
                               B.intermediate.bias);
    if (relu) {
      g2.act = GPS_ACT_RELU; g2.Cp = P.bb_u_p;
    }
    GPS_TRY(gemm(g2, sg));
    if (!relu) GPS_TRY(sigmoid_fwd(P.bb_u, N, d, P.bb_u_p, sg));
    // z2 = drop(u Wo^T + bo) + a   (BigBirdOutput)
    GemmParams g3 = linear_fwd(P, N, d, d, {P.bb_u, d, P.bb_u_p}, {B.output.weight, d, P.bb_out_p}, P.bb_z2, d,
                               B.output.bias);
    g3.R1 = P.bb_a; g3.ldr1 = (int)d;
    set_dropout(g3, P.drop(GPS_SITE_BB_OUTPUT));
    GPS_TRY(gemm(g3, sg));
    // hA = x + drop(LN2(z2)) with norm1_attn's column sums; GPS_NORM_NONE: s = x + drop(LN2(z2)) [+ x_loc] with planes
    float* dst = P.hA;
    Planes dstp;
    const float* r2 = nullptr;
    if (P.nonorm) {
      dst = P.s; dstp = P.s_p;
      if (two_branches) {
        r2 = P.xloc;
        GPS_TRY(sd->order(st, sg));
      }
    }
    GPS_TRY(layernorm_fwd(P.bb_z2, N, d, B.ln2.weight, B.ln2.bias, B.ln_eps, stat + 2 * N, stat + 3 * N, dst, dstp, a->x,
                          r2, P.drop(GPS_SITE_ATTN_OUT), stats(BN_A), sg));
  }

  if (two_branches) GPS_TRY(sd->order(sd->s3, st));

  // ---- s = norm1_local(x_loc) + norm1_attn(hA)   (gps_layer.py:194,217,222)
  if (!P.nonorm) {
    const float* first = P.loc ? P.xloc : P.hA;
    BnView bf = P.loc ? bn_view(P, BN_L, a->norm1_local, N) : bn_view(P, BN_A, a->norm1_attn, N);
    const float* second = (P.loc && P.glob) ? P.hA : nullptr;
    BnView bs = bn_view(P, BN_A, a->norm1_attn, N);
    GPS_TRY(bn_combine(first, bf, second, bs, P.s, N, d, st, P.s_p));
  }

  // ---- FFN: t = s + drop(W2 drop(act(W1 s + b1)) + b2)   (gps_layer.py:225, 253-257)
  {
    GemmParams g = linear_fwd(P, N, 2 * d, d, {P.s, d, P.s_p}, {a->ff1.weight, d, P.ff1_p}, P.hid, 2 * d, a->ff1.bias);
    g.act = act; g.C_pre = P.hid_pre; g.ldpre = (int)(2 * d); g.Cp = P.hid_p;
    set_dropout(g, P.drop(GPS_SITE_FF1));
    GPS_TRY(gemm(g, st));
    GemmParams g2 = linear_fwd(P, N, d, 2 * d, {P.hid, 2 * d, P.hid_p}, {a->ff2.weight, 2 * d, P.ff2_p}, P.t, d,
                               a->ff2.bias);
    g2.R1 = P.s; g2.ldr1 = (int)d; g2.stats = stats(BN_2);
    set_dropout(g2, P.drop(GPS_SITE_FF2));
    if (P.nonorm) {   // x_out = t (no norm2)
      g2.C = a->x_out;
      g2.Cp = out_planes(a->x_planes_out);
    }
    GPS_TRY(gemm(g2, st));
    if (!P.nonorm)
      GPS_TRY(bn_combine(P.t, bn_view(P, BN_2, a->norm2, N), nullptr, BnView(), a->x_out, N, d, st,
                         out_planes(a->x_planes_out)));  // :229
  }
  return GPS_OK;
}

// =================================================================================== backward
static int layer_backward(const GpsLayerArgs* a, cudaStream_t st) {
  Plan P;
  const GpsGat& gat = a->gat;   // the local model's parameters: read when local_type selects it
  const GpsGenConv& gen = a->genconv;
  const GpsPna& pna = a->pna;
  GPS_TRY(make_plan(a, &P, true));
  GPS_REQUIRE(a->saved && a->workspace, GPS_ERR_ARG, "saved/workspace buffers are required");
  GPS_REQUIRE(a->workspace_bytes >= P.bwd_bytes, GPS_ERR_ARG, "workspace too small (%lld < %lld)",
              (long long)a->workspace_bytes, (long long)P.bwd_bytes);
  GPS_TRY(check_params(a, P));
  GPS_REQUIRE(a->grad_x_out && a->grad_x, GPS_ERR_ARG, "grad_x_out / grad_x are required");
  GPS_REQUIRE(!P.gat || P.E == 0 || a->grad_edge_attr, GPS_ERR_ARG, "grad_edge_attr is required for GAT");
  GPS_REQUIRE(!P.gen || P.E == 0 || a->grad_edge_attr, GPS_ERR_ARG, "grad_edge_attr is required for GENConv");
  GPS_REQUIRE(!P.pna || P.E == 0 || a->grad_edge_attr, GPS_ERR_ARG, "grad_edge_attr is required for PNA");
  const int64_t N = P.N, E = P.E, d = P.d;
  const int act = a->act;
  DropCfg nodrop;
  auto sums = [&](int which) { return P.bsums + (int64_t)which * 2 * d; };
  GPS_CUDA(cudaMemsetAsync(P.bsums, 0, (size_t)P.nbn * 2 * d * sizeof(double), st));
  if (P.gen) GPS_CUDA(cudaMemsetAsync(P.gen_bsums, 0, (size_t)2 * 2 * d * sizeof(double), st));
  // weight-gradient GEMMs run on the side stream, each forked where its operands become final
  Side* sd;
  GPS_TRY(side_stream(&sd));
  cudaStream_t s2 = sd->s;
  auto wfork = [&](cudaStream_t from) -> int { return sd->order(from, s2); };
  const bool two_branches = P.loc && P.glob;
  cudaStream_t sa = two_branches ? sd->s3 : st;   // stream of the attention-branch backward
  cudaStream_t se = sd->s4;                       // stream of the edge BatchNorm backward (GatedGCN)
  // data-parallel hook: the caller's event is recorded on the weight-gradient stream once the early gradient group
  // (FFN, attention output projection, norm2 / norm1_local / norm1_attn) has been enqueued there
  // (recorded as EXTERNAL events under stream capture, so that collectives enqueued outside the captured graph can wait
  // on them after each replay: NCCL kernels inside a graph cost ~0.5 ms of host time per launch on this stack)
  auto record_ev = [&](void* ev, cudaStream_t s) -> int {
    if (!ev) return GPS_OK;
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    GPS_CUDA(cudaStreamIsCapturing(s, &cs));
    GPS_CUDA(cudaEventRecordWithFlags((cudaEvent_t)ev, s, cs == cudaStreamCaptureStatusActive ? cudaEventRecordExternal
                                                                                               : cudaEventRecordDefault));
    return GPS_OK;
  };
  auto early_done = [&]() -> int { return record_ev(a->ev_grads_early, s2); };
  auto mid_done = [&]() -> int { return record_ev(a->ev_grads_mid, s2); };   // after the local model's weight gradients
  // the accumulator of dWcat is zeroed now, while its stream is idle, instead of on the tail
  if (P.Wy) {
    GPS_TRY(wfork(st));
    GPS_CUDA(cudaMemsetAsync(P.gWcat, 0, (size_t)(P.Wy * d + P.Wy) * sizeof(float), s2));
  }

  // e_out = e + drop(act(BN_e(e^))) (gatedgcn_layer.py:76-83): g_e^ needs grad_edge_out alone -> off the critical path
  if (P.gated) {
    GPS_TRY(sd->order(st, se));
    BnView ve = bn_view(P, BN_E, a->bn_edge_e);
    if (a->grad_edge_out && E > 0) {
      GPS_TRY(bn_bwd_reduce(a->grad_edge_out, d, P.ehat, d, E, d, ve, act, P.drop(GPS_SITE_GCN_E), sums(BN_E), se));
      GPS_TRY(bn_bwd_apply(a->grad_edge_out, d, P.ehat, d, E, d, ve, act, P.drop(GPS_SITE_GCN_E), sums(BN_E), P.g_e, d,
                           a->bn_edge_e.grad_weight, a->bn_edge_e.grad_bias, se, P.grads_accumulate));
    } else {
      if (E > 0) GPS_CUDA(cudaMemsetAsync(P.g_e, 0, (size_t)(E * d) * sizeof(float), se));
      if (a->bn_edge_e.grad_weight && !P.grads_prezeroed)
        GPS_CUDA(cudaMemsetAsync(a->bn_edge_e.grad_weight, 0, d * sizeof(float), se));
      if (a->bn_edge_e.grad_bias && !P.grads_prezeroed)
        GPS_CUDA(cudaMemsetAsync(a->bn_edge_e.grad_bias, 0, d * sizeof(float), se));
    }
  }

  // ---- norm2 (gps_layer.py:229): g_t.  GPS_NORM_NONE: g_t = grad_x_out, whose planes the FF2 products read unless
  // the dropout in front of them writes its own
  const float* g_t = P.nonorm ? a->grad_x_out : P.g_t;
  if (!P.nonorm) {
    BnView v2 = bn_view(P, BN_2, a->norm2);
    GPS_TRY(bn_bwd_reduce(a->grad_x_out, d, P.t, d, N, d, v2, -1, nodrop, sums(BN_2), st));
    GPS_TRY(bn_bwd_apply(a->grad_x_out, d, P.t, d, N, d, v2, -1, nodrop, sums(BN_2), P.g_t, d, a->norm2.grad_weight,
                         a->norm2.grad_bias, st, P.grads_accumulate, P.gt_p));
  } else if (!(P.dropout.p > 0.f) && P.gt_p.hi && N > 0) {
    ToPlanesItem it{g_t, d, (int)N, (int)d, P.gt_p};
    GPS_TRY(to_planes(&it, 1, st));
  }
  // upstream gradients of x_loc and hA: norm1_local's / norm1_attn's input gradients, or g_s itself without them
  const float* g_xloc = P.nonorm ? P.g_s : P.g_xloc;
  const Planes g_xloc_p = P.nonorm ? P.gs_p : P.gl1_p;
  const float* g_hA = P.nonorm ? P.g_s : P.g_hA;
  const Planes g_hA_p = P.nonorm ? P.gs_p : P.ghA_p;

  // ---- FFN (gps_layer.py:253-257)
  {
    Operand g_ff2;   // gradient at the output of ff_linear2 (after ff_dropout2)
    GPS_TRY(dropmul(P, {g_t, d, P.gt_p}, P.g_tmp, P.gtmp_p, GPS_SITE_FF2, st, &g_ff2));
    // g_hid = (g_ff2 W2) * act'(pre) * drop1
    GemmParams g = linear_dgrad(P, N, 2 * d, d, g_ff2, {a->ff2.weight, 2 * d, P.ff2_p}, P.g_hid, 2 * d);
    set_act_mask(g, act, P.hid, P.hid_pre, 2 * d);
    set_dropout(g, P.drop(GPS_SITE_FF1));
    g.Cp = P.ghid_p;
    GPS_TRY(gemm(g, st));
    const Operand g_hid{P.g_hid, 2 * d, P.ghid_p};
    GPS_TRY(wfork(st));
    GPS_TRY(linear_wgrad(P, g_ff2, {P.hid, 2 * d, P.hid_p}, N, d, 2 * d, a->ff2.grad_weight, a->ff2.grad_bias, s2));
    GPS_TRY(linear_wgrad(P, g_hid, {P.s, d, P.s_p}, N, 2 * d, d, a->ff1.grad_weight, a->ff1.grad_bias, s2));
    // g_s = g_t + g_hid W1
    GemmParams g2 = linear_dgrad(P, N, d, 2 * d, g_hid, {a->ff1.weight, d, P.ff1_p}, P.g_s, d);
    g2.R1 = g_t; g2.ldr1 = (int)d;
    g2.Cp = P.gs_p;   // GPS_NORM_NONE only: the branches' products read g_s
    GPS_TRY(gemm(g2, st));
  }
  // the attention-branch backward needs g_s (and hA) only: it forks here and runs next to norm1_local's backward and
  // the local-model backward
  if (two_branches) GPS_TRY(sd->order(st, sa));

  // ---- norm1_local / norm1_attn (gps_layer.py:194,217): g_xloc, g_hA
  if (P.loc && !P.nonorm) {
    BnView v = bn_view(P, BN_L, a->norm1_local);
    GPS_TRY(bn_bwd_reduce(P.g_s, d, P.xloc, d, N, d, v, -1, nodrop, sums(BN_L), st));
    GPS_TRY(bn_bwd_apply(P.g_s, d, P.xloc, d, N, d, v, -1, nodrop, sums(BN_L), P.g_xloc, d,
                         a->norm1_local.grad_weight, a->norm1_local.grad_bias, st, P.grads_accumulate, P.gl1_p));
  }
  // norm1_local's gradients belong to the early group: the weight-gradient stream takes them in before the attention
  // branch (forked before them) records the group's event there; with no global model the group ends here
  const bool glob_model = P.attn || P.perf || P.bb;
  if (!glob_model || (P.loc && !P.nonorm)) GPS_TRY(wfork(st));
  if (!glob_model) GPS_TRY(early_done());
  if (P.attn) {
    if (!P.nonorm) {
      BnView v = bn_view(P, BN_A, a->norm1_attn);
      GPS_TRY(bn_bwd_reduce(P.g_s, d, P.hA, d, N, d, v, -1, nodrop, sums(BN_A), sa));
      GPS_TRY(bn_bwd_apply(P.g_s, d, P.hA, d, N, d, v, -1, nodrop, sums(BN_A), P.g_hA, d, a->norm1_attn.grad_weight,
                           a->norm1_attn.grad_bias, sa, P.grads_accumulate, P.ghA_p));
    }
    // hA = x + drop(O Wo^T + bo)
    Operand g_ao;
    GPS_TRY(dropmul(P, {g_hA, d, g_hA_p}, P.g_tmp2, P.gtmp2_p, GPS_SITE_ATTN_OUT, sa, &g_ao));
    // g_O = g_ao Wo
    GPS_TRY(gemm(linear_dgrad(P, N, d, d, g_ao, {a->attn_out.weight, d, P.out_p}, P.g_O, d), sa));
    GPS_TRY(wfork(sa));
    GPS_TRY(linear_wgrad(P, g_ao, {P.O, d, P.O_p}, N, d, d, a->attn_out.grad_weight, a->attn_out.grad_bias, s2));
    GPS_TRY(early_done());
    const float* Q = P.Y1 + P.qkv_off;
    float* gQ = P.gY1 + P.qkv_off;
    GPS_TRY(attention_bwd(a->graph, P.H, P.hd, Q, Q + d, Q + 2 * d, P.Wy, P.O, P.g_O, d, P.lse, P.delta, gQ, gQ + d,
                          gQ + 2 * d, P.Wy, P.pa, a->seed, a->offset, sa, (const unsigned long long*)a->offset_dev,
                          P.gY1_p.cols(P.qkv_off), P.gY1_p.cols(P.qkv_off + d), P.gY1_p.cols(P.qkv_off + 2 * d), P.bias));
  }

  if (P.perf) {
    const int64_t inner = P.inner, NH = N * P.H, dh = a->perf_dim_head;
    if (!P.nonorm) {
      BnView v = bn_view(P, BN_A, a->norm1_attn);
      GPS_TRY(bn_bwd_reduce(P.g_s, d, P.hA, d, N, d, v, -1, nodrop, sums(BN_A), sa));
      GPS_TRY(bn_bwd_apply(P.g_s, d, P.hA, d, N, d, v, -1, nodrop, sums(BN_A), P.g_hA, d, a->norm1_attn.grad_weight,
                           a->norm1_attn.grad_bias, sa, P.grads_accumulate));
    }
    Operand g_ao;   // hA = x + drop_pd(drop_pa(to_out(O)))
    GPS_TRY(dropmul(P, {g_hA, d}, P.g_tmp2, Planes(), GPS_SITE_ATTN_OUT, sa, &g_ao, P.pa, GPS_SITE_PERF_OUT));
    // g_O = g_ao Wout   [N, inner]
    GPS_TRY(gemm(linear_dgrad(P, N, inner, d, g_ao, {a->attn_out.weight, inner}, P.g_O, inner), sa));
    GPS_TRY(wfork(sa));
    GPS_TRY(linear_wgrad(P, g_ao, {P.O, inner}, N, d, inner, a->attn_out.grad_weight, a->attn_out.grad_bias, s2));
    GPS_TRY(early_done());
    // linear attention and feature maps (performer_layer.py:200-205, 119-144)
    if (P.perf_pairwise)
      GPS_TRY(perf_quad_bwd(a->graph, P.H, P.m, P.pnmax, P.pfq, P.pfk, P.pV, P.pgmax, P.O, P.pden, P.g_O, P.g_pden,
                            P.g_pfq, P.g_pfk, P.g_pV, P.g_pgrow, sa));
    else
      GPS_TRY(perf_linattn_bwd(a->graph, P.H, P.m, P.pnmax, P.pfq, P.pfk, P.pV, P.pgmax, P.g_O, P.g_pfq, P.g_pfk, P.g_pV,
                               P.g_pgmax, sa));
    GPS_TRY(perf_features_bwd(P.g_pfq, P.g_pfk, P.pfq, P.pfk, P.pQ, P.pK, P.g_pQ, P.g_pK, a->graph, P.H, P.m, P.pargq,
                              P.pargk, P.g_pgmax, P.g_pgrow, P.perf_pairwise, sa));
    float* gdd[2] = {P.g_pfq, P.g_pfk};
    float* gqk[2] = {P.g_pQ, P.g_pK};
    for (int i = 0; i < 2; ++i) {   // g_q += g_dd Pn   (dd = q Pn^T)
      GemmParams h = linear_dgrad(P, NH, dh, P.mp, {gdd[i], P.mp}, {P.pPn, dh}, gqk[i], dh);
      h.R1 = gqk[i]; h.ldr1 = (int)dh;
      GPS_TRY(gemm(h, sa));
    }
    // projections: dW = g^T x ;  g_xp = g_hA + gQ Wq + gK Wk + gV Wv
    const GpsLinear* lin[3] = {&a->perf_q, &a->perf_k, &a->perf_v};
    const float* gsrc[3] = {P.g_pQ, P.g_pK, P.g_pV};
    GPS_TRY(wfork(sa));
    for (int i = 0; i < 3; ++i) {
      GPS_TRY(linear_wgrad(P, {gsrc[i], inner}, {a->x, d}, N, inner, d, lin[i]->grad_weight, nullptr, s2));
      GemmParams h = linear_dgrad(P, N, d, inner, {gsrc[i], inner}, {lin[i]->weight, d}, P.g_xp, d);
      h.R1 = i == 0 ? g_hA : P.g_xp; h.ldr1 = (int)d;
      GPS_TRY(gemm(h, sa));
    }
  }

  if (P.bb) {
    const GpsBigBird& B = a->bigbird;
    if (!P.nonorm) {
      BnView v = bn_view(P, BN_A, a->norm1_attn);
      GPS_TRY(bn_bwd_reduce(P.g_s, d, P.hA, d, N, d, v, -1, nodrop, sums(BN_A), sa));
      GPS_TRY(bn_bwd_apply(P.g_s, d, P.hA, d, N, d, v, -1, nodrop, sums(BN_A), P.g_hA, d, a->norm1_attn.grad_weight,
                           a->norm1_attn.grad_bias, sa, P.grads_accumulate));
    }
    GPS_TRY(wfork(sa));
    GPS_TRY(early_done());
    const float* stat = P.bb_stat;
    // LN2 from g' = drop(g_hA): dz2 (the residual path into a) and g_od = drop(dz2), the gradient of output.dense
    GPS_TRY(layernorm_bwd(g_hA, P.drop(GPS_SITE_ATTN_OUT), P.bb_z2, N, d, B.ln2.weight, stat + 2 * N, stat + 3 * N,
                          P.bb_god, P.bb_god_p, P.drop(GPS_SITE_BB_OUTPUT), P.bb_dz2, nullptr, P.bb_part,
                          B.ln2.grad_weight, B.ln2.grad_bias, P.grads_accumulate, sa));
    // output.dense: g_u = (g_od Wo) * act'(u)
    const bool relu = B.hidden_act == GPS_BIGBIRD_RELU;
    const Operand g_od{P.bb_god, d, P.bb_god_p}, g_u{P.bb_gu, d, P.bb_gu_p};
    GemmParams g = linear_dgrad(P, N, d, d, g_od, {B.output.weight, d, P.bb_out_p}, P.bb_gu, d);
    if (relu) {
      set_act_mask(g, GPS_ACT_RELU, P.bb_u, nullptr, d);
      g.Cp = P.bb_gu_p;
    }
    GPS_TRY(gemm(g, sa));
    if (!relu) GPS_TRY(sigmoid_bwd(P.bb_gu, P.bb_u, N, d, P.bb_gu_p, sa));
    GPS_TRY(wfork(sa));
    GPS_TRY(linear_wgrad(P, g_od, {P.bb_u, d, P.bb_u_p}, N, d, d, B.output.grad_weight, B.output.grad_bias, s2));
    GPS_TRY(linear_wgrad(P, g_u, {P.bb_a, d, P.bb_a_p}, N, d, d, B.intermediate.grad_weight, B.intermediate.grad_bias,
                         s2));
    // intermediate.dense: g_a = g_u Wi + dz2
    GemmParams g2 = linear_dgrad(P, N, d, d, g_u, {B.intermediate.weight, d, P.bb_in_p}, P.bb_ga, d);
    g2.R1 = P.bb_dz2; g2.ldr1 = (int)d;
    GPS_TRY(gemm(g2, sa));
    // LN1: g_so = drop(dz1), the gradient of attention.output.dense; dz1 + g_hA is BigBird's share of grad_x
    GPS_TRY(layernorm_bwd(P.bb_ga, nodrop, P.bb_z1, N, d, B.ln1.weight, stat, stat + N, P.bb_gso, P.bb_gso_p,
                          P.drop(GPS_SITE_BB_SELF_OUT), P.bb_gx, g_hA, P.bb_part, B.ln1.grad_weight, B.ln1.grad_bias,
                          P.grads_accumulate, sa));
    const Operand g_so{P.bb_gso, d, P.bb_gso_p};
    GPS_TRY(gemm(linear_dgrad(P, N, d, d, g_so, {B.self_out.weight, d, P.bb_so_p}, P.g_O, d), sa));
    GPS_TRY(wfork(sa));   // the LayerNorm gradients are final here too
    GPS_TRY(linear_wgrad(P, g_so, {P.O, d, P.O_p}, N, d, d, B.self_out.grad_weight, B.self_out.grad_bias, s2));
    if (!P.loc) GPS_TRY(mid_done());
    // block-sparse attention: dQ | dK | dV into the in_proj columns of gY1
    const float* Q = P.Y1 + P.qkv_off;
    float* gQ = P.gY1 + P.qkv_off;
    GPS_TRY(bb_attn_bwd(a->graph, P.H, P.hd, B, Q, Q + d, Q + 2 * d, P.Wy, P.O, P.g_O, d, P.lse, P.delta, gQ, gQ + d,
                        gQ + 2 * d, P.Wy, sa));
    if (P.gY1_p.hi && N > 0) {
      ToPlanesItem it{gQ, P.Wy, (int)N, (int)(3 * d), P.gY1_p.cols(P.qkv_off)};
      GPS_TRY(to_planes(&it, 1, sa));
    }
  }

  // ---- local model backward
  const float* g_x_local = nullptr;  // direct gradient paths into x besides the projections
  if (P.gated) {
    // x_loc = x + drop(act(BN_x(x~))): g_x~ -> gY1[:, 0:d]  (gatedgcn_layer.py:72-83)
    BnView vx = bn_view(P, BN_X, a->bn_node_x);
    GPS_TRY(bn_bwd_reduce(g_xloc, d, P.xt, d, N, d, vx, act, P.drop(GPS_SITE_GCN_X), sums(BN_X), st));
    GPS_TRY(bn_bwd_apply(g_xloc, d, P.xt, d, N, d, vx, act, P.drop(GPS_SITE_GCN_X), sums(BN_X), P.gY1, P.Wy,
                         a->bn_node_x.grad_weight, a->bn_node_x.grad_bias, st, P.grads_accumulate, P.gY1_p));
    GPS_TRY(sd->order(se, st));
    // message/aggregate backward (SURVEY Appendix C)
    GPS_TRY(gatedgcn_bwd_dst(a->graph, d, P.gY1, P.Wy, P.ehat, P.Y1 + d, P.Wy, P.g_e, P.g_num, P.gY1 + 2 * d, st, P.ge_p,
                             P.gY1_p.cols(2 * d), P.pe_rho, P.g_den));
    // g_e, g_num and g_den are final here.  The EquivStableLapPE gate's mlp_r_ij gradients (mid group) and grad_pe need
    // g_num / g_den only, so they run on the (by now idle) edge-BatchNorm stream next to the src-ordered pass and the
    // weight gradients
    GPS_TRY(sd->order(st, se));
    if (P.eslap) {
      GPS_TRY(eslap_bwd(a->graph, a->pe, a->pe_dim, d, act, P.g_num, P.g_den, P.Y1 + d, P.Wy, P.ehat, P.pe_r, P.pe_rho,
                        a->pe_mlp0.weight, a->pe_mlp0.bias, a->pe_mlp1.weight, P.pe_gz, P.pe_gr, P.pe_part, a->grad_pe,
                        a->pe_mlp0.grad_weight, a->pe_mlp0.grad_bias, a->pe_mlp1.grad_weight, a->pe_mlp1.grad_bias,
                        P.grads_accumulate, se));
    }
    GPS_TRY(gatedgcn_bwd_src(a->graph, d, P.g_e, P.ehat, P.g_num, P.gY1 + 3 * d, P.gY1 + d, P.Wy, st, P.gY1_p.cols(3 * d),
                             P.gY1_p.cols(d), P.pe_rho));
    // C: dC = g_e^T e ; g_edge_attr = grad_edge_out + g_e C
    const Operand g_e{P.g_e, d, P.ge_p};
    GPS_TRY(wfork(st));
    GPS_TRY(linear_wgrad(P, g_e, {a->edge_attr, d, P.e_p}, E, d, d, a->gcn_C.grad_weight, a->gcn_C.grad_bias, s2));
    if (P.eslap) GPS_TRY(sd->order(se, s2));   // the mlp_r_ij gradients are final at ev_grads_mid; grad_pe joins at the end
    GPS_TRY(mid_done());
    // an output only: on the edge stream (after the gate's backward there), off the local branch and the weight-gradient
    // chain; joined at the end
    if (a->grad_edge_attr && E > 0) {
      GemmParams g = linear_dgrad(P, E, d, d, g_e, {a->gcn_C.weight, d, P.C_p}, a->grad_edge_attr, d);
      g.R1 = a->grad_edge_out; g.ldr1 = (int)d;
      GPS_TRY(gemm(g, se));
    }
    g_x_local = g_xloc;  // residual x_in + ...
  } else if (P.gine) {
    // x_loc = x + drop(h1 W1^T + b1)
    Operand g_l1;
    GPS_TRY(dropmul(P, {g_xloc, d, g_xloc_p}, P.g_tmp3, P.gtmp3_p, GPS_SITE_LOCAL, st, &g_l1));
    // g_h1 = (g_l1 W1) * act'(pre)
    GemmParams g = linear_dgrad(P, N, d, d, g_l1, {a->gine_lin1.weight, d, P.g1_p}, P.g_h1, d);
    set_act_mask(g, act, P.h1, P.h1_pre, d);
    g.Cp = P.gh1_p;
    GPS_TRY(gemm(g, st));
    const Operand g_h1{P.g_h1, d, P.gh1_p};
    GPS_TRY(wfork(st));
    GPS_TRY(linear_wgrad(P, g_l1, {P.h1, d, P.h1_p}, N, d, d, a->gine_lin1.grad_weight, a->gine_lin1.grad_bias, s2));
    GPS_TRY(linear_wgrad(P, g_h1, {P.agg, d, P.agg_p}, N, d, d, a->gine_lin0.grad_weight, a->gine_lin0.grad_bias, s2));
    GPS_TRY(mid_done());
    // g_agg = g_h1 W0
    GPS_TRY(gemm(linear_dgrad(P, N, d, d, g_h1, {a->gine_lin0.weight, d, P.g0_p}, P.g_agg, d), st));
    GPS_REQUIRE(a->grad_edge_attr || E == 0, GPS_ERR_ARG, "grad_edge_attr is required for GINE");
    GPS_TRY(gine_bwd_dst(a->graph, d, a->x, a->edge_attr, P.g_agg, a->grad_edge_attr, st));
    GPS_TRY(gine_bwd_src(a->graph, d, a->grad_edge_attr, P.g_agg, a->gine_eps, g_xloc, P.g_xl, st));
    g_x_local = P.g_xl;
  } else if (P.gcn) {
    // x_loc = x + drop(b + A_hat Y): g_h = drop * g_xloc; g_b = colsum(g_h); gY = A_hat^T g_h -> gY1[:, 0:d]
    Operand g_h;
    GPS_TRY(dropmul(P, {g_xloc, d}, P.g_tmp3, Planes(), GPS_SITE_LOCAL, st, &g_h));
    if (a->gcn_conv.grad_bias) {
      if (!P.grads_prezeroed) GPS_CUDA(cudaMemsetAsync(a->gcn_conv.grad_bias, 0, (size_t)d * sizeof(float), st));
      GPS_TRY(colsum(g_h.f, d, N, d, a->gcn_conv.grad_bias, st));
    }
    GPS_TRY(gcn_bwd(a->graph, d, g_h.f, P.dinv, P.gY1, P.Wy, st, P.gY1_p));
    GPS_TRY(wfork(st));
    GPS_TRY(mid_done());
    g_x_local = g_xloc;
  } else if (P.gat) {
    // x_loc = x + drop(GATConv(x) + b): g_h = drop * g_xloc -> gY1[:, 0:d], grad_edge_attr, att_* / bias / lin_edge
    Operand g_h;
    GPS_TRY(dropmul(P, {g_xloc, d}, P.g_tmp3, Planes(), GPS_SITE_LOCAL, st, &g_h));
    float* g_v = P.gat_ws;
    GPS_TRY(gat_bwd(a->graph, d, P.H, P.Y1, P.Wy, a->edge_attr, P.gat_v, gat.att_src, gat.att_dst,
                    gat_scores(P.gat_sc, N, E, P.H), g_h.f, P.gat_ws + P.H * d, P.gY1, P.Wy, P.gY1_p, a->grad_edge_attr,
                    g_v, gat.grad_att_src, gat.grad_att_dst, gat.lin_src.grad_bias, P.grads_accumulate, st));
    GPS_TRY(gat_fold_bwd(gat.lin_edge.weight, gat.att_edge, g_v, d, P.H, gat.lin_edge.grad_weight, gat.grad_att_edge,
                         P.grads_accumulate, st));
    GPS_TRY(wfork(st));
    GPS_TRY(mid_done());
    g_x_local = g_xloc;
  } else if (P.gen) {
    // x_loc = x + drop(r W4^T)
    Operand g_l;
    GPS_TRY(dropmul(P, {g_xloc, d, g_xloc_p}, P.g_tmp3, P.gtmp3_p, GPS_SITE_LOCAL, st, &g_l));
    // g_r = g_l W4 [N, 2d]
    GPS_TRY(gemm(linear_dgrad(P, N, 2 * d, d, g_l, {gen.lin1.weight, 2 * d, P.mlp4_p}, P.gen_gr, 2 * d), st));
    // r = relu(mlp.1(h1)): g_h1 and the mlp.1 gradients
    const BnView vb = gen_bn_view(P, gen.bn);
    GPS_TRY(bn_bwd_reduce(P.gen_gr, 2 * d, P.gen_h1, 2 * d, N, 2 * d, vb, GPS_ACT_RELU, nodrop, P.gen_bsums, st));
    GPS_TRY(bn_bwd_apply(P.gen_gr, 2 * d, P.gen_h1, 2 * d, N, 2 * d, vb, GPS_ACT_RELU, nodrop, P.gen_bsums, P.gen_gh1,
                         2 * d, gen.bn.grad_weight, gen.bn.grad_bias, st, P.grads_accumulate, P.gen_gh1_p));
    const Operand g_h1{P.gen_gh1, 2 * d, P.gen_gh1_p};
    GPS_TRY(wfork(st));
    GPS_TRY(linear_wgrad(P, g_l, {P.gen_r, 2 * d, P.gen_r_p}, N, d, 2 * d, gen.lin1.grad_weight, nullptr, s2));
    GPS_TRY(linear_wgrad(P, g_h1, {P.gen_u, d, P.gen_u_p}, N, 2 * d, d, gen.lin0.grad_weight, nullptr, s2));
    GPS_TRY(mid_done());
    // g_u = g_h1 W0; then grad_edge_attr (dst ordered) and g_x_local = g_u + sum_out grad_edge_attr + g_xloc
    GPS_TRY(gemm(linear_dgrad(P, N, d, 2 * d, g_h1, {gen.lin0.weight, d, P.mlp0_p}, P.gen_gu, d), st));
    GPS_TRY(genconv_bwd_dst(a->graph, d, a->x, a->edge_attr, P.agg, P.gen_lse, P.gen_gu, a->grad_edge_attr, st));
    GPS_TRY(gine_bwd_src(a->graph, d, a->grad_edge_attr, P.gen_gu, 0.f, g_xloc, P.g_xl, st));
    g_x_local = P.g_xl;
  } else if (P.pna) {
    // x_loc = x + drop(h W_lin^T + b_lin), h = Z W_post^T + b_post
    Operand g_l;
    GPS_TRY(dropmul(P, {g_xloc, d, g_xloc_p}, P.g_tmp3, P.gtmp3_p, GPS_SITE_LOCAL, st, &g_l));
    // g_h = g_l W_lin
    GemmParams g = linear_dgrad(P, N, d, d, g_l, {pna.lin.weight, d, P.lin_p}, P.pna_gh, d);
    g.Cp = P.pna_gh_p;
    GPS_TRY(gemm(g, st));
    const Operand g_h{P.pna_gh, d, P.pna_gh_p};
    GPS_TRY(wfork(st));
    GPS_TRY(linear_wgrad(P, g_l, {P.pna_h, d, P.pna_h_p}, N, d, d, pna.lin.grad_weight, pna.lin.grad_bias, s2));
    GPS_TRY(linear_wgrad(P, g_h, {P.pna_Z, 4 * d, P.pna_Z_p}, N, d, 4 * d, pna.post.grad_weight, pna.post.grad_bias,
                         s2));
    // g_Z = g_h W_post [N, 4d]
    GPS_TRY(gemm(linear_dgrad(P, N, 4 * d, d, g_h, {pna.post.weight, 4 * d, P.post_p}, P.pna_gZ, 4 * d), st));
    // g_q (every edge's g_m), g_P_dst | g_P_src -> gY1[:, 0:2d], g_x_local = g_xloc + g_Z[:, 0:d]
    GPS_TRY(pna_bwd(a->graph, d, P.pna_gZ, P.pna_arg, g_xloc, P.pna_gq, P.pna_gq_p, P.gY1, P.Wy, P.gY1_p, P.g_xl, st));
    // edge term: g_F = g_q^T e, g_c = colsum(g_q), unfolded into edge_encoder, pre's edge block and pre's bias
    const Operand g_q{P.pna_gq, d, P.pna_gq_p};
    float* g_F = P.pna_gF;
    float* g_c = P.pna_gF + d * P.de;
    GPS_TRY(wfork(st));
    GPS_CUDA(cudaMemsetAsync(g_F, 0, (size_t)(d * P.de + d) * sizeof(float), s2));
    GPS_TRY(wgrad_add(P, g_q, {a->edge_attr, P.de, P.e_p}, E, d, P.de, g_F, g_c, s2));
    GPS_TRY(pna_fold_bwd(pna.pre.weight, pna.edge_encoder.weight, pna.edge_encoder.bias, g_F, g_c, d, P.de,
                         pna.pre.grad_weight, pna.pre.grad_bias, pna.edge_encoder.grad_weight,
                         pna.edge_encoder.grad_bias, P.grads_accumulate, s2));
    GPS_TRY(mid_done());
    // grad_edge_attr = g_q F
    if (E > 0)
      GPS_TRY(gemm(linear_dgrad(P, E, P.de, d, g_q, {P.pna_F, P.de, P.pna_F_p}, a->grad_edge_attr, P.de), st));
    g_x_local = P.g_xl;
  }

  if (two_branches) GPS_TRY(sd->order(sa, st));

  // ---- g_x = [local paths] + [attention residual] + gY1 Wcat ;  d{A,B,D,E,in_proj}
  if (P.Wy) {
    const Operand gY1{P.gY1, P.Wy, P.gY1_p};
    GPS_TRY(wfork(st));
    // d Wcat (+ bias gradient) on s2, unpacked into the caller's A, B, D, E / conv / in_proj gradients
    GPS_TRY(wgrad_add(P, gY1, {a->x, d, P.x_p}, N, P.Wy, d, P.gWcat, P.gbcat, s2));
    PackDesc pdsc = pack_desc(P);
    k_unpack<<<(unsigned)P.Wy, 128, 0, s2>>>(pdsc, P.gWcat, P.gbcat, P.grads_accumulate ? 1 : 0);
    GPS_LAUNCH_CHECK();
    GemmParams g = linear_dgrad(P, N, d, P.Wy, gY1, {P.Wcat, d, P.Wcat_p}, a->grad_x, d);
    g.R1 = g_x_local; g.ldr1 = (int)d;
    g.R2 = P.attn ? g_hA : (P.perf ? P.g_xp : (P.bb ? P.bb_gx : nullptr)); g.ldr2 = (int)d;
    // grad_x is written by the product's epilogue, not accumulated into, and the launch policy picks any K-split: at
    // d = 304 none (one CTA per output tile reducing all 7d: 55 us fp32-grade / 33 us bf16, where the 4-way split-K
    // into a zeroed grad_x took 64 / 45 us; H100 SXM, 700 W), and the memset of grad_x goes
    GPS_TRY(gemm(g, st));
  } else if (g_x_local) {
    GPS_TRY(add3(g_x_local, d, P.perf ? P.g_xp : nullptr, d, nullptr, 0, a->grad_x, d, N, d, st));
  } else {
    GPS_TRY(add3(P.g_xp, d, nullptr, 0, nullptr, 0, a->grad_x, d, N, d, st));   // Performer only
  }
  GPS_TRY(sd->join(st));
  if (P.gated) GPS_TRY(sd->order(se, st));   // grad_edge_attr and the gate's grad_pe
  GPS_TRY(record_ev(a->ev_grads_done, st));
  return GPS_OK;
}

}  // namespace gps

// =================================================================================== C ABI
using namespace gps;

extern "C" const char* gps_last_error(void) { return g_err; }
extern "C" int gps_abi_version(void) { return GPS_ABI_VERSION; }
extern "C" const char* gps_build_arch(void) { return "sm_90a"; }
extern "C" unsigned long long gps_launch_count(void) { return g_launches.load(); }
extern "C" unsigned long long gps_fallback_count(void) { return g_fallbacks.load(); }

extern "C" int gps_to_planes(const float* src, int64_t ld, int64_t rows, int64_t cols, void* hi, void* lo, int64_t ldp,
                             void* stream) {
  GPS_REQUIRE(src && hi, GPS_ERR_ARG, "gps_to_planes: null argument");
  ToPlanesItem it{src, ld, (int)rows, (int)cols, Planes{(__nv_bfloat16*)hi, (__nv_bfloat16*)lo, ldp}};
  return to_planes(&it, 1, (cudaStream_t)stream);
}

extern "C" int gps_gemm_planes(const void* A_hi, const void* A_lo, int64_t lda, int32_t ta, const void* B_hi,
                               const void* B_lo, int64_t ldb, int32_t tb, float* C, int64_t ldc, void* C_hi, void* C_lo,
                               int64_t ldcp, int64_t M, int64_t N, int64_t K, int32_t splitk, int32_t precision,
                               float* colsum_a, void* stream) {
  GemmParams g;
  g.M = (int)M; g.N = (int)N; g.K = (int)K;
  g.ta = ta; g.tb = tb; g.C = C; g.ldc = (int)ldc;
  g.Ap = Planes{(__nv_bfloat16*)A_hi, (__nv_bfloat16*)A_lo, lda};
  g.Bp = Planes{(__nv_bfloat16*)B_hi, (__nv_bfloat16*)B_lo, ldb};
  g.Cp = Planes{(__nv_bfloat16*)C_hi, (__nv_bfloat16*)C_lo, ldcp};
  g.splitk = splitk < 1 ? 1 : splitk; g.precision = precision; g.colsum_a = colsum_a;
  int rc = gemm_tma(g, (cudaStream_t)stream);
  if (rc == GPS_ERR_UNSUPPORTED) set_error("gps_gemm_planes: the TMA kernel does not take this shape/alignment");
  return rc;
}
extern "C" int gps_gemm_epilogue(const GpsGemmArgs* a, int32_t impl, void* stream) {
  GPS_REQUIRE(a, GPS_ERR_ARG, "gps_gemm_epilogue: null args");
  const int64_t kMax = 0x7FFFFFFF;
  GPS_REQUIRE(a->M >= 0 && a->N >= 0 && a->K >= 0 && a->M <= kMax && a->N <= kMax && a->K <= kMax, GPS_ERR_ARG,
              "gps_gemm_epilogue: M, N, K must lie in [0, 2^31)");
  GPS_REQUIRE(impl >= 0 && impl <= 3, GPS_ERR_ARG, "gps_gemm_epilogue: impl %d is not 0..3", impl);
  GPS_REQUIRE(a->C || a->Cp.hi, GPS_ERR_ARG, "gps_gemm_epilogue: neither C nor Cp given");
  // the CUDA-core and register-staged kernels read the fp32 operands and write fp32 C only
  GPS_REQUIRE(!(impl == 1 || impl == 2) || !a->Cp.hi, GPS_ERR_ARG,
              "gps_gemm_epilogue: impl %d does not write output planes (Cp)", impl);
  GPS_REQUIRE(!(impl == 1 || impl == 2) || (a->A && a->B), GPS_ERR_ARG,
              "gps_gemm_epilogue: impl %d needs the fp32 operands A and B", impl);
  GemmParams g;
  g.M = (int)a->M; g.N = (int)a->N; g.K = (int)a->K;
  g.A = a->A; g.lda = (int)a->lda; g.ta = a->ta;
  g.B = a->B; g.ldb = (int)a->ldb; g.tb = a->tb;
  g.Ap = Planes{(__nv_bfloat16*)a->Ap.hi, (__nv_bfloat16*)a->Ap.lo, a->Ap.ld};
  g.Bp = Planes{(__nv_bfloat16*)a->Bp.hi, (__nv_bfloat16*)a->Bp.lo, a->Bp.ld};
  g.Cp = Planes{(__nv_bfloat16*)a->Cp.hi, (__nv_bfloat16*)a->Cp.lo, a->Cp.ld};
  g.C = a->C; g.ldc = (int)a->ldc; g.cp_hd = a->cp_hd; g.cp_hd_pad = a->cp_hd_pad;
  g.bias = a->bias; g.C_pre = a->C_pre; g.ldpre = (int)a->ldpre; g.act = a->act;
  g.mask_src = a->mask_src; g.ldmask = (int)a->ldmask; g.mask_act = a->mask_act; g.mask_is_post = a->mask_is_post;
  g.p_drop = a->p_drop; g.site = a->site; g.p_drop2 = a->p_drop2; g.site2 = a->site2;
  g.seed = a->seed; g.offset = a->offset; g.offset_dev = a->offset_dev;
  g.R1 = a->R1; g.ldr1 = (int)a->ldr1; g.R2 = a->R2; g.ldr2 = (int)a->ldr2;
  g.stats = a->stats; g.colsum_a = a->colsum_a; g.splitk = a->splitk < 1 ? 1 : a->splitk; g.precision = a->precision;
  const cudaStream_t st = (cudaStream_t)stream;
  int rc;
  switch (impl) {
    case 1: rc = gemm_simt(g, st); break;
    case 2: rc = gemm_tc(g, st); break;
    case 3: rc = gemm_tma(g, st); break;
    default: return gemm(g, st);
  }
  if (rc == GPS_ERR_UNSUPPORTED)
    set_error("gps_gemm_epilogue: impl %d does not take M=%d N=%d K=%d (ta=%d tb=%d) with these alignments", impl, g.M,
              g.N, g.K, g.ta, g.tb);
  return rc;
}

namespace {
struct StagePlan {   // all bn_view_at reads of a plan
  bool train;
};
}  // namespace

extern "C" int gps_rowwise_stage(const GpsRowwiseArgs* a, int32_t op, void* stream) {
  GPS_REQUIRE(a, GPS_ERR_ARG, "gps_rowwise_stage: null args");
  GPS_REQUIRE(op >= GPS_ROWWISE_BN_ACT_RESIDUAL && op <= GPS_ROWWISE_COLSUM, GPS_ERR_ARG,
              "gps_rowwise_stage: unknown op %d", op);
  const int64_t rows = a->rows, E = a->E, d = a->d;
  GPS_REQUIRE(rows >= 0 && E >= 0 && d >= 0, GPS_ERR_ARG, "gps_rowwise_stage: negative size (rows %lld, E %lld, d %lld)",
              (long long)rows, (long long)E, (long long)d);
  const bool bwd = op == GPS_ROWWISE_BN_BWD_REDUCE || op == GPS_ROWWISE_BN_BWD_APPLY;
  const int64_t ldx = a->ldx ? a->ldx : d, ldg = a->ldg ? a->ldg : d, ldo = a->ldo ? a->ldo : d;
  // the ops whose kernels take a pitch for x, g and out; every other tensor has pitch d
  const bool free_ldx = op == GPS_ROWWISE_BN_ACT_RESIDUAL || bwd || op == GPS_ROWWISE_COLSUM;
  const bool free_ldo = op == GPS_ROWWISE_BN_BWD_APPLY;
  const int64_t lds[3] = {ldx, ldg, ldo};
  const char* ldn[3] = {"ldx", "ldg", "ldo"};
  const bool ld_free[3] = {free_ldx, bwd, free_ldo};
  for (int i = 0; i < 3; ++i) {
    // ld == d is the dense layout, whose alignment is the kernels' d % 4 rule (GPS_ERR_UNSUPPORTED)
    GPS_REQUIRE(lds[i] >= d && (lds[i] == d || lds[i] % 4 == 0), GPS_ERR_ARG,
                "gps_rowwise_stage: %s = %lld must be d = %lld, or above it and a multiple of 4", ldn[i],
                (long long)lds[i], (long long)d);
    GPS_REQUIRE(ld_free[i] || lds[i] == d, GPS_ERR_ARG, "gps_rowwise_stage: op %d takes %s = d only (got %lld)", op,
                ldn[i], (long long)lds[i]);
  }
  // tensors over rows (E) may be NULL when there are none
  GPS_REQUIRE(rows == 0 || a->x, GPS_ERR_ARG, "gps_rowwise_stage: op %d needs x", op);
  GPS_REQUIRE(rows == 0 || op == GPS_ROWWISE_BN_BWD_REDUCE || a->out, GPS_ERR_ARG, "gps_rowwise_stage: op %d needs out",
              op);
  GPS_REQUIRE(rows == 0 || !bwd || a->g, GPS_ERR_ARG, "gps_rowwise_stage: op %d needs g", op);
  GPS_REQUIRE(E == 0 || op != GPS_ROWWISE_BN_ACT_RESIDUAL2 || (a->x2 && a->out2), GPS_ERR_ARG,
              "gps_rowwise_stage: BN_ACT_RESIDUAL2 needs x2 and out2");
  // the BatchNorms the op reads: what bn_view_at hands the kernels must be there
  const int nbn = op == GPS_ROWWISE_BN_ACT_RESIDUAL2 || (op == GPS_ROWWISE_BN_COMBINE && a->x2) ? 2
                  : op == GPS_ROWWISE_DROPMUL || op == GPS_ROWWISE_COLSUM                     ? 0
                                                                                              : 1;
  BnView v[2];
  for (int i = 0; i < nbn; ++i) {
    const GpsRowwiseBn& b = a->bn[i];
    const GpsBatchNorm& m = b.bn;
    GPS_REQUIRE(m.weight && m.bias, GPS_ERR_ARG, "gps_rowwise_stage: bn[%d] needs weight and bias", i);
    GPS_REQUIRE(b.train || (m.running_mean && m.running_var), GPS_ERR_ARG,
                "gps_rowwise_stage: bn[%d] in eval mode needs the running statistics", i);
    GPS_REQUIRE(!b.train || b.saved, GPS_ERR_ARG, "gps_rowwise_stage: bn[%d] in training mode needs saved", i);
    GPS_REQUIRE(!(bwd || b.train) || b.sums, GPS_ERR_ARG, "gps_rowwise_stage: bn[%d] needs sums", i);
    const StagePlan P{b.train != 0};
    const int64_t fwd_rows = bwd ? -1 : (i == 1 && op == GPS_ROWWISE_BN_ACT_RESIDUAL2 ? E : rows);
    v[i] = bn_view_at(P, b.saved, b.sums, d, a->bn[i].bn, fwd_rows);
  }
  DropCfg drop;
  drop.p = a->p; drop.seed = a->seed; drop.offset = a->offset; drop.site = a->site; drop.offset_dev = a->offset_dev;
  DropCfg drop2 = drop;
  drop2.site = a->site2;
  const Planes outp{(__nv_bfloat16*)a->planes.hi, (__nv_bfloat16*)a->planes.lo, a->planes.ld};
  const cudaStream_t st = (cudaStream_t)stream;
  switch (op) {
    case GPS_ROWWISE_BN_ACT_RESIDUAL:
      return bn_act_residual(a->x, ldx, a->R, a->out, rows, d, v[0], a->act, drop, a->stats, st, outp);
    case GPS_ROWWISE_BN_ACT_RESIDUAL2:
      return bn_act_residual2(a->x, a->R, a->out, rows, v[0], drop, a->stats, a->x2, a->R2, a->out2, E, v[1], drop2, outp,
                              d, a->act, st);
    case GPS_ROWWISE_BN_COMBINE:
      return bn_combine(a->x, v[0], a->x2, v[1], a->out, rows, d, st, outp);
    case GPS_ROWWISE_BN_BWD_REDUCE:
      return bn_bwd_reduce(a->g, ldg, a->x, ldx, rows, d, v[0], a->act, drop, a->bn[0].sums, st);
    case GPS_ROWWISE_BN_BWD_APPLY:
      return bn_bwd_apply(a->g, ldg, a->x, ldx, rows, d, v[0], a->act, drop, a->bn[0].sums, a->out, ldo,
                          a->bn[0].bn.grad_weight, a->bn[0].bn.grad_bias, st, a->accumulate != 0, outp);
    case GPS_ROWWISE_DROPMUL:
      return dropmul_rows(a->x, a->out, rows, d, drop, a->p2, a->site2, outp, st);
    default:
      return colsum(a->x, ldx, rows, d, a->out, st);
  }
}

extern "C" void gps_debug_set(int v) { gemm_tc_set_debug(v); }
// bring-up hooks of the TMA GEMM: forced tile width (0 = heuristic) and a device buffer of 256 x 16 uint64 phase stamps
extern "C" void gps_debug_tma(int force_bn, void* trace) {
  gemm_tma_set_force_bn(force_bn);
  gemm_tma_set_trace((unsigned long long*)trace);
}
extern "C" void gps_debug_tma_splits(int splits) { gemm_tma_set_force_splits(splits); }
extern "C" void gps_debug_attn(void* buf) { attention_tc_set_debug((float*)buf); }

extern "C" int gps_layer_plan(const GpsLayerArgs* args, GpsLayerPlan* plan) {
  GPS_REQUIRE(args && plan, GPS_ERR_ARG, "gps_layer_plan: null argument");
  Plan P;
  GPS_TRY(make_plan(args, &P, false));
  plan->saved_bytes = P.saved_bytes;
  plan->fwd_workspace_bytes = P.fwd_bytes;
  plan->bwd_workspace_bytes = P.bwd_bytes;
  plan->wplanes_bytes = P.wplanes_bytes;
  return GPS_OK;
}

extern "C" int gps_layer_forward(const GpsLayerArgs* args, void* stream) {
  GPS_REQUIRE(args, GPS_ERR_ARG, "gps_layer_forward: null args");
  return layer_forward(args, (cudaStream_t)stream);
}

extern "C" int gps_layer_backward(const GpsLayerArgs* args, void* stream) {
  GPS_REQUIRE(args, GPS_ERR_ARG, "gps_layer_backward: null args");
  return layer_backward(args, (cudaStream_t)stream);
}

// ---- stage entry points of the BigBird global model (bigbird.cu)
static int bb_stage(const GpsGraph* g, int64_t heads, int64_t hd, const GpsBigBird* bb, const char* what) {
  GPS_REQUIRE(g && bb, GPS_ERR_ARG, "%s: null argument", what);
  GPS_REQUIRE(hd >= 1 && heads >= 1, GPS_ERR_ARG, "%s: heads and hd must be >= 1", what);
  return bb_check(heads * hd, heads, bb);
}

extern "C" int gps_bigbird_attention_forward(const GpsGraph* g, int64_t heads, int64_t hd, const GpsBigBird* bb,
                                             const float* Q, const float* K, const float* V, int64_t ld, float* O,
                                             int64_t ldo, float* lse, void* stream) {
  GPS_TRY(bb_stage(g, heads, hd, bb, "bigbird_attention_forward"));
  GPS_REQUIRE(Q && K && V && O && lse, GPS_ERR_ARG, "bigbird_attention_forward: null argument");
  GPS_REQUIRE(ld >= heads * hd && ldo >= heads * hd, GPS_ERR_ARG, "bigbird_attention_forward: ld / ldo < heads * hd");
  return bb_attn_fwd(*g, heads, hd, *bb, Q, K, V, ld, O, ldo, lse, (cudaStream_t)stream);
}

extern "C" int gps_bigbird_attention_backward(const GpsGraph* g, int64_t heads, int64_t hd, const GpsBigBird* bb,
                                              const float* Q, const float* K, const float* V, int64_t ld,
                                              const float* O, const float* dO, int64_t ldo, const float* lse,
                                              float* delta, float* dQ, float* dK, float* dV, int64_t ldg,
                                              void* stream) {
  GPS_TRY(bb_stage(g, heads, hd, bb, "bigbird_attention_backward"));
  GPS_REQUIRE(Q && K && V && O && dO && lse && delta && dQ && dK && dV, GPS_ERR_ARG,
              "bigbird_attention_backward: null argument");
  GPS_REQUIRE(ld >= heads * hd && ldo >= heads * hd && ldg >= heads * hd, GPS_ERR_ARG,
              "bigbird_attention_backward: ld / ldo / ldg < heads * hd");
  return bb_attn_bwd(*g, heads, hd, *bb, Q, K, V, ld, O, dO, ldo, lse, delta, dQ, dK, dV, ldg, (cudaStream_t)stream);
}

extern "C" int gps_layernorm_forward(const float* z, int64_t rows, int64_t d, const float* gamma, const float* beta,
                                     float eps, float* y, float* mean, float* rstd, void* stream) {
  GPS_REQUIRE(z && gamma && beta && y && mean && rstd && rows >= 0 && eps >= 0.f, GPS_ERR_ARG,
              "layernorm_forward: null argument, rows < 0 or eps < 0");
  return layernorm_fwd(z, rows, d, gamma, beta, eps, mean, rstd, y, Planes(), nullptr, nullptr, DropCfg(), nullptr,
                       (cudaStream_t)stream);
}

extern "C" int gps_layernorm_backward(const float* g, const float* z, int64_t rows, int64_t d, const float* gamma,
                                      const float* mean, const float* rstd, float* dz, float* grad_gamma,
                                      float* grad_beta, void* workspace, int32_t accumulate, void* stream) {
  GPS_REQUIRE(g && z && gamma && mean && rstd && dz && workspace && rows >= 0, GPS_ERR_ARG,
              "layernorm_backward: null argument or rows < 0");
  return layernorm_bwd(g, DropCfg(), z, rows, d, gamma, mean, rstd, nullptr, Planes(), DropCfg(), dz, nullptr,
                       (float*)workspace, grad_gamma, grad_beta, accumulate != 0, (cudaStream_t)stream);
}

extern "C" int gps_linear_forward(const float* A, int64_t lda, const float* W, int64_t ldw, const float* bias,
                                  float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, int32_t act,
                                  int32_t precision, void* stream) {
  GemmParams g;
  g.M = (int)M; g.N = (int)N; g.K = (int)K;
  g.A = A; g.lda = (int)lda; g.B = W; g.ldb = (int)ldw; g.C = C; g.ldc = (int)ldc; g.bias = bias; g.act = act;
  g.precision = precision;
  return gemm(g, (cudaStream_t)stream);
}

extern "C" int gps_gemm(const float* A, int64_t lda, int32_t ta, const float* B, int64_t ldb, int32_t tb, float* C,
                        int64_t ldc, int64_t M, int64_t N, int64_t K, int32_t splitk, int32_t precision, int32_t impl,
                        void* stream) {
  GemmParams g;
  g.M = (int)M; g.N = (int)N; g.K = (int)K;
  g.A = A; g.lda = (int)lda; g.ta = ta; g.B = B; g.ldb = (int)ldb; g.tb = tb; g.C = C; g.ldc = (int)ldc;
  g.splitk = splitk < 1 ? 1 : splitk; g.precision = precision;
  if (impl == 1) return gemm_simt(g, (cudaStream_t)stream);
  if (impl == 2) {
    int rc = gemm_tc(g, (cudaStream_t)stream);
    if (rc == GPS_ERR_UNSUPPORTED) set_error("gps_gemm: the tensor-core kernel does not take this shape/alignment");
    return rc;
  }
  return gemm(g, (cudaStream_t)stream);
}

extern "C" int gps_gatedgcn_aggregate_forward(const GpsGraph* g, int64_t d, const float* Ax, const float* Bx,
                                              const float* Dx, const float* Ex, int64_t ldy, float* Ce, float* xt,
                                              double* stats_x, double* stats_e, void* stream) {
  GPS_REQUIRE(g && Ax && Bx && Dx && Ex && (Ce || g->E == 0) && xt, GPS_ERR_ARG, "gatedgcn_aggregate: null argument");
  return gatedgcn_fwd(*g, d, Ax, Bx, Dx, Ex, ldy, Ce, xt, stats_x, stats_e, (cudaStream_t)stream);
}

extern "C" int gps_gine_aggregate_forward(const GpsGraph* g, int64_t d, const float* x, const float* e, float eps,
                                          float* out, void* stream) {
  GPS_REQUIRE(g && x && out && (e || g->E == 0), GPS_ERR_ARG, "gine_aggregate: null argument");
  return gine_fwd(*g, d, x, e, eps, out, (cudaStream_t)stream);
}

// ---- stage entry points of the message-passing backward passes, the EquivStableLapPE gate and GCN.  Each validates
// its arguments before it enqueues anything: the sparse kernels take d > 0, d % 4 == 0, d <= 4096 (scatter.cu,
// node_geom), checked here up front because some of them launch a kernel before the first one that checks it.
static int stage_width(int64_t d, const char* what) {
  GPS_REQUIRE(d > 0 && d % 4 == 0 && d <= 4096, GPS_ERR_UNSUPPORTED, "%s needs d %% 4 == 0 and 0 < d <= 4096 (got %lld)",
              what, (long long)d);
  return GPS_OK;
}
// optional caller planes: hi == NULL means none; else a pitch that is a multiple of 8 and holds `cols` columns
static int stage_planes(const GpsPlanes* p, int64_t cols, Planes* out, const char* what) {
  *out = Planes();
  if (!p || !p->hi) return GPS_OK;
  GPS_REQUIRE(p->ld >= cols && p->ld % 8 == 0, GPS_ERR_ARG, "%s: plane pitch %lld must be a multiple of 8 and >= %lld",
              what, (long long)p->ld, (long long)cols);
  *out = Planes{(__nv_bfloat16*)p->hi, (__nv_bfloat16*)p->lo, p->ld};
  return GPS_OK;
}

extern "C" int gps_gatedgcn_aggregate_forward_gated(const GpsGraph* g, int64_t d, const float* Ax, const float* Bx,
                                                    const float* Dx, const float* Ex, int64_t ldy, float* Ce, float* xt,
                                                    double* stats_x, double* stats_e, const float* rho, void* stream) {
  GPS_REQUIRE(g && Ax && Bx && Dx && Ex && (Ce || g->E == 0) && xt, GPS_ERR_ARG, "gatedgcn_aggregate_gated: null argument");
  GPS_TRY(stage_width(d, "gatedgcn_aggregate_gated"));
  GPS_REQUIRE(ldy >= d, GPS_ERR_ARG, "gatedgcn_aggregate_gated: ldy < d");
  return gatedgcn_fwd(*g, d, Ax, Bx, Dx, Ex, ldy, Ce, xt, stats_x, stats_e, (cudaStream_t)stream, rho);
}

extern "C" int gps_gatedgcn_aggregate_backward(const GpsGraph* g, int64_t d, const float* ehat, const float* Bx,
                                               int64_t ldy, const float* rho, float* gY, int64_t ldg, float* g_e,
                                               float* g_num, float* g_den, const GpsPlanes* gY_planes,
                                               const GpsPlanes* g_e_planes, void* stream) {
  GPS_REQUIRE(g && gY && g_num && (g->E == 0 || (ehat && Bx && g_e)) && (!rho || g_den), GPS_ERR_ARG,
              "gatedgcn_aggregate_backward: null argument");
  GPS_TRY(stage_width(d, "gatedgcn_aggregate_backward"));
  GPS_REQUIRE(ldy >= d && ldg >= 4 * d, GPS_ERR_ARG, "gatedgcn_aggregate_backward: ldy < d or ldg < 4 d");
  Planes yp, ep;
  GPS_TRY(stage_planes(gY_planes, 4 * d, &yp, "gatedgcn_aggregate_backward gY_planes"));
  GPS_TRY(stage_planes(g_e_planes, d, &ep, "gatedgcn_aggregate_backward g_e_planes"));
  const cudaStream_t st = (cudaStream_t)stream;
  // as layer_backward: block 0 of gY is g_xt; the passes write g_Dx (block 2), then g_Ex (block 3) and g_Bx (block 1)
  GPS_TRY(gatedgcn_bwd_dst(*g, d, gY, ldg, ehat, Bx, ldy, g_e, g_num, gY + 2 * d, st, ep, yp.cols(2 * d), rho, g_den));
  return gatedgcn_bwd_src(*g, d, g_e, ehat, g_num, gY + 3 * d, gY + d, ldg, st, yp.cols(3 * d), yp.cols(d), rho);
}

extern "C" int gps_eslap_forward(const GpsGraph* g, const float* pe, int64_t k, int64_t d, int32_t act, const float* w1,
                                 const float* b1, const float* w2, const float* b2, float* r, float* rho, void* stream) {
  GPS_REQUIRE(g && (g->E == 0 || (pe && w1 && b1 && w2 && b2 && r && rho)), GPS_ERR_ARG, "eslap_forward: null argument");
  GPS_TRY(stage_width(d, "eslap_forward"));
  GPS_REQUIRE(k >= 1 && (act == GPS_ACT_RELU || act == GPS_ACT_GELU), GPS_ERR_ARG, "eslap_forward: k < 1 or unknown act");
  return eslap_fwd(*g, pe, k, d, act, w1, b1, w2, b2, r, rho, (cudaStream_t)stream);
}

// workspace of gps_eslap_backward: gz [E], gr [E], then part [ceil(E / chunk), 3d + 1] (floats)
extern "C" int64_t gps_eslap_workspace_bytes(int64_t E, int64_t d) {
  if (E <= 0) return 0;
  return (2 * E + ceil_div(E, eslap_wgrad_chunk(E)) * (3 * d + 1)) * (int64_t)sizeof(float);
}

extern "C" int gps_eslap_backward(const GpsGraph* g, const float* pe, int64_t k, int64_t d, int32_t act,
                                  const float* g_num, const float* g_den, const float* Bx, int64_t ldy, const float* ehat,
                                  const float* r, const float* rho, const float* w1, const float* b1, const float* w2,
                                  void* workspace, int64_t workspace_bytes, float* grad_pe, float* gw1, float* gb1,
                                  float* gw2, float* gb2, int32_t accumulate, void* stream) {
  const int64_t E = g ? g->E : 0;
  GPS_REQUIRE(g && (E == 0 || (g_num && g_den && Bx && ehat && r && rho && w1 && b1 && w2 && workspace)) &&
                  (pe || (E == 0 && !grad_pe)),
              GPS_ERR_ARG, "eslap_backward: null argument");
  GPS_TRY(stage_width(d, "eslap_backward"));
  GPS_REQUIRE(k >= 1 && (act == GPS_ACT_RELU || act == GPS_ACT_GELU) && ldy >= d, GPS_ERR_ARG,
              "eslap_backward: k < 1, unknown act or ldy < d");
  GPS_REQUIRE(workspace_bytes >= gps_eslap_workspace_bytes(E, d), GPS_ERR_ARG, "eslap_backward: workspace too small");
  float* ws = (float*)workspace;
  float* gz = E > 0 ? ws : nullptr;
  float* gr = E > 0 ? ws + E : nullptr;
  float* part = E > 0 ? ws + 2 * E : nullptr;
  return eslap_bwd(*g, pe, k, d, act, g_num, g_den, Bx, ldy, ehat, r, rho, w1, b1, w2, gz, gr, part, grad_pe, gw1, gb1,
                   gw2, gb2, accumulate != 0, (cudaStream_t)stream);
}

extern "C" int gps_gine_aggregate_backward(const GpsGraph* g, int64_t d, const float* x, const float* e,
                                           const float* g_out, float eps, const float* add, float* g_e, float* g_x,
                                           void* stream) {
  GPS_REQUIRE(g && g_out && g_x && (g->E == 0 || (x && e && g_e)), GPS_ERR_ARG, "gine_aggregate_backward: null argument");
  GPS_TRY(stage_width(d, "gine_aggregate_backward"));
  GPS_TRY(gine_bwd_dst(*g, d, x, e, g_out, g_e, (cudaStream_t)stream));
  return gine_bwd_src(*g, d, g_e, g_out, eps, add, g_x, (cudaStream_t)stream);
}

extern "C" int gps_gcn_aggregate_forward(const GpsGraph* g, int64_t d, const float* Y, int64_t ldy, const float* bias,
                                         const float* x, float* dinv, float* xloc, float p_drop, uint64_t seed,
                                         uint64_t offset, double* stats, void* stream) {
  GPS_REQUIRE(g && Y && bias && x && dinv && xloc, GPS_ERR_ARG, "gcn_aggregate_forward: null argument");
  GPS_TRY(stage_width(d, "gcn_aggregate_forward"));
  GPS_REQUIRE(ldy >= d && p_drop >= 0.f && p_drop < 1.f, GPS_ERR_ARG, "gcn_aggregate_forward: ldy < d or p_drop not in [0,1)");
  DropCfg drop;
  drop.p = p_drop; drop.seed = seed; drop.offset = offset; drop.site = GPS_SITE_LOCAL;
  GPS_TRY(gcn_dinv(*g, dinv, (cudaStream_t)stream));
  return gcn_fwd(*g, d, Y, ldy, dinv, bias, x, xloc, drop, stats, (cudaStream_t)stream);
}

extern "C" int gps_gcn_aggregate_backward(const GpsGraph* g, int64_t d, const float* g_h, const float* dinv, float* gY,
                                          int64_t ldg, const GpsPlanes* gY_planes, void* stream) {
  GPS_REQUIRE(g && g_h && dinv && gY, GPS_ERR_ARG, "gcn_aggregate_backward: null argument");
  GPS_TRY(stage_width(d, "gcn_aggregate_backward"));
  GPS_REQUIRE(ldg >= d, GPS_ERR_ARG, "gcn_aggregate_backward: ldg < d");
  Planes yp;
  GPS_TRY(stage_planes(gY_planes, d, &yp, "gcn_aggregate_backward gY_planes"));
  return gcn_bwd(*g, d, g_h, dinv, gY, ldg, (cudaStream_t)stream, yp);
}

// ---- stage entry points of the GAT local model (gat.cu).  Each validates its arguments before it enqueues anything.
extern "C" int gps_gat_fold_forward(const float* W_edge, const float* att_edge, int64_t d, int64_t H, float* v,
                                    void* stream) {
  GPS_REQUIRE(W_edge && att_edge && v, GPS_ERR_ARG, "gat_fold_forward: null argument");
  return gat_fold_fwd(W_edge, att_edge, d, H, v, (cudaStream_t)stream);
}

extern "C" int gps_gat_fold_backward(const float* W_edge, const float* att_edge, const float* g_v, int64_t d, int64_t H,
                                     float* g_W_edge, float* g_att_edge, int32_t accumulate, void* stream) {
  GPS_REQUIRE(W_edge && att_edge && g_v, GPS_ERR_ARG, "gat_fold_backward: null argument");
  return gat_fold_bwd(W_edge, att_edge, g_v, d, H, g_W_edge, g_att_edge, accumulate != 0, (cudaStream_t)stream);
}

extern "C" int gps_gat_forward(const GpsGraph* g, int64_t d, int64_t H, const float* Y, int64_t ldy,
                               const float* edge_attr, const float* v, const float* att_src, const float* att_dst,
                               const float* bias, const float* x, float* scores, float* xloc, float p_drop,
                               uint64_t seed, uint64_t offset, double* stats, void* stream) {
  GPS_REQUIRE(g && Y && v && att_src && att_dst && bias && x && scores && xloc && (edge_attr || g->E == 0), GPS_ERR_ARG,
              "gat_forward: null argument");
  GPS_TRY(gat_check(d, H));
  GPS_REQUIRE(ldy >= d && ldy % 4 == 0 && p_drop >= 0.f && p_drop < 1.f, GPS_ERR_ARG,
              "gat_forward: ldy < d, ldy %% 4 != 0 or p_drop not in [0,1)");
  DropCfg drop;
  drop.p = p_drop; drop.seed = seed; drop.offset = offset; drop.site = GPS_SITE_LOCAL;
  return gat_fwd(*g, d, H, Y, ldy, edge_attr, v, att_src, att_dst, bias, x, gat_scores(scores, g->N, g->E, H), xloc,
                 drop, stats, (cudaStream_t)stream);
}

extern "C" int64_t gps_gat_workspace_bytes(int64_t N, int64_t E, int64_t H, int64_t d) {
  return gat_bwd_workspace_floats(N, E, H, d) * (int64_t)sizeof(float);
}

extern "C" int gps_gat_backward(const GpsGraph* g, int64_t d, int64_t H, const float* Y, int64_t ldy,
                                const float* edge_attr, const float* v, const float* att_src, const float* att_dst,
                                const float* scores, const float* g_h, void* workspace, int64_t workspace_bytes,
                                float* gY, int64_t ldg, const GpsPlanes* gY_planes, float* grad_edge_attr, float* g_v,
                                float* g_att_src, float* g_att_dst, float* g_bias, int32_t accumulate, void* stream) {
  GPS_REQUIRE(g && Y && v && att_src && att_dst && scores && g_h && workspace && gY && g_v && (edge_attr || g->E == 0),
              GPS_ERR_ARG, "gat_backward: null argument");
  GPS_TRY(gat_check(d, H));
  GPS_REQUIRE(ldy >= d && ldg >= d && ldy % 4 == 0 && ldg % 4 == 0, GPS_ERR_ARG,
              "gat_backward: ldy / ldg < d or not a multiple of 4");
  GPS_REQUIRE(workspace_bytes >= gps_gat_workspace_bytes(g->N, g->E, H, d), GPS_ERR_ARG, "gat_backward: workspace too small");
  Planes yp;
  GPS_TRY(stage_planes(gY_planes, d, &yp, "gat_backward gY_planes"));
  return gat_bwd(*g, d, H, Y, ldy, edge_attr, v, att_src, att_dst, gat_scores((float*)scores, g->N, g->E, H), g_h,
                 (float*)workspace, gY, ldg, yp, grad_edge_attr, g_v, g_att_src, g_att_dst, g_bias, accumulate != 0,
                 (cudaStream_t)stream);
}

// ---- stage entry points of the GENConv message passing (genconv.cu; the backward's source-ordered pass is GINE's)
extern "C" int gps_genconv_aggregate_forward(const GpsGraph* g, int64_t d, const float* x, const float* e, float* agg,
                                             float* lse, float* u, void* stream) {
  GPS_REQUIRE(g && x && agg && lse && u && (e || g->E == 0), GPS_ERR_ARG, "genconv_aggregate_forward: null argument");
  GPS_TRY(stage_width(d, "genconv_aggregate_forward"));
  return genconv_fwd(*g, d, x, e, agg, lse, u, (cudaStream_t)stream);
}

extern "C" int gps_genconv_aggregate_backward(const GpsGraph* g, int64_t d, const float* x, const float* e,
                                              const float* agg, const float* lse, const float* g_u, const float* add,
                                              float* g_e, float* g_x, void* stream) {
  GPS_REQUIRE(g && x && agg && lse && g_u && g_x && (g->E == 0 || (e && g_e)), GPS_ERR_ARG,
              "genconv_aggregate_backward: null argument");
  GPS_TRY(stage_width(d, "genconv_aggregate_backward"));
  GPS_TRY(genconv_bwd_dst(*g, d, x, e, agg, lse, g_u, g_e, (cudaStream_t)stream));
  return gine_bwd_src(*g, d, g_e, g_u, 0.f, add, g_x, (cudaStream_t)stream);
}

// ---- stage entry points of the PNA edge fold and message passing (pna.cu)
extern "C" int gps_pna_fold_forward(const float* pre_w, const float* pre_b, const float* enc_w, const float* enc_b,
                                    int64_t d, int64_t de, float* F, float* c, void* stream) {
  GPS_REQUIRE(pre_w && pre_b && enc_w && enc_b && F && c, GPS_ERR_ARG, "pna_fold_forward: null argument");
  GPS_TRY(stage_width(d, "pna_fold_forward"));
  return pna_fold_fwd(pre_w, pre_b, enc_w, enc_b, d, de, F, c, (cudaStream_t)stream);
}

extern "C" int gps_pna_fold_backward(const float* pre_w, const float* enc_w, const float* enc_b, const float* g_F,
                                     const float* g_c, int64_t d, int64_t de, float* grad_pre_w, float* grad_pre_b,
                                     float* grad_enc_w, float* grad_enc_b, int32_t accumulate, void* stream) {
  GPS_REQUIRE(pre_w && enc_w && enc_b && g_F && g_c, GPS_ERR_ARG, "pna_fold_backward: null argument");
  GPS_TRY(stage_width(d, "pna_fold_backward"));
  return pna_fold_bwd(pre_w, enc_w, enc_b, g_F, g_c, d, de, grad_pre_w, grad_pre_b, grad_enc_w, grad_enc_b,
                      accumulate != 0, (cudaStream_t)stream);
}

extern "C" int gps_pna_aggregate_forward(const GpsGraph* g, int64_t d, const float* x, const float* Y, int64_t ldy,
                                         const float* q, float* Z, int32_t* arg, void* stream) {
  GPS_REQUIRE(g && x && Y && Z && arg && (q || g->E == 0), GPS_ERR_ARG, "pna_aggregate_forward: null argument");
  GPS_TRY(stage_width(d, "pna_aggregate_forward"));
  GPS_REQUIRE(ldy >= 2 * d && ldy % 4 == 0, GPS_ERR_ARG, "pna_aggregate_forward: ldy must be >= 2d and a multiple of 4");
  return pna_fwd(*g, d, x, Y, ldy, q, Z, Planes(), arg, (cudaStream_t)stream);
}

extern "C" int gps_pna_aggregate_backward(const GpsGraph* g, int64_t d, const float* g_Z, const int32_t* arg,
                                          const float* add, float* g_q, float* gY, int64_t ldg, float* g_x,
                                          void* stream) {
  GPS_REQUIRE(g && g_Z && arg && gY && g_x && (g_q || g->E == 0), GPS_ERR_ARG, "pna_aggregate_backward: null argument");
  GPS_TRY(stage_width(d, "pna_aggregate_backward"));
  GPS_REQUIRE(ldg >= 2 * d && ldg % 4 == 0, GPS_ERR_ARG, "pna_aggregate_backward: ldg must be >= 2d and a multiple of 4");
  return pna_bwd(*g, d, g_Z, arg, add, g_q, Planes(), gY, ldg, Planes(), g_x, (cudaStream_t)stream);
}

// ---- stage entry points of the Performer (performer.cu, performer_quad.cu).  Each validates its arguments before it
// enqueues anything: dim_head 64, 256 < m <= 272 (perf_supported), H > 0 and N * H * 272 < 2^31.
static int perf_stage(const GpsGraph* g, int64_t H, int64_t dim_head, int64_t m) {
  GPS_TRY(perf_supported(dim_head, m));
  return perf_index_range(g->N, H);
}

extern "C" int gps_performer_prep(const GpsGraph* g, int64_t H, int64_t dim_head, int64_t m, const float* P, float* Pn,
                                  int* nmax, float* gmax, int* argk, void* stream) {
  GPS_REQUIRE(g && P && Pn && nmax && gmax && argk, GPS_ERR_ARG, "performer_prep: null argument");
  GPS_TRY(perf_stage(g, H, dim_head, m));
  return perf_prep(P, m, Pn, *g, H, nmax, gmax, argk, (cudaStream_t)stream);
}

extern "C" int gps_performer_features_forward(const GpsGraph* g, int64_t H, int64_t dim_head, int64_t m, float* fq,
                                              float* fk, const float* Q, const float* K, float* gmax, int* argq,
                                              int* argk, void* stream) {
  GPS_REQUIRE(g && fq && fk && Q && K && gmax && argq && argk, GPS_ERR_ARG, "performer_features_forward: null argument");
  GPS_TRY(perf_stage(g, H, dim_head, m));
  return perf_features_fwd(fq, fk, Q, K, *g, H, m, gmax, argq, argk, (cudaStream_t)stream);
}

extern "C" int gps_performer_attention_forward(const GpsGraph* g, int64_t H, int64_t dim_head, int64_t m, int32_t form,
                                               const int* nmax, const float* qf, const float* kf, const float* V,
                                               const float* gmax, float* O, float* den, void* stream) {
  GPS_REQUIRE(form == 0 || form == 1, GPS_ERR_ARG, "performer_attention_forward: form must be 0 (context) or 1 (pairwise)");
  GPS_REQUIRE(g && nmax && qf && kf && V && gmax && O && (form == 0 || den), GPS_ERR_ARG,
              "performer_attention_forward: null argument");
  GPS_TRY(perf_stage(g, H, dim_head, m));
  if (form == 1) return perf_quad_fwd(*g, H, m, nmax, qf, kf, V, gmax, O, den, (cudaStream_t)stream);
  return perf_linattn_fwd(*g, H, m, nmax, qf, kf, V, gmax, O, (cudaStream_t)stream);
}

extern "C" int gps_performer_attention_backward(const GpsGraph* g, int64_t H, int64_t dim_head, int64_t m, int32_t form,
                                                const int* nmax, const float* qf, const float* kf, const float* V,
                                                const float* gmax, const float* O, const float* den, const float* gO,
                                                float* gden, float* g_qf, float* g_kf, float* gV, float* ggmax,
                                                float* gmrow, void* stream) {
  GPS_REQUIRE(form == 0 || form == 1, GPS_ERR_ARG, "performer_attention_backward: form must be 0 (context) or 1 (pairwise)");
  GPS_REQUIRE(g && nmax && qf && kf && V && gmax && gO && g_qf && g_kf && gV &&
                  (form == 0 ? ggmax != nullptr : (O && den && gden && gmrow)),
              GPS_ERR_ARG, "performer_attention_backward: null argument");
  GPS_TRY(perf_stage(g, H, dim_head, m));
  if (form == 1)
    return perf_quad_bwd(*g, H, m, nmax, qf, kf, V, gmax, O, den, gO, gden, g_qf, g_kf, gV, gmrow, (cudaStream_t)stream);
  return perf_linattn_bwd(*g, H, m, nmax, qf, kf, V, gmax, gO, g_qf, g_kf, gV, ggmax, (cudaStream_t)stream);
}

extern "C" int gps_performer_features_backward(const GpsGraph* g, int64_t H, int64_t dim_head, int64_t m, int32_t form,
                                               float* g_fq, float* g_fk, const float* fq, const float* fk, const float* Q,
                                               const float* K, float* gQ, float* gK, const int* argq, const int* argk,
                                               const float* ggmax, float* gmrow, void* stream) {
  GPS_REQUIRE(form == 0 || form == 1, GPS_ERR_ARG, "performer_features_backward: form must be 0 (context) or 1 (pairwise)");
  GPS_REQUIRE(g && g_fq && g_fk && fq && fk && Q && K && gQ && gK && argq && argk && gmrow && (form == 1 || ggmax),
              GPS_ERR_ARG, "performer_features_backward: null argument");
  GPS_TRY(perf_stage(g, H, dim_head, m));
  return perf_features_bwd(g_fq, g_fk, fq, fk, Q, K, gQ, gK, *g, H, m, argq, argk, ggmax, gmrow, form == 1,
                           (cudaStream_t)stream);
}

// The attention stages: one argument contract for gps_attention_stage and the six entry points that are calls of it.
static Planes attn_planes(const GpsPlanes& p) { return Planes{(__nv_bfloat16*)p.hi, (__nv_bfloat16*)p.lo, p.ld}; }

static int attn_check_planes(const GpsPlanes& p, int64_t min_ld, const char* name) {
  if (!p.hi && !p.lo) return GPS_OK;
  GPS_REQUIRE(p.hi, GPS_ERR_ARG, "gps_attention_stage: %s has lo without hi", name);
  GPS_REQUIRE(p.ld >= min_ld, GPS_ERR_ARG, "gps_attention_stage: %s pitch %lld is below %lld", name, (long long)p.ld,
              (long long)min_ld);
  GPS_REQUIRE(p.ld % 8 == 0, GPS_ERR_UNSUPPORTED, "gps_attention_stage: %s pitch %lld is not a multiple of 8", name,
              (long long)p.ld);
  return GPS_OK;
}

static int attn_check(const GpsAttnStageArgs* a, int32_t op) {
  GPS_REQUIRE(a, GPS_ERR_ARG, "gps_attention_stage: null args");
  GPS_REQUIRE(op == GPS_ATTN_FWD || op == GPS_ATTN_FWD_TC || op == GPS_ATTN_BWD, GPS_ERR_ARG,
              "gps_attention_stage: unknown op %d", op);
  const GpsGraph& g = a->graph;
  GPS_REQUIRE(g.N >= 0 && g.B >= 0 && g.N <= 0x7FFFFFFF && g.B <= 0x7FFFFFFF, GPS_ERR_ARG,
              "gps_attention_stage: N %lld and B %lld must lie in [0, 2^31)", (long long)g.N, (long long)g.B);
  GPS_REQUIRE(g.N == 0 || (g.B >= 1 && g.graph_ptr), GPS_ERR_ARG, "gps_attention_stage: %lld nodes need B >= 1 and graph_ptr",
              (long long)g.N);
  GPS_REQUIRE(a->heads >= 1, GPS_ERR_ARG, "gps_attention_stage: heads must be >= 1 (got %lld)", (long long)a->heads);
  GPS_REQUIRE(a->p_drop >= 0.f && a->p_drop < 1.f, GPS_ERR_ARG, "gps_attention_stage: p_drop %g is not in [0, 1)",
              (double)a->p_drop);
  if (a->bias) {
    GPS_REQUIRE(a->bias->bias, GPS_ERR_ARG, "gps_attention_stage: null attention bias");
    GPS_REQUIRE(a->bias->nmax >= 1, GPS_ERR_ARG, "gps_attention_stage: nmax must be >= 1 (got %lld)",
                (long long)a->bias->nmax);
  }
  const bool tc = op == GPS_ATTN_FWD_TC, bwd = op == GPS_ATTN_BWD;
  GPS_REQUIRE(a->O && a->lse, GPS_ERR_ARG, "gps_attention_stage: op %d needs O and lse", op);
  if (tc) {
    GPS_REQUIRE(a->qkv.hi, GPS_ERR_ARG, "gps_attention_stage: FWD_TC needs the qkv planes");
    GPS_REQUIRE(a->precision == GPS_PREC_FP32 || a->precision == GPS_PREC_BF16, GPS_ERR_ARG,
                "gps_attention_stage: precision %d is not GPS_PREC_FP32 or GPS_PREC_BF16", a->precision);
  } else {
    GPS_REQUIRE(a->Q && a->K && a->V, GPS_ERR_ARG, "gps_attention_stage: op %d needs Q, K and V", op);
  }
  GPS_REQUIRE(!bwd || (a->dO && a->delta && a->dQ && a->dK && a->dV), GPS_ERR_ARG,
              "gps_attention_stage: BWD needs dO, delta, dQ, dK and dV");
  GPS_REQUIRE(a->hd >= 1 && a->hd <= 192, GPS_ERR_UNSUPPORTED, "gps_attention_stage: head dim %lld must be in 1..192",
              (long long)a->hd);
  const int64_t D = a->heads * a->hd;
  GPS_REQUIRE(tc || a->ld >= D, GPS_ERR_ARG, "gps_attention_stage: ld %lld is below heads * hd = %lld", (long long)a->ld,
              (long long)D);
  GPS_REQUIRE(a->ldo >= D, GPS_ERR_ARG, "gps_attention_stage: ldo %lld is below heads * hd = %lld", (long long)a->ldo,
              (long long)D);
  GPS_REQUIRE(!bwd || a->ldg >= D, GPS_ERR_ARG, "gps_attention_stage: ldg %lld is below heads * hd = %lld",
              (long long)a->ldg, (long long)D);
  if (bwd) {
    GPS_TRY(attn_check_planes(a->dQ_planes, D, "dQ_planes"));
    GPS_TRY(attn_check_planes(a->dK_planes, D, "dK_planes"));
    GPS_TRY(attn_check_planes(a->dV_planes, D, "dV_planes"));
  } else {
    GPS_TRY(attn_check_planes(a->O_planes, D, "O_planes"));
  }
  if (tc) {
    GPS_REQUIRE(attention_tc_supported(a->hd), GPS_ERR_UNSUPPORTED,
                "gps_attention_stage: FWD_TC takes head dims that are a multiple of 4 up to 128 (got %lld)",
                (long long)a->hd);
    GPS_TRY(attn_check_planes(a->qkv, 3 * a->heads * attention_tc_hd_pad(a->hd), "qkv"));
    GPS_REQUIRE(a->precision != GPS_PREC_FP32 || a->qkv.lo, GPS_ERR_UNSUPPORTED,
                "gps_attention_stage: FWD_TC in GPS_PREC_FP32 needs qkv.lo");
  }
  return GPS_OK;
}

extern "C" int gps_attention_stage(const GpsAttnStageArgs* a, int32_t op, void* stream) {
  GPS_TRY(attn_check(a, op));
  const cudaStream_t st = (cudaStream_t)stream;
  switch (op) {
    case GPS_ATTN_FWD:
      return attention_fwd(a->graph, a->heads, a->hd, a->Q, a->K, a->V, a->ld, a->O, a->ldo, a->lse, a->p_drop, a->seed,
                           a->offset, st, a->offset_dev, attn_planes(a->O_planes), a->bias);
    case GPS_ATTN_FWD_TC:
      return attention_tc_fwd(a->graph, a->heads, a->hd, attn_planes(a->qkv), a->O, a->ldo, attn_planes(a->O_planes),
                              a->lse, a->p_drop, a->seed, a->offset, a->offset_dev, a->precision, st, a->bias);
    default:
      return attention_bwd(a->graph, a->heads, a->hd, a->Q, a->K, a->V, a->ld, a->O, a->dO, a->ldo, a->lse, a->delta,
                           a->dQ, a->dK, a->dV, a->ldg, a->p_drop, a->seed, a->offset, st, a->offset_dev,
                           attn_planes(a->dQ_planes), attn_planes(a->dK_planes), attn_planes(a->dV_planes), a->bias);
  }
}

// the six fixed-signature entry points: the stage call with the fields they take; the biased ones require a bias
static GpsAttnStageArgs attn_args(const GpsGraph* g, int64_t heads, int64_t hd, float p_drop, uint64_t seed,
                                  uint64_t offset, const GpsAttnBias* bias) {
  GpsAttnStageArgs a{};
  a.graph = *g;
  a.heads = heads; a.hd = hd; a.p_drop = p_drop; a.seed = seed; a.offset = offset; a.bias = bias;
  return a;
}
static int attn_fwd_call(const GpsGraph* g, int64_t heads, int64_t hd, const float* Q, const float* K, const float* V,
                         int64_t ld, float* O, int64_t ldo, float* lse, float p_drop, uint64_t seed, uint64_t offset,
                         const GpsAttnBias* bias, void* stream) {
  GPS_REQUIRE(g, GPS_ERR_ARG, "gps_attention_stage: null graph");
  GpsAttnStageArgs a = attn_args(g, heads, hd, p_drop, seed, offset, bias);
  a.Q = Q; a.K = K; a.V = V; a.ld = ld; a.O = O; a.ldo = ldo; a.lse = lse;
  return gps_attention_stage(&a, GPS_ATTN_FWD, stream);
}
static int attn_fwd_tc_call(const GpsGraph* g, int64_t heads, int64_t hd, const void* qkv_hi, const void* qkv_lo,
                            int64_t ld, float* O, int64_t ldo, float* lse, float p_drop, uint64_t seed, uint64_t offset,
                            int32_t precision, const GpsAttnBias* bias, void* stream) {
  GPS_REQUIRE(g, GPS_ERR_ARG, "gps_attention_stage: null graph");
  GpsAttnStageArgs a = attn_args(g, heads, hd, p_drop, seed, offset, bias);
  a.qkv = GpsPlanes{const_cast<void*>(qkv_hi), const_cast<void*>(qkv_lo), ld};
  a.precision = precision; a.O = O; a.ldo = ldo; a.lse = lse;
  return gps_attention_stage(&a, GPS_ATTN_FWD_TC, stream);
}
static int attn_bwd_call(const GpsGraph* g, int64_t heads, int64_t hd, const float* Q, const float* K, const float* V,
                         int64_t ld, const float* O, const float* dO, int64_t ldo, const float* lse, float* delta,
                         float* dQ, float* dK, float* dV, int64_t ldg, float p_drop, uint64_t seed, uint64_t offset,
                         const GpsAttnBias* bias, void* stream) {
  GPS_REQUIRE(g, GPS_ERR_ARG, "gps_attention_stage: null graph");
  GpsAttnStageArgs a = attn_args(g, heads, hd, p_drop, seed, offset, bias);
  a.Q = Q; a.K = K; a.V = V; a.ld = ld; a.O = const_cast<float*>(O); a.dO = dO; a.ldo = ldo;
  a.lse = const_cast<float*>(lse); a.delta = delta; a.dQ = dQ; a.dK = dK; a.dV = dV; a.ldg = ldg;
  return gps_attention_stage(&a, GPS_ATTN_BWD, stream);
}

extern "C" int gps_attention_forward(const GpsGraph* g, int64_t heads, int64_t hd, const float* Q, const float* K,
                                     const float* V, int64_t ld, float* O, int64_t ldo, float* lse, float p_drop,
                                     uint64_t seed, uint64_t offset, void* stream) {
  return attn_fwd_call(g, heads, hd, Q, K, V, ld, O, ldo, lse, p_drop, seed, offset, nullptr, stream);
}

extern "C" int gps_attention_forward_tc(const GpsGraph* g, int64_t heads, int64_t hd, const void* qkv_hi, const void* qkv_lo,
                                        int64_t ld, float* O, int64_t ldo, float* lse, float p_drop, uint64_t seed,
                                        uint64_t offset, int32_t precision, void* stream) {
  return attn_fwd_tc_call(g, heads, hd, qkv_hi, qkv_lo, ld, O, ldo, lse, p_drop, seed, offset, precision, nullptr, stream);
}

extern "C" int gps_attention_backward(const GpsGraph* g, int64_t heads, int64_t hd, const float* Q, const float* K,
                                      const float* V, int64_t ld, const float* O, const float* dO, int64_t ldo,
                                      const float* lse, float* delta, float* dQ, float* dK, float* dV, int64_t ldg,
                                      float p_drop, uint64_t seed, uint64_t offset, void* stream) {
  return attn_bwd_call(g, heads, hd, Q, K, V, ld, O, dO, ldo, lse, delta, dQ, dK, dV, ldg, p_drop, seed, offset, nullptr,
                       stream);
}

extern "C" int gps_attention_forward_biased(const GpsGraph* g, int64_t heads, int64_t hd, const float* Q,
                                            const float* K, const float* V, int64_t ld, float* O, int64_t ldo,
                                            float* lse, float p_drop, uint64_t seed, uint64_t offset,
                                            const GpsAttnBias* bias, void* stream) {
  GPS_REQUIRE(bias, GPS_ERR_ARG, "gps_attention_forward_biased: null attention bias");
  return attn_fwd_call(g, heads, hd, Q, K, V, ld, O, ldo, lse, p_drop, seed, offset, bias, stream);
}

extern "C" int gps_attention_forward_tc_biased(const GpsGraph* g, int64_t heads, int64_t hd, const void* qkv_hi,
                                               const void* qkv_lo, int64_t ld, float* O, int64_t ldo, float* lse,
                                               float p_drop, uint64_t seed, uint64_t offset, int32_t precision,
                                               const GpsAttnBias* bias, void* stream) {
  GPS_REQUIRE(bias, GPS_ERR_ARG, "gps_attention_forward_tc_biased: null attention bias");
  return attn_fwd_tc_call(g, heads, hd, qkv_hi, qkv_lo, ld, O, ldo, lse, p_drop, seed, offset, precision, bias, stream);
}

extern "C" int gps_attention_backward_biased(const GpsGraph* g, int64_t heads, int64_t hd, const float* Q,
                                             const float* K, const float* V, int64_t ld, const float* O,
                                             const float* dO, int64_t ldo, const float* lse, float* delta, float* dQ,
                                             float* dK, float* dV, int64_t ldg, float p_drop, uint64_t seed,
                                             uint64_t offset, const GpsAttnBias* bias, void* stream) {
  GPS_REQUIRE(bias, GPS_ERR_ARG, "gps_attention_backward_biased: null attention bias");
  return attn_bwd_call(g, heads, hd, Q, K, V, ld, O, dO, ldo, lse, delta, dQ, dK, dV, ldg, p_drop, seed, offset, bias,
                       stream);
}

extern "C" int gps_dropout_mask(float* mask, int64_t rows, int64_t cols, float p, uint64_t seed, uint64_t offset,
                                int32_t site, void* stream) {
  GPS_REQUIRE(mask && cols % 4 == 0, GPS_ERR_ARG, "dropout_mask: cols must be a multiple of 4");
  int64_t n4 = rows * cols / 4;
  if (n4 == 0) return GPS_OK;
  k_dropmask<<<(unsigned)std::min<int64_t>(ceil_div(n4, 256), kNumSMs * 8), 256, 0, (cudaStream_t)stream>>>(
      mask, n4, p, seed, offset, site);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}
