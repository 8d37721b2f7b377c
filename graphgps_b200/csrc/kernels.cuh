// kernels.cuh — internal launch API of the non-GEMM stages (implemented in elementwise.cu,
// scatter.cu, attention.cu).  All functions enqueue on `stream` and return GPS_* codes.
#pragma once
#include "common.cuh"

namespace gps {

// Per-column BatchNorm view used by consumers: y = gamma * (z - mean) * invstd + beta
// mode 0: mean/invstd arrays are final (backward, or after an explicit bn_finalize)
// mode 1: training forward — the consumer derives mean/invstd from the producer's double column sums itself and
//         its first CTA stores them (for backward) and applies torch.nn.BatchNorm1d's running-stat update, so no
//         separate finalize launch sits between producer and consumer
// mode 2: eval forward — running statistics
struct BnView {
  const float* mean = nullptr;
  const float* invstd = nullptr;
  const float* gamma = nullptr;
  const float* beta = nullptr;
  int mode = 0;
  const double* sums = nullptr;   // [2][d]
  double inv_n = 0.0, unbias = 1.0;
  int64_t d = 0;
  float* save_mean = nullptr;
  float* save_invstd = nullptr;
  float* running_mean = nullptr;
  float* running_var = nullptr;
  long long* nbt = nullptr;
};

#ifdef __CUDACC__
// Per-thread BatchNorm constants of the float4 column group c4 (the row-wise stages of elementwise.cu and rwse.cu).
// Mode 1 derives mean / invstd from the double column sums; the CTA with virtual block index 0 (blockIdx.x unless vb
// is given) and threadIdx.y == 0 stores them and applies the running-statistics update.
struct BnRegs {  // per-thread column constants: y = z * sc + sh ; zhat = (z - mean) * invstd
  float4 mean, invstd, gamma, beta;
  __device__ void load(const BnView& v, int c4, int vb = -1) {
    gamma = ld4(v.gamma + c4 * 4);
    beta = ld4(v.beta + c4 * 4);
    if (v.mode == 0) {
      mean = ld4(v.mean + c4 * 4);
      invstd = ld4(v.invstd + c4 * 4);
    } else if (v.mode == 2) {
      mean = ld4(v.running_mean + c4 * 4);
      const float4 rv = ld4(v.running_var + c4 * 4);
      invstd = make_float4(rsqrtf(rv.x + kBnEps), rsqrtf(rv.y + kBnEps), rsqrtf(rv.z + kBnEps), rsqrtf(rv.w + kBnEps));
    } else {
      float m[4], is[4], var[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const double mu = v.sums[c4 * 4 + j] * v.inv_n;
        double vv = v.sums[v.d + c4 * 4 + j] * v.inv_n - mu * mu;
        if (vv < 0.0) vv = 0.0;
        m[j] = (float)mu;
        var[j] = (float)(vv * v.unbias);
        is[j] = (float)(1.0 / sqrt(vv + (double)kBnEps));
      }
      mean = make_float4(m[0], m[1], m[2], m[3]);
      invstd = make_float4(is[0], is[1], is[2], is[3]);
      if ((vb < 0 ? (int)blockIdx.x : vb) == 0 && threadIdx.y == 0) {   // one CTA publishes the statistics and the running update
        st4(v.save_mean + c4 * 4, mean);
        st4(v.save_invstd + c4 * 4, invstd);
        if (v.running_mean) {
          const float4 rm = ld4(v.running_mean + c4 * 4);
          st4(v.running_mean + c4 * 4, make_float4((1.f - kBnMomentum) * rm.x + kBnMomentum * m[0],
                                                   (1.f - kBnMomentum) * rm.y + kBnMomentum * m[1],
                                                   (1.f - kBnMomentum) * rm.z + kBnMomentum * m[2],
                                                   (1.f - kBnMomentum) * rm.w + kBnMomentum * m[3]));
        }
        if (v.running_var) {
          const float4 rv = ld4(v.running_var + c4 * 4);
          st4(v.running_var + c4 * 4, make_float4((1.f - kBnMomentum) * rv.x + kBnMomentum * var[0],
                                                  (1.f - kBnMomentum) * rv.y + kBnMomentum * var[1],
                                                  (1.f - kBnMomentum) * rv.z + kBnMomentum * var[2],
                                                  (1.f - kBnMomentum) * rv.w + kBnMomentum * var[3]));
        }
        if (c4 == 0 && v.nbt) *v.nbt += 1;
      }
    }
  }
  __device__ float4 zhat(float4 z) const {
    return make_float4((z.x - mean.x) * invstd.x, (z.y - mean.y) * invstd.y, (z.z - mean.z) * invstd.z,
                       (z.w - mean.w) * invstd.w);
  }
  __device__ float4 apply(float4 z) const { return f4fma(zhat(z), gamma, beta); }
};
#endif  // __CUDACC__

struct DropCfg {
  float p = 0.f;
  uint64_t seed = 0, offset = 0;
  int site = 0;
  const unsigned long long* offset_dev = nullptr;  // optional device-resident addend (CUDA-graph replays)
};

// ---- forward row-wise stages ----------------------------------------------------------------
// out = R + dropout(act(BN(z)))  [+ column sums of out into stats]   (gatedgcn_layer.py:72-83)
int bn_act_residual(const float* z, int64_t ldz, const float* R, float* out, int64_t rows, int64_t d,
                    BnView bn, int act, DropCfg drop, double* stats, cudaStream_t stream, Planes outp = Planes());
int bn_act_residual2(const float* zx, const float* Rx, float* outx, int64_t N, BnView bnx, DropCfg dropx, double* statsx,
                     const float* ze, const float* Re, float* oute, int64_t E, BnView bne, DropCfg drope, Planes outep,
                     int64_t d, int act, cudaStream_t stream);
// out = BN_a(a) [+ BN_b(b)]   (gps_layer.py:194,217,222 and :229)
int bn_combine(const float* a, BnView bna, const float* b, BnView bnb, float* out, int64_t rows, int64_t d,
               cudaStream_t stream, Planes outp = Planes());

// ---- backward row-wise stages ---------------------------------------------------------------
// g' = g * [act'(BN(z))] * [dropout scale];  sums[0][c] += sum_r g', sums[1][c] += sum_r g' * zhat
int bn_bwd_reduce(const float* g, int64_t ldg, const float* z, int64_t ldz, int64_t rows, int64_t d, BnView bn,
                  int act /* -1: none */, DropCfg drop, double* sums, cudaStream_t stream);
// out = gamma*invstd*(g' - S1/n - zhat*S2/n) (+ add); also writes grad_gamma = S2, grad_beta = S1
int bn_bwd_apply(const float* g, int64_t ldg, const float* z, int64_t ldz, int64_t rows, int64_t d, BnView bn,
                 int act, DropCfg drop, const double* sums, float* out, int64_t ldo, float* grad_gamma,
                 float* grad_beta, cudaStream_t stream, bool accumulate = false, Planes outp = Planes());
// out = a + b (+ c)   row-wise with independent leading dimensions
int add3(const float* a, int64_t lda, const float* b, int64_t ldb, const float* c, int64_t ldc, float* out,
         int64_t ldo, int64_t rows, int64_t d, cudaStream_t stream);
// out[c] = sum_r a[r, c]  (float atomics into pre-zeroed out)
int colsum(const float* a, int64_t lda, int64_t rows, int64_t d, float* out, cudaStream_t stream);
// dst[r, :] = src[r, :] for a [rows, d] block with leading dimensions
int copy2d(const float* src, int64_t lds, float* dst, int64_t ldd, int64_t rows, int64_t d, cudaStream_t stream);

// ---- sparse (message passing) stages -------------------------------------------------------
// rho (optional, [E]): EquivStableLapPE edge gate, sigma_ij = sigmoid(e_ij) * rho_e (eslap.cu)
int gatedgcn_fwd(const GpsGraph& g, int64_t d, const float* Ax, const float* Bx, const float* Dx,
                 const float* Ex, int64_t ldy, float* Ce, float* xt, double* stats_x, double* stats_e,
                 cudaStream_t stream, const float* rho = nullptr);
// dst-ordered backward pass: reads g_xt (ld ldg), ehat, Bx; g_e holds the BN_e-path gradient on entry
// and the total gradient w.r.t. e_ij on exit; writes g_num [N,d] and g_Dx (ld ldg).  With rho: also g_den [N,d].
int gatedgcn_bwd_dst(const GpsGraph& g, int64_t d, const float* g_xt, int64_t ldg, const float* ehat,
                     const float* Bx, int64_t ldy, float* g_e, float* g_num, float* g_Dx,
                     cudaStream_t stream, Planes g_e_p = Planes(), Planes g_Dx_p = Planes(), const float* rho = nullptr,
                     float* g_den = nullptr);
// src-ordered backward pass: g_Ex_j = sum g_e_k, g_Bx_j = sum g_num[dst(k)] * sigmoid(ehat_k)
int gatedgcn_bwd_src(const GpsGraph& g, int64_t d, const float* g_e, const float* ehat, const float* g_num,
                     float* g_Ex, float* g_Bx, int64_t ldg, cudaStream_t stream, Planes g_Ex_p = Planes(),
                     Planes g_Bx_p = Planes(), const float* rho = nullptr);

// EquivStableLapPE edge gate (eslap.cu): PE [N,k] row-major; w1 = mlp_r_ij.0.weight [d,1], b1 [d], w2 = mlp_r_ij.2.weight
// [1,d], b2 [1].  Forward: r [E], rho [E].  Backward (after gatedgcn_bwd_dst with rho): per-edge scratch gz, gr [E] and
// part [ceil(E / eslap_wgrad_chunk(E)), 3d+1]; writes (or, accumulate, adds) the four mlp_r_ij gradients and writes grad_pe.
int64_t eslap_wgrad_chunk(int64_t E);
int eslap_fwd(const GpsGraph& g, const float* pe, int64_t k, int64_t d, int act, const float* w1, const float* b1,
              const float* w2, const float* b2, float* r, float* rho, cudaStream_t stream);
int eslap_bwd(const GpsGraph& g, const float* pe, int64_t k, int64_t d, int act, const float* g_num, const float* g_den,
              const float* Bx, int64_t ldy, const float* ehat, const float* r, const float* rho, const float* w1,
              const float* b1, const float* w2, float* gz, float* gr, float* part, float* grad_pe, float* gw1,
              float* gb1, float* gw2, float* gb2, bool accumulate, cudaStream_t stream);
int gine_fwd(const GpsGraph& g, int64_t d, const float* x, const float* e, float eps, float* out,
             cudaStream_t stream, Planes outp = Planes());
// g_e[k] = g_o[dst(k)] * [x_src + e_k > 0];  (dst ordered)
int gine_bwd_dst(const GpsGraph& g, int64_t d, const float* x, const float* e, const float* g_o, float* g_e,
                 cudaStream_t stream);
// g_x[j] = (1+eps) g_o[j] + sum_{k: src=j} g_e[k]  (+ add[j])
int gine_bwd_src(const GpsGraph& g, int64_t d, const float* g_e, const float* g_o, float eps, const float* add,
                 float* g_x, cudaStream_t stream);

// GCN (PyG GCNConv): dinv_i = (1 + #non-self in-edges)^-1/2; x_loc = x + drop(b + A_hat Y) [+ column sums of x_loc];
// backward gY = A_hat^T g_h
int gcn_dinv(const GpsGraph& g, float* dinv, cudaStream_t stream);
int gcn_fwd(const GpsGraph& g, int64_t d, const float* Y, int64_t ldy, const float* dinv, const float* bias,
            const float* x, float* xloc, DropCfg drop, double* stats, cudaStream_t stream);
int gcn_bwd(const GpsGraph& g, int64_t d, const float* g_h, const float* dinv, float* gY, int64_t ldg,
            cudaStream_t stream, Planes gYp = Planes());

// GAT (PyG GATConv, gat.cu).  H heads of C = d / H channels; Y [N, ldy] = x W_src^T; v [H, d] = fold(W_edge, att_edge).
// Scores saved by the forward, in one buffer of (4 N + E) H floats: a_src, a_dst, a_self (the added self loop's edge
// score), lse (log-sum-exp of each (node, head) softmax), each [N, H], then a_edge [E, H] in edge-id order.
struct GatScores {
  float *a_src, *a_dst, *a_self, *lse, *a_edge;
};
GatScores gat_scores(float* base, int64_t N, int64_t E, int64_t H);
// H > 0 with d % H == 0 (else GPS_ERR_ARG), d % 4 == 0 and d <= 4096 (else GPS_ERR_UNSUPPORTED)
int gat_check(int64_t d, int64_t H);
int gat_fold_fwd(const float* W_edge, const float* att_edge, int64_t d, int64_t H, float* v, cudaStream_t stream);
// g_W_edge[hC+c, :] = att_edge[hC+c] g_v[h];  g_att_edge[hC+c] = W_edge[hC+c, :] . g_v[h]  (written, or added)
int gat_fold_bwd(const float* W_edge, const float* att_edge, const float* g_v, int64_t d, int64_t H, float* gW,
                 float* gatt, bool accumulate, cudaStream_t stream);
// x_loc = x + drop(GATConv(x) + bias) [+ column sums of x_loc]
int gat_fwd(const GpsGraph& g, int64_t d, int64_t H, const float* Y, int64_t ldy, const float* ea, const float* v,
            const float* att_src, const float* att_dst, const float* bias, const float* x, GatScores s, float* xloc,
            DropCfg drop, double* stats, cudaStream_t stream);
// floats of scratch gat_bwd needs
int64_t gat_bwd_workspace_floats(int64_t N, int64_t E, int64_t H, int64_t d);
// from g_h (the gradient of the aggregation output, bias included): gY [N, ldg] (+ planes), grad_ea [E, d] (NULL = not
// needed), g_v [H, d] (written), and g_att_src / g_att_dst / g_bias (each NULL = not needed; written, or added)
int gat_bwd(const GpsGraph& g, int64_t d, int64_t H, const float* Y, int64_t ldy, const float* ea, const float* v,
            const float* att_src, const float* att_dst, GatScores s, const float* g_h, float* ws, float* gY, int64_t ldg,
            Planes gYp, float* grad_ea, float* g_v, float* g_att_src, float* g_att_dst, float* g_bias, bool accumulate,
            cudaStream_t stream);

// GENConv (PyG GENConv, softmax aggregation, genconv.cu).  Forward: agg, lse (log-sum-exp of each (node, channel)
// segment, 0 without in-edges) and u = agg + x, all [N, d], plus u's planes.  Backward, dst ordered:
// g_e[k] = g_u[dst] alpha_k (1 + m_k - agg[dst]) [x_src + e_k > 0]; the src-ordered pass is gine_bwd_src with eps = 0.
int genconv_fwd(const GpsGraph& g, int64_t d, const float* x, const float* e, float* agg, float* lse, float* u,
                cudaStream_t stream, Planes up = Planes());
int genconv_bwd_dst(const GpsGraph& g, int64_t d, const float* x, const float* e, const float* agg, const float* lse,
                    const float* g_u, float* g_e, cudaStream_t stream);

// PNA (PyG PNAConv, mean / max / sum aggregation, pna.cu).  pna_check: 0 < de <= d, de % 4 == 0.  Fold: F = W_e W_enc
// [d, de] and c = W_e b_enc + b_pre [d], W_e the column block 2d..3d of W_pre [d, 3d]; its backward writes (or, with
// accumulate, adds) the gradients of W_pre's block 2d..3d, b_pre, W_enc and b_enc from g_F [d, de] and g_c [d] (each
// output NULL = not needed).  Forward: m_k = Y[i, 0:d] + Y[j, d:2d] + q[k] (Y = [P_dst | P_src | ...] with pitch ldy),
// Z = [x | mean | max | sum] [N, 4d] (fp32 when Z != NULL, planes when Zp.hi), arg [N, d] = edge id of the first
// maximiser (-1 without in-edges).  Backward from g_Z [N, 4d]: g_q [E, d] (+ planes), g_P_dst into gY[:, 0:d] and
// g_P_src into gY[:, d:2d] (+ planes), g_x = add + g_Z[:, 0:d] (add NULL = none).
int pna_check(int64_t d, int64_t de);
int pna_fold_fwd(const float* Wpre, const float* bpre, const float* Wenc, const float* benc, int64_t d, int64_t de,
                 float* F, float* cvec, cudaStream_t st);
int pna_fold_bwd(const float* Wpre, const float* Wenc, const float* benc, const float* gF, const float* gc, int64_t d,
                 int64_t de, float* gWpre, float* gbpre, float* gWenc, float* gbenc, bool accumulate, cudaStream_t st);
int pna_fwd(const GpsGraph& g, int64_t d, const float* x, const float* Y, int64_t ldy, const float* q, float* Z,
            Planes Zp, int* arg, cudaStream_t stream);
int pna_bwd(const GpsGraph& g, int64_t d, const float* gZ, const int* arg, const float* add, float* g_q, Planes gqp,
            float* gY, int64_t ldg, Planes gYp, float* g_x, cudaStream_t stream);

// ---- attention ------------------------------------------------------------------------------
int attention_fwd(const GpsGraph& g, int64_t heads, int64_t hd, const float* Q, const float* K, const float* V,
                  int64_t ld, float* O, int64_t ldo, float* lse, float p_drop, uint64_t seed, uint64_t offset,
                  cudaStream_t stream, const unsigned long long* offset_dev = nullptr, Planes Op = Planes(),
                  const GpsAttnBias* bias = nullptr);
// bias (BiasedTransformer): NULL = none; its grad_bias, when set, is written whole by attention_bwd (padding zeroed)
int attention_bwd(const GpsGraph& g, int64_t heads, int64_t hd, const float* Q, const float* K, const float* V,
                  int64_t ld, const float* O, const float* dO, int64_t ldo, const float* lse, float* delta,
                  float* dQ, float* dK, float* dV, int64_t ldg, float p_drop, uint64_t seed, uint64_t offset,
                  cudaStream_t stream, const unsigned long long* offset_dev = nullptr, Planes dQp = Planes(),
                  Planes dKp = Planes(), Planes dVp = Planes(), const GpsAttnBias* bias = nullptr);

// BigBird (bigbird.cu).  bb_check: a usable GpsBigBird for d / H (GPS_ERR_ARG, or GPS_ERR_UNSUPPORTED for hd > 128).
// Block-sparse attention over the packed rows: forward O, lse [N, H]; backward delta [N, H], then dQ, dK, dV written
// whole.  LayerNorm: out = [R1 +] drop(LN(z)) [+ R2] (+ planes, + double column sums into stats [2][d]), mean / rstd
// [rows] saved.  Its backward from g' = gdrop(g): out1 = drop1(dz) (+ planes), out2 = dz (+ add) (each NULL = not
// wanted), grad_gamma / grad_beta through part (layernorm_part_floats(d) floats), written or added.
int bb_check(int64_t d, int64_t H, const GpsBigBird* bb);
int bb_attn_fwd(const GpsGraph& g, int64_t H, int64_t hd, const GpsBigBird& bb, const float* Q, const float* K,
                const float* V, int64_t ld, float* O, int64_t ldo, float* lse, cudaStream_t stream);
int bb_attn_bwd(const GpsGraph& g, int64_t H, int64_t hd, const GpsBigBird& bb, const float* Q, const float* K,
                const float* V, int64_t ld, const float* O, const float* dO, int64_t ldo, const float* lse, float* delta,
                float* dQ, float* dK, float* dV, int64_t ldg, cudaStream_t stream);
int64_t layernorm_part_floats(int64_t d);
int layernorm_fwd(const float* z, int64_t rows, int64_t d, const float* gamma, const float* beta, float eps, float* mean,
                  float* rstd, float* out, Planes outp, const float* R1, const float* R2, DropCfg drop, double* stats,
                  cudaStream_t stream);
int layernorm_bwd(const float* g, DropCfg gdrop, const float* z, int64_t rows, int64_t d, const float* gamma,
                  const float* mean, const float* rstd, float* out1, Planes out1p, DropCfg drop1, float* out2,
                  const float* add, float* part, float* grad_gamma, float* grad_beta, bool accumulate,
                  cudaStream_t stream);
// sigmoid in place (+ planes); its backward g *= s (1 - s) in place (+ planes)
int sigmoid_fwd(float* x, int64_t rows, int64_t d, Planes p, cudaStream_t stream);
int sigmoid_bwd(float* g, const float* s, int64_t rows, int64_t d, Planes p, cudaStream_t stream);

// wgmma version (attention_tc.cu): Q, K, V from bf16 hi/lo planes in the per-head padded layout
// column (which * H + h) * hd_pad + k, hd_pad = attention_tc_hd_pad(hd), pad columns zero
void attention_tc_set_debug(float* buf);   // bring-up: 3 x 128 x 128 floats (S, P, raw O of CTA (0,0))
bool attention_tc_supported(int64_t hd);
int64_t attention_tc_hd_pad(int64_t hd);
int attention_tc_fwd(const GpsGraph& g, int64_t heads, int64_t hd, Planes qkv, float* O, int64_t ldo, Planes Op, float* lse,
                     float p_drop, uint64_t seed, uint64_t offset, const unsigned long long* offset_dev, int precision,
                     cudaStream_t stream, const GpsAttnBias* bias = nullptr);

}  // namespace gps
