// graphormer.cu — host-side orchestration of the Graphormer layer (graphgps/layer/graphormer_layer.py:39-49) and its C
// ABI.  Every stage is an existing kernel:
//   forward:  LN_in (+ planes of h) -> [Q|K|V] = h W_in^T + b_in (+ the padded per-head planes of the wgmma attention)
//             -> attention (+ bias) -> x1 = x + drop_10(O Wo^T + bo) -> LN_mlp (+ planes)
//             -> hid = drop_11(GELU(h2 W1^T + b1)) (+ planes) -> x_out = x1 + drop_12(hid W2^T + b2)
//   backward: the mirror image; the weight products run on the side stream, the LayerNorm parameter gradients go
//             through layernorm_bwd's per-CTA partials.  No float atomics.
#include <string.h>

#include "layer_ops.cuh"

namespace gps {

namespace {

constexpr float kLnEps = 1e-5f;   // nn.LayerNorm's default, as the reference builds input_norm and mlp.0

struct GrPlan {
  int64_t N, d, H, hd;
  int prec;
  bool train, grads_prezeroed, grads_accumulate, use_planes, attn_tc;
  DropCfg drop_attn, drop_mlp, drop_out;   // sites 10, 11, 12 (p = 0 in eval mode)
  float pa;                                // attention dropout, 0 in eval mode
  // saved: row statistics mean_in | rstd_in | mean_mlp | rstd_mlp [4][N], h = LN_in(x), Y = [Q|K|V] [N, 3d], O, lse
  // [N, H], x1, h2 = LN_mlp(x1), hid (after GELU and dropout), hid_pre; the weight planes
  float *stat, *h, *Y, *O, *lse, *x1, *h2, *hid, *hid_pre;
  Planes h_p, O_p, h2_p, hid_p, win_p, wout_p, w1_p, w2_p;
  int64_t saved_bytes;
  // forward workspace: Q | K | V as padded per-head planes (wgmma attention only)
  Planes qkv_p;
  int64_t fwd_bytes;
  // backward workspace
  float *g_a, *g_hid, *g_h2, *g_x1, *g_b, *g_O, *delta, *gY, *g_h, *part;
  Planes ga_p, ghid_p, gb_p, gY_p;
  int64_t bwd_bytes;
};

int make_plan(const GpsGraphormerArgs* a, GrPlan* P, bool bind) {
  memset(P, 0, sizeof(*P));
  GPS_REQUIRE(a, GPS_ERR_ARG, "graphormer: null args");
  GPS_REQUIRE(a->heads > 0 && a->d > 0 && a->d % a->heads == 0, GPS_ERR_ARG,
              "graphormer: embed_dim %lld must be a positive multiple of num_heads %lld", (long long)a->d,
              (long long)a->heads);
  GPS_REQUIRE(a->d % 4 == 0 && a->d <= 4096, GPS_ERR_UNSUPPORTED,
              "graphormer: embed_dim must be a multiple of 4 and <= 4096 (got %lld)", (long long)a->d);
  GPS_REQUIRE(a->d / a->heads <= 192, GPS_ERR_UNSUPPORTED, "graphormer: head dim %lld > 192 is not built",
              (long long)(a->d / a->heads));
  GPS_REQUIRE(a->precision == GPS_PREC_FP32 || a->precision == GPS_PREC_BF16, GPS_ERR_ARG,
              "graphormer: unknown precision %d", a->precision);
  GPS_REQUIRE(a->graph.N >= 0 && a->graph.B >= 0, GPS_ERR_ARG, "graphormer: negative graph sizes");
  GPS_REQUIRE(a->dropout >= 0.f && a->dropout < 1.f && a->attn_dropout >= 0.f && a->attn_dropout < 1.f &&
                  a->mlp_dropout >= 0.f && a->mlp_dropout < 1.f,
              GPS_ERR_ARG, "graphormer: dropout probabilities must be in [0,1)");
  const int64_t N = a->graph.N, d = a->d;
  P->N = N; P->d = d; P->H = a->heads; P->hd = d / a->heads;
  P->prec = a->precision;
  P->train = a->training != 0;
  set_grad_flags(P, a->flags);
  P->drop_attn = drop_cfg(a->dropout, P->train, a->seed, a->offset, a->offset_dev, GPS_SITE_GR_ATTN);
  P->drop_mlp = drop_cfg(a->mlp_dropout, P->train, a->seed, a->offset, a->offset_dev, GPS_SITE_GR_MLP);
  P->drop_out = drop_cfg(a->dropout, P->train, a->seed, a->offset, a->offset_dev, GPS_SITE_GR_OUT);
  P->pa = P->train ? a->attn_dropout : 0.f;
  P->use_planes = d % 8 == 0;
  const bool lo = a->precision == GPS_PREC_FP32;

  Arena S(bind ? a->saved : nullptr, a->saved_bytes);
  P->stat = S.alloc<float>(4 * N);
  P->h = S.alloc<float>(N * d);
  P->Y = S.alloc<float>(N * 3 * d);
  P->O = S.alloc<float>(N * d);
  P->lse = S.alloc<float>(N * P->H);
  P->x1 = S.alloc<float>(N * d);
  P->h2 = S.alloc<float>(N * d);
  P->hid = S.alloc<float>(N * d);
  P->hid_pre = S.alloc<float>(N * d);
  if (P->use_planes) {
    P->h_p = arena_planes(S, N, d, lo);
    P->O_p = arena_planes(S, N, d, lo);
    P->h2_p = arena_planes(S, N, d, lo);
    P->hid_p = arena_planes(S, N, d, lo);
    P->win_p = arena_planes(S, 3 * d, d, lo);
    P->wout_p = arena_planes(S, d, d, lo);
    P->w1_p = arena_planes(S, d, d, lo);
    P->w2_p = arena_planes(S, d, d, lo);
  }
  P->saved_bytes = S.used;
  GPS_REQUIRE(!S.overflow, GPS_ERR_ARG, "graphormer: saved buffer too small (%lld < %lld)", (long long)a->saved_bytes,
              (long long)S.used);

  // the wgmma forward when the graphs fill its tiles (as GPSLayer decides, layer.cu)
  P->attn_tc = P->use_planes && attention_tc_supported(P->hd) && a->graph.B > 0 && N >= 64 * a->graph.B;
  Arena F(bind ? a->workspace : nullptr, a->workspace_bytes);
  if (P->attn_tc) P->qkv_p = arena_planes(F, N, 3 * P->H * attention_tc_hd_pad(P->hd), lo);
  P->fwd_bytes = F.used;

  Arena Bk(bind ? a->workspace : nullptr, a->workspace_bytes);
  P->g_a = Bk.alloc<float>(N * d);
  P->g_hid = Bk.alloc<float>(N * d);
  P->g_h2 = Bk.alloc<float>(N * d);
  P->g_x1 = Bk.alloc<float>(N * d);
  P->g_b = Bk.alloc<float>(N * d);
  P->g_O = Bk.alloc<float>(N * d);
  P->delta = Bk.alloc<float>(N * P->H);
  P->gY = Bk.alloc<float>(N * 3 * d);
  P->g_h = Bk.alloc<float>(N * d);
  P->part = Bk.alloc<float>(layernorm_part_floats(d));
  if (P->use_planes) {
    P->ga_p = arena_planes(Bk, N, d, lo);
    P->ghid_p = arena_planes(Bk, N, d, lo);
    P->gb_p = arena_planes(Bk, N, d, lo);
    P->gY_p = arena_planes(Bk, N, 3 * d, lo);
  }
  P->bwd_bytes = Bk.used;
  return GPS_OK;
}

int check_params(const GpsGraphormerArgs* a) {
  const struct { const GpsLinear* l; const char* name; } ps[] = {
      {&a->input_norm, "input_norm"}, {&a->attn_in, "attention.in_proj"}, {&a->attn_out, "attention.out_proj"},
      {&a->mlp_norm, "mlp.0"},        {&a->mlp_lin1, "mlp.1"},             {&a->mlp_lin2, "mlp.4"}};
  for (const auto& p : ps)
    GPS_REQUIRE(p.l->weight && p.l->bias, GPS_ERR_ARG, "graphormer: missing parameter %s.{weight,bias}", p.name);
  return GPS_OK;
}

int check_bias(const GpsAttnBias* bias) {
  if (!bias) return GPS_OK;
  GPS_REQUIRE(bias->bias, GPS_ERR_ARG, "graphormer: null attention bias pointer");
  GPS_REQUIRE(bias->nmax >= 1, GPS_ERR_ARG, "graphormer: attention bias nmax must be >= 1 (got %lld)",
              (long long)bias->nmax);
  return GPS_OK;
}

// plan, buffers and parameters of one call, all before any CUDA call
int prepare(const GpsGraphormerArgs* a, const GpsAttnBias* bias, bool fwd, GrPlan* P) {
  GPS_TRY(make_plan(a, P, true));
  GPS_TRY(check_params(a));
  GPS_TRY(check_bias(bias));
  GPS_REQUIRE(a->x && a->saved && a->workspace, GPS_ERR_ARG, "graphormer: x, saved and workspace are required");
  const int64_t ws = fwd ? P->fwd_bytes : P->bwd_bytes;
  GPS_REQUIRE(a->workspace_bytes >= ws, GPS_ERR_ARG, "graphormer: workspace too small (%lld < %lld)",
              (long long)a->workspace_bytes, (long long)ws);
  if (fwd) GPS_REQUIRE(a->x_out, GPS_ERR_ARG, "graphormer: x_out is required");
  else GPS_REQUIRE(a->grad_x_out && a->grad_x, GPS_ERR_ARG, "graphormer: grad_x_out and grad_x are required");
  return GPS_OK;
}

// =================================================================================== forward
int graphormer_forward(const GpsGraphormerArgs* a, const GpsAttnBias* bias, cudaStream_t st) {
  GrPlan P;
  GPS_TRY(prepare(a, bias, true, &P));
  const int64_t N = P.N, d = P.d;
  if (N == 0) return GPS_OK;
  float* stat = P.stat;
  if (P.use_planes) {   // the four weights -> bf16 hi/lo planes, one launch
    const ToPlanesItem it[4] = {{a->attn_in.weight, d, (int)(3 * d), (int)d, P.win_p},
                                {a->attn_out.weight, d, (int)d, (int)d, P.wout_p},
                                {a->mlp_lin1.weight, d, (int)d, (int)d, P.w1_p},
                                {a->mlp_lin2.weight, d, (int)d, (int)d, P.w2_p}};
    GPS_TRY(to_planes(it, 4, st));
  }
  // h = input_norm(x)
  GPS_TRY(layernorm_fwd(a->x, N, d, a->input_norm.weight, a->input_norm.bias, kLnEps, stat, stat + N, P.h, P.h_p,
                        nullptr, nullptr, DropCfg(), nullptr, st));
  // [Q|K|V] = h W_in^T + b_in  (MHA in_proj)
  GemmParams gq = linear_fwd(P, N, 3 * d, d, {P.h, d, P.h_p}, {a->attn_in.weight, d, P.win_p}, P.Y, 3 * d,
                             a->attn_in.bias);
  if (P.attn_tc) {
    gq.Cp = P.qkv_p; gq.cp_hd = (int)P.hd; gq.cp_hd_pad = (int)attention_tc_hd_pad(P.hd);
  }
  GPS_TRY(gemm(gq, st));
  // attention over each graph's own nodes (to_dense_batch + key_padding_mask + [real_nodes])
  const unsigned long long* odev = (const unsigned long long*)a->offset_dev;
  if (P.attn_tc)
    GPS_TRY(attention_tc_fwd(a->graph, P.H, P.hd, P.qkv_p, P.O, d, P.O_p, P.lse, P.pa, a->seed, a->offset, odev, P.prec,
                             st, bias));
  else
    GPS_TRY(attention_fwd(a->graph, P.H, P.hd, P.Y, P.Y + d, P.Y + 2 * d, 3 * d, P.O, d, P.lse, P.pa, a->seed,
                          a->offset, st, odev, P.O_p, bias));
  // x1 = x + drop(O Wo^T + bo)
  GemmParams g = linear_fwd(P, N, d, d, {P.O, d, P.O_p}, {a->attn_out.weight, d, P.wout_p}, P.x1, d, a->attn_out.bias);
  g.R1 = a->x; g.ldr1 = (int)d;
  set_dropout(g, P.drop_attn);
  GPS_TRY(gemm(g, st));
  // h2 = mlp.0(x1)
  GPS_TRY(layernorm_fwd(P.x1, N, d, a->mlp_norm.weight, a->mlp_norm.bias, kLnEps, stat + 2 * N, stat + 3 * N, P.h2,
                        P.h2_p, nullptr, nullptr, DropCfg(), nullptr, st));
  // hid = mlp.3(GELU(mlp.1(h2)))
  GemmParams g1 = linear_fwd(P, N, d, d, {P.h2, d, P.h2_p}, {a->mlp_lin1.weight, d, P.w1_p}, P.hid, d, a->mlp_lin1.bias);
  g1.act = GPS_ACT_GELU; g1.C_pre = P.hid_pre; g1.ldpre = (int)d; g1.Cp = P.hid_p;
  set_dropout(g1, P.drop_mlp);
  GPS_TRY(gemm(g1, st));
  // x_out = x1 + mlp.5(mlp.4(hid))
  GemmParams g2 = linear_fwd(P, N, d, d, {P.hid, d, P.hid_p}, {a->mlp_lin2.weight, d, P.w2_p}, a->x_out, d,
                             a->mlp_lin2.bias);
  g2.R1 = P.x1; g2.ldr1 = (int)d;
  set_dropout(g2, P.drop_out);
  return gemm(g2, st);
}

// The [N, d] gradient g in front of the dropout c, with planes: dropmul_rows into tmp when the dropout is active, else
// g itself with its planes converted into tmp_p.  One launch either way.
int dropped_operand(const GrPlan& P, const float* g, const DropCfg& c, float* tmp, Planes tmp_p, cudaStream_t st,
                    Operand* out) {
  if (c.p > 0.f) {
    *out = Operand{tmp, P.d, tmp_p};
    return dropmul_rows(g, tmp, P.N, P.d, c, 0.f, 0, tmp_p, st);
  }
  *out = Operand{g, P.d, tmp_p};
  if (!tmp_p.hi) return GPS_OK;
  ToPlanesItem it{g, P.d, (int)P.N, (int)P.d, tmp_p};
  return to_planes(&it, 1, st);
}

// =================================================================================== backward
int graphormer_backward(const GpsGraphormerArgs* a, const GpsAttnBias* bias, cudaStream_t st) {
  GrPlan P;
  GPS_TRY(prepare(a, bias, false, &P));
  const int64_t N = P.N, d = P.d;
  const float* stat = P.stat;
  const DropCfg nodrop;
  Side* sd;
  GPS_TRY(side_stream(&sd));
  cudaStream_t s2 = sd->s;
  if (N == 0) {   // no rows: the parameter gradients are zero (or unchanged when accumulating)
    if (!P.grads_prezeroed) {
      const GpsLinear* ls[6] = {&a->input_norm, &a->attn_in, &a->attn_out, &a->mlp_norm, &a->mlp_lin1, &a->mlp_lin2};
      const int64_t rows[6] = {d, 3 * d, d, d, d, d}, cols[6] = {1, d, d, 1, d, d};
      GPS_TRY(zero_linear_grads(ls, rows, cols, 6, st));
    }
    if (bias && bias->grad_bias)
      GPS_CUDA(cudaMemsetAsync(bias->grad_bias, 0, (size_t)(a->graph.B * P.H * bias->nmax * bias->nmax) * sizeof(float),
                               st));
    return GPS_OK;
  }
  // x_out = x1 + drop_12(hid W2^T + b2): g_a = drop_12(g_out), the gradient of mlp.4's output
  Operand g_a;
  GPS_TRY(dropped_operand(P, a->grad_x_out, P.drop_out, P.g_a, P.ga_p, st, &g_a));
  // g_hid = (g_a W2) * GELU'(pre) * drop_11
  GemmParams g = linear_dgrad(P, N, d, d, g_a, {a->mlp_lin2.weight, d, P.w2_p}, P.g_hid, d);
  set_act_mask(g, GPS_ACT_GELU, P.hid, P.hid_pre, d);
  set_dropout(g, P.drop_mlp);
  g.Cp = P.ghid_p;
  GPS_TRY(gemm(g, st));
  const Operand g_hid{P.g_hid, d, P.ghid_p};
  GPS_TRY(sd->fork(st));
  GPS_TRY(linear_wgrad(P, g_a, {P.hid, d, P.hid_p}, N, d, d, a->mlp_lin2.grad_weight, a->mlp_lin2.grad_bias, s2));
  GPS_TRY(linear_wgrad(P, g_hid, {P.h2, d, P.h2_p}, N, d, d, a->mlp_lin1.grad_weight, a->mlp_lin1.grad_bias, s2));
  // g_h2 = g_hid W1; mlp.0: g_x1 = LN_mlp'(g_h2) + g_out
  GPS_TRY(gemm(linear_dgrad(P, N, d, d, g_hid, {a->mlp_lin1.weight, d, P.w1_p}, P.g_h2, d), st));
  GPS_TRY(layernorm_bwd(P.g_h2, nodrop, P.x1, N, d, a->mlp_norm.weight, stat + 2 * N, stat + 3 * N, nullptr, Planes(),
                        nodrop, P.g_x1, a->grad_x_out, P.part, a->mlp_norm.grad_weight, a->mlp_norm.grad_bias,
                        P.grads_accumulate, st));
  // x1 = x + drop_10(O Wo^T + bo): g_b = drop_10(g_x1); g_O = g_b Wo
  Operand g_b;
  GPS_TRY(dropped_operand(P, P.g_x1, P.drop_attn, P.g_b, P.gb_p, st, &g_b));
  GPS_TRY(gemm(linear_dgrad(P, N, d, d, g_b, {a->attn_out.weight, d, P.wout_p}, P.g_O, d), st));
  GPS_TRY(sd->fork(st));
  GPS_TRY(linear_wgrad(P, g_b, {P.O, d, P.O_p}, N, d, d, a->attn_out.grad_weight, a->attn_out.grad_bias, s2));
  // attention: dQ | dK | dV into gY (+ planes), grad_bias
  GPS_TRY(attention_bwd(a->graph, P.H, P.hd, P.Y, P.Y + d, P.Y + 2 * d, 3 * d, P.O, P.g_O, d, P.lse, P.delta, P.gY,
                        P.gY + d, P.gY + 2 * d, 3 * d, P.pa, a->seed, a->offset, st,
                        (const unsigned long long*)a->offset_dev, P.gY_p.cols(0), P.gY_p.cols(d), P.gY_p.cols(2 * d),
                        bias));
  const Operand gY{P.gY, 3 * d, P.gY_p};
  GPS_TRY(sd->fork(st));
  GPS_TRY(linear_wgrad(P, gY, {P.h, d, P.h_p}, N, 3 * d, d, a->attn_in.grad_weight, a->attn_in.grad_bias, s2));
  // g_h = gY W_in; input_norm: grad_x = LN_in'(g_h) + g_x1
  GPS_TRY(gemm(linear_dgrad(P, N, d, 3 * d, gY, {a->attn_in.weight, d, P.win_p}, P.g_h, d), st));
  GPS_TRY(layernorm_bwd(P.g_h, nodrop, a->x, N, d, a->input_norm.weight, stat, stat + N, nullptr, Planes(), nodrop,
                        a->grad_x, P.g_x1, P.part, a->input_norm.grad_weight, a->input_norm.grad_bias,
                        P.grads_accumulate, st));
  return sd->join(st);
}

}  // namespace

}  // namespace gps

// =================================================================================== C ABI
using namespace gps;

extern "C" int gps_graphormer_plan(const GpsGraphormerArgs* args, GpsGraphormerPlan* plan) {
  GPS_REQUIRE(args && plan, GPS_ERR_ARG, "gps_graphormer_plan: null argument");
  GrPlan P;
  GPS_TRY(make_plan(args, &P, false));
  plan->saved_bytes = P.saved_bytes;
  plan->fwd_workspace_bytes = P.fwd_bytes;
  plan->bwd_workspace_bytes = P.bwd_bytes;
  return GPS_OK;
}

extern "C" int gps_graphormer_forward(const GpsGraphormerArgs* args, const GpsAttnBias* bias, void* stream) {
  return graphormer_forward(args, bias, (cudaStream_t)stream);
}

extern "C" int gps_graphormer_backward(const GpsGraphormerArgs* args, const GpsAttnBias* bias, void* stream) {
  return graphormer_backward(args, bias, (cudaStream_t)stream);
}
