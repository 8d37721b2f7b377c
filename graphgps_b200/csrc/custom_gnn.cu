// custom_gnn.cu — the message-passing layers of CustomGNN (graphgps/network/custom_gnn.py:31-37) as the LRGB GatedGCN
// and GINE configs stack them: GatedGCNLayer (gatedgcn_layer.py:11-136) and GINEConvLayer (gine_conv_layer.py:90-116),
// forward and backward, one C call per direction, and their C ABI.
//
// Widths.  The sparse and row-wise kernels take d % 4 == 0 and the TMA GEMM takes operand planes with a pitch that is a
// multiple of 8, but the configs use d = 108, 138, 166 and 208.  So every intermediate runs at the pitch
// dp = round_up(d, 8) with its pad columns exactly zero, and the existing kernels run unchanged at width dp:
//   - the weight planes get zero pad rows and columns and the biases zero pad entries, so every pre-activation, Ce and
//     e_ij is 0 in the pad columns; sigmoid(0) Bx_pad = 0, so xt_pad = Ax_pad = 0;
//   - a BatchNorm over an all-zero column gives beta_pad = 0 (the padded gamma / beta are zero), relu(0) = gelu(0) = 0,
//     and the residual adds the zero pad columns of the input;
//   - in the backward the incoming gradients are zero in the pad columns and stay so through every stage, and the pad
//     rows / columns of the weight gradients are dropped.
// Only the boundary is new: k_pad copies [rows, d] blocks at pitch d into zero-padded blocks at pitch dp (and / or their
// bf16 planes), and back; the BatchNorms read [dp] copies of gamma, beta and the running statistics, whose [d] part is
// written back to the module's buffers in the same call.  At d % 8 == 0 (dp = d) the caller's tensors are used in place.
// Padding 108 (d % 8 == 4) also keeps its weight gradients off the fp32 split-K path, which accumulates with atomics.
//
// GatedGCN:  forward  pack -> [Ax|Bx|Dx|Ex] = x Wcat^T + b (Ce = e C^T + bC on the side stream) -> gatedgcn_fwd (both
//                     BatchNorms' column sums) -> bn_act_residual2 -> unpack
//            backward the edge BatchNorm on its own stream next to the node BatchNorm -> gatedgcn_bwd_dst / _src ->
//                     grad_x = gY Wcat (+ grad_x_out), grad_edge_attr = g_e C (+ grad_edge_out); weight products on
//                     the side stream -> unpack
// GINE:      forward  pack -> gine_fwd -> h = relu(agg W0^T + b0) -> x_out = [x +] drop(relu(h W1^T + b1)) -> unpack
//            backward g2 = g_out drop relu'(.) (k_gine_gout) -> g_h -> g_agg -> gine_bwd_dst / _src -> unpack
#include <string.h>

#include "layer_ops.cuh"

namespace gps {

namespace {

// ------------------------------------------------------------------------------- pad / unpad (PadList: layer_ops.cuh)
struct PadDesc {
  PadItem it[kPadItems];
  int start[kPadItems + 1];   // first block of each item in the 1-D grid
  int n;
};

// one thread per 4 consecutive columns of a row; scalar loads, since the source pitch may be odd
__global__ void k_pad(PadDesc d) {
  int item = 0;
  while (item + 1 < d.n && (int)blockIdx.x >= d.start[item + 1]) ++item;
  const PadItem& it = d.it[item];
  const int g4 = (it.cols_p + 3) >> 2;
  const int64_t idx = ((int64_t)blockIdx.x - d.start[item]) * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)it.rows_p * g4) return;
  const int64_t r = idx / g4;
  const int c = (int)(idx - r * g4) * 4;
  float v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = r < it.rows && c + j < it.cols ? it.src[r * it.lds + c + j] : 0.f;
  if (it.dst) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (c + j < it.cols_p) it.dst[r * it.ldd + c + j] = v[j];
  }
  if (it.p.hi) planes_store4(it.p, r, c, make_float4(v[0], v[1], v[2], v[3]));
}

// GINE backward head: g2 = g_out * drop * [pre > 0] at pitch dp (+ planes), with g_out read at pitch ldg and its
// columns >= d taken as zero; gpad != NULL: also the zero-padded copy of g_out (the residual's share of grad_x)
__global__ void k_gine_gout(const float* __restrict__ g, int64_t ldg, int d, const float* __restrict__ pre, int dp,
                            int64_t N, DropCfg drop, float* __restrict__ g2, Planes g2p, float* __restrict__ gpad) {
  const int C4 = dp >> 2;
  if (drop.p > 0.f && drop.offset_dev) drop.offset += *drop.offset_dev;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N * C4; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / C4;
    const int c = (int)(i - r * C4) * 4;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = c + j < d ? g[r * ldg + c + j] : 0.f;
    const float4 gv = make_float4(v[0], v[1], v[2], v[3]);
    if (gpad) st4(gpad + r * dp + c, gv);
    const float4 p = ld4(pre + r * dp + c);
    float4 o = make_float4(p.x > 0.f ? gv.x : 0.f, p.y > 0.f ? gv.y : 0.f, p.z > 0.f ? gv.z : 0.f, p.w > 0.f ? gv.w : 0.f);
    if (drop.p > 0.f) o = f4mul(o, dropout_scale4(drop.p, drop.seed, drop.offset, drop.site, (uint64_t)i));
    st4(g2 + r * dp + c, o);
    if (g2p.hi) planes_store4(g2p, r, c, o);
  }
}

// =================================================================================== plan
struct CgPlan {
  int64_t N, E, d, dp;
  int kind, act, prec;
  bool train, pad, residual, gated;
  bool grads_prezeroed = true;   // linear_wgrad: the gradient region is zeroed once per backward call
  float eps;
  DropCfg drop_x, drop_e;        // sites 15, 4095 (p = 0 in eval mode)
  // persistent (wplanes): GatedGCN W = [A|B|D|E] [4dp, dp], W2 = C; GINE W = nn.0, W2 = nn.2; biases b1 / b2 of the
  // same row counts; GatedGCN's BatchNorm affine parameters bnw = gamma_x | beta_x | gamma_e | beta_e [4][dp]
  Planes W_p, W2_p;
  float *b1, *b2, *bnw;
  int64_t wplanes_bytes;
  // saved: the padded inputs (pad only) and their planes, GatedGCN's Y [N, 4dp], ehat [E, dp], xt [N, dp], saved
  // BatchNorm statistics bnbuf [2][2dp] and padded running statistics rs [4][dp] (pad only); GINE's agg, h, pre2
  float *x, *e, *Y, *ehat, *xt, *bnbuf, *rs, *agg, *h, *pre2;
  Planes x_p, e_p, agg_p, h_p;
  int64_t saved_bytes;
  // forward workspace: BatchNorm column sums [2][2dp], the unread column sums of x_out, padded outputs (pad only)
  double *fstats, *sink;
  float *xo, *eo;
  int64_t fwd_bytes;
  // backward workspace
  double* bsums;
  float *gxo, *geo, *gx, *gea, *gY, *ge, *gnum, *g2, *gh, *gagg;
  Planes gY_p, ge_p, g2_p, gh_p;
  float* grads;          // every parameter gradient at pitch dp, zeroed as one region
  int64_t grads_bytes;
  int64_t bwd_bytes;
};

int make_plan(const GpsCustomGnnArgs* a, CgPlan* P, bool bind) {
  memset(P, 0, sizeof(*P));
  P->grads_prezeroed = true;
  GPS_REQUIRE(a, GPS_ERR_ARG, "custom_gnn: null args");
  GPS_REQUIRE(a->kind == GPS_CUSTOM_GATEDGCN || a->kind == GPS_CUSTOM_GINE, GPS_ERR_ARG, "custom_gnn: unknown kind %d",
              a->kind);
  GPS_REQUIRE(a->d > 0, GPS_ERR_ARG, "custom_gnn: d must be positive (got %lld)", (long long)a->d);
  GPS_REQUIRE(a->d <= 4096, GPS_ERR_UNSUPPORTED, "custom_gnn: d <= 4096 (got %lld)", (long long)a->d);
  GPS_REQUIRE(a->precision == GPS_PREC_FP32 || a->precision == GPS_PREC_BF16, GPS_ERR_ARG,
              "custom_gnn: unknown precision %d", a->precision);
  GPS_REQUIRE(a->kind != GPS_CUSTOM_GATEDGCN || a->act == GPS_ACT_RELU || a->act == GPS_ACT_GELU, GPS_ERR_ARG,
              "custom_gnn: unknown act %d", a->act);
  GPS_REQUIRE(a->graph.N >= 0 && a->graph.E >= 0 && a->graph.B >= 0, GPS_ERR_ARG, "custom_gnn: negative graph sizes");
  GPS_REQUIRE(a->dropout >= 0.f && a->dropout < 1.f, GPS_ERR_ARG, "custom_gnn: dropout must be in [0,1)");
  GPS_REQUIRE(a->flags == 0, GPS_ERR_ARG, "custom_gnn: flags are reserved (got %d)", a->flags);
  const int64_t N = a->graph.N, E = a->graph.E, d = a->d, dp = round_up(d, 8);
  P->N = N; P->E = E; P->d = d; P->dp = dp;
  P->kind = a->kind; P->gated = a->kind == GPS_CUSTOM_GATEDGCN;
  P->act = P->gated ? a->act : GPS_ACT_RELU;
  P->prec = a->precision;
  P->train = a->training != 0;
  P->pad = dp != d;
  P->residual = a->residual != 0;
  P->eps = a->gine_eps;
  P->drop_x = drop_cfg(a->dropout, P->train, a->seed, a->offset, a->offset_dev, GPS_SITE_CG_X);
  P->drop_e = drop_cfg(a->dropout, P->train, a->seed, a->offset, a->offset_dev, GPS_SITE_CG_E);
  const bool lo = a->precision == GPS_PREC_FP32;
  const int64_t wrows = P->gated ? 4 * dp : dp;   // rows of the first product's weight

  Arena W(bind ? a->wplanes : nullptr, a->wplanes_bytes);
  P->W_p = arena_planes(W, wrows, dp, lo);
  P->W2_p = arena_planes(W, dp, dp, lo);
  P->b1 = W.alloc<float>(wrows);
  P->b2 = W.alloc<float>(dp);
  if (P->gated) P->bnw = W.alloc<float>(4 * dp);
  P->wplanes_bytes = W.used;
  GPS_REQUIRE(!bind || !W.overflow, GPS_ERR_ARG, "custom_gnn: wplanes buffer too small (%lld < %lld)",
              (long long)a->wplanes_bytes, (long long)W.used);

  Arena S(bind ? a->saved : nullptr, a->saved_bytes);
  if (P->pad) {
    P->x = S.alloc<float>(N * dp);
    P->e = S.alloc<float>(E * dp);
  }
  if (P->gated) {
    P->x_p = arena_planes(S, N, dp, lo);
    P->e_p = arena_planes(S, E, dp, lo);
    P->Y = S.alloc<float>(N * 4 * dp);
    P->ehat = S.alloc<float>(E * dp);
    P->xt = S.alloc<float>(N * dp);
    P->bnbuf = S.alloc<float>(4 * dp);
    if (P->pad) P->rs = S.alloc<float>(4 * dp);
  } else {
    P->agg = S.alloc<float>(N * dp);
    P->agg_p = arena_planes(S, N, dp, lo);
    P->h = S.alloc<float>(N * dp);
    P->h_p = arena_planes(S, N, dp, lo);
    P->pre2 = S.alloc<float>(N * dp);
  }
  P->saved_bytes = S.used;
  GPS_REQUIRE(!bind || !S.overflow, GPS_ERR_ARG, "custom_gnn: saved buffer too small (%lld < %lld)",
              (long long)a->saved_bytes, (long long)S.used);

  Arena F(bind ? a->workspace : nullptr, a->workspace_bytes);
  P->fstats = F.alloc<double>(4 * dp);
  P->sink = F.alloc<double>(2 * dp);
  if (P->pad) {
    P->xo = F.alloc<float>(N * dp);
    if (P->gated) P->eo = F.alloc<float>(E * dp);
  }
  P->fwd_bytes = F.used;

  Arena Bk(bind ? a->workspace : nullptr, a->workspace_bytes);
  P->bsums = Bk.alloc<double>(4 * dp);
  const int64_t g0 = Bk.used;
  P->grads = Bk.alloc<float>(wrows * dp);   // then, consecutive in the arena: b1, W2, b2 (and the BatchNorms)
  Bk.alloc<float>(wrows);
  Bk.alloc<float>(dp * dp);
  Bk.alloc<float>(dp);
  if (P->gated) Bk.alloc<float>(4 * dp);
  P->grads_bytes = Bk.used - g0;
  if (P->pad) {
    P->gxo = Bk.alloc<float>(N * dp);
    P->gx = Bk.alloc<float>(N * dp);
    P->gea = Bk.alloc<float>(E * dp);
    if (P->gated) P->geo = Bk.alloc<float>(E * dp);
  }
  P->ge = Bk.alloc<float>(E * dp);
  if (P->gated) {
    P->gY = Bk.alloc<float>(N * 4 * dp);
    P->gY_p = arena_planes(Bk, N, 4 * dp, lo);
    P->ge_p = arena_planes(Bk, E, dp, lo);
    P->gnum = Bk.alloc<float>(N * dp);
  } else {
    P->g2 = Bk.alloc<float>(N * dp);
    P->g2_p = arena_planes(Bk, N, dp, lo);
    P->gh = Bk.alloc<float>(N * dp);
    P->gh_p = arena_planes(Bk, N, dp, lo);
    P->gagg = Bk.alloc<float>(N * dp);
  }
  P->bwd_bytes = Bk.used;
  return GPS_OK;
}

// gradient slots inside P.grads, at pitch dp, in arena order
struct CgGrads {
  float *W, *b1, *W2, *b2, *bn;
};
CgGrads grad_slots(const CgPlan& P) {
  auto next = [](float* p, int64_t n) { return p + round_up(n * (int64_t)sizeof(float), 256) / (int64_t)sizeof(float); };
  const int64_t dp = P.dp, wrows = P.gated ? 4 * dp : dp;
  CgGrads g;
  g.W = P.grads;
  g.b1 = next(g.W, wrows * dp);
  g.W2 = next(g.b1, wrows);
  g.b2 = next(g.W2, dp * dp);
  g.bn = P.gated ? next(g.b2, dp) : nullptr;
  return g;
}

int check_params(const GpsCustomGnnArgs* a, const CgPlan& P) {
  if (P.gated) {
    const struct { const GpsLinear* l; const char* name; } ps[] = {
        {&a->A, "A"}, {&a->B, "B"}, {&a->C, "C"}, {&a->D, "D"}, {&a->E, "E"}};
    for (const auto& p : ps)
      GPS_REQUIRE(p.l->weight && p.l->bias, GPS_ERR_ARG, "custom_gnn: missing parameter %s.weight / %s.bias", p.name,
                  p.name);
    for (const GpsBatchNorm* b : {&a->bn_node_x, &a->bn_edge_e})
      GPS_REQUIRE(b->weight && b->bias && b->running_mean && b->running_var, GPS_ERR_ARG,
                  "custom_gnn: missing parameter or buffer of %s", b == &a->bn_node_x ? "bn_node_x" : "bn_edge_e");
  } else {
    GPS_REQUIRE(a->nn0.weight && a->nn0.bias && a->nn2.weight && a->nn2.bias, GPS_ERR_ARG,
                "custom_gnn: missing parameter of model.nn.0 / model.nn.2");
  }
  return GPS_OK;
}

// plan, buffers and parameters of one call, all before any CUDA call
int prepare(const GpsCustomGnnArgs* a, bool fwd, CgPlan* P) {
  GPS_REQUIRE(a, GPS_ERR_ARG, "custom_gnn: null args");
  GPS_REQUIRE(a->x && a->saved && a->workspace && a->wplanes, GPS_ERR_ARG,
              "custom_gnn: x, saved, workspace and wplanes are required");
  GPS_TRY(make_plan(a, P, true));
  GPS_TRY(check_params(a, *P));
  GPS_REQUIRE(P->E == 0 || a->edge_attr, GPS_ERR_ARG, "custom_gnn: edge_attr is required");
  const int64_t ws = fwd ? P->fwd_bytes : P->bwd_bytes;
  GPS_REQUIRE(a->workspace_bytes >= ws, GPS_ERR_ARG, "custom_gnn: workspace too small (%lld < %lld)",
              (long long)a->workspace_bytes, (long long)ws);
  if (fwd) {
    GPS_REQUIRE(a->x_out, GPS_ERR_ARG, "custom_gnn: x_out is required");
    GPS_REQUIRE(!P->gated || P->E == 0 || a->edge_out, GPS_ERR_ARG, "custom_gnn: edge_out is required (GatedGCN)");
  } else {
    GPS_REQUIRE(a->grad_x_out && a->grad_x, GPS_ERR_ARG, "custom_gnn: grad_x_out and grad_x are required");
  }
  return GPS_OK;
}

// GatedGCN BatchNorm i (0: bn_node_x, 1: bn_edge_e) over the padded copies of its parameters and, with padding, of its
// running statistics
BnView bn_slot(const CgPlan& P, const GpsCustomGnnArgs* a, int i, int64_t fwd_rows = -1) {
  GpsBatchNorm b = i ? a->bn_edge_e : a->bn_node_x;
  b.weight = P.bnw + 2 * i * P.dp;
  b.bias = P.bnw + (2 * i + 1) * P.dp;
  if (P.pad) {
    b.running_mean = P.rs + 2 * i * P.dp;
    b.running_var = P.rs + (2 * i + 1) * P.dp;
  }
  return bn_view_at(P, P.bnbuf + 2 * i * P.dp, P.fstats + 2 * i * P.dp, P.dp, b, fwd_rows);
}

// =================================================================================== forward
int gated_forward(const GpsCustomGnnArgs* a, const CgPlan& P, cudaStream_t st) {
  const int64_t N = P.N, E = P.E, d = P.d, dp = P.dp;
  if (P.train) GPS_CUDA(cudaMemsetAsync(P.fstats, 0, (size_t)4 * dp * sizeof(double), st));
  // the inputs (+ planes), the running statistics and, unless the caller's copy is current, the weights: one launch
  const GpsBatchNorm* bns[2] = {&a->bn_node_x, &a->bn_edge_e};
  PadList L;
  L.add(a->x, d, N, d, P.x, dp, N, dp, P.x_p);
  L.add(a->edge_attr, d, E, d, P.e, dp, E, dp, P.e_p);
  if (P.pad)
    for (int i = 0; i < 2; ++i) {
      L.add(bns[i]->running_mean, d, 1, d, P.rs + 2 * i * dp, dp, 1, dp);
      L.add(bns[i]->running_var, d, 1, d, P.rs + (2 * i + 1) * dp, dp, 1, dp);
    }
  if (!a->wplanes_valid) {
    const GpsLinear* node[4] = {&a->A, &a->B, &a->D, &a->E};
    for (int i = 0; i < 4; ++i) {
      L.add(node[i]->weight, d, d, d, nullptr, 0, dp, dp, P.W_p.rows(i * dp));
      L.add(node[i]->bias, d, 1, d, P.b1 + i * dp, dp, 1, dp);
    }
    L.add(a->C.weight, d, d, d, nullptr, 0, dp, dp, P.W2_p);
    L.add(a->C.bias, d, 1, d, P.b2, dp, 1, dp);
    for (int i = 0; i < 2; ++i) {
      L.add(bns[i]->weight, d, 1, d, P.bnw + 2 * i * dp, dp, 1, dp);
      L.add(bns[i]->bias, d, 1, d, P.bnw + (2 * i + 1) * dp, dp, 1, dp);
    }
  }
  GPS_TRY(L.run(st));
  const float* x = P.pad ? P.x : a->x;
  const float* e = P.pad ? P.e : a->edge_attr;
  // Ce = e C^T + bC on the side stream, next to the node product
  Side* sd;
  GPS_TRY(side_stream(&sd));
  if (E > 0) {
    GPS_TRY(sd->fork(st));
    GPS_TRY(gemm(linear_fwd(P, E, dp, dp, {e, dp, P.e_p}, {nullptr, dp, P.W2_p}, P.ehat, dp, P.b2), sd->s));
  }
  // [Ax | Bx | Dx | Ex] = x Wcat^T + bcat
  GPS_TRY(gemm(linear_fwd(P, N, 4 * dp, dp, {x, dp, P.x_p}, {nullptr, dp, P.W_p}, P.Y, 4 * dp, P.b1), st));
  if (E > 0) GPS_TRY(sd->join(st));
  GPS_TRY(gatedgcn_fwd(a->graph, dp, P.Y, P.Y + dp, P.Y + 2 * dp, P.Y + 3 * dp, 4 * dp, P.ehat, P.xt,
                       P.train ? P.fstats : nullptr, P.train ? P.fstats + 2 * dp : nullptr, st));
  // x_out = [x +] drop(act(BN_x(xt))), e_out = [e +] drop(act(BN_e(e_ij))) in one launch; x_out's column sums are not
  // needed, they land in the sink
  float* xo = P.pad ? P.xo : a->x_out;
  float* eo = P.pad ? P.eo : a->edge_out;
  GPS_TRY(bn_act_residual2(P.xt, P.residual ? x : nullptr, xo, N, bn_slot(P, a, 0, N), P.drop_x, P.sink, P.ehat,
                           P.residual ? e : nullptr, eo, E, bn_slot(P, a, 1, E), P.drop_e, Planes(), dp, P.act, st));
  if (!P.pad) return GPS_OK;
  PadList U;
  U.add(xo, dp, N, d, a->x_out, d, N, d);
  U.add(eo, dp, E, d, a->edge_out, d, E, d);
  if (P.train)
    for (int i = 0; i < 2; ++i) {
      U.add(P.rs + 2 * i * dp, dp, 1, d, bns[i]->running_mean, d, 1, d);
      U.add(P.rs + (2 * i + 1) * dp, dp, 1, d, bns[i]->running_var, d, 1, d);
    }
  return U.run(st);
}

int gine_forward(const GpsCustomGnnArgs* a, const CgPlan& P, cudaStream_t st) {
  const int64_t N = P.N, E = P.E, d = P.d, dp = P.dp;
  PadList L;
  L.add(a->x, d, N, d, P.x, dp, N, dp);
  L.add(a->edge_attr, d, E, d, P.e, dp, E, dp);
  if (!a->wplanes_valid) {
    L.add(a->nn0.weight, d, d, d, nullptr, 0, dp, dp, P.W_p);
    L.add(a->nn0.bias, d, 1, d, P.b1, dp, 1, dp);
    L.add(a->nn2.weight, d, d, d, nullptr, 0, dp, dp, P.W2_p);
    L.add(a->nn2.bias, d, 1, d, P.b2, dp, 1, dp);
  }
  GPS_TRY(L.run(st));
  const float* x = P.pad ? P.x : a->x;
  const float* e = P.pad ? P.e : a->edge_attr;
  // agg = (1 + eps) x + sum_j relu(x_j + e_ij)  (+ planes)
  GPS_TRY(gine_fwd(a->graph, dp, x, e, P.eps, P.agg, st, P.agg_p));
  // h = relu(agg W0^T + b0)  (+ planes)
  GemmParams g = linear_fwd(P, N, dp, dp, {P.agg, dp, P.agg_p}, {nullptr, dp, P.W_p}, P.h, dp, P.b1);
  g.act = GPS_ACT_RELU; g.Cp = P.h_p;
  GPS_TRY(gemm(g, st));
  // x_out = [x +] drop(relu(h W1^T + b1)), with the pre-activation kept for relu'
  float* xo = P.pad ? P.xo : a->x_out;
  GemmParams g2 = linear_fwd(P, N, dp, dp, {P.h, dp, P.h_p}, {nullptr, dp, P.W2_p}, xo, dp, P.b2);
  g2.act = GPS_ACT_RELU; g2.C_pre = P.pre2; g2.ldpre = (int)dp;
  set_dropout(g2, P.drop_x);
  if (P.residual) {
    g2.R1 = x; g2.ldr1 = (int)dp;
  }
  GPS_TRY(gemm(g2, st));
  if (!P.pad) return GPS_OK;
  PadList U;
  U.add(xo, dp, N, d, a->x_out, d, N, d);
  return U.run(st);
}

int cg_forward(const GpsCustomGnnArgs* a, cudaStream_t st) {
  CgPlan P;
  GPS_TRY(prepare(a, true, &P));
  if (P.N == 0) return GPS_OK;
  return P.gated ? gated_forward(a, P, st) : gine_forward(a, P, st);
}

// =================================================================================== backward
// the parameter gradients at pitch dp -> the caller's [d, d] / [d] buffers, with grad_x / grad_edge_attr when padded
void unpack_grads(const GpsCustomGnnArgs* a, const CgPlan& P, PadList& U) {
  const int64_t d = P.d, dp = P.dp;
  const CgGrads g = grad_slots(P);
  auto lin = [&](const GpsLinear& l, const float* gw, const float* gb) {
    U.add(gw, dp, d, d, l.grad_weight, d, d, d);
    U.add(gb, dp, 1, d, l.grad_bias, d, 1, d);
  };
  if (P.gated) {
    const GpsLinear* node[4] = {&a->A, &a->B, &a->D, &a->E};
    for (int i = 0; i < 4; ++i) lin(*node[i], g.W + i * dp * dp, g.b1 + i * dp);
    lin(a->C, g.W2, g.b2);
    const GpsBatchNorm* bns[2] = {&a->bn_node_x, &a->bn_edge_e};
    for (int i = 0; i < 2; ++i) {
      U.add(g.bn + 2 * i * dp, dp, 1, d, bns[i]->grad_weight, d, 1, d);
      U.add(g.bn + (2 * i + 1) * dp, dp, 1, d, bns[i]->grad_bias, d, 1, d);
    }
  } else {
    lin(a->nn0, g.W, g.b1);
    lin(a->nn2, g.W2, g.b2);
  }
  if (P.pad) {
    U.add(P.gx, dp, P.N, d, a->grad_x, d, P.N, d);
    U.add(P.gea, dp, P.E, d, a->grad_edge_attr, d, P.E, d);
  }
}

int gated_backward(const GpsCustomGnnArgs* a, const CgPlan& P, cudaStream_t st) {
  const int64_t N = P.N, E = P.E, d = P.d, dp = P.dp;
  const CgGrads gr = grad_slots(P);
  Side* sd;
  GPS_TRY(side_stream(&sd));
  cudaStream_t s2 = sd->s, se = sd->s4;
  GPS_CUDA(cudaMemsetAsync(P.bsums, 0, (size_t)4 * dp * sizeof(double), st));
  GPS_CUDA(cudaMemsetAsync(P.grads, 0, (size_t)P.grads_bytes, st));
  if (P.pad) {
    PadList L;
    L.add(a->grad_x_out, d, N, d, P.gxo, dp, N, dp);
    L.add(a->grad_edge_out, d, E, d, P.geo, dp, E, dp);
    GPS_TRY(L.run(st));
  }
  const float* gxo = P.pad ? P.gxo : a->grad_x_out;
  const float* geo = a->grad_edge_out ? (P.pad ? P.geo : a->grad_edge_out) : nullptr;
  const float* x = P.pad ? P.x : a->x;
  const float* e = P.pad ? P.e : a->edge_attr;
  // edge side: g_e = BN_e backward of grad_edge_out, on its own stream (it needs grad_edge_out alone)
  GPS_TRY(sd->order(st, se));
  if (E > 0) {
    const BnView ve = bn_slot(P, a, 1);
    if (geo) {
      GPS_TRY(bn_bwd_reduce(geo, dp, P.ehat, dp, E, dp, ve, P.act, P.drop_e, P.bsums + 2 * dp, se));
      GPS_TRY(bn_bwd_apply(geo, dp, P.ehat, dp, E, dp, ve, P.act, P.drop_e, P.bsums + 2 * dp, P.ge, dp,
                           gr.bn + 2 * dp, gr.bn + 3 * dp, se));
    } else {
      GPS_CUDA(cudaMemsetAsync(P.ge, 0, (size_t)(E * dp) * sizeof(float), se));
    }
  }
  // node side: g_xt -> gY[:, 0:dp] (+ planes)
  const BnView vx = bn_slot(P, a, 0);
  GPS_TRY(bn_bwd_reduce(gxo, dp, P.xt, dp, N, dp, vx, P.act, P.drop_x, P.bsums, st));
  GPS_TRY(bn_bwd_apply(gxo, dp, P.xt, dp, N, dp, vx, P.act, P.drop_x, P.bsums, P.gY, 4 * dp, gr.bn, gr.bn + dp, st,
                       false, P.gY_p));
  GPS_TRY(sd->order(se, st));
  // message / aggregate backward: g_Dx, g_e (total), then g_Ex, g_Bx
  GPS_TRY(gatedgcn_bwd_dst(a->graph, dp, P.gY, 4 * dp, P.ehat, P.Y + dp, 4 * dp, P.ge, P.gnum, P.gY + 2 * dp, st,
                           P.ge_p, P.gY_p.cols(2 * dp)));
  GPS_TRY(gatedgcn_bwd_src(a->graph, dp, P.ge, P.ehat, P.gnum, P.gY + 3 * dp, P.gY + dp, 4 * dp, st,
                           P.gY_p.cols(3 * dp), P.gY_p.cols(dp)));
  // weight products on the side stream: [A|B|D|E] from gY and x, C from g_e and e
  const Operand gY{P.gY, 4 * dp, P.gY_p}, ge{P.ge, dp, P.ge_p};
  GPS_TRY(sd->fork(st));
  GPS_TRY(linear_wgrad(P, gY, {x, dp, P.x_p}, N, 4 * dp, dp, gr.W, gr.b1, s2));
  GPS_TRY(linear_wgrad(P, ge, {e, dp, P.e_p}, E, dp, dp, gr.W2, gr.b2, s2));
  // grad_x = gY Wcat [+ grad_x_out]; grad_edge_attr = g_e C [+ grad_edge_out]
  GemmParams gx = linear_dgrad(P, N, dp, 4 * dp, gY, {nullptr, dp, P.W_p}, P.pad ? P.gx : a->grad_x, dp);
  if (P.residual) {
    gx.R1 = gxo; gx.ldr1 = (int)dp;
  }
  GPS_TRY(gemm(gx, st));
  if (a->grad_edge_attr && E > 0) {
    GemmParams g = linear_dgrad(P, E, dp, dp, ge, {nullptr, dp, P.W2_p}, P.pad ? P.gea : a->grad_edge_attr, dp);
    if (P.residual && geo) {
      g.R1 = geo; g.ldr1 = (int)dp;
    }
    GPS_TRY(gemm(g, st));
  }
  GPS_TRY(sd->join(st));
  PadList U;
  unpack_grads(a, P, U);
  return U.run(st);
}

int gine_backward(const GpsCustomGnnArgs* a, const CgPlan& P, cudaStream_t st) {
  const int64_t N = P.N, E = P.E, d = P.d, dp = P.dp;
  const CgGrads gr = grad_slots(P);
  Side* sd;
  GPS_TRY(side_stream(&sd));
  cudaStream_t s2 = sd->s;
  GPS_CUDA(cudaMemsetAsync(P.grads, 0, (size_t)P.grads_bytes, st));
  const float* x = P.pad ? P.x : a->x;
  const float* e = P.pad ? P.e : a->edge_attr;
  // g2 = grad_x_out * drop * relu'(pre2) (+ planes), and the padded grad_x_out for the residual
  const int64_t n4 = N * (dp / 4);
  k_gine_gout<<<(unsigned)std::min<int64_t>(ceil_div(n4, 256), kNumSMs * 8), 256, 0, st>>>(
      a->grad_x_out, d, (int)d, P.pre2, (int)dp, N, P.drop_x, P.g2, P.g2_p, P.pad && P.residual ? P.gxo : nullptr);
  GPS_LAUNCH_CHECK();
  const float* gxo = P.pad ? P.gxo : a->grad_x_out;
  // g_h = (g2 W1) * relu'(h)  (+ planes)
  const Operand g2{P.g2, dp, P.g2_p}, gh{P.gh, dp, P.gh_p};
  GemmParams g = linear_dgrad(P, N, dp, dp, g2, {nullptr, dp, P.W2_p}, P.gh, dp);
  set_act_mask(g, GPS_ACT_RELU, P.h, nullptr, dp);
  g.Cp = P.gh_p;
  GPS_TRY(gemm(g, st));
  GPS_TRY(sd->fork(st));
  GPS_TRY(linear_wgrad(P, g2, {P.h, dp, P.h_p}, N, dp, dp, gr.W2, gr.b2, s2));
  GPS_TRY(linear_wgrad(P, gh, {P.agg, dp, P.agg_p}, N, dp, dp, gr.W, gr.b1, s2));
  // g_agg = g_h W0, then the aggregation's backward: g_e (dst ordered), grad_x = (1 + eps) g_agg + sum g_e [+ g_out]
  GPS_TRY(gemm(linear_dgrad(P, N, dp, dp, gh, {nullptr, dp, P.W_p}, P.gagg, dp), st));
  float* ge = !P.pad && a->grad_edge_attr ? a->grad_edge_attr : (P.pad ? P.gea : P.ge);
  if (E > 0) GPS_TRY(gine_bwd_dst(a->graph, dp, x, e, P.gagg, ge, st));
  GPS_TRY(gine_bwd_src(a->graph, dp, ge, P.gagg, P.eps, P.residual ? gxo : nullptr, P.pad ? P.gx : a->grad_x, st));
  GPS_TRY(sd->join(st));
  PadList U;
  unpack_grads(a, P, U);
  return U.run(st);
}

int cg_backward(const GpsCustomGnnArgs* a, cudaStream_t st) {
  CgPlan P;
  GPS_TRY(prepare(a, false, &P));
  if (P.N == 0) {   // no rows: every gradient is zero
    PadList U;
    GPS_CUDA(cudaMemsetAsync(P.grads, 0, (size_t)P.grads_bytes, st));
    unpack_grads(a, P, U);
    return U.run(st);
  }
  return P.gated ? gated_backward(a, P, st) : gine_backward(a, P, st);
}

}  // namespace

int PadList::run(cudaStream_t st) const {
  GPS_REQUIRE(!overflow, GPS_ERR_ARG, "pad: more than %d pad items in one launch", kPadItems);
  PadDesc d;
  int total = 0;
  for (int i = 0; i < n; ++i) {
    d.it[i] = it[i];
    d.start[i] = total;
    total += (int)ceil_div((int64_t)it[i].rows_p * ((it[i].cols_p + 3) / 4), 256);
  }
  d.n = n;
  d.start[n] = total;
  if (total == 0) return GPS_OK;
  k_pad<<<(unsigned)total, 256, 0, st>>>(d);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

}  // namespace gps

// =================================================================================== C ABI
using namespace gps;

extern "C" int gps_custom_gnn_plan(const GpsCustomGnnArgs* args, GpsCustomGnnPlan* plan) {
  GPS_REQUIRE(args && plan, GPS_ERR_ARG, "gps_custom_gnn_plan: null argument");
  CgPlan P;
  GPS_TRY(make_plan(args, &P, false));
  plan->saved_bytes = P.saved_bytes;
  plan->fwd_workspace_bytes = P.fwd_bytes;
  plan->bwd_workspace_bytes = P.bwd_bytes;
  plan->wplanes_bytes = P.wplanes_bytes;
  return GPS_OK;
}

extern "C" int gps_custom_gnn_forward(const GpsCustomGnnArgs* args, void* stream) {
  return cg_forward(args, (cudaStream_t)stream);
}

extern "C" int gps_custom_gnn_backward(const GpsCustomGnnArgs* args, void* stream) {
  return cg_backward(args, (cudaStream_t)stream);
}
