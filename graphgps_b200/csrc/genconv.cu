// genconv.cu — the message passing of the GENConv local model (PyG 2.2 GENConv(dim_h, dim_h), gps_layer.py:60-61).
//
// With the defaults the reference uses (aggr='softmax', t = 1, learn_t=False, msg_norm=False, in == out, edge_dim None):
//   m_k    = relu(x[src_k] + e_k) + 1e-7                               (GENConv.message)
//   alpha  = exp(m_k - max_i) / (sum_i exp(m_k - max_i) + 1e-16)       per target i and channel c (utils.softmax)
//   agg_i  = sum_k alpha_k m_k   (0 for a node without in-edges)       (SoftmaxAggregation)
//   u_i    = agg_i + x_i                                               (GENConv.forward: out + x_dst, then mlp(u))
// The MLP (Linear, BatchNorm1d, ReLU, Linear) runs in the layer (layer.cu) on the dense-product and row-wise stages.
//
// A thread owns (node, 4 channels) and walks the node's dst-sorted segment in edge-id order with an online softmax,
// so no atomics touch feature data and every run gives the same bits.  The forward saves lse = max + log(sum) per
// (node, channel); the backward recomputes alpha = exp(m - lse) per edge.  S >= 1 after the first edge, so the 1e-16 of
// the denominator vanishes in fp32 and exp(m - lse) is alpha.  With t = 1:
//   d agg_i / d m_k = alpha_k (1 + m_k - agg_i),  grad_e_k = g_u_i alpha_k (1 + m_k - agg_i) [x_src + e_k > 0]
// and g_x_j = g_u_j + sum over j's out-edges of grad_e_k (+ the caller's upstream), which is gine_bwd_src with eps = 0.
#include "kernels.cuh"

namespace gps {

namespace {

constexpr float kGenMsgEps = 1e-7f;   // GENConv(eps=1e-7), added to every message after the ReLU

__device__ __forceinline__ float4 gen_msg(float4 pre) {
  return make_float4(fmaxf(pre.x, 0.f) + kGenMsgEps, fmaxf(pre.y, 0.f) + kGenMsgEps, fmaxf(pre.z, 0.f) + kGenMsgEps,
                     fmaxf(pre.w, 0.f) + kGenMsgEps);
}

// one channel of the online softmax: running max M, sum S = sum exp(m - M), weighted sum A = sum exp(m - M) m
__device__ __forceinline__ void online_step(float m, float& M, float& S, float& A) {
  const float Mn = fmaxf(M, m);
  const float a = expf(M - Mn), b = expf(m - Mn);   // a = 0 for the first edge (M = -inf)
  S = fmaf(S, a, b);
  A = fmaf(A, a, b * m);
  M = Mn;
}

__global__ void k_genconv_fwd(GpsGraph g, int d, const float* __restrict__ x, const float* __restrict__ e,
                              float* __restrict__ agg, float* __restrict__ lse, float* __restrict__ u, Planes up) {
  const int c = threadIdx.x * 4, ry = threadIdx.y, RY = blockDim.y;
  for (int64_t i = (int64_t)blockIdx.x * RY + ry; i < g.N; i += (int64_t)gridDim.x * RY) {
    float4 M = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY), S = f4zero(), A = f4zero();
    const int kb = g.dst_ptr[i], ke = g.dst_ptr[i + 1];
    for (int k = kb; k < ke; ++k) {
      const int j = g.dst_src[k];
      const int64_t eid = g.dst_eid[k];
      const float4 m = gen_msg(f4add(ld4(x + (int64_t)j * d + c), ld4(e + eid * d + c)));
      online_step(m.x, M.x, S.x, A.x);
      online_step(m.y, M.y, S.y, A.y);
      online_step(m.z, M.z, S.z, A.z);
      online_step(m.w, M.w, S.w, A.w);
    }
    float4 a = f4zero(), l = f4zero();
    if (ke > kb) {
      a = make_float4(A.x / (S.x + 1e-16f), A.y / (S.y + 1e-16f), A.z / (S.z + 1e-16f), A.w / (S.w + 1e-16f));
      l = make_float4(M.x + logf(S.x), M.y + logf(S.y), M.z + logf(S.z), M.w + logf(S.w));
    }
    const float4 v = f4add(a, ld4(x + i * d + c));
    st4(agg + i * d + c, a);
    st4(lse + i * d + c, l);
    st4(u + i * d + c, v);
    if (up.hi) planes_store4(up, i, c, v);
  }
}

__device__ __forceinline__ float gen_grad(float pre, float gu, float ag, float l) {
  const float m = fmaxf(pre, 0.f) + kGenMsgEps;
  return pre > 0.f ? gu * expf(m - l) * (1.f + m - ag) : 0.f;
}

__global__ void k_genconv_bwd_dst(GpsGraph g, int d, const float* __restrict__ x, const float* __restrict__ e,
                                  const float* __restrict__ agg, const float* __restrict__ lse,
                                  const float* __restrict__ g_u, float* __restrict__ g_e) {
  const int c = threadIdx.x * 4, ry = threadIdx.y, RY = blockDim.y;
  for (int64_t i = (int64_t)blockIdx.x * RY + ry; i < g.N; i += (int64_t)gridDim.x * RY) {
    const int kb = g.dst_ptr[i], ke = g.dst_ptr[i + 1];
    if (kb == ke) continue;
    const float4 gu = ld4(g_u + i * d + c), ag = ld4(agg + i * d + c), l = ld4(lse + i * d + c);
    for (int k = kb; k < ke; ++k) {
      const int j = g.dst_src[k];
      const int64_t eid = g.dst_eid[k];
      const float4 pre = f4add(ld4(x + (int64_t)j * d + c), ld4(e + eid * d + c));
      st4(g_e + eid * d + c, make_float4(gen_grad(pre.x, gu.x, ag.x, l.x), gen_grad(pre.y, gu.y, ag.y, l.y),
                                         gen_grad(pre.z, gu.z, ag.z, l.z), gen_grad(pre.w, gu.w, ag.w, l.w)));
    }
  }
}

// (node, float4 column group) per thread, as the other message-passing kernels (scatter.cu node_geom without statistics)
static int gen_geom(int64_t N, int64_t d, dim3* grid, dim3* block) {
  GPS_REQUIRE(d > 0 && d % 4 == 0 && d / 4 <= 1024, GPS_ERR_UNSUPPORTED,
              "genconv needs d %% 4 == 0 and d <= 4096 (got %lld)", (long long)d);
  const int C4 = (int)(d / 4);
  const int RY = C4 >= 256 ? 1 : 256 / C4;
  int64_t blocks = ceil_div(N > 0 ? N : 1, (int64_t)RY * 2);
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  *grid = dim3((unsigned)blocks);
  *block = dim3(C4, RY);
  return GPS_OK;
}

}  // namespace

int genconv_fwd(const GpsGraph& g, int64_t d, const float* x, const float* e, float* agg, float* lse, float* u,
                cudaStream_t stream, Planes up) {
  if (g.N == 0) return GPS_OK;
  dim3 grid, block;
  GPS_TRY(gen_geom(g.N, d, &grid, &block));
  k_genconv_fwd<<<grid, block, 0, stream>>>(g, (int)d, x, e, agg, lse, u, up);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int genconv_bwd_dst(const GpsGraph& g, int64_t d, const float* x, const float* e, const float* agg, const float* lse,
                    const float* g_u, float* g_e, cudaStream_t stream) {
  if (g.N == 0 || g.E == 0) return GPS_OK;
  dim3 grid, block;
  GPS_TRY(gen_geom(g.N, d, &grid, &block));
  k_genconv_bwd_dst<<<grid, block, 0, stream>>>(g, (int)d, x, e, agg, lse, g_u, g_e);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

}  // namespace gps
