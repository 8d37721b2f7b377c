// pna.cu — the message passing of the PNA local model (PyG 2.2 PNAConv(dim_h, dim_h, aggregators=['mean','max','sum'],
// scalers=['identity'], edge_dim=de, towers=1, pre_layers=1, post_layers=1, divide_input=False), gps_layer.py:75-90).
//
// For edge k from j to i, with W_pre = [W_dst | W_src | W_e] (column blocks of pre_nns.0.0.weight [d, 3d]):
//   m_k = W_dst x_i + W_src x_j + W_e (W_enc e_k + b_enc) + b_pre
// The layer computes P_dst = x W_dst^T and P_src = x W_src^T as two segments of the fused node projection, and the edge
// term as one product q = e F^T + c with the fold F = W_e W_enc [d, de], c = W_e b_enc + b_pre (k_pna_fold), so
//   m_k = P_dst[i] + P_src[j] + q[k].
// Per target i and channel: mean, max and sum over i's in-edges (0 in all three for a node without any), and
//   Z_i = [x_i | mean | max | sum]   [N, 4d], the operand of post_nns.0.0.
// The max follows torch_scatter's scatter_max: the first maximising in-edge in edge-id order wins (strict >; the
// dst-sorted segments are in edge-id order), and the whole max gradient goes to it.  The forward saves its edge id
// (-1 without in-edges).  Backward, per in-edge k of i:
//   g_m_k = g_mean_i / cnt_i + g_sum_i + [k == argmax_i] g_max_i
// written to g_q[k] (edge-id order); g_P_dst[i] = sum_k g_m_k; and, in the CSC pass, g_P_src[j] = sum over j's
// out-edges of g_m_k.  A thread owns (node, 4 channels) and walks its segment in order: no atomics touch feature data,
// and every run gives the same bits.
#include <algorithm>

#include "kernels.cuh"

namespace gps {

namespace {

// F[r, c] = sum_k W_e[r, k] W_enc[k, c] (r < d, c < de); cvec[r] = sum_k W_e[r, k] b_enc[k] + b_pre[r].  One row r per
// block; thread c == de computes cvec[r].  W_e is the column block 2d..3d of W_pre (row pitch 3d).
__global__ void k_pna_fold(const float* __restrict__ Wpre, const float* __restrict__ bpre, const float* __restrict__ Wenc,
                           const float* __restrict__ benc, int d, int de, float* __restrict__ F, float* __restrict__ cvec) {
  const int r = blockIdx.x;
  const float* we = Wpre + (int64_t)r * 3 * d + 2 * d;
  for (int c = threadIdx.x; c <= de; c += blockDim.x) {
    float acc = 0.f;
    if (c < de) {
      for (int k = 0; k < d; ++k) acc = fmaf(we[k], Wenc[(int64_t)k * de + c], acc);
      F[(int64_t)r * de + c] = acc;
    } else {
      for (int k = 0; k < d; ++k) acc = fmaf(we[k], benc[k], acc);
      cvec[r] = acc + bpre[r];
    }
  }
}

// The fold's backward, from g_F [d, de] and g_c [d]:
//   g_W_e[r, k] = sum_c g_F[r, c] W_enc[k, c] + g_c[r] b_enc[k]      blocks 0 .. d-1 (row r)
//   g_W_enc[k, c] = sum_r W_e[r, k] g_F[r, c],  g_b_enc[k] = sum_r W_e[r, k] g_c[r]   blocks d .. 2d-1 (row k)
//   g_b_pre = g_c                                                     block 0
// Every output element is one fixed-order dot product; accumulate adds it to the caller's buffer.
__global__ void k_pna_unfold(const float* __restrict__ Wpre, const float* __restrict__ Wenc,
                             const float* __restrict__ benc, const float* __restrict__ gF, const float* __restrict__ gc,
                             int d, int de, float* __restrict__ gWpre, float* __restrict__ gbpre,
                             float* __restrict__ gWenc, float* __restrict__ gbenc, int accumulate) {
  auto put = [&](float* p, float v) { *p = accumulate ? *p + v : v; };
  if ((int)blockIdx.x < d) {
    const int r = blockIdx.x;
    if (gWpre) {   // one warp per output: lanes stride the contiguous c of both rows, then a fixed-order warp sum
      const float* gf = gF + (int64_t)r * de;
      const int lane = threadIdx.x & 31, nw = blockDim.x >> 5;
      for (int k = threadIdx.x >> 5; k < d; k += nw) {
        const float* wk = Wenc + (int64_t)k * de;
        float acc = 0.f;
        for (int c = lane; c < de; c += 32) acc = fmaf(gf[c], wk[c], acc);
        acc = warp_sum(acc);
        if (lane == 0) put(gWpre + (int64_t)r * 3 * d + 2 * d + k, fmaf(gc[r], benc[k], acc));
      }
    }
    if (r == 0 && gbpre)
      for (int i = threadIdx.x; i < d; i += blockDim.x) put(gbpre + i, gc[i]);
  } else {
    const int k = blockIdx.x - d;
    for (int c = threadIdx.x; c <= de; c += blockDim.x) {
      float acc = 0.f;
      if (c < de) {
        if (!gWenc) continue;
        for (int r = 0; r < d; ++r) acc = fmaf(Wpre[(int64_t)r * 3 * d + 2 * d + k], gF[(int64_t)r * de + c], acc);
        put(gWenc + (int64_t)k * de + c, acc);
      } else if (gbenc) {
        for (int r = 0; r < d; ++r) acc = fmaf(Wpre[(int64_t)r * 3 * d + 2 * d + k], gc[r], acc);
        put(gbenc + k, acc);
      }
    }
  }
}

__device__ __forceinline__ void max_step(float m, int eid, float& M, int& A) {
  if (m > M) {   // strict: the first maximiser in edge-id order keeps the argmax
    M = m;
    A = eid;
  }
}

__global__ void k_pna_fwd(GpsGraph g, int d, const float* __restrict__ x, const float* __restrict__ Y, int64_t ldy,
                          const float* __restrict__ q, float* __restrict__ Z, Planes Zp, int* __restrict__ arg) {
  const int c = threadIdx.x * 4, ry = threadIdx.y, RY = blockDim.y;
  for (int64_t i = (int64_t)blockIdx.x * RY + ry; i < g.N; i += (int64_t)gridDim.x * RY) {
    const int kb = g.dst_ptr[i], ke = g.dst_ptr[i + 1];
    const float4 pd = ld4(Y + i * ldy + c);
    float4 S = f4zero(), M = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    int4 A = make_int4(-1, -1, -1, -1);
    for (int k = kb; k < ke; ++k) {
      const int j = g.dst_src[k];
      const int eid = g.dst_eid[k];
      const float4 m = f4add(f4add(pd, ld4(Y + (int64_t)j * ldy + d + c)), ld4(q + (int64_t)eid * d + c));
      S = f4add(S, m);
      max_step(m.x, eid, M.x, A.x);
      max_step(m.y, eid, M.y, A.y);
      max_step(m.z, eid, M.z, A.z);
      max_step(m.w, eid, M.w, A.w);
    }
    float4 mean = f4zero(), mx = f4zero();
    if (ke > kb) {
      const float n = (float)(ke - kb);
      mean = make_float4(S.x / n, S.y / n, S.z / n, S.w / n);
      mx = M;
    }
    const float4 xv = ld4(x + i * d + c);
    if (Z) {
      float* z = Z + i * 4 * d;
      st4(z + c, xv);
      st4(z + d + c, mean);
      st4(z + 2 * d + c, mx);
      st4(z + 3 * d + c, S);
    }
    if (Zp.hi) {
      planes_store4(Zp, i, c, xv);
      planes_store4(Zp, i, d + c, mean);
      planes_store4(Zp, i, 2 * d + c, mx);
      planes_store4(Zp, i, 3 * d + c, S);
    }
    *reinterpret_cast<int4*>(arg + i * d + c) = A;
  }
}

__device__ __forceinline__ float pick(int eid, int a, float gmax) { return eid == a ? gmax : 0.f; }

__global__ void k_pna_bwd_dst(GpsGraph g, int d, const float* __restrict__ gZ, const int* __restrict__ arg,
                              const float* __restrict__ add, float* __restrict__ g_q, Planes gqp,
                              float* __restrict__ gP, int64_t ldg, Planes gPp, float* __restrict__ g_x) {
  const int c = threadIdx.x * 4, ry = threadIdx.y, RY = blockDim.y;
  for (int64_t i = (int64_t)blockIdx.x * RY + ry; i < g.N; i += (int64_t)gridDim.x * RY) {
    const float* gz = gZ + i * 4 * d;
    st4(g_x + i * d + c, add ? f4add(ld4(add + i * d + c), ld4(gz + c)) : ld4(gz + c));
    const int kb = g.dst_ptr[i], ke = g.dst_ptr[i + 1];
    float4 acc = f4zero();
    if (ke > kb) {
      const float n = (float)(ke - kb);
      const float4 gmean = ld4(gz + d + c), gmax = ld4(gz + 2 * d + c), gsum = ld4(gz + 3 * d + c);
      const float4 base = make_float4(gmean.x / n + gsum.x, gmean.y / n + gsum.y, gmean.z / n + gsum.z,
                                      gmean.w / n + gsum.w);
      const int4 a = *reinterpret_cast<const int4*>(arg + i * d + c);
      for (int k = kb; k < ke; ++k) {
        const int eid = g.dst_eid[k];
        const float4 gm = make_float4(base.x + pick(eid, a.x, gmax.x), base.y + pick(eid, a.y, gmax.y),
                                      base.z + pick(eid, a.z, gmax.z), base.w + pick(eid, a.w, gmax.w));
        st4(g_q + (int64_t)eid * d + c, gm);
        if (gqp.hi) planes_store4(gqp, eid, c, gm);
        acc = f4add(acc, gm);
      }
    }
    st4(gP + i * ldg + c, acc);
    if (gPp.hi) planes_store4(gPp, i, c, acc);
  }
}

__global__ void k_pna_bwd_src(GpsGraph g, int d, const float* __restrict__ g_q, float* __restrict__ gP, int64_t ldg,
                              Planes gPp) {
  const int c = threadIdx.x * 4, ry = threadIdx.y, RY = blockDim.y;
  for (int64_t j = (int64_t)blockIdx.x * RY + ry; j < g.N; j += (int64_t)gridDim.x * RY) {
    float4 acc = f4zero();
    const int kb = g.src_ptr[j], ke = g.src_ptr[j + 1];
    for (int k = kb; k < ke; ++k) acc = f4add(acc, ld4(g_q + (int64_t)g.src_eid[k] * d + c));
    st4(gP + j * ldg + c, acc);
    if (gPp.hi) planes_store4(gPp, j, c, acc);
  }
}

// (node, float4 column group) per thread, as the other message-passing kernels
static int pna_geom(int64_t N, int64_t d, dim3* grid, dim3* block) {
  GPS_REQUIRE(d > 0 && d % 4 == 0 && d / 4 <= 1024, GPS_ERR_UNSUPPORTED,
              "PNA needs d %% 4 == 0 and d <= 4096 (got %lld)", (long long)d);
  const int C4 = (int)(d / 4);
  const int RY = C4 >= 256 ? 1 : 256 / C4;
  int64_t blocks = ceil_div(N > 0 ? N : 1, (int64_t)RY * 2);
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  *grid = dim3((unsigned)blocks);
  *block = dim3(C4, RY);
  return GPS_OK;
}

}  // namespace

int pna_check(int64_t d, int64_t de) {
  GPS_REQUIRE(de > 0 && de <= d && de % 4 == 0, GPS_ERR_UNSUPPORTED,
              "PNA needs 0 < edge_dim <= dim_h and edge_dim %% 4 == 0 (got edge_dim %lld, dim_h %lld)", (long long)de,
              (long long)d);
  return GPS_OK;
}

int pna_fold_fwd(const float* Wpre, const float* bpre, const float* Wenc, const float* benc, int64_t d, int64_t de,
                 float* F, float* cvec, cudaStream_t st) {
  GPS_TRY(pna_check(d, de));
  // one thread per column of F plus one for c: a single pass over the row for de <= 992
  const int threads = (int)std::min<int64_t>(1024, round_up(de + 1, (int64_t)32));
  k_pna_fold<<<(unsigned)d, threads, 0, st>>>(Wpre, bpre, Wenc, benc, (int)d, (int)de, F, cvec);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int pna_fold_bwd(const float* Wpre, const float* Wenc, const float* benc, const float* gF, const float* gc, int64_t d,
                 int64_t de, float* gWpre, float* gbpre, float* gWenc, float* gbenc, bool accumulate, cudaStream_t st) {
  GPS_TRY(pna_check(d, de));
  k_pna_unfold<<<(unsigned)(2 * d), 256, 0, st>>>(Wpre, Wenc, benc, gF, gc, (int)d, (int)de, gWpre, gbpre, gWenc, gbenc,
                                                  accumulate ? 1 : 0);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int pna_fwd(const GpsGraph& g, int64_t d, const float* x, const float* Y, int64_t ldy, const float* q, float* Z,
            Planes Zp, int* arg, cudaStream_t stream) {
  if (g.N == 0) return GPS_OK;
  dim3 grid, block;
  GPS_TRY(pna_geom(g.N, d, &grid, &block));
  k_pna_fwd<<<grid, block, 0, stream>>>(g, (int)d, x, Y, ldy, q, Z, Zp, arg);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int pna_bwd(const GpsGraph& g, int64_t d, const float* gZ, const int* arg, const float* add, float* g_q, Planes gqp,
            float* gY, int64_t ldg, Planes gYp, float* g_x, cudaStream_t stream) {
  if (g.N == 0) return GPS_OK;
  dim3 grid, block;
  GPS_TRY(pna_geom(g.N, d, &grid, &block));
  k_pna_bwd_dst<<<grid, block, 0, stream>>>(g, (int)d, gZ, arg, add, g_q, gqp, gY, ldg, gYp, g_x);
  GPS_LAUNCH_CHECK();
  k_pna_bwd_src<<<grid, block, 0, stream>>>(g, (int)d, g_q, gY + d, ldg, gYp.cols(d));
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

}  // namespace gps
