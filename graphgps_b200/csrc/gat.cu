// gat.cu — the GAT local model: PyG 2.2 GATConv(dim_h, dim_h / H, heads=H, edge_dim=dim_h) as built at
// graphgps/layer/gps_layer.py:70-74 and called at :183-189 with its defaults (concat, negative_slope 0.2, no attention
// dropout, add_self_loops with fill_value 'mean', bias).
//
// For node i, head h (C = d / H channels per head), Y = x W_src^T (a column block of the fused node projection):
//   a_src[i,h] = Y[i,h,:] . att_src[h]     a_dst[i,h] = Y[i,h,:] . att_dst[h]
//   a_edge[e,h] = (W_edge e_e)[h,:] . att_edge[h] = e_e . v[h],   v[h] = W_edge[hC:(h+1)C, :]^T att_edge[h]   (fold)
//   self loops: every j -> i with j == i is dropped; one loop (i, i) per node is added whose attribute is the mean of
//   i's remaining in-edge attributes (0 without any), so its score is the mean of their a_edge.
//   z_ji = leaky_relu(a_src[j] + a_dst[i] + a_edge[ji], 0.2);  alpha = softmax of z over the in-edges of i and its loop
//   x_loc_i = x_i + drop(sum_j alpha_ji Y[j] + bias)
// The forward saves the scores and the per-(node, head) log-sum-exp; alpha is recomputed from them.  Every reduction
// runs in a fixed order (warp butterflies, edge-id-ordered segments, fixed row chunks summed in chunk order), so two
// runs give the same bits; the only atomics are the double column sums of the BatchNorm statistics, as in scatter.cu.
#include "kernels.cuh"

namespace gps {

namespace {

constexpr int kWarpsPerBlock = 8;
constexpr float kSlope = 0.2f;

__device__ __forceinline__ float lrelu(float z) { return z > 0.f ? z : kSlope * z; }
// torch's leaky_relu backward takes the negative slope at exactly 0
__device__ __forceinline__ float lrelu_d(float z) { return z > 0.f ? 1.f : kSlope; }

// thread geometry of the (node, 4 channels) kernels, as scatter.cu's node_geom
struct Geom {
  dim3 block, grid;
  size_t smem;
};
static int gat_geom(int64_t N, int64_t d, bool stats, Geom* g) {
  GPS_REQUIRE(d > 0 && d % 4 == 0 && d / 4 <= 1024, GPS_ERR_UNSUPPORTED,
              "GAT needs d %% 4 == 0 and d <= 4096 (got %lld)", (long long)d);
  const int C4 = (int)(d / 4);
  int RY = C4 >= 256 ? 1 : 256 / C4;
  int64_t cap = kNumSMs * 16;
  if (stats) {   // same-address double atomics serialise: few, fat CTAs
    RY = C4 >= 1024 ? 1 : 1024 / C4;
    if (RY > 16) RY = 16;
    const int smem_cap = (int)(48 * 1024 / (2 * (size_t)C4 * sizeof(float4)));
    if (RY > smem_cap) RY = smem_cap < 1 ? 1 : smem_cap;
    cap = kNumSMs;
  }
  int64_t blocks = ceil_div(N > 0 ? N : 1, (int64_t)RY * 2);
  if (blocks > cap) blocks = cap;
  g->block = dim3(C4, RY, 1);
  g->grid = dim3((unsigned)blocks, 1, 1);
  g->smem = stats && RY > 1 ? 2 * (size_t)RY * C4 * sizeof(float4) : 0;
  return GPS_OK;
}

// v[h, k] = sum_c W_edge[h*C + c, k] * att_edge[h*C + c]
__global__ void k_gat_fold(const float* __restrict__ W, const float* __restrict__ att, int d, int C,
                           float* __restrict__ v) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int H = d / C;
  if (idx >= (int64_t)H * d) return;
  const int h = (int)(idx / d), k = (int)(idx % d);
  float s = 0.f;
  for (int c = 0; c < C; ++c) s = fmaf(W[(int64_t)(h * C + c) * d + k], att[h * C + c], s);
  v[idx] = s;
}

// one warp per row r = h*C + c of W_edge: g_W[r, :] = att[r] g_v[h, :],  g_att[r] = W[r, :] . g_v[h, :]
__global__ void k_gat_fold_bwd(const float* __restrict__ W, const float* __restrict__ att, const float* __restrict__ gv,
                               int d, int C, float* gW, float* gatt, int accumulate) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (r >= d) return;
  const int h = r / C;
  const float a = att[r];
  float s = 0.f;
  for (int k = lane; k < d; k += 32) {
    const float g = gv[(int64_t)h * d + k];
    s = fmaf(W[(int64_t)r * d + k], g, s);
    if (gW) {
      float* p = gW + (int64_t)r * d + k;
      *p = accumulate ? *p + a * g : a * g;
    }
  }
  s = warp_sum(s);
  if (lane == 0 && gatt) gatt[r] = accumulate ? gatt[r] + s : s;
}

// a_src, a_dst [N, H]: one warp per node
__global__ void k_gat_node_scores(int64_t N, int d, int C, const float* __restrict__ Y, int64_t ldy,
                                  const float* __restrict__ att_src, const float* __restrict__ att_dst,
                                  float* __restrict__ a_src, float* __restrict__ a_dst) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (i >= N) return;
  const int H = d / C;
  for (int h = 0; h < H; ++h) {
    float s = 0.f, t = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float y = Y[i * ldy + h * C + c];
      s = fmaf(y, att_src[h * C + c], s);
      t = fmaf(y, att_dst[h * C + c], t);
    }
    s = warp_sum(s);
    t = warp_sum(t);
    if (lane == 0) {
      a_src[i * H + h] = s;
      a_dst[i * H + h] = t;
    }
  }
}

// a_edge [E, H] = e_e . v[h]: one warp per edge (edge-id order)
__global__ void k_gat_edge_scores(int64_t E, int d, int H, const float* __restrict__ ea, const float* __restrict__ v,
                                  float* __restrict__ a_edge) {
  const int lane = threadIdx.x & 31;
  const int64_t e = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (e >= E) return;
  for (int h = 0; h < H; ++h) {
    float s = 0.f;
    for (int k = lane; k < d; k += 32) s = fmaf(ea[e * d + k], v[(int64_t)h * d + k], s);
    s = warp_sum(s);
    if (lane == 0) a_edge[e * H + h] = s;
  }
}

// per (node, head): the self loop's score a_self = mean of a_edge over the non-self in-edges (0 without any) and the
// log-sum-exp of z over those edges and the loop.  One warp per node, lanes over heads, edges in CSR (edge-id) order.
__global__ void k_gat_softmax_stats(GpsGraph g, int H, const float* __restrict__ a_src, const float* __restrict__ a_dst,
                                    const float* __restrict__ a_edge, float* __restrict__ a_self, float* __restrict__ lse) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (i >= g.N) return;
  const int b = g.dst_ptr[i], en = g.dst_ptr[i + 1];
  for (int h = lane; h < H; h += 32) {
    float se = 0.f;
    int deg = 0;
    for (int q = b; q < en; ++q) {
      if (g.dst_src[q] == (int)i) continue;
      se += a_edge[(int64_t)g.dst_eid[q] * H + h];
      ++deg;
    }
    const float as = deg > 0 ? se / (float)deg : 0.f;
    const float ad = a_dst[i * H + h];
    float m = lrelu(a_src[i * H + h] + ad + as), s = 1.f;
    for (int q = b; q < en; ++q) {
      const int j = g.dst_src[q];
      if (j == (int)i) continue;
      const float z = lrelu(a_src[(int64_t)j * H + h] + ad + a_edge[(int64_t)g.dst_eid[q] * H + h]);
      if (z > m) {
        s = fmaf(s, expf(m - z), 1.f);
        m = z;
      } else {
        s += expf(z - m);
      }
    }
    a_self[i * H + h] = as;
    lse[i * H + h] = m + logf(s);
  }
}

// head of each of the 4 channels c..c+3 and their attention weights for score base `pre - a_src`: when the four share a
// head (C % 4 == 0) one exp serves all
struct Heads4 {
  int h[4];
  bool same;
};
__device__ __forceinline__ Heads4 heads4(int c, int C) {
  Heads4 r;
#pragma unroll
  for (int k = 0; k < 4; ++k) r.h[k] = (c + k) / C;
  r.same = r.h[0] == r.h[3];
  return r;
}
// alpha for the four channels of edge j -> i with edge score ae[h] (row of [*, H])
__device__ __forceinline__ float4 alpha4(const Heads4& hs, const float* __restrict__ asj, const float* __restrict__ adi,
                                         const float* __restrict__ ae, const float* __restrict__ lsei) {
  float a[4];
  if (hs.same) {
    const int h = hs.h[0];
    a[0] = a[1] = a[2] = a[3] = expf(lrelu(asj[h] + adi[h] + ae[h]) - lsei[h]);
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int h = hs.h[k];
      a[k] = expf(lrelu(asj[h] + adi[h] + ae[h]) - lsei[h]);
    }
  }
  return make_float4(a[0], a[1], a[2], a[3]);
}

// x_loc_i = x_i + drop(alpha_ii Y_i + sum_{j->i, j != i} alpha_ji Y_j + bias)  [+ column sums of x_loc]
template <bool STATS>
__global__ void __launch_bounds__(1024) k_gat_fwd(GpsGraph g, int d, int C, const float* __restrict__ Y, int64_t ldy,
                                                  const float* __restrict__ a_src, const float* __restrict__ a_dst,
                                                  const float* __restrict__ a_edge, const float* __restrict__ a_self,
                                                  const float* __restrict__ lse, const float* __restrict__ bias,
                                                  const float* __restrict__ x, float* __restrict__ xloc, DropCfg drop,
                                                  double* stats) {
  extern __shared__ float4 sm[];
  const int c = threadIdx.x * 4, ry = threadIdx.y, RY = blockDim.y, C4 = blockDim.x;
  const int H = d / C;
  const uint64_t offs = drop.offset + ((drop.p > 0.f && drop.offset_dev) ? *drop.offset_dev : 0ull);
  const float4 b4 = ld4(bias + c);
  const Heads4 hs = heads4(c, C);
  float4 acc[2] = {f4zero(), f4zero()};
  for (int64_t i = (int64_t)blockIdx.x * RY + ry; i < g.N; i += (int64_t)gridDim.x * RY) {
    const float* adi = a_dst + i * H;
    const float* lsei = lse + i * H;
    float4 a = f4mul(alpha4(hs, a_src + i * H, adi, a_self + i * H, lsei), ld4(Y + i * ldy + c));
    for (int k = g.dst_ptr[i]; k < g.dst_ptr[i + 1]; ++k) {
      const int j = g.dst_src[k];
      if (j == (int)i) continue;
      const float4 al = alpha4(hs, a_src + (int64_t)j * H, adi, a_edge + (int64_t)g.dst_eid[k] * H, lsei);
      a = f4fma(al, ld4(Y + (int64_t)j * ldy + c), a);
    }
    float4 h = f4add(a, b4);
    if (drop.p > 0.f) h = f4mul(h, dropout_scale4(drop.p, drop.seed, offs, drop.site, ((uint64_t)i * (uint64_t)d + c) >> 2));
    const float4 v = f4add(ld4(x + i * d + c), h);
    st4(xloc + i * d + c, v);
    if (STATS) {
      acc[0] = f4add(acc[0], v);
      acc[1] = f4fma(v, v, acc[1]);
    }
  }
  if (STATS) {   // CTA reduction over threadIdx.y, then double atomics (as scatter.cu's block_stats)
    if (RY > 1) {
      sm[ry * C4 + threadIdx.x] = acc[0];
      sm[(RY + ry) * C4 + threadIdx.x] = acc[1];
      __syncthreads();
      if (ry == 0)
        for (int y = 1; y < RY; ++y) {
          acc[0] = f4add(acc[0], sm[y * C4 + threadIdx.x]);
          acc[1] = f4add(acc[1], sm[(RY + y) * C4 + threadIdx.x]);
        }
    }
    if (ry == 0) {
      const float* s0 = reinterpret_cast<const float*>(&acc[0]);
      const float* s1 = reinterpret_cast<const float*>(&acc[1]);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        atomic_add_f64(stats + c + k, (double)s0[k]);
        atomic_add_f64(stats + d + c + k, (double)s1[k]);
      }
    }
  }
}

__device__ __forceinline__ float warp_dot_head(const float* __restrict__ p, const float* __restrict__ q, int C, int lane) {
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s = fmaf(p[c], q[c], s);
  return warp_sum(s);
}

// Backward, destination pass: one warp per node i, heads in turn.  g_alpha_ji = g_h[i,h] . Y[j,h];
// Delta = sum alpha g_alpha;  g_z = alpha (g_alpha - Delta) leaky_relu'(pre);  g_a_dst[i] = sum g_z (loop included);
// per edge g_a_edge = g_z + g_z_loop / deg_i.  Writes alpha, g_z, g_a_edge [E, H] (0 on removed self loops) and
// alpha_loop, g_z_loop, g_a_dst [N, H]; then grad_edge_attr[e] = sum_h g_a_edge[e,h] v[h] (0 on removed self loops).
__global__ void k_gat_bwd_dst(GpsGraph g, int d, int C, const float* __restrict__ Y, int64_t ldy,
                              const float* __restrict__ a_src, const float* __restrict__ a_dst,
                              const float* __restrict__ a_edge, const float* __restrict__ a_self,
                              const float* __restrict__ lse, const float* __restrict__ g_h, const float* __restrict__ v,
                              float* __restrict__ alpha, float* __restrict__ gz, float* __restrict__ gae,
                              float* __restrict__ alpha_loop, float* __restrict__ gz_loop, float* __restrict__ gad,
                              float* __restrict__ grad_ea) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (i >= g.N) return;
  const int H = d / C;
  const int b = g.dst_ptr[i], en = g.dst_ptr[i + 1];
  int deg = 0;
  for (int q = b; q < en; ++q) deg += g.dst_src[q] != (int)i;
  const float* ghi = g_h + i * d;
  for (int h = 0; h < H; ++h) {
    const float ad = a_dst[i * H + h], L = lse[i * H + h];
    const float pre_s = a_src[i * H + h] + ad + a_self[i * H + h];
    const float al_s = expf(lrelu(pre_s) - L);
    const float ga_s = warp_dot_head(ghi + h * C, Y + i * ldy + h * C, C, lane);
    float delta = al_s * ga_s;
    for (int q = b; q < en; ++q) {   // g_alpha per edge, parked in gz
      const int j = g.dst_src[q];
      if (j == (int)i) continue;
      const int64_t e = g.dst_eid[q];
      const float ga = warp_dot_head(ghi + h * C, Y + (int64_t)j * ldy + h * C, C, lane);
      delta = fmaf(expf(lrelu(a_src[(int64_t)j * H + h] + ad + a_edge[e * H + h]) - L), ga, delta);
      if (lane == 0) gz[e * H + h] = ga;
    }
    __syncwarp();
    const float gz_s = al_s * (ga_s - delta) * lrelu_d(pre_s);
    float sum = 0.f;
    for (int q = b + lane; q < en; q += 32) {
      const int j = g.dst_src[q];
      const int64_t e = g.dst_eid[q];
      if (j == (int)i) {
        alpha[e * H + h] = 0.f;
        gz[e * H + h] = 0.f;
        continue;
      }
      const float pre = a_src[(int64_t)j * H + h] + ad + a_edge[e * H + h];
      const float al = expf(lrelu(pre) - L);
      const float gzv = al * (gz[e * H + h] - delta) * lrelu_d(pre);
      alpha[e * H + h] = al;
      gz[e * H + h] = gzv;
      sum += gzv;
    }
    sum = warp_sum(sum) + gz_s;
    const float share = deg > 0 ? gz_s / (float)deg : 0.f;   // the loop's score is the mean of the in-edge scores
    for (int q = b + lane; q < en; q += 32) {
      const int64_t e = g.dst_eid[q];
      gae[e * H + h] = g.dst_src[q] == (int)i ? 0.f : gz[e * H + h] + share;
    }
    if (lane == 0) {
      alpha_loop[i * H + h] = al_s;
      gz_loop[i * H + h] = gz_s;
      gad[i * H + h] = sum;
    }
    __syncwarp();
  }
  if (!grad_ea) return;
  for (int q = b; q < en; ++q) {
    const int64_t e = g.dst_eid[q];
    const bool self = g.dst_src[q] == (int)i;
    for (int k = lane * 4; k < d; k += 128) {
      float4 acc = f4zero();
      if (!self)
        for (int h = 0; h < H; ++h) {
          const float w = gae[e * H + h];
          acc = f4fma(make_float4(w, w, w, w), ld4(v + (int64_t)h * d + k), acc);
        }
      st4(grad_ea + e * d + k, acc);
    }
  }
}

// Backward, source pass: thread (node j, 4 channels) over j's out-edges in CSC (edge-id) order.
//   gY[j,h,:] = alpha_jj g_h[j,h,:] + sum_{j->i, i != j} alpha_ji g_h[i,h,:] + G_src[j,h] att_src[h] + g_a_dst[j,h] att_dst[h]
//   G_src[j,h] = g_z_loop[j,h] + sum_{j->i, i != j} g_z[ji,h]   (written to gsrc [N, H])
__global__ void k_gat_bwd_src(GpsGraph g, int d, int C, const float* __restrict__ g_h, const float* __restrict__ alpha,
                              const float* __restrict__ gz, const float* __restrict__ alpha_loop,
                              const float* __restrict__ gz_loop, const float* __restrict__ gad,
                              const float* __restrict__ att_src, const float* __restrict__ att_dst, float* __restrict__ gY,
                              int64_t ldg, Planes gYp, float* __restrict__ gsrc) {
  const int c = threadIdx.x * 4, ry = threadIdx.y, RY = blockDim.y;
  const int H = d / C;
  const Heads4 hs = heads4(c, C);
  const float4 as4 = ld4(att_src + c), ad4 = ld4(att_dst + c);
  for (int64_t j = (int64_t)blockIdx.x * RY + ry; j < g.N; j += (int64_t)gridDim.x * RY) {
    float al[4], G[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      al[k] = alpha_loop[j * H + hs.h[k]];
      G[k] = gz_loop[j * H + hs.h[k]];
    }
    const float4 gj = ld4(g_h + j * d + c);
    float4 a = f4mul(make_float4(al[0], al[1], al[2], al[3]), gj);
    for (int q = g.src_ptr[j]; q < g.src_ptr[j + 1]; ++q) {
      const int i = g.src_dst[q];
      if (i == (int)j) continue;
      const int64_t e = g.src_eid[q];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        al[k] = alpha[e * H + hs.h[k]];
        G[k] += gz[e * H + hs.h[k]];
      }
      a = f4fma(make_float4(al[0], al[1], al[2], al[3]), ld4(g_h + (int64_t)i * d + c), a);
    }
    float gd[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) gd[k] = gad[j * H + hs.h[k]];
    a = f4fma(make_float4(G[0], G[1], G[2], G[3]), as4, a);
    a = f4fma(make_float4(gd[0], gd[1], gd[2], gd[3]), ad4, a);
    st4(gY + j * ldg + c, a);
    if (gYp.hi) planes_store4(gYp, j, c, a);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if ((c + k) % C == 0) gsrc[j * H + hs.h[k]] = G[k];
  }
}

// Parameter gradients, stage 1 over node chunks: part[b] = [g_att_src (d) | g_att_dst (d) | g_bias (d)] of the rows
// [b*chunk, (b+1)*chunk), in row order
__global__ void k_gat_wgrad_nodes(int64_t N, int64_t chunk, int d, int C, const float* __restrict__ Y, int64_t ldy,
                                  const float* __restrict__ gsrc, const float* __restrict__ gad,
                                  const float* __restrict__ g_h, float* __restrict__ part) {
  const int64_t r0 = (int64_t)blockIdx.x * chunk;
  const int64_t r1 = r0 + chunk < N ? r0 + chunk : N;
  const int H = d / C;
  float* out = part + (int64_t)blockIdx.x * 3 * d;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    const int h = c / C;
    float s1 = 0.f, s2 = 0.f, s3 = 0.f;
    for (int64_t r = r0; r < r1; ++r) {
      const float y = Y[r * ldy + c];
      s1 = fmaf(gsrc[r * H + h], y, s1);
      s2 = fmaf(gad[r * H + h], y, s2);
      s3 += g_h[r * d + c];
    }
    out[c] = s1;
    out[d + c] = s2;
    out[2 * d + c] = s3;
  }
}

// stage 1 over edge chunks: part[b] = g_v [H, d] = sum_e g_a_edge[e,h] e_e over the edges [b*chunk, (b+1)*chunk)
__global__ void k_gat_wgrad_edges(int64_t E, int64_t chunk, int d, int H, const float* __restrict__ gae,
                                  const float* __restrict__ ea, float* __restrict__ part) {
  const int64_t e0 = (int64_t)blockIdx.x * chunk;
  const int64_t e1 = e0 + chunk < E ? e0 + chunk : E;
  float* out = part + (int64_t)blockIdx.x * H * d;
  for (int q = threadIdx.x; q < H * d; q += blockDim.x) {
    const int h = q / d, k = q % d;
    float s = 0.f;
    for (int64_t e = e0; e < e1; ++e) s = fmaf(gae[e * H + h], ea[e * d + k], s);
    out[q] = s;
  }
}

// stage 2: column sums of the parts in chunk order; column col goes to out[col / w][col % w] (NULL: not needed),
// written or, accumulate, added
__global__ void k_gat_wgrad_sum(int64_t nparts, int w, int nout, const float* __restrict__ part, float* o0, float* o1,
                                float* o2, int accumulate) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  const int ncols = w * nout;
  if (col >= ncols) return;
  float s = 0.f;
#pragma unroll 8
  for (int64_t b = 0; b < nparts; ++b) s += part[b * ncols + col];
  float* base = col < w ? o0 : (col < 2 * w ? o1 : o2);
  if (!base) return;
  float* dst = base + col % w;
  *dst = accumulate ? *dst + s : s;
}

}  // namespace

// rows per stage-1 block: about one block per SM (at least 32 rows each), a function of the row count alone
static int64_t gat_chunk(int64_t rows) {
  const int64_t c = ceil_div(rows, (int64_t)kNumSMs);
  return c > 32 ? c : 32;
}

int gat_check(int64_t d, int64_t H) {
  GPS_REQUIRE(H > 0 && d % H == 0, GPS_ERR_ARG, "GAT: dim_h %lld is not a multiple of heads %lld", (long long)d,
              (long long)H);
  GPS_REQUIRE(d > 0 && d % 4 == 0 && d <= 4096, GPS_ERR_UNSUPPORTED, "GAT needs d %% 4 == 0 and 0 < d <= 4096 (got %lld)",
              (long long)d);
  return GPS_OK;
}

GatScores gat_scores(float* base, int64_t N, int64_t E, int64_t H) {
  GatScores s;
  s.a_src = base;
  s.a_dst = base ? base + N * H : nullptr;
  s.a_self = base ? base + 2 * N * H : nullptr;
  s.lse = base ? base + 3 * N * H : nullptr;
  s.a_edge = base ? base + 4 * N * H : nullptr;
  (void)E;
  return s;
}

int64_t gat_bwd_workspace_floats(int64_t N, int64_t E, int64_t H, int64_t d) {
  return 3 * E * H + 4 * N * H + ceil_div(N, gat_chunk(N)) * 3 * d + ceil_div(E, gat_chunk(E)) * H * d;
}

int gat_fold_fwd(const float* W_edge, const float* att_edge, int64_t d, int64_t H, float* v, cudaStream_t st) {
  GPS_TRY(gat_check(d, H));
  k_gat_fold<<<(unsigned)ceil_div(H * d, (int64_t)256), 256, 0, st>>>(W_edge, att_edge, (int)d, (int)(d / H), v);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int gat_fold_bwd(const float* W_edge, const float* att_edge, const float* g_v, int64_t d, int64_t H, float* gW,
                 float* gatt, bool accumulate, cudaStream_t st) {
  GPS_TRY(gat_check(d, H));
  if (!gW && !gatt) return GPS_OK;
  k_gat_fold_bwd<<<(unsigned)ceil_div(d, (int64_t)kWarpsPerBlock), 32 * kWarpsPerBlock, 0, st>>>(
      W_edge, att_edge, g_v, (int)d, (int)(d / H), gW, gatt, accumulate ? 1 : 0);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int gat_fwd(const GpsGraph& g, int64_t d, int64_t H, const float* Y, int64_t ldy, const float* ea, const float* v,
            const float* att_src, const float* att_dst, const float* bias, const float* x, GatScores s, float* xloc,
            DropCfg drop, double* stats, cudaStream_t st) {
  GPS_TRY(gat_check(d, H));
  const int C = (int)(d / H);
  if (g.E > 0) {
    k_gat_edge_scores<<<(unsigned)ceil_div(g.E, (int64_t)kWarpsPerBlock), 32 * kWarpsPerBlock, 0, st>>>(
        g.E, (int)d, (int)H, ea, v, s.a_edge);
    GPS_LAUNCH_CHECK();
  }
  if (g.N == 0) return GPS_OK;
  const unsigned node_blocks = (unsigned)ceil_div(g.N, (int64_t)kWarpsPerBlock);
  k_gat_node_scores<<<node_blocks, 32 * kWarpsPerBlock, 0, st>>>(g.N, (int)d, C, Y, ldy, att_src, att_dst, s.a_src,
                                                                 s.a_dst);
  GPS_LAUNCH_CHECK();
  k_gat_softmax_stats<<<node_blocks, 32 * kWarpsPerBlock, 0, st>>>(g, (int)H, s.a_src, s.a_dst, s.a_edge, s.a_self, s.lse);
  GPS_LAUNCH_CHECK();
  Geom gm;
  GPS_TRY(gat_geom(g.N, d, stats != nullptr, &gm));
  if (stats)
    k_gat_fwd<true><<<gm.grid, gm.block, gm.smem, st>>>(g, (int)d, C, Y, ldy, s.a_src, s.a_dst, s.a_edge, s.a_self, s.lse,
                                                        bias, x, xloc, drop, stats);
  else
    k_gat_fwd<false><<<gm.grid, gm.block, 0, st>>>(g, (int)d, C, Y, ldy, s.a_src, s.a_dst, s.a_edge, s.a_self, s.lse,
                                                   bias, x, xloc, drop, nullptr);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int gat_bwd(const GpsGraph& g, int64_t d, int64_t H, const float* Y, int64_t ldy, const float* ea, const float* v,
            const float* att_src, const float* att_dst, GatScores s, const float* g_h, float* ws, float* gY, int64_t ldg,
            Planes gYp, float* grad_ea, float* g_v, float* g_att_src, float* g_att_dst, float* g_bias, bool accumulate,
            cudaStream_t st) {
  GPS_TRY(gat_check(d, H));
  const int64_t N = g.N, E = g.E;
  const int C = (int)(d / H);
  float* alpha = ws;
  float* gz = alpha + E * H;
  float* gae = gz + E * H;
  float* alpha_loop = gae + E * H;
  float* gz_loop = alpha_loop + N * H;
  float* gad = gz_loop + N * H;
  float* gsrc = gad + N * H;
  float* part_n = gsrc + N * H;
  const int64_t chunk_n = gat_chunk(N), parts_n = ceil_div(N, chunk_n);
  float* part_e = part_n + parts_n * 3 * d;
  const int64_t chunk_e = gat_chunk(E), parts_e = ceil_div(E, chunk_e);
  if (N > 0) {
    const unsigned node_blocks = (unsigned)ceil_div(N, (int64_t)kWarpsPerBlock);
    k_gat_bwd_dst<<<node_blocks, 32 * kWarpsPerBlock, 0, st>>>(g, (int)d, C, Y, ldy, s.a_src, s.a_dst, s.a_edge, s.a_self,
                                                               s.lse, g_h, v, alpha, gz, gae, alpha_loop, gz_loop, gad,
                                                               grad_ea);
    GPS_LAUNCH_CHECK();
    Geom gm;
    GPS_TRY(gat_geom(N, d, false, &gm));
    k_gat_bwd_src<<<gm.grid, gm.block, 0, st>>>(g, (int)d, C, g_h, alpha, gz, alpha_loop, gz_loop, gad, att_src, att_dst,
                                                gY, ldg, gYp, gsrc);
    GPS_LAUNCH_CHECK();
    k_gat_wgrad_nodes<<<(unsigned)parts_n, 256, 0, st>>>(N, chunk_n, (int)d, C, Y, ldy, gsrc, gad, g_h, part_n);
    GPS_LAUNCH_CHECK();
  }
  if (E > 0) {
    k_gat_wgrad_edges<<<(unsigned)parts_e, 256, 0, st>>>(E, chunk_e, (int)d, (int)H, gae, ea, part_e);
    GPS_LAUNCH_CHECK();
  }
  if (g_att_src || g_att_dst || g_bias) {   // N = 0: writes zeros (or adds nothing)
    k_gat_wgrad_sum<<<(unsigned)ceil_div(3 * d, (int64_t)128), 128, 0, st>>>(N > 0 ? parts_n : 0, (int)d, 3, part_n,
                                                                            g_att_src, g_att_dst, g_bias,
                                                                            accumulate ? 1 : 0);
    GPS_LAUNCH_CHECK();
  }
  if (g_v) {
    k_gat_wgrad_sum<<<(unsigned)ceil_div(H * d, (int64_t)128), 128, 0, st>>>(E > 0 ? parts_e : 0, (int)(H * d), 1, part_e,
                                                                            g_v, nullptr, nullptr, 0);
    GPS_LAUNCH_CHECK();
  }
  return GPS_OK;
}

}  // namespace gps
