// bigbird.cu — the BigBird global model's own stages (graphgps/layer/bigbird_layer.py:1116-1356,1667-1706 of the
// reference): block-sparse attention over each graph's packed rows, forward and backward, row-wise LayerNorm forward and
// backward, and the sigmoid hidden activation.  The dense products around them run on the TMA GEMM (layer.cu).
//
// Attention works on the packed [N, d] Q / K / V rows: local position p of graph g is node graph_ptr[g] + p, and a
// position >= n_g is a masked key (the reference adds -10000 to it, which in fp32 is an exclusion unless two logits
// differ by ~1e4).  Query block i of head h attends to the key blocks key_idx[key_ptr[h][i] .. key_ptr[h][i+1]), a
// multiset: a block listed twice enters numerator and denominator twice.  One warp per (graph, head, block); keys (or,
// in the key-major backward, queries) go across the lanes in chunks of 32, and the head's hd columns across the lanes
// for the weighted sums.  Every sum runs in a fixed order: the same bits in every run, and no atomics.
#include "kernels.cuh"

namespace gps {

namespace {

constexpr int kWarps = 4;     // warps per CTA of the attention kernels
constexpr int kMaxHd = 128;   // head dim bound: kMaxHd / 32 accumulators per lane
constexpr int kAcc = kMaxHd / 32;

struct BbGeom {
  const int* gptr;
  int B, H, hd, bs, nb;
  const int* ptr;   // key_ptr (query-major) or query_ptr (key-major)
  const int* idx;
  float scale;
};

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// sum_k a[k] * b[k] over hd columns (a in shared memory, b a row in global memory), in column order
__device__ __forceinline__ float dot_row(const float* a, const float* __restrict__ b, int hd) {
  float s = 0.f;
  for (int k = 0; k < hd; ++k) s = fmaf(a[k], b[k], s);
  return s;
}

// the (graph, head, block) of this warp; false when the warp has no work
__device__ __forceinline__ bool bb_item(const BbGeom& G, int& g, int& h, int& blk, int& n0, int& n) {
  const int64_t item = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (item >= (int64_t)G.B * G.H * G.nb) return false;
  blk = (int)(item % G.nb);
  h = (int)((item / G.nb) % G.H);
  g = (int)(item / ((int64_t)G.nb * G.H));
  n0 = G.gptr[g];
  n = G.gptr[g + 1] - n0;
  return blk * G.bs < n;
}

// global node of flattened entry t of a block list (t / bs: list slot, t % bs: position in the block); -1 if masked
__device__ __forceinline__ int list_node(const BbGeom& G, int lb, int t, int n0, int n) {
  const int p = G.idx[lb + t / G.bs] * G.bs + t % G.bs;
  return p < n ? n0 + p : -1;
}

// ---------------------------------------------------------------------------------------------- forward
// O[q] = sum_k w_k exp(s_qk - m) V[k] / sum_k w_k exp(s_qk - m), s = (q . k) / sqrt(hd), w = multiplicity;
// lse[q, h] = m + log(sum) (online over chunks of 32 keys)
__global__ void __launch_bounds__(kWarps * 32) k_bb_fwd(BbGeom G, const float* __restrict__ Q, const float* __restrict__ K,
                                                         const float* __restrict__ V, int64_t ld, float* __restrict__ O,
                                                         int64_t ldo, float* __restrict__ lse) {
  __shared__ float s_q[kWarps][kMaxHd];
  __shared__ float s_p[kWarps][32];
  __shared__ int s_j[kWarps][32];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int g, h, blk, n0, n;
  if (!bb_item(G, g, h, blk, n0, n)) return;
  const int lb = G.ptr[h * (G.nb + 1) + blk], L = (G.ptr[h * (G.nb + 1) + blk + 1] - lb) * G.bs;
  const int64_t col = (int64_t)h * G.hd;
  const int qend = min(blk * G.bs + G.bs, n);
  for (int qp = blk * G.bs; qp < qend; ++qp) {
    const int64_t row = n0 + qp;
    __syncwarp();
    for (int k = lane; k < G.hd; k += 32) s_q[w][k] = Q[row * ld + col + k] * G.scale;
    __syncwarp();
    float m = -INFINITY, l = 0.f, acc[kAcc];
#pragma unroll
    for (int a = 0; a < kAcc; ++a) acc[a] = 0.f;
    for (int c = 0; c < L; c += 32) {
      const int t = c + lane;
      const int j = t < L ? list_node(G, lb, t, n0, n) : -1;
      const float s = j >= 0 ? dot_row(s_q[w], K + (int64_t)j * ld + col, G.hd) : -INFINITY;
      const float mn = fmaxf(m, warp_max(s));
      const float corr = m == -INFINITY ? 0.f : expf(m - mn);
      const float p = j >= 0 ? expf(s - mn) : 0.f;
      l = l * corr + warp_sum(p);
      s_p[w][lane] = p;
      s_j[w][lane] = j;
      __syncwarp();
      const int cnt = min(32, L - c);
#pragma unroll
      for (int a = 0; a < kAcc; ++a) acc[a] *= corr;
      for (int u = 0; u < cnt; ++u) {
        const int ju = s_j[w][u];
        if (ju < 0) continue;
        const float pu = s_p[w][u];
        const float* vr = V + (int64_t)ju * ld + col;
#pragma unroll
        for (int a = 0; a < kAcc; ++a)
          if (lane + 32 * a < G.hd) acc[a] = fmaf(pu, vr[lane + 32 * a], acc[a]);
      }
      __syncwarp();
      m = mn;
    }
    const float inv = 1.f / l;
#pragma unroll
    for (int a = 0; a < kAcc; ++a)
      if (lane + 32 * a < G.hd) O[row * ldo + col + lane + 32 * a] = acc[a] * inv;
    if (lane == 0) lse[row * G.H + h] = m + logf(l);
  }
}

// ---------------------------------------------------------------------------------------------- backward
// query-major: delta[q] = dO[q] . O[q]; dQ[q] = scale sum_k w_k p_qk (dO[q] . V[k] - delta[q]) K[k]
__global__ void __launch_bounds__(kWarps * 32) k_bb_bwd_q(BbGeom G, const float* __restrict__ Q,
                                                           const float* __restrict__ K, const float* __restrict__ V,
                                                           int64_t ld, const float* __restrict__ O,
                                                           const float* __restrict__ dO, int64_t ldo,
                                                           const float* __restrict__ lse, float* __restrict__ delta,
                                                           float* __restrict__ dQ, int64_t ldg) {
  __shared__ float s_q[kWarps][kMaxHd];
  __shared__ float s_do[kWarps][kMaxHd];
  __shared__ float s_p[kWarps][32];
  __shared__ int s_j[kWarps][32];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int g, h, blk, n0, n;
  if (!bb_item(G, g, h, blk, n0, n)) return;
  const int lb = G.ptr[h * (G.nb + 1) + blk], L = (G.ptr[h * (G.nb + 1) + blk + 1] - lb) * G.bs;
  const int64_t col = (int64_t)h * G.hd;
  const int qend = min(blk * G.bs + G.bs, n);
  for (int qp = blk * G.bs; qp < qend; ++qp) {
    const int64_t row = n0 + qp;
    __syncwarp();
    float dl = 0.f;
    for (int k = lane; k < G.hd; k += 32) {
      s_q[w][k] = Q[row * ld + col + k] * G.scale;
      const float go = dO[row * ldo + col + k];
      s_do[w][k] = go;
      dl = fmaf(go, O[row * ldo + col + k], dl);
    }
    dl = warp_sum(dl);
    if (lane == 0) delta[row * G.H + h] = dl;
    const float ls = lse[row * G.H + h];
    __syncwarp();
    float acc[kAcc];
#pragma unroll
    for (int a = 0; a < kAcc; ++a) acc[a] = 0.f;
    for (int c = 0; c < L; c += 32) {
      const int t = c + lane;
      const int j = t < L ? list_node(G, lb, t, n0, n) : -1;
      float ds = 0.f;
      if (j >= 0) {
        const float p = expf(dot_row(s_q[w], K + (int64_t)j * ld + col, G.hd) - ls);
        ds = p * (dot_row(s_do[w], V + (int64_t)j * ld + col, G.hd) - dl);
      }
      s_p[w][lane] = ds;
      s_j[w][lane] = j;
      __syncwarp();
      const int cnt = min(32, L - c);
      for (int u = 0; u < cnt; ++u) {
        const int ju = s_j[w][u];
        if (ju < 0) continue;
        const float du = s_p[w][u];
        const float* kr = K + (int64_t)ju * ld + col;
#pragma unroll
        for (int a = 0; a < kAcc; ++a)
          if (lane + 32 * a < G.hd) acc[a] = fmaf(du, kr[lane + 32 * a], acc[a]);
      }
      __syncwarp();
    }
#pragma unroll
    for (int a = 0; a < kAcc; ++a)
      if (lane + 32 * a < G.hd) dQ[row * ldg + col + lane + 32 * a] = acc[a] * G.scale;
  }
}

// key-major over the transposed lists: dV[k] = sum_q w p_qk dO[q], dK[k] = scale sum_q w ds_qk Q[q]
__global__ void __launch_bounds__(kWarps * 32) k_bb_bwd_kv(BbGeom G, const float* __restrict__ Q,
                                                            const float* __restrict__ K, const float* __restrict__ V,
                                                            int64_t ld, const float* __restrict__ dO, int64_t ldo,
                                                            const float* __restrict__ lse,
                                                            const float* __restrict__ delta, float* __restrict__ dK,
                                                            float* __restrict__ dV, int64_t ldg) {
  __shared__ float s_k[kWarps][kMaxHd];
  __shared__ float s_v[kWarps][kMaxHd];
  __shared__ float s_p[kWarps][32];
  __shared__ float s_d[kWarps][32];
  __shared__ int s_i[kWarps][32];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int g, h, blk, n0, n;
  if (!bb_item(G, g, h, blk, n0, n)) return;
  const int lb = G.ptr[h * (G.nb + 1) + blk], L = (G.ptr[h * (G.nb + 1) + blk + 1] - lb) * G.bs;
  const int64_t col = (int64_t)h * G.hd;
  const int kend = min(blk * G.bs + G.bs, n);
  for (int kp = blk * G.bs; kp < kend; ++kp) {
    const int64_t row = n0 + kp;
    __syncwarp();
    for (int k = lane; k < G.hd; k += 32) {
      s_k[w][k] = K[row * ld + col + k];
      s_v[w][k] = V[row * ld + col + k];
    }
    __syncwarp();
    float ak[kAcc], av[kAcc];
#pragma unroll
    for (int a = 0; a < kAcc; ++a) ak[a] = av[a] = 0.f;
    for (int c = 0; c < L; c += 32) {
      const int t = c + lane;
      const int i = t < L ? list_node(G, lb, t, n0, n) : -1;
      float p = 0.f, ds = 0.f;
      if (i >= 0) {
        // the score as the forward computed it: (scale q) . k in column order
        const float* qr = Q + (int64_t)i * ld + col;
        float s = 0.f;
        for (int k = 0; k < G.hd; ++k) s = fmaf(qr[k] * G.scale, s_k[w][k], s);
        p = expf(s - lse[(int64_t)i * G.H + h]);
        ds = p * (dot_row(s_v[w], dO + (int64_t)i * ldo + col, G.hd) - delta[(int64_t)i * G.H + h]);
      }
      s_p[w][lane] = p;
      s_d[w][lane] = ds;
      s_i[w][lane] = i;
      __syncwarp();
      const int cnt = min(32, L - c);
      for (int u = 0; u < cnt; ++u) {
        const int iu = s_i[w][u];
        if (iu < 0) continue;
        const float pu = s_p[w][u], du = s_d[w][u];
        const float* qr = Q + (int64_t)iu * ld + col;
        const float* gr = dO + (int64_t)iu * ldo + col;
#pragma unroll
        for (int a = 0; a < kAcc; ++a)
          if (lane + 32 * a < G.hd) {
            av[a] = fmaf(pu, gr[lane + 32 * a], av[a]);
            ak[a] = fmaf(du, qr[lane + 32 * a], ak[a]);
          }
      }
      __syncwarp();
    }
#pragma unroll
    for (int a = 0; a < kAcc; ++a)
      if (lane + 32 * a < G.hd) {
        dK[row * ldg + col + lane + 32 * a] = ak[a] * G.scale;
        dV[row * ldg + col + lane + 32 * a] = av[a];
      }
  }
}

BbGeom bb_geom(const GpsGraph& g, int64_t H, int64_t hd, const GpsBigBird& bb, bool key_major) {
  BbGeom G;
  G.gptr = g.graph_ptr;
  G.B = (int)g.B; G.H = (int)H; G.hd = (int)hd; G.bs = (int)bb.block_size; G.nb = (int)bb.num_blocks;
  G.ptr = key_major ? bb.query_ptr : bb.key_ptr;
  G.idx = key_major ? bb.query_idx : bb.key_idx;
  G.scale = (float)(1.0 / sqrt((double)hd));
  return G;
}

unsigned bb_grid(const BbGeom& G) { return (unsigned)ceil_div((int64_t)G.B * G.H * G.nb, kWarps); }

// ---------------------------------------------------------------------------------------------- LayerNorm
// one warp per row; lanes own float4 column groups c4 = lane + 32 k.  Column statistics / parameter-gradient partials
// go through per-warp shared-memory rows that each lane updates in its own columns only, then are summed over the
// warps in order: deterministic.
int ln_warps(int64_t d) {
  int64_t w = 6144 / d;   // 2 * d floats per warp within 48 KB
  return (int)(w > 8 ? 8 : (w < 1 ? 1 : w));
}

struct LnFwd {
  const float* z; const float* gamma; const float* beta; float eps;
  float* mean; float* rstd;
  float* out; Planes outp;
  const float* R1; const float* R2; DropCfg drop;
  double* stats;
  int64_t rows, d;
};

__global__ void __launch_bounds__(256) k_ln_fwd(LnFwd a) {
  extern __shared__ float sm[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, W = blockDim.x >> 5;
  const int C4 = (int)(a.d >> 2);
  float* st = sm + (int64_t)w * 2 * a.d;
  if (a.stats)
    for (int c = lane; c < 2 * a.d; c += 32) st[c] = 0.f;
  __syncwarp();
  if (a.drop.p > 0.f && a.drop.offset_dev) a.drop.offset += *a.drop.offset_dev;
  for (int64_t r = (int64_t)blockIdx.x * W + w; r < a.rows; r += (int64_t)gridDim.x * W) {
    const float* zr = a.z + r * a.d;
    float s = 0.f;
    for (int c4 = lane; c4 < C4; c4 += 32) {
      const float4 v = ld4(zr + c4 * 4);
      s += (v.x + v.y) + (v.z + v.w);
    }
    const float mu = warp_sum(s) / (float)a.d;
    float q = 0.f;
    for (int c4 = lane; c4 < C4; c4 += 32) {
      const float4 v = ld4(zr + c4 * 4);
      const float x0 = v.x - mu, x1 = v.y - mu, x2 = v.z - mu, x3 = v.w - mu;
      q += (x0 * x0 + x1 * x1) + (x2 * x2 + x3 * x3);
    }
    const float rs = 1.f / sqrtf(warp_sum(q) / (float)a.d + a.eps);
    if (lane == 0) {
      a.mean[r] = mu;
      a.rstd[r] = rs;
    }
    for (int c4 = lane; c4 < C4; c4 += 32) {
      const float4 v = ld4(zr + c4 * 4);
      const float4 gm = ld4(a.gamma + c4 * 4), bt = ld4(a.beta + c4 * 4);
      float4 y = make_float4((v.x - mu) * rs * gm.x + bt.x, (v.y - mu) * rs * gm.y + bt.y, (v.z - mu) * rs * gm.z + bt.z,
                             (v.w - mu) * rs * gm.w + bt.w);
      if (a.drop.p > 0.f)
        y = f4mul(y, dropout_scale4(a.drop.p, a.drop.seed, a.drop.offset, a.drop.site, (uint64_t)r * C4 + c4));
      if (a.R1) y = f4add(y, ld4(a.R1 + r * a.d + c4 * 4));
      if (a.R2) y = f4add(y, ld4(a.R2 + r * a.d + c4 * 4));
      st4(a.out + r * a.d + c4 * 4, y);
      if (a.outp.hi) planes_store4(a.outp, r, c4 * 4, y);
      if (a.stats) {
        float* s0 = st + c4 * 4;
        float* s1 = st + a.d + c4 * 4;
        s0[0] += y.x; s0[1] += y.y; s0[2] += y.z; s0[3] += y.w;
        s1[0] += y.x * y.x; s1[1] += y.y * y.y; s1[2] += y.z * y.z; s1[3] += y.w * y.w;
      }
    }
  }
  if (!a.stats) return;
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * a.d; c += blockDim.x) {
    float t = 0.f;
    for (int k = 0; k < W; ++k) t += sm[(int64_t)k * 2 * a.d + c];
    atomic_add_f64(a.stats + c, (double)t);
  }
}

struct LnBwd {
  const float* g; DropCfg gdrop;           // upstream gradient and the dropout in front of the LayerNorm's output
  const float* z; const float* gamma; const float* mean; const float* rstd;
  float* out1; Planes out1p; DropCfg drop1; // out1 = drop1(dz)
  float* out2; const float* add;           // out2 = dz (+ add)
  float* part;                             // [gridDim.x][2][d]: per-CTA sums of g' * xhat and g'
  int64_t rows, d;
};

__global__ void __launch_bounds__(256) k_ln_bwd(LnBwd a) {
  extern __shared__ float sm[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, W = blockDim.x >> 5;
  const int C4 = (int)(a.d >> 2);
  float* st = sm + (int64_t)w * 2 * a.d;
  for (int c = lane; c < 2 * a.d; c += 32) st[c] = 0.f;
  __syncwarp();
  if (a.gdrop.p > 0.f && a.gdrop.offset_dev) a.gdrop.offset += *a.gdrop.offset_dev;
  if (a.drop1.p > 0.f && a.drop1.offset_dev) a.drop1.offset += *a.drop1.offset_dev;
  const float inv_d = 1.f / (float)a.d;
  for (int64_t r = (int64_t)blockIdx.x * W + w; r < a.rows; r += (int64_t)gridDim.x * W) {
    const float mu = a.mean[r], rs = a.rstd[r];
    auto gprime = [&](int c4) {
      float4 gv = ld4(a.g + r * a.d + c4 * 4);
      if (a.gdrop.p > 0.f)
        gv = f4mul(gv, dropout_scale4(a.gdrop.p, a.gdrop.seed, a.gdrop.offset, a.gdrop.site, (uint64_t)r * C4 + c4));
      return gv;
    };
    auto xhat = [&](int c4) {
      const float4 v = ld4(a.z + r * a.d + c4 * 4);
      return make_float4((v.x - mu) * rs, (v.y - mu) * rs, (v.z - mu) * rs, (v.w - mu) * rs);
    };
    float c1 = 0.f, c2 = 0.f;
    for (int c4 = lane; c4 < C4; c4 += 32) {
      const float4 gv = gprime(c4), xh = xhat(c4), gm = ld4(a.gamma + c4 * 4);
      const float4 dx = f4mul(gv, gm);
      c1 += (dx.x + dx.y) + (dx.z + dx.w);
      c2 += (dx.x * xh.x + dx.y * xh.y) + (dx.z * xh.z + dx.w * xh.w);
      float* s0 = st + c4 * 4;
      float* s1 = st + a.d + c4 * 4;
      s0[0] += gv.x * xh.x; s0[1] += gv.y * xh.y; s0[2] += gv.z * xh.z; s0[3] += gv.w * xh.w;
      s1[0] += gv.x; s1[1] += gv.y; s1[2] += gv.z; s1[3] += gv.w;
    }
    c1 = warp_sum(c1) * inv_d;
    c2 = warp_sum(c2) * inv_d;
    for (int c4 = lane; c4 < C4; c4 += 32) {
      const float4 gv = gprime(c4), xh = xhat(c4), gm = ld4(a.gamma + c4 * 4);
      const float4 dz = make_float4(rs * (gv.x * gm.x - c1 - xh.x * c2), rs * (gv.y * gm.y - c1 - xh.y * c2),
                                    rs * (gv.z * gm.z - c1 - xh.z * c2), rs * (gv.w * gm.w - c1 - xh.w * c2));
      if (a.out2) st4(a.out2 + r * a.d + c4 * 4, a.add ? f4add(dz, ld4(a.add + r * a.d + c4 * 4)) : dz);
      if (a.out1) {
        float4 o = dz;
        if (a.drop1.p > 0.f)
          o = f4mul(o, dropout_scale4(a.drop1.p, a.drop1.seed, a.drop1.offset, a.drop1.site, (uint64_t)r * C4 + c4));
        st4(a.out1 + r * a.d + c4 * 4, o);
        if (a.out1p.hi) planes_store4(a.out1p, r, c4 * 4, o);
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * a.d; c += blockDim.x) {
    float t = 0.f;
    for (int k = 0; k < W; ++k) t += sm[(int64_t)k * 2 * a.d + c];
    a.part[(int64_t)blockIdx.x * 2 * a.d + c] = t;
  }
}

// grad_gamma[c] (+)= sum_k part[k][0][c], grad_beta[c] (+)= sum_k part[k][1][c], k in order
__global__ void k_ln_grads(const float* __restrict__ part, int nparts, int64_t d, float* gg, float* gb, int accumulate) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= 2 * d) return;
  float t = 0.f;
  for (int k = 0; k < nparts; ++k) t += part[(int64_t)k * 2 * d + c];
  float* dst = c < d ? gg : gb;
  const int64_t j = c < d ? c : c - d;
  if (dst) dst[j] = accumulate ? dst[j] + t : t;
}

// sigmoid in place (+ planes), and its backward g *= s (1 - s) from the stored output s (+ planes)
__global__ void k_sigmoid(float* __restrict__ x, const float* __restrict__ s, int64_t n4, int64_t c4n, Planes p) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 v = ld4(x + i * 4);
    if (s) {
      const float4 sv = ld4(s + i * 4);
      v = make_float4(v.x * sv.x * (1.f - sv.x), v.y * sv.y * (1.f - sv.y), v.z * sv.z * (1.f - sv.z),
                      v.w * sv.w * (1.f - sv.w));
    } else {
      v = make_float4(1.f / (1.f + expf(-v.x)), 1.f / (1.f + expf(-v.y)), 1.f / (1.f + expf(-v.z)),
                      1.f / (1.f + expf(-v.w)));
    }
    st4(x + i * 4, v);
    if (p.hi) planes_store4(p, i / c4n, (i % c4n) * 4, v);
  }
}

}  // namespace

int bb_check(int64_t d, int64_t H, const GpsBigBird* bb) {
  GPS_REQUIRE(bb, GPS_ERR_ARG, "BigBird: null GpsBigBird");
  GPS_REQUIRE(H > 0 && d % H == 0, GPS_ERR_ARG, "BigBird: dim_h %lld not divisible by num_heads %lld", (long long)d,
              (long long)H);
  GPS_REQUIRE(d / H <= kMaxHd, GPS_ERR_UNSUPPORTED, "BigBird: head dim %lld > %d is not built", (long long)(d / H),
              kMaxHd);
  GPS_REQUIRE(bb->block_size >= 1 && bb->num_blocks >= 4, GPS_ERR_ARG,
              "BigBird: block_size must be >= 1 and num_blocks >= 4 (got %lld, %lld)", (long long)bb->block_size,
              (long long)bb->num_blocks);
  GPS_REQUIRE(bb->key_ptr && bb->key_idx && bb->query_ptr && bb->query_idx, GPS_ERR_ARG, "BigBird: null block list");
  GPS_REQUIRE(bb->hidden_act == GPS_BIGBIRD_RELU || bb->hidden_act == GPS_BIGBIRD_SIGMOID, GPS_ERR_ARG,
              "BigBird: unknown hidden_act %d", bb->hidden_act);
  return GPS_OK;
}

int bb_attn_fwd(const GpsGraph& g, int64_t H, int64_t hd, const GpsBigBird& bb, const float* Q, const float* K,
                const float* V, int64_t ld, float* O, int64_t ldo, float* lse, cudaStream_t st) {
  if (g.N == 0 || g.B == 0) return GPS_OK;
  const BbGeom G = bb_geom(g, H, hd, bb, false);
  k_bb_fwd<<<bb_grid(G), kWarps * 32, 0, st>>>(G, Q, K, V, ld, O, ldo, lse);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int bb_attn_bwd(const GpsGraph& g, int64_t H, int64_t hd, const GpsBigBird& bb, const float* Q, const float* K,
                const float* V, int64_t ld, const float* O, const float* dO, int64_t ldo, const float* lse, float* delta,
                float* dQ, float* dK, float* dV, int64_t ldg, cudaStream_t st) {
  if (g.N == 0 || g.B == 0) return GPS_OK;
  const BbGeom Gq = bb_geom(g, H, hd, bb, false);
  k_bb_bwd_q<<<bb_grid(Gq), kWarps * 32, 0, st>>>(Gq, Q, K, V, ld, O, dO, ldo, lse, delta, dQ, ldg);
  GPS_LAUNCH_CHECK();
  const BbGeom Gk = bb_geom(g, H, hd, bb, true);
  k_bb_bwd_kv<<<bb_grid(Gk), kWarps * 32, 0, st>>>(Gk, Q, K, V, ld, dO, ldo, lse, delta, dK, dV, ldg);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int64_t layernorm_part_floats(int64_t d) { return (int64_t)2 * kNumSMs * d; }

static int ln_width(int64_t d) {
  GPS_REQUIRE(d > 0 && d % 4 == 0 && d <= 4096, GPS_ERR_UNSUPPORTED,
              "LayerNorm needs d %% 4 == 0 and 0 < d <= 4096 (got %lld)", (long long)d);
  return GPS_OK;
}

int layernorm_fwd(const float* z, int64_t rows, int64_t d, const float* gamma, const float* beta, float eps, float* mean,
                  float* rstd, float* out, Planes outp, const float* R1, const float* R2, DropCfg drop, double* stats,
                  cudaStream_t st) {
  GPS_TRY(ln_width(d));
  if (rows == 0) return GPS_OK;
  LnFwd a{z, gamma, beta, eps, mean, rstd, out, outp, R1, R2, drop, stats, rows, d};
  const int W = stats ? ln_warps(d) : 8;
  int64_t grid = ceil_div(rows, W);
  if (stats && grid > kNumSMs / 2) grid = kNumSMs / 2;   // column sums: few CTAs, as the row-wise stages
  k_ln_fwd<<<(unsigned)grid, W * 32, stats ? (size_t)W * 2 * d * sizeof(float) : 0, st>>>(a);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int layernorm_bwd(const float* g, DropCfg gdrop, const float* z, int64_t rows, int64_t d, const float* gamma,
                  const float* mean, const float* rstd, float* out1, Planes out1p, DropCfg drop1, float* out2,
                  const float* add, float* part, float* grad_gamma, float* grad_beta, bool accumulate, cudaStream_t st) {
  GPS_TRY(ln_width(d));
  int nparts = 0;
  if (rows > 0) {
    LnBwd a{g, gdrop, z, gamma, mean, rstd, out1, out1p, drop1, out2, add, part, rows, d};
    const int W = ln_warps(d);
    int64_t grid = ceil_div(rows, W);
    if (grid > kNumSMs) grid = kNumSMs;
    nparts = (int)grid;
    k_ln_bwd<<<(unsigned)grid, W * 32, (size_t)W * 2 * d * sizeof(float), st>>>(a);
    GPS_LAUNCH_CHECK();
  }
  if (grad_gamma || grad_beta) {
    k_ln_grads<<<(unsigned)ceil_div(2 * d, 256), 256, 0, st>>>(part, nparts, d, grad_gamma, grad_beta,
                                                                accumulate ? 1 : 0);
    GPS_LAUNCH_CHECK();
  }
  return GPS_OK;
}

static unsigned elementwise_grid(int64_t n4) {
  const int64_t b = ceil_div(n4, 256);
  return (unsigned)(b < kNumSMs * 8 ? b : kNumSMs * 8);
}

int sigmoid_fwd(float* x, int64_t rows, int64_t d, Planes p, cudaStream_t st) {
  const int64_t n4 = rows * d / 4;
  if (n4 == 0) return GPS_OK;
  k_sigmoid<<<elementwise_grid(n4), 256, 0, st>>>(x, nullptr, n4, d / 4, p);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int sigmoid_bwd(float* g, const float* s, int64_t rows, int64_t d, Planes p, cudaStream_t st) {
  const int64_t n4 = rows * d / 4;
  if (n4 == 0) return GPS_OK;
  k_sigmoid<<<elementwise_grid(n4), 256, 0, st>>>(g, s, n4, d / 4, p);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

}  // namespace gps
