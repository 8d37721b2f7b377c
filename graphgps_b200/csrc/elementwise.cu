// elementwise.cu — row-wise stages of the GPS layer: BatchNorm apply / statistics / backward,
// residual adds, activation, dropout (gps_layer.py:188-194,212-217,222-229; gatedgcn_layer.py:72-83).
//
// One skeleton (k_rowwise): a thread owns one float4 column group and strides over rows, so the
// per-column BatchNorm constants live in registers and the column statistics are reduced
// per-thread -> per-CTA (shared memory) -> global (double atomics).  All loads/stores are 128-bit.
#include <cooperative_groups.h>

#include "kernels.cuh"

namespace gps {

namespace {

struct RowGeom {
  dim3 block, grid;
  size_t smem;
};

static int row_geom(int64_t rows, int64_t d, int nstat, RowGeom* g) {
  GPS_REQUIRE(d > 0 && d % 4 == 0 && d / 4 <= 1024, GPS_ERR_UNSUPPORTED,
              "row-wise stage needs d %% 4 == 0 and d <= 4096 (got %lld)", (long long)d);
  int C4 = (int)(d / 4);
  // Kernels that end with column statistics add 2*NS*d doubles per CTA onto the same d addresses, and
  // same-address L2 atomics serialise (~50 ns each: 300 CTAs cost ~17 us for a 4.4 MB reduce whose loads
  // need ~3 us).  So: few, fat CTAs (up to 1024 threads) when there are statistics, many small ones otherwise.
  int RY = C4 >= 256 ? 1 : 256 / C4;
  int64_t cap = kNumSMs * 8;
  if (nstat > 0) {
    RY = C4 >= 1024 ? 1 : 1024 / C4;
    if (RY > 16) RY = 16;
    const int smem_cap = (int)(48 * 1024 / ((size_t)nstat * C4 * sizeof(float4)));   // static 48 KB limit
    if (RY > smem_cap) RY = smem_cap < 1 ? 1 : smem_cap;
    cap = kNumSMs / 2;
  }
  int64_t blocks = ceil_div(rows > 0 ? rows : 1, (int64_t)RY * 4);
  if (blocks > cap) blocks = cap;
  g->block = dim3(C4, RY, 1);
  g->grid = dim3((unsigned)blocks, 1, 1);
  g->smem = RY > 1 ? (size_t)nstat * RY * C4 * sizeof(float4) : 0;
  return GPS_OK;
}

// body of one row-wise stage run by blocks [0, vgrid) (virtual block index vb: two stages can share one launch)
template <class Op>
__device__ __forceinline__ void rowwise_body(Op& op, int64_t rows, int vb, int vgrid, float4* sm) {
  const int c4 = threadIdx.x, ry = threadIdx.y, RY = blockDim.y, C4 = blockDim.x;
  constexpr int NS = Op::NS;
  float4 acc[NS > 0 ? NS : 1];
#pragma unroll
  for (int s = 0; s < (NS > 0 ? NS : 1); ++s) acc[s] = f4zero();
  op.prepare(c4);
#pragma unroll 4
  for (int64_t r = (int64_t)vb * RY + ry; r < rows; r += (int64_t)vgrid * RY) op.row(r, c4, acc);
  if (NS > 0) {
    if (RY > 1) {
#pragma unroll
      for (int s = 0; s < NS; ++s) sm[(s * RY + ry) * C4 + c4] = acc[s];
      __syncthreads();
      if (ry == 0) {
#pragma unroll
        for (int s = 0; s < NS; ++s)
          for (int y = 1; y < RY; ++y) acc[s] = f4add(acc[s], sm[(s * RY + y) * C4 + c4]);
      }
    }
    if (ry == 0) {
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        double* p = op.stat_ptr(s);
        if (p) {
          atomic_add_f64(p + c4 * 4 + 0, (double)acc[s].x);
          atomic_add_f64(p + c4 * 4 + 1, (double)acc[s].y);
          atomic_add_f64(p + c4 * 4 + 2, (double)acc[s].z);
          atomic_add_f64(p + c4 * 4 + 3, (double)acc[s].w);
        }
      }
    }
  }
  op.finish(c4, ry);
}

template <class Op>
__global__ void __launch_bounds__(1024) k_rowwise(Op op, int64_t rows) {
  extern __shared__ float4 sm[];
  rowwise_body(op, rows, (int)blockIdx.x, (int)gridDim.x, sm);
}

// two independent row-wise stages in one launch: blocks [0, ga) run `a`, the rest run `b` (same block shape)
template <class OpA, class OpB>
__global__ void __launch_bounds__(1024) k_rowwise2(OpA a, int64_t rowsA, int ga, OpB b, int64_t rowsB) {
  extern __shared__ float4 sm[];
  if ((int)blockIdx.x < ga) {
    a.vb = (int)blockIdx.x;
    rowwise_body(a, rowsA, (int)blockIdx.x, ga, sm);
  } else {
    b.vb = (int)blockIdx.x - ga;
    rowwise_body(b, rowsB, (int)blockIdx.x - ga, (int)gridDim.x - ga, sm);
  }
}

__device__ __forceinline__ float4 act4(int act, float4 v) {
  if (act < 0) return v;
  return make_float4(act_fwd_rt(act, v.x), act_fwd_rt(act, v.y), act_fwd_rt(act, v.z), act_fwd_rt(act, v.w));
}
__device__ __forceinline__ float4 dact4(int act, float4 v) {
  return make_float4(act_bwd_rt(act, v.x), act_bwd_rt(act, v.y), act_bwd_rt(act, v.z), act_bwd_rt(act, v.w));
}

// ---------------------------------------------------------------- forward: R + drop(act(BN(z)))
template <bool STATS>
struct OpBnActRes {
  static constexpr int NS = STATS ? 2 : 0;
  const float* z; int64_t ldz;
  const float* R; float* out; int64_t d;
  BnView bn; int act; DropCfg drop; double* stats; Planes outp;
  BnRegs reg;
  int vb = -1;   // virtual block index when two stages share a launch (k_rowwise2)
  __device__ void prepare(int c4) {
    reg.load(bn, c4, vb);
    if (drop.p > 0.f && drop.offset_dev) drop.offset += *drop.offset_dev;
  }
  __device__ void row(int64_t r, int c4, float4* acc) {
    float4 v = act4(act, reg.apply(ld4(z + r * ldz + c4 * 4)));
    if (drop.p > 0.f)
      v = f4mul(v, dropout_scale4(drop.p, drop.seed, drop.offset, drop.site, (uint64_t)r * (d >> 2) + c4));
    if (R) v = f4add(v, ld4(R + r * d + c4 * 4));
    st4(out + r * d + c4 * 4, v);
    if (outp.hi) planes_store4(outp, r, c4 * 4, v);
    if (STATS) {
      acc[0] = f4add(acc[0], v);
      acc[1] = f4fma(v, v, acc[1]);
    }
  }
  __device__ double* stat_ptr(int s) { return stats ? stats + (int64_t)s * d : nullptr; }
  __device__ void finish(int, int) {}
};

// ---------------------------------------------------------------- forward: BN(a) [+ BN(b)]
struct OpCombine {
  static constexpr int NS = 0;
  const float* a; const float* b; float* out; int64_t d;
  BnView bna, bnb; Planes outp;
  BnRegs ra, rb;
  __device__ void prepare(int c4) {
    ra.load(bna, c4);
    if (b) rb.load(bnb, c4);
  }
  __device__ void row(int64_t r, int c4, float4*) {
    float4 v = ra.apply(ld4(a + r * d + c4 * 4));
    if (b) v = f4add(v, rb.apply(ld4(b + r * d + c4 * 4)));
    st4(out + r * d + c4 * 4, v);
    if (outp.hi) planes_store4(outp, r, c4 * 4, v);
  }
  __device__ double* stat_ptr(int) { return nullptr; }
  __device__ void finish(int, int) {}
};

// ---------------------------------------------------------------- backward of BatchNorm (+act, +dropout)
__device__ __forceinline__ float4 bn_bwd_gprime(const float* g, int64_t ldg, int64_t r, int c4, float4 zh,
                                                const BnRegs& reg, int act, const DropCfg& drop, int64_t d) {
  float4 gp = ld4(g + r * ldg + c4 * 4);
  if (drop.p > 0.f)
    gp = f4mul(gp, dropout_scale4(drop.p, drop.seed, drop.offset, drop.site, (uint64_t)r * (d >> 2) + c4));
  if (act >= 0) gp = f4mul(gp, dact4(act, f4fma(zh, reg.gamma, reg.beta)));
  return gp;
}

struct OpBnBwdReduce {
  static constexpr int NS = 2;
  const float* g; int64_t ldg; const float* z; int64_t ldz; int64_t d;
  BnView bn; int act; DropCfg drop; double* sums;
  BnRegs reg;
  __device__ void prepare(int c4) {
    reg.load(bn, c4);
    if (drop.p > 0.f && drop.offset_dev) drop.offset += *drop.offset_dev;
  }
  __device__ void row(int64_t r, int c4, float4* acc) {
    float4 zh = reg.zhat(ld4(z + r * ldz + c4 * 4));
    float4 gp = bn_bwd_gprime(g, ldg, r, c4, zh, reg, act, drop, d);
    acc[0] = f4add(acc[0], gp);
    acc[1] = f4fma(gp, zh, acc[1]);
  }
  __device__ double* stat_ptr(int s) { return sums + (int64_t)s * d; }
  __device__ void finish(int, int) {}
};

struct OpBnBwdApply {
  static constexpr int NS = 0;
  const float* g; int64_t ldg; const float* z; int64_t ldz; int64_t d;
  BnView bn; int act; DropCfg drop; const double* sums; float inv_n;
  float* out; int64_t ldo; float* grad_gamma; float* grad_beta; int accumulate; Planes outp;
  BnRegs reg;
  float4 m1, m2, gs;  // S1/n, S2/n, gamma*invstd
  float4 s1raw, s2raw;
  __device__ void prepare(int c4) {
    reg.load(bn, c4);
    if (drop.p > 0.f && drop.offset_dev) drop.offset += *drop.offset_dev;
    const double* a = sums + c4 * 4;
    const double* b = sums + d + c4 * 4;
    s1raw = make_float4((float)a[0], (float)a[1], (float)a[2], (float)a[3]);
    s2raw = make_float4((float)b[0], (float)b[1], (float)b[2], (float)b[3]);
    m1 = f4scale(s1raw, inv_n);
    m2 = f4scale(s2raw, inv_n);
    if (bn.mode == 2) m1 = m2 = f4zero();   // eval mode: the statistics are constants, dz = g' * gamma * invstd
    gs = f4mul(reg.gamma, reg.invstd);
  }
  __device__ void row(int64_t r, int c4, float4*) {
    float4 zh = reg.zhat(ld4(z + r * ldz + c4 * 4));
    float4 gp = bn_bwd_gprime(g, ldg, r, c4, zh, reg, act, drop, d);
    float4 v = make_float4(gs.x * (gp.x - m1.x - zh.x * m2.x), gs.y * (gp.y - m1.y - zh.y * m2.y),
                           gs.z * (gp.z - m1.z - zh.z * m2.z), gs.w * (gp.w - m1.w - zh.w * m2.w));
    st4(out + r * ldo + c4 * 4, v);
    if (outp.hi) planes_store4(outp, r, c4 * 4, v);
  }
  __device__ double* stat_ptr(int) { return nullptr; }
  __device__ void finish(int c4, int ry) {
    if (blockIdx.x == 0 && ry == 0) {
      if (grad_gamma) st4(grad_gamma + c4 * 4, accumulate ? f4add(ld4(grad_gamma + c4 * 4), s2raw) : s2raw);
      if (grad_beta) st4(grad_beta + c4 * 4, accumulate ? f4add(ld4(grad_beta + c4 * 4), s1raw) : s1raw);
    }
  }
};

struct OpAdd3 {
  static constexpr int NS = 0;
  const float* a; int64_t lda; const float* b; int64_t ldb; const float* c; int64_t ldc;
  float* out; int64_t ldo;
  __device__ void prepare(int) {}
  __device__ void row(int64_t r, int c4, float4*) {
    float4 v = ld4(a + r * lda + c4 * 4);
    if (b) v = f4add(v, ld4(b + r * ldb + c4 * 4));
    if (c) v = f4add(v, ld4(c + r * ldc + c4 * 4));
    st4(out + r * ldo + c4 * 4, v);
  }
  __device__ double* stat_ptr(int) { return nullptr; }
  __device__ void finish(int, int) {}
};

// out[c] += sum_r a[r, c]: thread -> CTA (shared memory over threadIdx.y) -> the kColsumCtas CTAs of one cluster
// (grid y), in rank order through distributed shared memory -> one float add per column, so the sum is the same in every
// run.  grid x walks column chunks of blockDim.x float4 columns.
constexpr int kColsumCtas = 8;
__global__ void __launch_bounds__(1024) k_colsum(const float* __restrict__ a, int64_t lda, int64_t rows, int C4,
                                                 float* __restrict__ out) {
  extern __shared__ float4 sm[];
  const int ry = threadIdx.y, RY = blockDim.y, CB = blockDim.x;
  const int c4 = blockIdx.x * CB + threadIdx.x;
  const bool col_ok = c4 < C4;
  float4 acc = f4zero();
  if (col_ok)
    for (int64_t r = (int64_t)blockIdx.y * RY + ry; r < rows; r += (int64_t)gridDim.y * RY)
      acc = f4add(acc, ld4(a + r * lda + c4 * 4));
  if (RY > 1) {
    sm[ry * CB + threadIdx.x] = acc;
    __syncthreads();
    if (ry == 0)
      for (int y = 1; y < RY; ++y) acc = f4add(acc, sm[y * CB + threadIdx.x]);
  }
  if (ry == 0) sm[threadIdx.x] = acc;   // row-0 slots: read above only by the thread that now overwrites them
  cooperative_groups::cluster_group cluster = cooperative_groups::this_cluster();
  cluster.sync();
  if (blockIdx.y == 0 && ry == 0 && col_ok) {
    float4 tot = f4zero();
    for (int k = 0; k < (int)gridDim.y; ++k) tot = f4add(tot, cluster.map_shared_rank(sm, k)[threadIdx.x]);
    atomicAdd(out + c4 * 4 + 0, tot.x);   // the only adder of this element
    atomicAdd(out + c4 * 4 + 1, tot.y);
    atomicAdd(out + c4 * 4 + 2, tot.z);
    atomicAdd(out + c4 * 4 + 3, tot.w);
  }
  cluster.sync();   // no CTA leaves while rank 0 still reads its shared memory
}

template <class Op>
static int launch_rowwise(Op op, int64_t rows, int64_t d, cudaStream_t stream) {
  if (rows == 0) return GPS_OK;
  RowGeom g;
  GPS_TRY(row_geom(rows, d, Op::NS, &g));
  k_rowwise<Op><<<g.grid, g.block, g.smem, stream>>>(op, rows);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

}  // namespace

int bn_act_residual(const float* z, int64_t ldz, const float* R, float* out, int64_t rows, int64_t d, BnView bn,
                    int act, DropCfg drop, double* stats, cudaStream_t stream, Planes outp) {
  if (stats) {
    OpBnActRes<true> op{z, ldz, R, out, d, bn, act, drop, stats, outp};
    return launch_rowwise(op, rows, d, stream);
  }
  OpBnActRes<false> op{z, ldz, R, out, d, bn, act, drop, nullptr, outp};
  return launch_rowwise(op, rows, d, stream);
}

// both GatedGCN outputs in one launch: x_loc = x + drop(act(BN_x(x~))) with column sums, e_out = e + drop(act(BN_e(e^)))
int bn_act_residual2(const float* zx, const float* Rx, float* outx, int64_t N, BnView bnx, DropCfg dropx, double* statsx,
                     const float* ze, const float* Re, float* oute, int64_t E, BnView bne, DropCfg drope, Planes outep,
                     int64_t d, int act, cudaStream_t stream) {
  if (N == 0 || E == 0 || !statsx) {   // degenerate sizes / eval mode: two plain launches
    GPS_TRY(bn_act_residual(zx, d, Rx, outx, N, d, bnx, act, dropx, statsx, stream));
    return bn_act_residual(ze, d, Re, oute, E, d, bne, act, drope, nullptr, stream, outep);
  }
  RowGeom g;
  GPS_TRY(row_geom(N, d, 2, &g));                    // the statistics stage fixes the (fat) block shape
  const int RY = (int)g.block.y;
  int64_t gb = ceil_div(E, (int64_t)RY * 4);
  if (gb > kNumSMs * 2) gb = kNumSMs * 2;
  OpBnActRes<true> opx{zx, d, Rx, outx, d, bnx, act, dropx, statsx, Planes()};
  OpBnActRes<false> ope{ze, d, Re, oute, d, bne, act, drope, nullptr, outep};
  k_rowwise2<<<dim3((unsigned)(g.grid.x + gb)), g.block, g.smem, stream>>>(opx, N, (int)g.grid.x, ope, E);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int bn_combine(const float* a, BnView bna, const float* b, BnView bnb, float* out, int64_t rows, int64_t d,
               cudaStream_t stream, Planes outp) {
  OpCombine op{a, b, out, d, bna, bnb, outp};
  return launch_rowwise(op, rows, d, stream);
}

int bn_bwd_reduce(const float* g, int64_t ldg, const float* z, int64_t ldz, int64_t rows, int64_t d, BnView bn,
                  int act, DropCfg drop, double* sums, cudaStream_t stream) {
  OpBnBwdReduce op{g, ldg, z, ldz, d, bn, act, drop, sums};
  return launch_rowwise(op, rows, d, stream);
}

int bn_bwd_apply(const float* g, int64_t ldg, const float* z, int64_t ldz, int64_t rows, int64_t d, BnView bn,
                 int act, DropCfg drop, const double* sums, float* out, int64_t ldo, float* grad_gamma,
                 float* grad_beta, cudaStream_t stream, bool accumulate, Planes outp) {
  OpBnBwdApply op{g, ldg, z, ldz, d, bn, act, drop, sums, 1.f / (float)(rows > 0 ? rows : 1),
                  out, ldo, grad_gamma, grad_beta, accumulate ? 1 : 0, outp};
  if (rows == 0) {
    // no rows: gradients of gamma/beta are zero
    if (grad_gamma && !accumulate) GPS_CUDA(cudaMemsetAsync(grad_gamma, 0, d * sizeof(float), stream));
    if (grad_beta && !accumulate) GPS_CUDA(cudaMemsetAsync(grad_beta, 0, d * sizeof(float), stream));
    return GPS_OK;
  }
  return launch_rowwise(op, rows, d, stream);
}

int add3(const float* a, int64_t lda, const float* b, int64_t ldb, const float* c, int64_t ldc, float* out,
         int64_t ldo, int64_t rows, int64_t d, cudaStream_t stream) {
  OpAdd3 op{a, lda, b, ldb, c, ldc, out, ldo};
  return launch_rowwise(op, rows, d, stream);
}

int colsum(const float* a, int64_t lda, int64_t rows, int64_t d, float* out, cudaStream_t stream) {
  if (rows == 0) return GPS_OK;
  GPS_REQUIRE(d > 0 && d % 4 == 0, GPS_ERR_UNSUPPORTED, "colsum needs d %% 4 == 0 (got %lld)", (long long)d);
  const int C4 = (int)(d / 4);
  const int CB = C4 < 128 ? C4 : 128;                // float4 columns per CTA
  const int RY = 1024 / CB < 16 ? 1024 / CB : 16;    // row lanes per CTA
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)ceil_div(C4, CB), kColsumCtas);   // one cluster per column chunk
  cfg.blockDim = dim3(CB, RY);
  cfg.dynamicSmemBytes = (size_t)RY * CB * sizeof(float4);
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1;
  attr[0].val.clusterDim.y = kColsumCtas;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  GPS_CUDA(cudaLaunchKernelEx(&cfg, k_colsum, a, lda, rows, C4, out));
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int copy2d(const float* src, int64_t lds, float* dst, int64_t ldd, int64_t rows, int64_t d, cudaStream_t stream) {
  if (rows == 0) return GPS_OK;
  GPS_CUDA(cudaMemcpy2DAsync(dst, ldd * sizeof(float), src, lds * sizeof(float), d * sizeof(float), rows,
                             cudaMemcpyDeviceToDevice, stream));
  return GPS_OK;
}

}  // namespace gps
