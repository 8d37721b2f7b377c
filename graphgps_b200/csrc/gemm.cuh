// gemm.cuh — parameter block shared by the dense-product kernels (gemm_simt.cu, gemm_tc.cu).
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace gps {

// C[m,n] (+)= epilogue( sum_k Aop[m,k] * Bop[k,n] )
//   ta == 0: Aop[m,k] = A[m*lda + k]      ta == 1: Aop[m,k] = A[k*lda + m]
//   tb == 0: Bop[k,n] = B[n*ldb + k]      tb == 1: Bop[k,n] = B[k*ldb + n]
// Epilogue order: +bias[n] -> (store pre-activation) -> act -> *act'(mask_src) -> dropout ->
//                 +R1 +R2 -> store -> column statistics (sum, sum of squares, double atomics).
// With splitk > 1 the partial products are atomically added into a pre-zeroed C and only the
// plain product is supported.  (With splitk <= 1 the TMA kernel may still split K when its launch policy finds that
// faster: a cluster whose ranks sum their partial tiles in rank order and then run the whole epilogue on their own
// rows, so C is written, not added to.)
struct GemmParams {
  int M = 0, N = 0, K = 0;
  const float* A = nullptr; int lda = 0; int ta = 0;
  const float* B = nullptr; int ldb = 0; int tb = 0;
  float* C = nullptr; int ldc = 0;
  const float* bias = nullptr;
  float* C_pre = nullptr; int ldpre = 0;   // optional copy of the pre-activation value
  int act = -1;                            // -1 none, GPS_ACT_*
  const float* mask_src = nullptr; int ldmask = 0; int mask_act = -1;  // multiply by act'(mask_src)
  int mask_is_post = 0;                    // relu only: mask_src holds the post-activation value
  float p_drop = 0.f; uint64_t seed = 0, offset = 0; int site = 0;    // dropout on the result
  const unsigned long long* offset_dev = nullptr;                     // optional device-resident addend to offset
  float p_drop2 = 0.f; int site2 = 0;      // optional inner dropout applied before the one above (Performer: attn_dropout
                                           // on to_out(O) inside SelfAttention, then GPSLayer.dropout_attn)
  const float* R1 = nullptr; int ldr1 = 0;
  const float* R2 = nullptr; int ldr2 = 0;
  double* stats = nullptr;                 // [2][N] column sum / sum of squares of the stored C
  int splitk = 1;
  float* colsum_a = nullptr;               // ta==1 only: += sum_k Aop[m,k]  (bias gradient), [M]
  int precision = GPS_PREC_FP32;
  // bf16 hi/lo planes of the operands as stored (A: [M,K] or, ta == 1, [K,M]; B: [N,K] or, tb == 1, [K,N]): when both
  // are given the TMA-fed kernel (gemm_tma.cu) runs and A/B (fp32) are not read.  Cp: optional plane copy of the
  // result for the next GEMM; C may then be null (planes-only output).
  Planes Ap, Bp, Cp;
  // Cp column remap for the attention operands: output column c lands at (c / cp_hd) * cp_hd_pad + c % cp_hd and the
  // cp_hd_pad - cp_hd pad columns of every head are written as zeros (per-head layout padded to a multiple of 16)
  int cp_hd = 0, cp_hd_pad = 0;
};

struct ToPlanesItem { const float* src; int64_t ld; int rows; int cols; Planes dst; };
// fp32 [rows, cols] (pitch ld) -> bf16 hi/lo planes, up to 16 matrices per launch
int to_planes(const ToPlanesItem* items, int n, cudaStream_t stream);
// TMA-fed wgmma product on plane operands; GPS_ERR_UNSUPPORTED when the planes are missing / misaligned
int gemm_tma(const GemmParams& p, cudaStream_t stream);
// rank-3 tensor map {cols, rows, planes} over a plane pair with a {64, box_rows, 1} SWIZZLE_128B box (cached)
int make_tensor_map(const __nv_bfloat16* hi, const __nv_bfloat16* lo, int planes, int64_t rows, int64_t cols, int64_t ld,
                    int box_rows, CUtensorMap* out);
void gemm_tma_set_force_bn(int bn);
void gemm_tma_set_force_splits(int s);   // K-splits of every launch that runs the epilogue (0 = the launch policy)
void gemm_tma_set_trace(unsigned long long* buf);   // bring-up: per-CTA phase timestamps (tools/gemm_trace.py)

// exact fp32 CUDA-core product (validation path and shapes the tensor-core kernel does not take)
int gemm_simt(const GemmParams& p, cudaStream_t stream);
// register-staged wgmma tensor-core product; returns GPS_ERR_UNSUPPORTED for shapes it does not take
int gemm_tc(const GemmParams& p, cudaStream_t stream);
void gemm_tc_set_debug(int v);   // bits 8.. : forced tile width (0 = heuristic)
// dispatcher used by the layer
int gemm(const GemmParams& p, cudaStream_t stream);

}  // namespace gps
