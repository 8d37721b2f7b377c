// eslap.cu — the EquivStableLapPE edge gate of GatedGCN (graphgps/layer/gatedgcn_layer.py:29-35, 65-70, 90-126).
//
// For edge e = j -> i with positional encoding PE [N, k]:
//   r_e = sum_c (PE_i[c] - PE_j[c])^2 ;  rho_e = sigmoid(w2 . act(w1 r_e + b1) + b2)     (mlp_r_ij, 1 -> d -> 1)
// and the GatedGCN gate becomes sigma_ij = sigmoid(e_ij) * rho_e (scatter.cu, PE instantiations).
// Backward (per edge, g_sigma = g_num_i * Bx_j + g_den_i formed from what k_gatedgcn_bwd_dst stores):
//   g_rho = sum_c g_sigma[c] sigmoid(e_ij)[c] ;  g_z = g_rho rho (1 - rho) ;  g_r = g_z sum_m w2[m] act'(w1[m] r + b1[m]) w1[m]
//   g_PE_n = sum_{e: dst=n} 2 g_r (PE_n - PE_src) + sum_{e: src=n} 2 g_r (PE_n - PE_dst)
//   mlp_r_ij gradients: column sums over the edges of g_z h_e, g_z, g_pre r_e, g_pre (g_pre = g_z w2 act'(pre)).
// Nothing of size [E, d] is stored: h_e and g_pre are recomputed from the two scalars (r_e, g_z_e).  Every reduction
// runs in a fixed order (warp butterflies, edge-id-ordered segments, fixed edge chunks summed in chunk order), so two
// runs give the same bits, and there are no atomics.
#include "kernels.cuh"

namespace gps {

namespace {

constexpr int kWarpsPerBlock = 8;

__device__ __forceinline__ float pe_dist2(const float* __restrict__ pe, int64_t k, int64_t a, int64_t b, int lane) {
  float acc = 0.f;
  for (int64_t c = lane; c < k; c += 32) {
    const float t = pe[a * k + c] - pe[b * k + c];
    acc = fmaf(t, t, acc);
  }
  return warp_sum(acc);
}

// r_e, rho_e: one warp per destination node, its in-edges in CSR (edge-id) order
template <int ACT>
__global__ void k_eslap_fwd(GpsGraph g, const float* __restrict__ pe, int64_t k, int d, const float* __restrict__ w1,
                            const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
                            float* __restrict__ r_out, float* __restrict__ rho_out) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (i >= g.N) return;
  const float bias2 = b2[0];
  for (int q = g.dst_ptr[i]; q < g.dst_ptr[i + 1]; ++q) {
    const int j = g.dst_src[q];
    const int64_t e = g.dst_eid[q];
    const float r = pe_dist2(pe, k, i, j, lane);
    float z = 0.f;
    for (int m = lane; m < d; m += 32) z = fmaf(w2[m], act_fwd<ACT>(fmaf(w1[m], r, b1[m])), z);
    z = warp_sum(z) + bias2;
    if (lane == 0) {
      r_out[e] = r;
      rho_out[e] = sigmoidf_(z);
    }
  }
}

// g_z_e and g_r_e: one warp per destination node (g_num_i / g_den_i rows reused across its in-edges)
template <int ACT>
__global__ void k_eslap_bwd_edge(GpsGraph g, int d, const float* __restrict__ g_num, const float* __restrict__ g_den,
                                 const float* __restrict__ Bx, int64_t ldy, const float* __restrict__ ehat,
                                 const float* __restrict__ r_in, const float* __restrict__ rho_in,
                                 const float* __restrict__ w1, const float* __restrict__ b1,
                                 const float* __restrict__ w2, float* __restrict__ gz_out, float* __restrict__ gr_out) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (i >= g.N) return;
  for (int q = g.dst_ptr[i]; q < g.dst_ptr[i + 1]; ++q) {
    const int64_t j = g.dst_src[q];
    const int64_t e = g.dst_eid[q];
    float acc = 0.f;
    for (int c = lane * 4; c < d; c += 128) {
      const float4 gn = ld4(g_num + i * d + c), gd = ld4(g_den + i * d + c), bx = ld4(Bx + j * ldy + c);
      const float4 eh = ld4(ehat + e * d + c);
      acc = fmaf(fmaf(gn.x, bx.x, gd.x), sigmoidf_(eh.x), acc);
      acc = fmaf(fmaf(gn.y, bx.y, gd.y), sigmoidf_(eh.y), acc);
      acc = fmaf(fmaf(gn.z, bx.z, gd.z), sigmoidf_(eh.z), acc);
      acc = fmaf(fmaf(gn.w, bx.w, gd.w), sigmoidf_(eh.w), acc);
    }
    const float g_rho = warp_sum(acc);
    const float rho = rho_in[e], r = r_in[e];
    const float gz = g_rho * rho * (1.f - rho);
    float s = 0.f;
    for (int m = lane; m < d; m += 32) s = fmaf(w2[m] * act_bwd<ACT>(fmaf(w1[m], r, b1[m])), w1[m], s);
    s = warp_sum(s);
    if (lane == 0) {
      gz_out[e] = gz;
      gr_out[e] = gz * s;
    }
  }
}

// grad_pe: one warp per node, lanes over the k channels; in-edges (CSR) then out-edges (CSC), each in edge-id order
__global__ void k_eslap_bwd_pe(GpsGraph g, const float* __restrict__ pe, int64_t k, const float* __restrict__ gr,
                               float* __restrict__ grad_pe) {
  const int lane = threadIdx.x & 31;
  const int64_t n = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (n >= g.N) return;
  const int db = g.dst_ptr[n], de = g.dst_ptr[n + 1], sb = g.src_ptr[n], se = g.src_ptr[n + 1];
  for (int64_t c = lane; c < k; c += 32) {
    const float p = pe[n * k + c];
    float acc = 0.f;
    for (int q = db; q < de; ++q) acc = fmaf(2.f * gr[g.dst_eid[q]], p - pe[(int64_t)g.dst_src[q] * k + c], acc);
    for (int q = sb; q < se; ++q) acc = fmaf(2.f * gr[g.src_eid[q]], p - pe[(int64_t)g.src_dst[q] * k + c], acc);
    grad_pe[n * k + c] = acc;
  }
}

// mlp_r_ij gradients, stage 1: block b sums its chunk of edges [b*chunk, (b+1)*chunk) in edge-id order.
// part[b] = [g_w2 (d) | g_w1 (d) | g_b1 (d) | g_b2 (1)]
template <int ACT>
__global__ void k_eslap_wgrad_part(int64_t E, int64_t chunk, int d, const float* __restrict__ r_in,
                                   const float* __restrict__ gz_in, const float* __restrict__ w1,
                                   const float* __restrict__ b1, const float* __restrict__ w2, float* __restrict__ part) {
  const int64_t e0 = (int64_t)blockIdx.x * chunk;
  const int64_t e1 = e0 + chunk < E ? e0 + chunk : E;
  float* out = part + (int64_t)blockIdx.x * (3 * d + 1);
  for (int m = threadIdx.x; m < d; m += blockDim.x) {
    const float a = w1[m], b = b1[m], w = w2[m];
    float gw2 = 0.f, gw1 = 0.f, gb1 = 0.f;
    for (int64_t e = e0; e < e1; ++e) {
      const float r = r_in[e], gz = gz_in[e];
      const float pre = fmaf(a, r, b);
      gw2 = fmaf(gz, act_fwd<ACT>(pre), gw2);
      const float gpre = gz * w * act_bwd<ACT>(pre);
      gw1 = fmaf(gpre, r, gw1);
      gb1 += gpre;
    }
    out[m] = gw2;
    out[d + m] = gw1;
    out[2 * d + m] = gb1;
  }
  if (threadIdx.x == 0) {
    float gb2 = 0.f;
    for (int64_t e = e0; e < e1; ++e) gb2 += gz_in[e];
    out[3 * d] = gb2;
  }
}

// stage 2: column sums of the parts in chunk order, written (or added) into the caller's gradient buffers
__global__ void k_eslap_wgrad_sum(int64_t nparts, int d, const float* __restrict__ part, float* gw2, float* gw1,
                                  float* gb1, float* gb2, int accumulate) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col > 3 * d) return;
  float s = 0.f;
#pragma unroll 8
  for (int64_t b = 0; b < nparts; ++b) s += part[b * (3 * d + 1) + col];
  float* base = col < d ? gw2 : (col < 2 * d ? gw1 : (col < 3 * d ? gb1 : gb2));
  if (!base) return;
  float* dst = base + (col < 3 * d ? col % d : 0);
  *dst = accumulate ? *dst + s : s;
}

}  // namespace

// edges per stage-1 block: about one block per SM (at least 32 edges each), a function of E alone
int64_t eslap_wgrad_chunk(int64_t E) {
  const int64_t c = ceil_div(E, (int64_t)kNumSMs);
  return c > 32 ? c : 32;
}

int eslap_fwd(const GpsGraph& g, const float* pe, int64_t k, int64_t d, int act, const float* w1, const float* b1,
              const float* w2, const float* b2, float* r, float* rho, cudaStream_t stream) {
  if (g.N == 0 || g.E == 0) return GPS_OK;
  const unsigned blocks = (unsigned)ceil_div(g.N, (int64_t)kWarpsPerBlock);
  if (act == GPS_ACT_RELU)
    k_eslap_fwd<GPS_ACT_RELU><<<blocks, 32 * kWarpsPerBlock, 0, stream>>>(g, pe, k, (int)d, w1, b1, w2, b2, r, rho);
  else
    k_eslap_fwd<GPS_ACT_GELU><<<blocks, 32 * kWarpsPerBlock, 0, stream>>>(g, pe, k, (int)d, w1, b1, w2, b2, r, rho);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int eslap_bwd(const GpsGraph& g, const float* pe, int64_t k, int64_t d, int act, const float* g_num, const float* g_den,
              const float* Bx, int64_t ldy, const float* ehat, const float* r, const float* rho, const float* w1,
              const float* b1, const float* w2, float* gz, float* gr, float* part, float* grad_pe, float* gw1,
              float* gb1, float* gw2, float* gb2, bool accumulate, cudaStream_t stream) {
  const unsigned node_blocks = (unsigned)ceil_div(g.N, (int64_t)kWarpsPerBlock);
  const int64_t chunk = eslap_wgrad_chunk(g.E), nparts = ceil_div(g.E, chunk);
  if (g.E > 0) {
    if (act == GPS_ACT_RELU)
      k_eslap_bwd_edge<GPS_ACT_RELU><<<node_blocks, 32 * kWarpsPerBlock, 0, stream>>>(
          g, (int)d, g_num, g_den, Bx, ldy, ehat, r, rho, w1, b1, w2, gz, gr);
    else
      k_eslap_bwd_edge<GPS_ACT_GELU><<<node_blocks, 32 * kWarpsPerBlock, 0, stream>>>(
          g, (int)d, g_num, g_den, Bx, ldy, ehat, r, rho, w1, b1, w2, gz, gr);
    GPS_LAUNCH_CHECK();
    if (act == GPS_ACT_RELU)
      k_eslap_wgrad_part<GPS_ACT_RELU><<<(unsigned)nparts, 256, 0, stream>>>(g.E, chunk, (int)d, r, gz, w1, b1, w2, part);
    else
      k_eslap_wgrad_part<GPS_ACT_GELU><<<(unsigned)nparts, 256, 0, stream>>>(g.E, chunk, (int)d, r, gz, w1, b1, w2, part);
    GPS_LAUNCH_CHECK();
  }
  if (gw1 || gb1 || gw2 || gb2) {   // E = 0: writes zeros (or adds nothing)
    k_eslap_wgrad_sum<<<(unsigned)ceil_div(3 * d + 1, (int64_t)128), 128, 0, stream>>>(g.E > 0 ? nparts : 0, (int)d, part,
                                                                                     gw2, gw1, gb1, gb2, accumulate ? 1 : 0);
    GPS_LAUNCH_CHECK();
  }
  if (grad_pe && g.N > 0) {
    k_eslap_bwd_pe<<<node_blocks, 32 * kWarpsPerBlock, 0, stream>>>(g, pe, k, gr, grad_pe);
    GPS_LAUNCH_CHECK();
  }
  return GPS_OK;
}

}  // namespace gps
