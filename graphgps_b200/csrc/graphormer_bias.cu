// graphormer_bias.cu — Graphormer's attention-bias encoder (graphgps/encoder/graphormer_encoder.py:103-183) and its
// C ABI.  The reference embeds every path position ([P, S, H]), scatters it into a dense [B, N, N, S, H] tensor and
// contracts it with edge_dis_encoder by bmm.  Here the contraction is folded into a table first:
//   Tab[k, t, h] = sum_h' edge_weight[t, h'] W[k, h', h]                (S*T*H floats, in shared memory)
// so a pair is S table lookups and one plain store per head, and nothing of size P*S*H exists.
//   forward:  the output's padding and graph-token rows (one memset or one fill launch), then one pass over the pairs
//   backward: one pass over the pairs into per-thread shared-memory slots keyed by (k, t) and by spatial type, summed
//             over the CTA's lanes in order into per-CTA partials (with the token's row-0 / column-0 partials), then
//             one CTA sums the partials in CTA order and runs the two small contractions
//               dW[k, h', h] = sum_t E[t, h'] Sig[k, t, h],   dE[t, h'] = sum_k sum_h W[k, h', h] Sig[k, t, h]
//             No float atomics: two runs give the same bits.
#include <string.h>

#include <algorithm>

#include "common.cuh"

namespace gps {

namespace {

constexpr int64_t kMaxHeads = 32;             // at least 4 lanes per head in a backward CTA
constexpr int64_t kMaxSpatialTable = 4096;    // (S+1)*H floats
constexpr int64_t kMaxEdgeTable = 8192;       // S*T*H floats
constexpr int64_t kMaxSlots = 384;            // S*T + S + 1 keys per backward thread
constexpr int kFwdThreads = 256;
constexpr int kBwdThreads = 128;
constexpr int kSlotPitch = kBwdThreads + 1;   // slot k of thread tid at k * kSlotPitch + tid: no bank conflicts
constexpr int kFinalThreads = 512;
constexpr int64_t kPairsPerCta = 1024;
constexpr int64_t kMaxBwdCtas = 8 * kNumSMs;

struct BiasGeom {
  int64_t P, B, nmax, H, S, T, np;   // np = N', the side of each graph's block
  int off;                           // 1 with the graph token
  bool edges;                        // shortest_path_types given
  int64_t ET, K;                     // edge keys S*T (0 without edges); keys per head K = ET + S + 1
  int64_t ctas;                      // CTAs of the backward pair pass
  int64_t part_floats;               // ctas * H * K
  int64_t bwd_bytes;
};

int make_geom(const GpsGraphormerBiasArgs* a, BiasGeom* g) {
  memset(g, 0, sizeof(*g));
  GPS_REQUIRE(a, GPS_ERR_ARG, "graphormer_bias: null args");
  GPS_REQUIRE(a->num_pairs >= 0 && a->num_graphs >= 0 && a->nmax >= 0, GPS_ERR_ARG,
              "graphormer_bias: negative sizes (pairs %lld, graphs %lld, nmax %lld)", (long long)a->num_pairs,
              (long long)a->num_graphs, (long long)a->nmax);
  GPS_REQUIRE(a->heads >= 1 && a->num_spatial_types >= 1 && a->num_edge_types >= 0, GPS_ERR_ARG,
              "graphormer_bias: need heads >= 1, num_spatial_types >= 1, num_edge_types >= 0 (got %lld, %lld, %lld)",
              (long long)a->heads, (long long)a->num_spatial_types, (long long)a->num_edge_types);
  GPS_REQUIRE(a->use_graph_token == 0 || a->use_graph_token == 1, GPS_ERR_ARG,
              "graphormer_bias: use_graph_token must be 0 or 1");
  GPS_REQUIRE(a->num_graphs == 0 || a->nmax >= 1, GPS_ERR_ARG, "graphormer_bias: nmax must be >= 1 with graphs");
  g->P = a->num_pairs; g->B = a->num_graphs; g->nmax = a->nmax;
  g->H = a->heads; g->S = a->num_spatial_types; g->T = a->num_edge_types;
  g->off = a->use_graph_token;
  g->np = a->nmax + g->off;
  g->edges = a->shortest_path_types != nullptr;
  GPS_REQUIRE(!g->edges || g->T >= 1, GPS_ERR_ARG, "graphormer_bias: shortest_path_types with num_edge_types 0");
  GPS_REQUIRE(g->H <= kMaxHeads, GPS_ERR_UNSUPPORTED, "graphormer_bias: heads %lld > %lld is not built",
              (long long)g->H, (long long)kMaxHeads);
  GPS_REQUIRE((g->S + 1) * g->H <= kMaxSpatialTable, GPS_ERR_UNSUPPORTED,
              "graphormer_bias: (num_spatial_types + 1) * heads = %lld > %lld is not built",
              (long long)((g->S + 1) * g->H), (long long)kMaxSpatialTable);
  g->ET = g->edges ? g->S * g->T : 0;
  GPS_REQUIRE(g->ET * g->H <= kMaxEdgeTable, GPS_ERR_UNSUPPORTED,
              "graphormer_bias: num_spatial_types * num_edge_types * heads = %lld > %lld is not built",
              (long long)(g->ET * g->H), (long long)kMaxEdgeTable);
  g->K = g->ET + g->S + 1;
  GPS_REQUIRE(g->K <= kMaxSlots, GPS_ERR_UNSUPPORTED,
              "graphormer_bias: num_spatial_types * (num_edge_types + 1) + 1 = %lld > %lld is not built",
              (long long)g->K, (long long)kMaxSlots);
  const int64_t work = g->P > g->B * (2 * g->np - 1) ? g->P : g->B * (2 * g->np - 1);
  g->ctas = ceil_div(work > 0 ? work : 1, kPairsPerCta);
  if (g->ctas > kMaxBwdCtas) g->ctas = kMaxBwdCtas;
  g->part_floats = g->ctas * g->H * g->K;
  Arena W(nullptr, 0);
  W.alloc<float>(g->part_floats);
  W.alloc<float>(g->ctas * g->H);
  g->bwd_bytes = W.used;
  return GPS_OK;
}

int check_tensors(const GpsGraphormerBiasArgs* a, const BiasGeom& g, bool fwd) {
  GPS_REQUIRE(g.P == 0 || (a->spatial_types && a->graph_index), GPS_ERR_ARG,
              "graphormer_bias: spatial_types and graph_index are required");
  GPS_REQUIRE(a->node_ptr, GPS_ERR_ARG, "graphormer_bias: node_ptr is required");
  GPS_REQUIRE(a->spatial_weight, GPS_ERR_ARG, "graphormer_bias: spatial_weight is required");
  GPS_REQUIRE(!g.edges || (a->edge_dis_weight && a->edge_weight), GPS_ERR_ARG,
              "graphormer_bias: edge_dis_weight and edge_weight are required with shortest_path_types");
  GPS_REQUIRE(!g.off || a->graph_token, GPS_ERR_ARG, "graphormer_bias: graph_token is required with use_graph_token");
  if (fwd) {
    GPS_REQUIRE(a->attn_bias || g.B == 0, GPS_ERR_ARG, "graphormer_bias: attn_bias is required");
  } else {
    GPS_REQUIRE(a->grad_attn_bias || g.B == 0, GPS_ERR_ARG, "graphormer_bias: grad_attn_bias is required");
    GPS_REQUIRE(a->workspace && a->workspace_bytes >= g.bwd_bytes, GPS_ERR_ARG,
                "graphormer_bias: workspace too small (%lld < %lld)", (long long)a->workspace_bytes,
                (long long)g.bwd_bytes);
  }
  return GPS_OK;
}

// The graph of pair (i, j) and the local indices, or false when either node lies outside [node_ptr[0], node_ptr[B])
// or j is not in i's graph.  Binary search with ptr[lo] <= i < ptr[hi]: empty graphs are stepped over.
__device__ __forceinline__ bool locate(const int64_t* __restrict__ ptr, int64_t B, int64_t nmax, int64_t i, int64_t j,
                                       int64_t* b, int64_t* il, int64_t* jl) {
  if (B <= 0 || i < __ldg(ptr) || i >= __ldg(ptr + B)) return false;
  int64_t lo = 0, hi = B;
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (__ldg(ptr + mid) <= i) lo = mid;
    else hi = mid;
  }
  const int64_t base = __ldg(ptr + lo), end = __ldg(ptr + lo + 1);
  if (j < base || j >= end || end - base > nmax) return false;
  *b = lo; *il = i - base; *jl = j - base;
  return true;
}

// Every entry of [B*H, np, np]: graph_token[h] in row 0 and column 0, 0 elsewhere (the pass over the pairs then
// overwrites the entries they cover).
__global__ void k_bias_fill_token(float* __restrict__ out, int64_t total, int64_t np, int64_t H,
                                  const float* __restrict__ tok) {
  const int64_t plane = np * np;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t rc = e % plane;
    out[e] = (rc < np || rc % np == 0) ? __ldg(tok + (e / plane) % H) : 0.f;
  }
}

__global__ void __launch_bounds__(kFwdThreads) k_bias_fwd(GpsGraphormerBiasArgs a, int64_t np, int off) {
  extern __shared__ float sm[];
  const int64_t P = a.num_pairs, B = a.num_graphs, H = a.heads, S = a.num_spatial_types, T = a.num_edge_types;
  const int64_t* __restrict__ spt = a.shortest_path_types;
  float* sp = sm;                     // [S+1, H]
  float* tab = sm + (S + 1) * H;      // [S, T, H]
  for (int64_t e = threadIdx.x; e < (S + 1) * H; e += blockDim.x) sp[e] = __ldg(a.spatial_weight + e);
  if (spt) {
    for (int64_t e = threadIdx.x; e < S * T * H; e += blockDim.x) {
      const int64_t k = e / (T * H), t = (e / H) % T, h = e % H;
      float acc = 0.f;
      for (int64_t hp = 0; hp < H; ++hp)
        acc = fmaf(__ldg(a.edge_weight + t * H + hp), __ldg(a.edge_dis_weight + (k * H + hp) * H + h), acc);
      tab[e] = acc;
    }
  }
  __syncthreads();
  const int64_t plane = np * np;
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < P; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t s = __ldg(a.spatial_types + p);
    int64_t b, il, jl;
    if (s < 0 || s > S || !locate(a.node_ptr, B, a.nmax, __ldg(a.graph_index + p), __ldg(a.graph_index + P + p), &b,
                                  &il, &jl))
      continue;
    float* o = a.attn_bias + b * H * plane + (il + off) * np + (jl + off);
    const float sd = (float)(s > 1 ? s : 1);
    for (int64_t h0 = 0; h0 < H; h0 += 8) {
      float acc[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) acc[u] = 0.f;
      if (spt) {
        for (int64_t k = 0; k < S; ++k) {
          const int64_t t = __ldg(spt + p * S + k);
          if (t < 0 || t >= T) continue;
          const float* r = tab + (k * T + t) * H + h0;
#pragma unroll
          for (int u = 0; u < 8; ++u)
            if (h0 + u < H) acc[u] += r[u];
        }
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int64_t h = h0 + u;
        if (h < H) o[h * plane] = spt ? sp[s * H + h] + acc[u] / sd : sp[s * H + h];
      }
    }
  }
}

// Per-CTA partials: part[(cta * H + h) * K + key] with key (k * T + t) for the edge keys and ET + s for spatial type s;
// tok_part[cta * H + h] = this CTA's share of row 0 and column 0 of grad_attn_bias.
__global__ void __launch_bounds__(kBwdThreads) k_bias_bwd_part(GpsGraphormerBiasArgs a, int64_t np, int off,
                                                                int64_t K, int64_t ET, int64_t chunk,
                                                                float* __restrict__ part,
                                                                float* __restrict__ tok_part) {
  extern __shared__ float slots[];   // [K][kSlotPitch]
  __shared__ float red[kBwdThreads / 32];
  const int64_t P = a.num_pairs, B = a.num_graphs, H = a.heads, S = a.num_spatial_types, T = a.num_edge_types;
  const int64_t* __restrict__ spt = a.shortest_path_types;
  const float* __restrict__ G = a.grad_attn_bias;
  const int tid = threadIdx.x;
  const int L = kBwdThreads / (int)H;           // lanes per head; threads tid >= H * L stay idle
  const int64_t h = tid / L, lane = tid % L;
  for (int64_t k = 0; k < K; ++k) slots[k * kSlotPitch + tid] = 0.f;
  const int64_t plane = np * np;
  if (h < H) {
    const int64_t p0 = blockIdx.x * chunk, p1 = p0 + chunk < P ? p0 + chunk : P;
    for (int64_t p = p0 + lane; p < p1; p += L) {
      const int64_t s = __ldg(a.spatial_types + p);
      int64_t b, il, jl;
      if (s < 0 || s > S || !locate(a.node_ptr, B, a.nmax, __ldg(a.graph_index + p), __ldg(a.graph_index + P + p), &b,
                                    &il, &jl))
        continue;
      const float g = __ldg(G + (b * H + h) * plane + (il + off) * np + (jl + off));
      slots[(ET + s) * kSlotPitch + tid] += g;
      if (spt) {
        const float gt = g / (float)(s > 1 ? s : 1);
        for (int64_t k = 0; k < S; ++k) {
          const int64_t t = __ldg(spt + p * S + k);
          if (t >= 0 && t < T) slots[(k * T + t) * kSlotPitch + tid] += gt;
        }
      }
    }
  }
  __syncthreads();
  for (int64_t o = tid; o < H * K; o += kBwdThreads) {
    const int64_t hh = o / K, k = o % K;
    const float* row = slots + k * kSlotPitch + hh * L;
    float acc = 0.f;
    for (int l = 0; l < L; ++l) acc += row[l];
    part[blockIdx.x * H * K + o] = acc;
  }
  if (!tok_part) return;
  const int64_t per = 2 * np - 1, n = B * per;
  for (int64_t hh = 0; hh < H; ++hh) {
    float acc = 0.f;
    for (int64_t e = blockIdx.x * (int64_t)kBwdThreads + tid; e < n; e += (int64_t)gridDim.x * kBwdThreads) {
      const int64_t b = e / per, r = e % per;
      const float* gb = G + (b * H + hh) * plane;
      acc += r < np ? __ldg(gb + r) : __ldg(gb + (r - np + 1) * np);
    }
    acc = warp_sum(acc);
    if ((tid & 31) == 0) red[tid >> 5] = acc;
    __syncthreads();
    if (tid == 0) {
      float s = 0.f;
      for (int w = 0; w < kBwdThreads / 32; ++w) s += red[w];
      tok_part[blockIdx.x * H + hh] = s;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kFinalThreads) k_bias_bwd_final(GpsGraphormerBiasArgs a, int64_t K, int64_t ET,
                                                                   int64_t ctas, const float* __restrict__ part,
                                                                   const float* __restrict__ tok_part) {
  extern __shared__ float sig[];     // [S, T, H]
  const int64_t H = a.heads, S = a.num_spatial_types, T = a.num_edge_types;
  const int tid = threadIdx.x;
  for (int64_t o = tid; o < H * K; o += kFinalThreads) {
    const int64_t hh = o / K, k = o % K;
    float acc = 0.f;
    for (int64_t c = 0; c < ctas; ++c) acc += __ldg(part + c * H * K + o);
    if (k < ET) sig[k * H + hh] = acc;
    else if (a.grad_spatial_weight) a.grad_spatial_weight[(k - ET) * H + hh] = acc;
  }
  if (tok_part && a.grad_graph_token) {
    for (int64_t hh = tid; hh < H; hh += kFinalThreads) {
      float acc = 0.f;
      for (int64_t c = 0; c < ctas; ++c) acc += __ldg(tok_part + c * H + hh);
      a.grad_graph_token[hh] = acc;
    }
  }
  if (ET == 0) return;
  __syncthreads();
  if (a.grad_edge_dis_weight) {
    for (int64_t o = tid; o < S * H * H; o += kFinalThreads) {
      const int64_t k = o / (H * H), hp = (o / H) % H, hh = o % H;
      float acc = 0.f;
      for (int64_t t = 0; t < T; ++t) acc = fmaf(__ldg(a.edge_weight + t * H + hp), sig[(k * T + t) * H + hh], acc);
      a.grad_edge_dis_weight[o] = acc;
    }
  }
  if (a.grad_edge_weight) {
    for (int64_t o = tid; o < T * H; o += kFinalThreads) {
      const int64_t t = o / H, hp = o % H;
      float acc = 0.f;
      for (int64_t k = 0; k < S; ++k)
        for (int64_t hh = 0; hh < H; ++hh)
          acc = fmaf(__ldg(a.edge_dis_weight + (k * H + hp) * H + hh), sig[(k * T + t) * H + hh], acc);
      a.grad_edge_weight[o] = acc;
    }
  }
}

int bias_forward(const GpsGraphormerBiasArgs* a, cudaStream_t st) {
  BiasGeom g;
  GPS_TRY(make_geom(a, &g));
  GPS_TRY(check_tensors(a, g, true));
  const int64_t total = g.B * g.H * g.np * g.np;
  if (total == 0) return GPS_OK;
  if (g.off) {
    const int64_t blocks = std::min<int64_t>(ceil_div(total, 256), kNumSMs * 16);
    k_bias_fill_token<<<(unsigned)blocks, 256, 0, st>>>(a->attn_bias, total, g.np, g.H, a->graph_token);
    GPS_LAUNCH_CHECK();
  } else {
    GPS_CUDA(cudaMemsetAsync(a->attn_bias, 0, (size_t)total * sizeof(float), st));
  }
  if (g.P == 0) return GPS_OK;
  const size_t smem = (size_t)((g.S + 1) * g.H + g.ET * g.H) * sizeof(float);
  if (smem > 48 * 1024)
    GPS_CUDA(cudaFuncSetAttribute(k_bias_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t blocks = std::min<int64_t>(ceil_div(g.P, kFwdThreads), kNumSMs * 8);
  k_bias_fwd<<<(unsigned)blocks, kFwdThreads, smem, st>>>(*a, g.np, g.off);
  GPS_LAUNCH_CHECK();
  return GPS_OK;
}

int bias_backward(const GpsGraphormerBiasArgs* a, cudaStream_t st) {
  BiasGeom g;
  GPS_TRY(make_geom(a, &g));
  GPS_TRY(check_tensors(a, g, false));
  float* part = reinterpret_cast<float*>(a->workspace);
  float* tok_part = part + round_up(g.part_floats, 64);
  const bool tok = g.off && a->grad_graph_token;
  const size_t slot_bytes = (size_t)(g.K * kSlotPitch) * sizeof(float);
  if (slot_bytes > 48 * 1024)
    GPS_CUDA(cudaFuncSetAttribute(k_bias_bwd_part, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)slot_bytes));
  k_bias_bwd_part<<<(unsigned)g.ctas, kBwdThreads, slot_bytes, st>>>(*a, g.np, g.off, g.K, g.ET,
                                                                     ceil_div(g.P, g.ctas), part,
                                                                     tok ? tok_part : nullptr);
  GPS_LAUNCH_CHECK();
  const size_t sig_bytes = (size_t)(g.ET * g.H) * sizeof(float);
  k_bias_bwd_final<<<1, kFinalThreads, sig_bytes, st>>>(*a, g.K, g.ET, g.ctas, part, tok ? tok_part : nullptr);
  GPS_LAUNCH_CHECK();
  if (!g.edges) {   // no edge term: its parameters do not enter the output
    if (a->grad_edge_dis_weight)
      GPS_CUDA(cudaMemsetAsync(a->grad_edge_dis_weight, 0, (size_t)(g.S * g.H * g.H) * sizeof(float), st));
    if (a->grad_edge_weight)
      GPS_CUDA(cudaMemsetAsync(a->grad_edge_weight, 0, (size_t)(g.T * g.H) * sizeof(float), st));
  }
  if (!g.off && a->grad_graph_token)
    GPS_CUDA(cudaMemsetAsync(a->grad_graph_token, 0, (size_t)g.H * sizeof(float), st));
  return GPS_OK;
}

}  // namespace

}  // namespace gps

// =================================================================================== C ABI
using namespace gps;

extern "C" int gps_graphormer_bias_plan(const GpsGraphormerBiasArgs* args, GpsGraphormerBiasPlan* plan) {
  GPS_REQUIRE(args && plan, GPS_ERR_ARG, "gps_graphormer_bias_plan: null argument");
  BiasGeom g;
  GPS_TRY(make_geom(args, &g));
  plan->fwd_workspace_bytes = 0;
  plan->bwd_workspace_bytes = g.bwd_bytes;
  return GPS_OK;
}

extern "C" int gps_graphormer_bias_forward(const GpsGraphormerBiasArgs* args, void* stream) {
  return bias_forward(args, (cudaStream_t)stream);
}

extern "C" int gps_graphormer_bias_backward(const GpsGraphormerBiasArgs* args, void* stream) {
  return bias_backward(args, (cudaStream_t)stream);
}
