/*
 * gps_b200.h — C ABI of libgps_b200.so: an H100 (sm_90a) implementation of the GraphGPS
 * `GPSLayer` forward+backward hot path.
 *
 * The reference (rampasek/GraphGPS) is pure Python and has NO FFI of its own (SURVEY.md §8b);
 * the boundary it offers is the Python module `graphgps.layer.gps_layer.GPSLayer`
 * (graphgps/layer/gps_layer.py:16-264).  The entry points below are what a binding for that
 * module calls; each cites the reference lines it replaces.  INTEGRATION.md shows the
 * ctypes binding and the GraphGym-side patch.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in `_host`;
 *   - the caller (PyTorch) owns every buffer; the library never allocates tensor memory.
 *     Scratch/saved sizes come from gps_layer_plan();
 *   - all work is enqueued on `stream` (a cudaStream_t passed as void*); no hidden
 *     synchronisation, no default-stream use; calls are re-entrant;
 *   - return value: 0 = ok, -1 = bad argument, -2 = unsupported shape/variant,
 *     -3 = CUDA error.  gps_last_error() returns a thread-local message.  No C++ exception
 *     crosses this boundary;
 *   - matrices are row-major float32; weights are `[out, in]` as in torch.nn.Linear
 *     (y = x · Wᵀ + b);
 *   - edge j→i: src = edge_index[0] = j, dst = edge_index[1] = i (PyG source_to_target flow,
 *     graphgps/layer/gatedgcn_layer.py:90-126).
 */
#ifndef GPS_B200_H_
#define GPS_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GPS_ABI_VERSION 4

enum { GPS_OK = 0, GPS_ERR_ARG = -1, GPS_ERR_UNSUPPORTED = -2, GPS_ERR_CUDA = -3 };

/* local_gnn_type / global_model_type of GPSLayer.__init__ (gps_layer.py:20-24,44-122) */
enum { GPS_LOCAL_NONE = 0, GPS_LOCAL_GATEDGCN = 1, GPS_LOCAL_GINE = 2, GPS_LOCAL_GCN = 3, GPS_LOCAL_GAT = 4,
       GPS_LOCAL_GENCONV = 5, GPS_LOCAL_PNA = 6 };
enum { GPS_GLOBAL_NONE = 0, GPS_GLOBAL_TRANSFORMER = 1, GPS_GLOBAL_PERFORMER = 2,
       GPS_GLOBAL_BIGBIRD = 3 };
/* register.act_dict keys used by shipped configs (gps_layer.py:33) */
enum { GPS_ACT_RELU = 0, GPS_ACT_GELU = 1 };
/* arithmetic of the dense products: FP32 = fp32-grade result (split-bf16 x3 on the tensor cores,
 * tolerance 1e-3 vs the reference); BF16 = single bf16 pass, fp32 accumulate (tolerance 1e-2) */
enum { GPS_PREC_FP32 = 0, GPS_PREC_BF16 = 1 };
/* GpsLayerArgs.norm_type: cfg.gt.batch_norm = True / False with cfg.gt.layer_norm = False (gps_layer.py:125-151) */
enum { GPS_NORM_BATCH = 0, GPS_NORM_NONE = 1 };

const char* gps_last_error(void);
int gps_abi_version(void);
/* compiled-for architecture string, e.g. "sm_100a" */
const char* gps_build_arch(void);
/* number of CUDA kernels this library has launched in the calling process (bench.py reports the
 * delta over its timed region as `gpu_launches`) */
unsigned long long gps_launch_count(void);
/* tuning hook of the register-staged wgmma GEMM (tools/gemm_tune.py): bits 8.. = forced tile width. 0 = normal. */
void gps_debug_set(int v);
/* bring-up hook of the TMA-fed GEMM (tools/gemm_trace.py): force_bn = forced tile width (0 = the launch policy; 64, 128,
 * 152 for a K-major B, 256 for a K-major A; a width the operand layout cannot take makes the product fail with
 * GPS_ERR_UNSUPPORTED); trace = device
 * buffer of 256 x 16 uint64 that the first 256 CTAs of each launch fill with globaltimer phase stamps (NULL = off) */
void gps_debug_tma(int force_bn, void* trace);
/* test hook of the TMA-fed GEMM: K-splits of every product that runs its epilogue (splitk <= 1), summed across the
 * cluster before the epilogue; 0 = the launch policy.  The count is clamped to [1, 8] and to the k-blocks of K. */
void gps_debug_tma_splits(int splits);
/* bring-up hook of the wgmma attention: device buffer of 3 x 128 x 128 floats that CTA (0,0) fills with its first
 * S tile, P tile and raw O accumulator (NULL = off) */
void gps_debug_attn(void* buf);

/* ------------------------------------------------------------------------------------------
 * Graph structure of one mini-batch (constant across the L layers and across fwd/bwd).
 * Replaces, per layer, PyG `MessagePassing.propagate`'s index handling
 * (gatedgcn_layer.py:67-70), torch_scatter's atomics (gatedgcn_layer.py:118-123) and
 * `to_dense_batch`'s bincount/cumsum/max (gps_layer.py:199).
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  int64_t N, E, B;
  const int32_t* dst_ptr;   /* [N+1] CSR by destination                          */
  const int32_t* dst_src;   /* [E]   source node of the k-th dst-sorted edge      */
  const int32_t* dst_eid;   /* [E]   original edge id of the k-th dst-sorted edge */
  const int32_t* src_ptr;   /* [N+1] CSC by source                               */
  const int32_t* src_dst;   /* [E]   destination node of the k-th src-sorted edge */
  const int32_t* src_eid;   /* [E]   original edge id                            */
  const int32_t* graph_ptr; /* [B+1] node offsets of each graph                  */
} GpsGraph;

/* bytes of int32 scratch the caller must provide to gps_graph_build (all arrays above) */
int64_t gps_graph_bytes(int64_t N, int64_t E, int64_t B);
/* Builds the CSR/CSC/graph_ptr arrays inside `storage` (>= gps_graph_bytes) from int64
 * edge_index [2,E] and sorted int64 batch [N]; fills *out with pointers into storage.
 * Within a node's segment edges are ordered by original edge id, so every reduction over
 * a segment is deterministic. */
int gps_graph_build(const int64_t* edge_index, const int64_t* batch, int64_t N, int64_t E,
                    int64_t B, void* storage, int64_t storage_bytes, GpsGraph* out,
                    void* stream);

/* ------------------------------------------------------------------------------------------
 * One BatchNorm1d (torch.nn.BatchNorm1d: gps_layer.py:136-138,150-151; gatedgcn_layer.py:37-38)
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  const float* weight;       /* gamma [d]                       */
  const float* bias;         /* beta  [d]                       */
  float* running_mean;       /* [d] updated in training mode    */
  float* running_var;        /* [d]                             */
  int64_t* num_batches_tracked; /* [1] or NULL                  */
  float* grad_weight;        /* [d] backward output (may be NULL in forward) */
  float* grad_bias;          /* [d]                             */
} GpsBatchNorm;

/* One Linear (weight [out,in], bias [out] or NULL) with its gradient outputs */
typedef struct {
  const float* weight;
  const float* bias;
  float* grad_weight;
  float* grad_bias;
} GpsLinear;

/* bf16 hi/lo planes of an fp32 [rows, cols] tensor: row-major, pitch ld elements (multiple of 8); lo may be NULL in
 * GPS_PREC_BF16 mode */
typedef struct {
  void* hi;
  void* lo;
  int64_t ld;
} GpsPlanes;

/* ------------------------------------------------------------------------------------------
 * GPSLayer forward / backward  (gps_layer.py:155-257; GatedGCN gatedgcn_layer.py:45-136)
 * state_dict names in comments are the reference's (SURVEY.md §8b).  GpsLayerArgs carries every local and global
 * model; local_type / global_type choose which of its members are read.  The structs below are members of it.
 * ---------------------------------------------------------------------------------------- */

/* Additive attention bias of the BiasedTransformer global model (gps_layer.py:104-106,202-204,234-241; Graphormer's
 * batch.attn_bias): bias [B*heads, nmax, nmax] row-major float32, row g*heads + h of graph g and head h, entry (il, jl)
 * for local query il and local key jl; nmax >= the largest graph of the batch (to_dense_batch's Nmax).  The scores
 * become S = (q . k) / sqrt(hd) + bias[g*heads + h, il, jl]; padded entries (il or jl >= n_g) are not read.  grad_bias
 * (backward; NULL = not needed) has the same layout and is written whole: dL/dS at every in-graph entry, 0 at every
 * padded one. */
typedef struct {
  const float* bias;
  int64_t nmax;
  float* grad_bias;
} GpsAttnBias;

/* GAT local model (local_type == GPS_LOCAL_GAT): PyG 2.2 GATConv(dim_h, dim_h / heads, heads=heads, edge_dim=dim_h)
 * with its defaults (concat, negative_slope 0.2, no attention dropout, add_self_loops with fill_value 'mean', bias),
 * gps_layer.py:70-74,183-189.  H = GpsLayerArgs.heads heads of C = d / H channels each (d % H != 0 is GPS_ERR_ARG).
 * Existing self-loop edges are dropped and one loop per node is added whose edge attribute is the mean of the node's
 * remaining in-edge attributes (0 without any); their grad_edge_attr rows are 0.  edge_attr and, in the backward,
 * grad_edge_attr are required (non-NULL when E > 0) and batch.edge_attr is not updated.  Parameters (non-NULL, else
 * GPS_ERR_ARG):
 *   lin_src   weight = local_model.lin_src.weight [d,d] (lin_dst is the same module), bias = local_model.bias [d]
 *             (added after the aggregation); its gradients: grad_weight with the fused node projection (final at
 *             ev_grads_done), grad_bias final at ev_grads_mid;
 *   lin_edge  weight = local_model.lin_edge.weight [d,d] (no bias);
 *   att_src / att_dst / att_edge = local_model.att_{src,dst,edge} [1,H,C], and their gradients, final at ev_grads_mid. */
typedef struct {
  GpsLinear lin_src;
  GpsLinear lin_edge;
  const float* att_src;
  const float* att_dst;
  const float* att_edge;
  float* grad_att_src;
  float* grad_att_dst;
  float* grad_att_edge;
} GpsGat;

/* GENConv local model (local_type == GPS_LOCAL_GENCONV): PyG 2.2 GENConv(dim_h, dim_h) with its defaults (softmax
 * aggregation with t = 1, no message norm, eps 1e-7, MLP d -> 2d -> d with BatchNorm, no bias), gps_layer.py:60-61,
 * 183-189.  For target i and channel c: m_k = relu(x[src_k] + e_k) + 1e-7, agg_i = sum_k softmax_k(m)_c m_kc over i's
 * in-edges (0 without any; self loops and duplicates are ordinary edges), u = agg + x and
 * h = lin1(relu(bn(lin0(u)))); x_loc = x + dropout(h).  edge_attr [E, d] and, in the backward, grad_edge_attr are
 * required (non-NULL when E > 0) and batch.edge_attr is not updated.  d % 4 == 0 and d <= 2048 (the 2d-wide BatchNorm
 * runs on the row-wise stages), else GPS_ERR_UNSUPPORTED.  Parameters (all non-NULL, else GPS_ERR_ARG), whose
 * gradients are final at ev_grads_mid:
 *   lin0 = local_model.mlp.0 [2d, d], bias NULL;
 *   bn   = local_model.mlp.1 [2d]: weight, bias, running_mean, running_var (num_batches_tracked optional); training
 *          mode normalises with the batch statistics and updates the running ones as torch.nn.BatchNorm1d;
 *   lin1 = local_model.mlp.4 [d, 2d], bias NULL.  The MLP's activation is ReLU whatever GpsLayerArgs.act is. */
typedef struct {
  GpsLinear lin0;
  GpsBatchNorm bn;
  GpsLinear lin1;
} GpsGenConv;

/* PNA local model (local_type == GPS_LOCAL_PNA): PyG 2.2 PNAConv(dim_h, dim_h, aggregators=['mean','max','sum'],
 * scalers=['identity'], edge_dim=edge_dim, towers=1, pre_layers=1, post_layers=1, divide_input=False),
 * gps_layer.py:75-90,183-189.  For edge k from j to i:
 *   m_k = pre.weight [x_i ; x_j ; edge_encoder(e_k)] + pre.bias
 * and per target i and channel the mean, max and sum of m over i's in-edges (0 in all three without any; self loops
 * and duplicates are ordinary edges); x_loc = x + dropout(lin(post([x | mean | max | sum]))).  The max gradient goes
 * whole to the first maximising in-edge in edge_index order (torch_scatter's scatter_max).  The degree histogram never
 * enters the arithmetic with the identity scaler, so it is not an argument.  edge_attr and grad_edge_attr are
 * [E, edge_dim] and required (non-NULL when E > 0); batch.edge_attr is not updated.  0 < edge_dim <= d and
 * edge_dim % 4 == 0, else GPS_ERR_UNSUPPORTED; gps_layer_plan does not read edge_dim and sizes for its bound d.
 * Parameters (weights and biases non-NULL, else GPS_ERR_ARG):
 *   edge_encoder = local_model.edge_encoder [d, edge_dim] + [d]; gradients final at ev_grads_mid;
 *   pre  = local_model.pre_nns.0.0 [d, 3d] + [d] (column blocks: destination, source, encoded edge); gradients final
 *          at ev_grads_done (the first two blocks come with the fused node projection);
 *   post = local_model.post_nns.0.0 [d, 4d] + [d]; gradients final at ev_grads_mid;
 *   lin  = local_model.lin [d, d] + [d]; gradients final at ev_grads_mid. */
typedef struct {
  GpsLinear edge_encoder;
  GpsLinear pre;
  GpsLinear post;
  GpsLinear lin;
  int64_t edge_dim;
} GpsPna;

/* BigBird global model (global_type == GPS_GLOBAL_BIGBIRD): the reference's SingleBigBirdLayer, one BigBirdLayer with
 * block-sparse self-attention (gps_layer.py:115-119,207-208; bigbird_layer.py:1667-1706).  For graph g of n_g nodes,
 * local position p is node graph_ptr[g] + p; the batch is padded to S = num_blocks * block_size positions (to_dense_batch's
 * Nmax rounded up to the block size) and positions >= n_g are masked keys, never queries.  Head h of query block i
 * attends to the multiset of key blocks key_idx[key_ptr[h*(nb+1) + i] .. key_ptr[h*(nb+1) + i + 1]) (a block listed
 * twice counts twice in the softmax); query_ptr / query_idx is its transpose (the query blocks of every key block, in
 * ascending order, with the same multiplicities).  nb = num_blocks >= 4, block_size >= 1 and the four lists non-NULL,
 * else GPS_ERR_ARG.  Scale 1/sqrt(hd), hd = d / heads (any hd >= 1 up to 128; d % heads != 0 is GPS_ERR_ARG), no
 * attention dropout.  With ctx the attention output [N, d]:
 *   a   = LN1(drop_8(ctx Wso^T + bso) + x)          (attention.output; dropout site 8 = GPS_SITE_BB_SELF_OUT)
 *   u   = act(a Wi^T + bi)                           (intermediate; act = hidden_act: 0 relu, 1 sigmoid)
 *   out = LN2(drop_9(u Wo^T + bo) + a)               (output; dropout site 9 = GPS_SITE_BB_OUTPUT)
 * LN = nn.LayerNorm(d, eps = ln_eps) over each row; both dropouts use GpsLayerArgs.dropout.  out then takes the place of
 * the attention output in the GPS layer: hA = x + drop_4(out), norm1_attn, as for the Transformer.  Parameters
 * (self_attn.encoder.layers.0.*; weights [d, d]; non-NULL, else GPS_ERR_ARG): query / key / value =
 * attention.self.{query,key,value} (bias NULL unless use_bias), self_out = attention.output.dense, ln1 =
 * attention.output.LayerNorm (weight = gamma, bias = beta), intermediate = intermediate.dense, output = output.dense,
 * ln2 = output.LayerNorm.  Gradients: query / key / value are final at ev_grads_done (one weight-gradient product with
 * the node projections); the other five at ev_grads_mid.  gps_layer_plan sizes BigBird from N, d and heads alone. */
enum { GPS_BIGBIRD_RELU = 0, GPS_BIGBIRD_SIGMOID = 1 };
typedef struct {
  int64_t block_size;
  int64_t num_blocks;          /* nb of the batch: ceil(Nmax / block_size) */
  int32_t hidden_act;          /* GPS_BIGBIRD_* */
  float ln_eps;                /* layer_norm_eps */
  const int32_t* key_ptr;      /* [heads * (nb + 1)], offsets into key_idx */
  const int32_t* key_idx;
  const int32_t* query_ptr;    /* [heads * (nb + 1)], offsets into query_idx */
  const int32_t* query_idx;
  GpsLinear query, key, value, self_out, ln1, intermediate, output, ln2;
} GpsBigBird;

/* GpsLayerArgs.flags (backward) */
enum {
  GPS_FLAG_GRADS_ZEROED = 1,     /* the parameter-gradient buffers are already zero */
  GPS_FLAG_GRADS_ACCUMULATE = 2  /* parameter gradients are added to the buffers (implies GPS_FLAG_GRADS_ZEROED) */
};

typedef struct {
  /* configuration */
  int64_t d;                 /* dim_h                                               */
  int64_t heads;             /* num_heads                                           */
  int32_t local_type;        /* GPS_LOCAL_*                                         */
  int32_t global_type;       /* GPS_GLOBAL_*                                        */
  int32_t act;               /* GPS_ACT_*                                           */
  int32_t training;          /* 1: batch statistics + dropout; 0: running stats     */
  int32_t precision;         /* GPS_PREC_*                                          */
  int32_t flags;             /* GPS_FLAG_* (backward)                               */
  float dropout;             /* cfg.gt.dropout       (gps_layer.py:92-96,139-140,152-153) */
  float attn_dropout;        /* cfg.gt.attn_dropout  (gps_layer.py:105-106,112-114)       */
  uint64_t seed;             /* Philox key for this call's dropout masks            */
  uint64_t offset;           /* Philox counter base (caller advances per call)      */
  float gine_eps;            /* local_model.eps buffer value (GINE)                 */
  /* normalisation of the GPSLayer (gps_layer.py:125-151, 191-229), GPS_NORM_*.  BATCH: norm1_local, norm1_attn and
   * norm2 are BatchNorm1d.  NONE (batch_norm=False, layer_norm=False): the three modules do not exist and are not read;
   * x_loc = x + local(x), hA = x + MHA(x), s = x_loc + hA, x_out = s + FFN(s).  GatedGCN's bn_node_x / bn_edge_e belong
   * to the local model and are required in both modes.  Any other value makes gps_layer_plan / _forward / _backward
   * return GPS_ERR_UNSUPPORTED. */
  int32_t norm_type;

  GpsGraph graph;

  /* inputs / outputs, row-major [N,d] / [E,d] */
  const float* x;            /* batch.x                                             */
  const float* edge_attr;    /* batch.edge_attr                                     */
  float* x_out;              /* new batch.x                                         */
  float* edge_out;           /* new batch.edge_attr (GatedGCN only, else unused)    */

  /* parameters */
  GpsLinear gcn_A, gcn_B, gcn_C, gcn_D, gcn_E;      /* local_model.{A,B,C,D,E}        */
  GpsBatchNorm bn_node_x, bn_edge_e;                /* local_model.bn_node_x / bn_edge_e */
  GpsLinear gine_lin0, gine_lin1;                   /* local_model.nn.0 / nn.2 (GINE) */
  GpsLinear attn_in;                                /* self_attn.in_proj_{weight,bias} [3d,d]   */
  GpsLinear attn_out;                               /* self_attn.out_proj / to_out              */
  GpsLinear perf_q, perf_k, perf_v;                 /* self_attn.to_{q,k,v} (no bias)           */
  const float* perf_proj;                           /* fast_attention.projection_matrix [m,64]  */
  int64_t perf_features;                            /* m (266)                                  */
  int64_t perf_dim_head;                            /* 64                                       */
  GpsBatchNorm norm1_local, norm1_attn, norm2;
  GpsLinear ff1, ff2;                               /* ff_linear1 [2d,d], ff_linear2 [d,2d]     */

  /* gradients w.r.t. outputs (backward input) and inputs (backward output) */
  const float* grad_x_out;   /* [N,d]                                               */
  const float* grad_edge_out;/* [E,d] or NULL (treated as zero)                     */
  float* grad_x;             /* [N,d]                                               */
  float* grad_edge_attr;     /* [E,d]                                               */

  /* caller-owned scratch; sizes from gps_layer_plan() */
  void* saved;   int64_t saved_bytes;     /* written by forward, read by backward   */
  void* workspace; int64_t workspace_bytes; /* transient; may be shared between calls on one stream */

  /* optional device-resident addend for `offset` (uint64 on the device, read by the kernels at run time):
   * lets a captured CUDA graph draw fresh dropout masks on every replay. NULL = use `offset` only. */
  const uint64_t* offset_dev;

  /* PyG GCNConv(dim_h, dim_h) local model (gps_layer.py:49-51): weight = local_model.lin.weight [d,d] (its Linear has
   * no bias), bias = local_model.bias [d], added after the normalised aggregation. */
  GpsLinear gcn_conv;

  /* backward, optional: a cudaEvent_t the library records as soon as the "early" parameter gradients are final -
   * ff_linear1/2, the attention output projection, norm2, norm1_local, norm1_attn - a few hundred microseconds before
   * the pass ends.  A data-parallel caller makes its communication stream wait on it and all-reduces that part of the
   * gradient bucket under the rest of the backward pass (graphgps_b200/dp.py).  NULL = not recorded. */
  void* ev_grads_early;

  /* optional: operand-plane hand-off between consecutive layers of a GPSModel (network/gps_model.py:100,105-108) and
   * persistent weight planes.  A plane pair is the bf16 hi/lo image of an fp32 tensor (see gps_to_planes).
   *  x_planes_in / e_planes_in   planes of x / edge_attr written by the previous layer: the layer skips its own
   *                              conversion of the inputs (hi == NULL: convert here, into `saved`);
   *  x_planes_out / e_planes_out caller-owned plane buffers the layer fills next to x_out / edge_out;
   *  wplanes                     caller-owned buffer (GpsLayerPlan.wplanes_bytes) for the planes of every weight;
   *                              wplanes_valid != 0: it already holds this layer's current weights (packed once per
   *                              optimiser step instead of once per forward call). */
  GpsPlanes x_planes_in, e_planes_in, x_planes_out, e_planes_out;
  void* wplanes; int64_t wplanes_bytes; int32_t wplanes_valid; int32_t reserved2 /* padding */;

  /* backward, optional: two more cudaEvent_t of the same kind as ev_grads_early.  ev_grads_mid: the local model's
   * gradients outside the fused node projection (C / GINE nn / GCN bias, bn_node_x, bn_edge_e) are final; A, B, D, E /
   * GCN lin share one weight-gradient GEMM with in_proj at the end of the pass.  ev_grads_done: every gradient of this
   * layer is final. */
  void* ev_grads_mid;
  void* ev_grads_done;

  /* optional: the EquivStableLapPE edge gate of GatedGCN (equivstable_pe=True, gatedgcn_layer.py:29-35,101-104).
   * pe = batch.pe_EquivStableLapPE, row-major contiguous [N, pe_dim], pe_dim >= 1.  For edge j->i:
   * r = sum_c (pe_i - pe_j)^2, rho = mlp_r_ij(r) and the gate becomes sigmoid(e_ij) * rho.  pe == NULL: no gate (the
   * fields below are not read).  pe != NULL with a local_type other than GPS_LOCAL_GATEDGCN is GPS_ERR_ARG.  Backward
   * writes grad_pe [N, pe_dim] (NULL = not needed) and the gradients of pe_mlp0 / pe_mlp1, which are final when
   * ev_grads_mid fires. */
  const float* pe; int64_t pe_dim;
  float* grad_pe;
  GpsLinear pe_mlp0 /* mlp_r_ij.0 [d,1] */, pe_mlp1 /* mlp_r_ij.2 [1,d] */;

  /* BiasedTransformer: bias == NULL is the unbiased Transformer (nmax and grad_bias must then be 0 / NULL).  A non-NULL
   * bias needs global_type == GPS_GLOBAL_TRANSFORMER and nmax >= 1, else GPS_ERR_ARG.  gps_layer_plan does not read it;
   * forward and backward must see the same bias tensor. */
  GpsAttnBias attn_bias;
  GpsGat gat;                /* read when local_type == GPS_LOCAL_GAT                */
  GpsGenConv genconv;        /* read when local_type == GPS_LOCAL_GENCONV            */
  GpsPna pna;                /* read when local_type == GPS_LOCAL_PNA                */
  GpsBigBird bigbird;        /* read when global_type == GPS_GLOBAL_BIGBIRD         */
} GpsLayerArgs;

typedef struct {
  int64_t saved_bytes;          /* activations kept for backward (0 needed if eval-only) */
  int64_t fwd_workspace_bytes;
  int64_t bwd_workspace_bytes;
  int64_t wplanes_bytes;        /* size of the optional persistent weight-plane buffer (GpsLayerArgs.wplanes) */
} GpsLayerPlan;

/* Sizes for the given configuration/graph (only sizes and type fields of args are read). */
int gps_layer_plan(const GpsLayerArgs* args, GpsLayerPlan* plan);
int gps_layer_forward(const GpsLayerArgs* args, void* stream);
int gps_layer_backward(const GpsLayerArgs* args, void* stream);

/* BigBird stage entry points.  Q, K, V: [N, heads*hd] slices with row stride ld; O / dO [N, heads*hd] (stride ldo);
 * lse / delta [N, heads] (per-row log-sum-exp / rowsum(dO * O)); dQ, dK, dV written whole (stride ldg).  Only bb's
 * geometry and lists are read.  The forward is one warp per (graph, head, query block); the backward a query-major pass
 * for dQ and a key-major pass over the transposed lists for dK / dV: no atomics, the same bits in every run. */
int gps_bigbird_attention_forward(const GpsGraph* g, int64_t heads, int64_t hd, const GpsBigBird* bb, const float* Q,
                                  const float* K, const float* V, int64_t ld, float* O, int64_t ldo, float* lse,
                                  void* stream);
int gps_bigbird_attention_backward(const GpsGraph* g, int64_t heads, int64_t hd, const GpsBigBird* bb, const float* Q,
                                   const float* K, const float* V, int64_t ld, const float* O, const float* dO,
                                   int64_t ldo, const float* lse, float* delta, float* dQ, float* dK, float* dV,
                                   int64_t ldg, void* stream);
/* Row-wise LayerNorm [rows, d] (d % 4 == 0, d <= 4096): y = (z - mean) * rstd * gamma + beta, mean / rstd [rows] saved.
 * Backward from g: dz [rows, d], and grad_gamma / grad_beta [d] (each NULL = not needed; written, or added when
 * accumulate != 0) reduced through per-CTA partials in a fixed order; workspace: 264 * d floats. */
int gps_layernorm_forward(const float* z, int64_t rows, int64_t d, const float* gamma, const float* beta, float eps,
                          float* y, float* mean, float* rstd, void* stream);
int gps_layernorm_backward(const float* g, const float* z, int64_t rows, int64_t d, const float* gamma, const float* mean,
                           const float* rstd, float* dz, float* grad_gamma, float* grad_beta, void* workspace,
                           int32_t accumulate, void* stream);

/* ------------------------------------------------------------------------------------------
 * Graphormer layer (graphgps/layer/graphormer_layer.py:5-49), the building block of GraphormerModel:
 *   h   = input_norm(x)                                    LayerNorm(d), eps 1e-5
 *   a   = MHA(h) over each graph's own nodes                scale 1/sqrt(hd), + attn_bias after scaling when given,
 *                                                           attn_dropout on the probabilities (site 16 + head)
 *   x1  = x + drop_10(a)                                    dropout, site 10
 *   out = x1 + drop_12(W2 drop_11(GELU(W1 mlp_norm(x1) + b1)) + b2)
 *                                                           mlp_dropout at site 11, dropout at site 12
 * Any head dim hd = d / heads (d % heads != 0 is GPS_ERR_ARG); d % 4 == 0 and d <= 4096, hd <= 192, else
 * GPS_ERR_UNSUPPORTED.  Parameters (all non-NULL, else GPS_ERR_ARG):
 *   input_norm = input_norm (weight = gamma, bias = beta), attn_in = attention.in_proj_{weight,bias} [3d, d],
 *   attn_out = attention.out_proj [d, d], mlp_norm = mlp.0 (gamma / beta), mlp_lin1 = mlp.1, mlp_lin2 = mlp.4 [d, d].
 * Backward writes grad_x and every non-NULL parameter gradient; the weight products run on a side stream that joins the
 * caller's stream before the call returns; the LayerNorm gradients are reduced through per-CTA partials in a fixed
 * order.  No float atomics: two runs give the same bits.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  int64_t d;                 /* embed_dim                                                     */
  int64_t heads;             /* num_heads                                                     */
  int32_t training;          /* 1: dropout active                                             */
  int32_t precision;         /* GPS_PREC_*                                                    */
  float dropout;             /* after the attention and after the MLP (sites 10, 12)          */
  float attn_dropout;        /* on the attention probabilities                                */
  float mlp_dropout;         /* inside the MLP, after GELU (site 11)                          */
  int32_t flags;             /* GPS_FLAG_* (backward), as GpsLayerArgs.flags                  */
  uint64_t seed;             /* Philox key of this call's dropout masks                      */
  uint64_t offset;           /* Philox counter base                                           */
  const uint64_t* offset_dev;/* optional device-resident addend to offset (CUDA-graph replays); NULL = none */
  GpsGraph graph;
  const float* x;            /* [N, d] batch.x                                                */
  float* x_out;              /* [N, d] new batch.x (forward)                                  */
  const float* grad_x_out;   /* [N, d] (backward)                                             */
  float* grad_x;             /* [N, d] (backward)                                             */
  void* saved; int64_t saved_bytes;         /* written by forward, read by backward           */
  void* workspace; int64_t workspace_bytes; /* transient                                      */
  GpsLinear input_norm, attn_in, attn_out, mlp_norm, mlp_lin1, mlp_lin2;
} GpsGraphormerArgs;

typedef struct {
  int64_t saved_bytes;
  int64_t fwd_workspace_bytes;
  int64_t bwd_workspace_bytes;
} GpsGraphormerPlan;

/* Sizes for the configuration and graph of args (only d, heads, precision and graph.N / graph.B are read). */
int gps_graphormer_plan(const GpsGraphormerArgs* args, GpsGraphormerPlan* plan);
/* bias: GpsAttnBias (layout as for the BiasedTransformer: [B*heads, nmax, nmax], row g*heads + h), or NULL for none.
 * The backward writes bias->grad_bias when it is not NULL. */
int gps_graphormer_forward(const GpsGraphormerArgs* args, const GpsAttnBias* bias, void* stream);
int gps_graphormer_backward(const GpsGraphormerArgs* args, const GpsAttnBias* bias, void* stream);

/* ------------------------------------------------------------------------------------------
 * Graphormer's attention-bias encoder (graphgps/encoder/graphormer_encoder.py:103-183, BiasEncoder), the producer of
 * the GpsAttnBias both consumers above read.  Inputs are graphormer_pre_processing's attributes, PyG-collated: pair p
 * has global nodes i = graph_index[0, p], j = graph_index[1, p] of one graph b (node_ptr[b] <= i, j < node_ptr[b+1]),
 * spatial type s_p = spatial_types[p] in [0, S] and, when shortest_path_types is not NULL, path types
 * t_pk = shortest_path_types[p * S + k] in [0, T).  With sd_p = max(1, s_p), il = i - node_ptr[b], jl = j - node_ptr[b]
 * and o = 1 with the graph token (else 0):
 *   attn_bias[b*H + h, o + il, o + jl] = spatial_weight[s_p, h]
 *                     + (1 / sd_p) sum_{k<S} sum_{h'} edge_weight[t_pk, h'] edge_dis_weight[(k*H + h')*H + h]
 * (the edge term only with shortest_path_types).  The output [B*H, N', N'], N' = nmax + o, is written whole: entries
 * no pair covers are 0 and, with the graph token, row 0 and column 0 of every graph hold graph_token[h].
 * Precondition: each ordered pair of a graph appears at most once (as graphormer_pre_processing emits them); each pair
 * is written with a plain store and their order is free.  A pair whose nodes or spatial type are out of range is
 * skipped, and a path type out of range adds nothing: no input is dereferenced out of bounds (the Python module rejects
 * such inputs before the call).
 * Backward from grad_attn_bias writes (each NULL = not needed) grad_spatial_weight [S+1, H], grad_edge_dis_weight
 * [S*H*H], grad_edge_weight [T, H] and grad_graph_token [H] through per-CTA partials summed in a fixed order: no float
 * atomics, two runs give the same bits.
 * Staged sizes: H <= 32, (S+1)*H <= 4096 and S*T*H <= 8192 floats, S*T + S + 1 <= 384 per-thread slots of the backward
 * (S*T counted only with shortest_path_types); anything larger is GPS_ERR_UNSUPPORTED.  Pair x position offsets are
 * 64-bit.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  int64_t num_pairs;         /* P                                                             */
  int64_t num_graphs;        /* B = batch.max() + 1 (to_dense_adj's batch size)               */
  int64_t nmax;              /* largest graph of the batch                                    */
  int64_t heads;             /* H = num_heads                                                 */
  int64_t num_spatial_types; /* S                                                             */
  int64_t num_edge_types;    /* T                                                             */
  int32_t use_graph_token;   /* 1: pad by one row and column and write graph_token there      */
  int32_t reserved;
  const int64_t* spatial_types;       /* [P]                                                  */
  const int64_t* graph_index;         /* [2, P] global node ids                               */
  const int64_t* shortest_path_types; /* [P, S] or NULL (no edge term)                        */
  const int64_t* node_ptr;            /* [B+1] first node of each graph                       */
  const float* spatial_weight;        /* spatial_encoder.weight [S+1, H]                      */
  const float* edge_dis_weight;       /* edge_dis_encoder.weight [S*H*H, 1]                   */
  const float* edge_weight;           /* edge_encoder.weight [T, H]                           */
  const float* graph_token;           /* graph_token [1, H, 1] (use_graph_token)              */
  float* attn_bias;                   /* [B*H, N', N'] (forward)                              */
  const float* grad_attn_bias;        /* [B*H, N', N'] (backward)                             */
  float* grad_spatial_weight;
  float* grad_edge_dis_weight;
  float* grad_edge_weight;
  float* grad_graph_token;
  void* workspace; int64_t workspace_bytes; /* transient (backward)                           */
} GpsGraphormerBiasArgs;

typedef struct {
  int64_t fwd_workspace_bytes;
  int64_t bwd_workspace_bytes;
} GpsGraphormerBiasPlan;

/* Sizes for args (only the sizes, use_graph_token and whether shortest_path_types is NULL are read). */
int gps_graphormer_bias_plan(const GpsGraphormerBiasArgs* args, GpsGraphormerBiasPlan* plan);
int gps_graphormer_bias_forward(const GpsGraphormerBiasArgs* args, void* stream);
int gps_graphormer_bias_backward(const GpsGraphormerBiasArgs* args, void* stream);

/* ------------------------------------------------------------------------------------------
 * Inductive link-prediction head (graphgps/head/inductive_edge.py, GNNInductiveEdgeHead) with edge_decoding "dot" and
 * layers_post_mp 1, the head of every PCQM-Contact config:
 *   y = x W^T + b                          (layer_post_mp.model.0.model, [d, d] and [d]; replaces batch.x)
 *   pred[k] = <y[s_k], y[t_k]>             (s_k, t_k) = column k of edge_index_labeled [2, K]
 * `pairs` is gps_graph_build(edge_index_labeled, batch, N, K, B): CSR by target, CSC by source, graph_ptr.
 * Eval (training == 0) also writes stats [4] float64 = hits@1, hits@3, hits@10, mrr averaged over the B graphs: for a
 * positive pair (i, j) (edge_label == 1) of graph g, rank = 1 + #{k in g, k != j : <y_i, y_k> > <y_i, y_j>} (the rank a
 * stable descending sort gives: ties count in the positive's favour); a graph's values are the means over its positives
 * of rank <= 1, <= 3, <= 10 and 1 / rank, and 0 when it has none.  A positive whose target lies outside its source's
 * graph is not counted (the Python module rejects such batches in eval).
 * Backward: dy = grad_y + sum_k g_k (y[t_k] e_{s_k} + y[s_k] e_{t_k}) as two segmented sums in pair order, then
 * dW = dy^T x, db = sum dy (deterministic split-K) and grad_x = dy W: no float atomics in fp32, two runs give the same
 * bits.  Indices out of [0, N) are never dereferenced.  d <= 4096.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  int64_t d;                 /* dim_in                                                        */
  int32_t training;          /* 1: training (no stats), 0: eval (stats)                       */
  int32_t precision;         /* GPS_PREC_*                                                    */
  int32_t flags;             /* reserved, 0                                                   */
  int32_t label_bytes;       /* 4 or 8: edge_label is int32 or int64                          */
  uint64_t seed;             /* unused (the head has no dropout)                              */
  GpsGraph pairs;            /* N = nodes, E = K labeled pairs, B = graphs                    */
  const int64_t* edge_index_labeled; /* [2, K]                                                */
  const void* edge_label;    /* [K] (eval)                                                    */
  const float* x;            /* [N, d]                                                        */
  GpsLinear lin;             /* layer_post_mp.model.0.model: weight [d, d], bias [d], grads   */
  float* y;                  /* [N, d] (forward)                                              */
  float* pred;               /* [K] (forward)                                                 */
  double* stats;             /* [4] (eval forward)                                            */
  const float* grad_y;       /* [N, d] or NULL (backward)                                     */
  const float* grad_pred;    /* [K] or NULL (backward)                                        */
  float* grad_x;             /* [N, d] (backward)                                             */
  void* saved; int64_t saved_bytes;         /* forward -> backward                            */
  void* workspace; int64_t workspace_bytes; /* transient                                      */
} GpsLinkHeadArgs;

typedef struct {
  int64_t saved_bytes;
  int64_t fwd_workspace_bytes;
  int64_t bwd_workspace_bytes;
} GpsLinkHeadPlan;

/* Sizes for args (only d, precision, training and the pair graph's N, E and B are read). */
int gps_link_head_plan(const GpsLinkHeadArgs* args, GpsLinkHeadPlan* plan);
int gps_link_head_forward(const GpsLinkHeadArgs* args, void* stream);
int gps_link_head_backward(const GpsLinkHeadArgs* args, void* stream);
/* Stage entry: the eval statistics above for node rows y [N, d] at pitch ld >= d, into stats [4]; workspace >= 32 * B
 * bytes (per-graph values). */
int gps_link_rank_metrics(const GpsGraph* pairs, const float* y, int64_t ld, int64_t d, const void* edge_label,
                          int32_t label_bytes, double* stats, void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Graph-prediction heads, the head of every graph-level config:
 *   GPS_GRAPH_HEAD_SAN (graphgps/head/san_graph.py, SANGraphHead(dim_in, dim_out, L)):
 *     h_0 = pool(x)                           [B, dim_in]
 *     h_{l+1} = act(h_l W_l^T + b_l), l < L   fc[l]: [dim_in >> (l+1), dim_in >> l]
 *     pred = h_L W_L^T + b_L                  fc[L]: [dim_out, dim_in >> L]
 *   GPS_GRAPH_HEAD_GRAPHORMER (graphgps/head/graphormer_graph.py, GraphormerHead(dim_in, dim_out)), L = 0:
 *     pred = pool(LayerNorm(x)) W^T + b       ln: gamma / beta [dim_in], eps 1e-5; fc[0]: [dim_out, dim_in]
 * Pooling over the graphs of `graph` (graph_ptr [B+1] read; rows sorted by graph): mean = per-graph sum / max(count, 1),
 * add = per-graph sum, graph_token = each graph's first row; an empty graph gives a zero row.  Under graph_token the
 * LayerNorm runs on the B token rows only (it is row-wise), so grad_x is zero off the token rows; an empty graph's row
 * stays zero after it, as pooling after the LayerNorm leaves it, so its pred is b and it adds nothing to ln's gradients.
 * Built: SAN head with mean / add / graph_token and act relu / gelu (exact erf), any L >= 0 with dim_in >> L >= 1;
 * Graphormer head with graph_token and dim_in % 4 == 0; 1 <= dim_in, dim_out <= 4096.  Anything else is
 * GPS_ERR_UNSUPPORTED, bad sizes or missing pointers GPS_ERR_ARG, all before any CUDA call.
 * Widths run at the next multiple of 8 with zero pad columns.  Per-graph sums walk each graph's rows in a fixed order
 * (a graph spread over several CTAs is combined from their partials in row order) and the weight gradients take the
 * deterministic split-K path: no float atomics in fp32, two runs give the same bits.  Backward writes grad_x [N, dim_in]
 * whole and every parameter gradient (the head has no dropout and no running statistics: training is not read).
 * ---------------------------------------------------------------------------------------- */
enum { GPS_GRAPH_HEAD_SAN = 0, GPS_GRAPH_HEAD_GRAPHORMER = 1 };
enum { GPS_POOL_MEAN = 0, GPS_POOL_ADD = 1, GPS_POOL_GRAPH_TOKEN = 2 };
#define GPS_GRAPH_HEAD_MAX_L 12 /* dim_in <= 4096 leaves a nonzero width for L <= 12 */

typedef struct {
  int32_t kind;              /* GPS_GRAPH_HEAD_*                                              */
  int32_t pooling;           /* GPS_POOL_*                                                    */
  int32_t act;               /* GPS_ACT_* (SAN head; not read by the Graphormer head)         */
  int32_t L;                 /* hidden layers of the SAN head; 0 for the Graphormer head      */
  int64_t dim_in, dim_out;
  int32_t training;          /* not read                                                      */
  int32_t precision;         /* GPS_PREC_*                                                    */
  int32_t flags;             /* reserved, 0                                                   */
  int32_t reserved;
  uint64_t seed;             /* unused (the head has no dropout)                              */
  GpsGraph graph;            /* N = rows of x, B = graphs, graph_ptr                          */
  const float* x;            /* [N, dim_in]                                                   */
  float* pred;               /* [B, dim_out] (forward)                                        */
  const float* grad_pred;    /* [B, dim_out] (backward)                                       */
  float* grad_x;             /* [N, dim_in] (backward)                                        */
  GpsLinear ln;              /* Graphormer head: ln.weight / ln.bias [dim_in] and their grads */
  GpsLinear fc[GPS_GRAPH_HEAD_MAX_L + 1]; /* FC_layers.{0..L} / layers.0, with their grads    */
  void* saved; int64_t saved_bytes;         /* forward -> backward                            */
  void* workspace; int64_t workspace_bytes; /* transient                                      */
} GpsGraphHeadArgs;

typedef struct {
  int64_t saved_bytes;
  int64_t fwd_workspace_bytes;
  int64_t bwd_workspace_bytes;
} GpsGraphHeadPlan;

/* Sizes for args (only kind, pooling, act, L, the widths, precision and the graph's N and B are read). */
int gps_graph_head_plan(const GpsGraphHeadArgs* args, GpsGraphHeadPlan* plan);
int gps_graph_head_forward(const GpsGraphHeadArgs* args, void* stream);
int gps_graph_head_backward(const GpsGraphHeadArgs* args, void* stream);
/* Stage entries: the pooling alone.  Forward writes out [B, d] at pitch ldo >= d (the columns beyond d are not
 * written); mean and add need a 16-byte aligned workspace >= 8 * ceil(N / 64) * round_up(d, 4) bytes (per-CTA
 * partials), graph_token none.
 * Backward writes grad_x [N, d] whole from grad_out [B, d] at pitch ldg >= d. */
int gps_graph_pool_forward(const GpsGraph* graph, int32_t pooling, const float* x, int64_t d, float* out, int64_t ldo,
                           void* workspace, int64_t workspace_bytes, void* stream);
int gps_graph_pool_backward(const GpsGraph* graph, int32_t pooling, const float* grad_out, int64_t ldg, int64_t d,
                            float* grad_x, void* stream);

/* ------------------------------------------------------------------------------------------
 * Node-prediction heads, the head of every node-level config: GraphGym's MLP (layers_post_mp = L) under
 * graphgps/head/inductive_node.py (GNNInductiveNodeHead) and GraphGym's GNNNodeHead (`node`):
 *   h_0 = x                                                  [N, dim_in]
 *   h_{l+1} = normalize(relu(h_l W_l^T + b_l)), l < L - 1    fc[l]: [dim_inner, dim_in (l = 0) or dim_inner]
 *   y = h_{L-1} W_{L-1}^T + b_{L-1}                          fc[L-1]: [dim_out, dim_in (L = 1) or dim_inner]
 *   pred = y[rows]                                           rows != NULL: M distinct row indices (int64)
 * normalize(r) = r / max(||r||_2, 1e-12) per row (F.normalize(p=2, dim=1), which GraphGym's hidden layers apply).
 * Backward: grad_y (NULL = 0) plus grad_pred (NULL = 0) added into rows; grad_x [N, dim_in] and every parameter
 * gradient written whole.  The normalisation's backward is g_in = (g - h (h.g)) / n for n = ||r|| >= 1e-12 and
 * g / 1e-12 below, times the ReLU mask.  Widths run at the next multiple of 8 with zero pad columns; every product is
 * the TMA GEMM, row sums run in a fixed order and the weight gradients take the deterministic split-K path: two runs
 * give the same bits.  Built: 1 <= L <= GPS_NODE_HEAD_MAX_L, 1 <= dim_in, dim_inner, dim_out <= 4096.  Anything else
 * is GPS_ERR_UNSUPPORTED, bad sizes or missing pointers GPS_ERR_ARG, all before any CUDA call.  Row indices outside
 * [0, N) are never dereferenced.
 * ---------------------------------------------------------------------------------------- */
#define GPS_NODE_HEAD_MAX_L 8

typedef struct {
  int32_t L;                 /* layers_post_mp                                                */
  int32_t precision;         /* GPS_PREC_*                                                    */
  int32_t flags;             /* reserved, 0                                                   */
  int32_t training;          /* not read (the head has no dropout and no running statistics)  */
  uint64_t seed;             /* unused                                                        */
  int64_t dim_in, dim_inner, dim_out;
  int64_t N;                 /* rows of x                                                     */
  int64_t M;                 /* entries of rows (0 without rows)                              */
  const float* x;            /* [N, dim_in]                                                   */
  const int64_t* rows;       /* [M] or NULL                                                   */
  float* y;                  /* [N, dim_out] (forward)                                        */
  float* pred;               /* [M, dim_out] (forward, with rows)                             */
  const float* grad_y;       /* [N, dim_out] or NULL (backward)                               */
  const float* grad_pred;    /* [M, dim_out] or NULL (backward)                               */
  float* grad_x;             /* [N, dim_in] (backward)                                        */
  GpsLinear fc[GPS_NODE_HEAD_MAX_L]; /* the L Linears in order, with their grads             */
  void* saved; int64_t saved_bytes;         /* forward -> backward                            */
  void* workspace; int64_t workspace_bytes; /* transient                                      */
} GpsNodeHeadArgs;

typedef struct {
  int64_t saved_bytes;
  int64_t fwd_workspace_bytes;
  int64_t bwd_workspace_bytes;
} GpsNodeHeadPlan;

/* Sizes for args (only L, the widths, precision and N are read). */
int gps_node_head_plan(const GpsNodeHeadArgs* args, GpsNodeHeadPlan* plan);
int gps_node_head_forward(const GpsNodeHeadArgs* args, void* stream);
int gps_node_head_backward(const GpsNodeHeadArgs* args, void* stream);
/* Stage entries: the row normalisation alone, over rows x d at pitch ld (d % 4 == 0, ld % 4 == 0, ld >= d, d <= 4096,
 * else GPS_ERR_UNSUPPORTED).  Forward: out = r / max(||r||, 1e-12) and norm [rows] = ||r||.  Backward from the forward's
 * out and norm: grad_in = the formula above times the ReLU mask (out > 0).  out may alias r, grad_in may alias g. */
int gps_row_l2norm_forward(const float* r, int64_t rows, int64_t d, int64_t ld, float* out, float* norm, void* stream);
int gps_row_l2norm_backward(const float* g, const float* out, const float* norm, int64_t rows, int64_t d, int64_t ld,
                            float* grad_in, void* stream);

/* The node losses (GraphGym's compute_loss with loss_fun cross_entropy, and graphgps/loss/weighted_cross_entropy.py):
 *   C > 1    pred_score = log_softmax(pred); loss = sum_i w_{y_i} (-pred_score[i, y_i]) / sum_i w_{y_i}
 *   C == 1   pred_score = sigmoid(pred); loss = sum_i w_{y_i} bce(pred_i, y_i) / M   (weighted only)
 * weighted: w_c = (M - count_c) / M * [count_c > 0] in float32 (count_c = labels equal to c, over max(C, 2) classes);
 * otherwise w = 1.  label: int64 [M] in [0, max(C, 2)).  The loss stays on the device (float32 [1]).  Counts use
 * integer atomics; every floating-point sum is fp64 through per-CTA partials added in a fixed order: two runs give
 * the same bits.  A batch whose weights sum to 0 (one class, or M = 0) gives NaN, as torch does.
 * Backward: grad_pred [M, C] from grad_loss (float32 [1], NULL = 0) and grad_score ([M, C], NULL = 0), reading the
 * forward's pred_score and saved buffer.  Built: 1 <= C <= GPS_NODE_LOSS_MAX_C (else GPS_ERR_UNSUPPORTED); C == 1
 * needs weighted. */
#define GPS_NODE_LOSS_MAX_C 4096

typedef struct {
  int64_t M;                 /* rows of pred                                                  */
  int64_t C;                 /* columns of pred; 1 = binary                                   */
  int32_t weighted;          /* 1: weighted_cross_entropy, 0: cross_entropy                   */
  int32_t flags;             /* reserved, 0                                                   */
  const float* pred;         /* [M, C]                                                        */
  const int64_t* label;      /* [M]                                                           */
  float* loss;               /* [1] (forward)                                                 */
  float* pred_score;         /* [M, C] (written by forward, read by backward)                 */
  const float* grad_loss;    /* [1] or NULL (backward)                                        */
  const float* grad_score;   /* [M, C] or NULL (backward)                                     */
  float* grad_pred;          /* [M, C] (backward)                                             */
  void* saved; int64_t saved_bytes;         /* forward -> backward                            */
  void* workspace; int64_t workspace_bytes; /* transient                                      */
} GpsNodeLossArgs;

typedef struct {
  int64_t saved_bytes;
  int64_t fwd_workspace_bytes;
  int64_t bwd_workspace_bytes;
} GpsNodeLossPlan;

/* Sizes for args (only M, C and weighted are read). */
int gps_node_loss_plan(const GpsNodeLossArgs* args, GpsNodeLossPlan* plan);
int gps_node_loss_forward(const GpsNodeLossArgs* args, void* stream);
int gps_node_loss_backward(const GpsNodeLossArgs* args, void* stream);

/* ------------------------------------------------------------------------------------------
 * RWSE, the random-walk structural encoding (graphgps/transform/posenc_stats.py:get_rw_landing_probs and
 * graphgps/encoder/kernel_pos_encoder.py:KernelPENodeEncoder).
 *
 * gps_rwse_landing: out[i, j] = (P^ksteps[j])[i, i] for every node i of `graph`, out [N, nk] float32, with
 * P = D_out^-1 A built from the graph's edges as the reference builds it from edge_index: A[s, d] counts the edges
 * s -> d (duplicates add up, self-loops count), D_out is the out-degree, a node without out-edges has a zero row, and
 * P^0 = I.  P is block-diagonal over the graphs (graph_ptr), so each graph's walks stay inside it.  `ksteps` is a host
 * array of nk values, copied into the launch arguments: any order, repeats and 0 are allowed.  nmax is the size of the
 * largest graph (GraphStructure.nmax).  workspace >= 8 * N bytes, 8-byte aligned (the inverse out-degrees in fp64).
 * Each entry is a fixed-order sum in CSR order, accumulated in fp64 and stored in fp32 after every step: no atomics,
 * two runs give the same bits.  Limits (else GPS_ERR_UNSUPPORTED): 1 <= nk <= GPS_RWSE_MAX_COLS,
 * 0 <= ksteps[j] <= GPS_RWSE_MAX_STEPS, and one walk row of the largest graph fits on chip (nmax <= about 28 000).
 * Bad sizes, missing pointers or a misaligned workspace are GPS_ERR_ARG; both before any CUDA call.
 * ---------------------------------------------------------------------------------------- */
#define GPS_RWSE_MAX_COLS 64
#define GPS_RWSE_MAX_STEPS 256
int gps_rwse_landing(const GpsGraph* graph, const int32_t* ksteps, int32_t nk, int32_t nmax, float* out,
                     void* workspace, int64_t workspace_bytes, void* stream);

/* KernelPENodeEncoder (model "linear"), w = dim_emb - dim_pe:
 *   forward    z = BN(pestat) (batch_norm; the raw statistics otherwise)    pestat [N, K], raw_norm over K columns
 *              out = [h | z Wp^T + bp]                                      out [N, dim_emb]; pe_encoder Wp [dim_pe, K]
 *              h = x Wx^T + bx with expand_x (linear_x Wx [w, dim_in]), else h = x (dim_in == w)
 *   backward   grad_x = g[:, :w] Wx (expand_x) or g[:, :w]; the gradients of Wp, bp, Wx, bx and of the BatchNorm's
 *              weight and bias (pestat is data and gets no gradient)
 * BatchNorm as torch.nn.BatchNorm1d: training normalises by the batch statistics (eps 1e-5) and updates running_mean /
 * running_var (unbiased, momentum 0.1) and num_batches_tracked; eval uses the running statistics.  Every column and
 * weight-gradient sum runs through per-CTA partials added in a fixed order: no float atomics, two runs give the same
 * bits.  Built: 1 <= K <= GPS_RWSE_MAX_COLS, 1 <= dim_pe <= dim_emb <= 4096, 1 <= dim_in <= 4096; training with
 * batch_norm needs N >= 2.  Anything else is GPS_ERR_UNSUPPORTED, bad sizes or missing pointers GPS_ERR_ARG, all
 * before any CUDA call.  Backward writes grad_x and every parameter gradient whole.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  int64_t N;                 /* rows of pestat, x and out                                     */
  int64_t K;                 /* columns of pestat (len(kernel.times))                         */
  int64_t dim_in;            /* columns of x                                                  */
  int64_t dim_emb;           /* columns of out                                                */
  int64_t dim_pe;            /* columns of the encoded statistics                             */
  int32_t expand_x;          /* 1: h = linear_x(x); 0: h = x                                  */
  int32_t batch_norm;        /* 1: raw_norm is a BatchNorm1d(K); 0: none                      */
  int32_t training;          /* BatchNorm: batch statistics and running update (1) or eval (0) */
  int32_t flags;             /* reserved, 0                                                   */
  const float* pestat;       /* [N, K]                                                        */
  const float* x;            /* [N, dim_in]                                                   */
  float* out;                /* [N, dim_emb] (forward)                                        */
  const float* grad_out;     /* [N, dim_emb] (backward)                                       */
  float* grad_x;             /* [N, dim_in] (backward)                                        */
  GpsLinear linear_x;        /* linear_x.weight [w, dim_in] / .bias [w] and grads (expand_x)  */
  GpsLinear pe_encoder;      /* pe_encoder.weight [dim_pe, K] / .bias [dim_pe] and grads      */
  GpsBatchNorm raw_norm;     /* raw_norm.* [K] (batch_norm)                                   */
  void* saved; int64_t saved_bytes;         /* forward -> backward                            */
  void* workspace; int64_t workspace_bytes; /* transient                                      */
} GpsKernelPeArgs;

typedef struct {
  int64_t saved_bytes;
  int64_t fwd_workspace_bytes;
  int64_t bwd_workspace_bytes;
} GpsKernelPePlan;

/* Sizes for args (only N, K, the widths, expand_x, batch_norm and training are read). */
int gps_kernel_pe_plan(const GpsKernelPeArgs* args, GpsKernelPePlan* plan);
int gps_kernel_pe_forward(const GpsKernelPeArgs* args, void* stream);
int gps_kernel_pe_backward(const GpsKernelPeArgs* args, void* stream);

/* ------------------------------------------------------------------------------------------
 * SAN layer (graphgps/layer/san_layer.py:10-210), the building block of SANTransformer, as every shipped config runs
 * it (full_graph, batch_norm, residual, no layer_norm, no Linear biases in the attention, in_dim == out_dim == d):
 *   [Q|K|V|Q2|K2] = x W^T, E = edge_attr W_E^T, E2 = W_E2 fake_edge_emb
 *   attn = sum over real edges j->i and fake pairs of s V[j] / (sum s + 1e-6), per head of hd = d / heads channels:
 *     real edge k: s = exp(clamp(sum_c K[j] Q[i] E[k] / sqrt(hd), -5, 5)) / (gamma + 1)   (per edge: duplicates count
 *                  twice, self loops are real edges)
 *     fake pair:   s = gamma exp(clamp(sum_c K2[j] Q2[i] E2 / sqrt(hd), -5, 5)) / (gamma + 1), for every j != i of i's
 *                  graph without a real edge j -> i
 *   h1  = BN1(x + O_h(drop_13(attn)))                     dropout site 13
 *   out = BN2(h1 + FFN2(drop_14(relu(FFN1(h1)))))         dropout site 14, FFN1 [2d, d], FFN2 [d, 2d]
 * d % heads != 0 is GPS_ERR_ARG; d % 4 == 0, d <= 4096 and hd <= 192, else GPS_ERR_UNSUPPORTED.  nmax is the size of
 * the largest graph of the batch (to_dense_batch's Nmax); the exclusion bitmap is [N, ceil(nmax / 32)] words of saved
 * memory.  Parameters (weights non-NULL, else GPS_ERR_ARG): Q, K, V, Q2, K2, E, E2 = attention.{Q,K,V,Q_2,K_2,E,E_2}
 * [d, d], bias NULL; O_h [d, d], ffn1, ffn2 with biases; bn1, bn2 = batch_norm{1,2}_h with running statistics (updated
 * in training mode as torch.nn.BatchNorm1d, momentum 0.1); fake_edge_emb [d] (attention.fake_edge_emb.weight, one row).
 * Backward writes grad_x, grad_edge_attr (NULL = not needed), every non-NULL parameter gradient and
 * grad_fake_edge_emb; the weight products run on a side stream that joins the caller's stream before the call
 * returns.  When Q..K2's grad_weight buffers are consecutive [5d, d] (K = Q + d*d, ...) they take one product.  No
 * float atomics: two runs give the same bits.
 *
 * variant 1 is SAN2Layer (graphgps/layer/san2_layer.py, the same trunk): the attention is a softmax (running max, no
 * clamp) taken separately over the real in-edges and over the fake pairs of each destination, mixed by the learned
 * float64 gamma = *gamma_param, read on the device by the kernels (an optimiser step or a CUDA-graph replay sees the
 * current value):
 *     real edge k: alpha = softmax over i's real in-edges of sum_c K[j] Q[i] E[k] / sqrt(hd)       (+1e-16 in the sum)
 *     fake pair:   beta  = softmax over i's fake pairs of sum_c K2[j] Q2[i] E2 / sqrt(hd)           (+1e-16 in the sum)
 *     attn[i] = (sum alpha V[j] + gamma sum beta V[j]) / (gamma + 1)      (an empty set contributes 0)
 * The gamma field is not read; gamma_param is required (GPS_ERR_ARG); backward writes *grad_gamma (added with
 * GPS_FLAG_GRADS_ACCUMULATE), reduced in float64 in a fixed order.  Any other variant is GPS_ERR_UNSUPPORTED.  All
 * these checks happen before any CUDA call.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  int64_t d;                 /* in_dim == out_dim                                              */
  int64_t heads;             /* num_heads                                                      */
  int32_t training;          /* 1: batch statistics and dropout; 0: running statistics         */
  int32_t precision;         /* GPS_PREC_*                                                     */
  float gamma;               /* cfg.gt.gamma, a constant (variant 0; not read by variant 1)    */
  float dropout;             /* sites 13 and 14                                                */
  int32_t flags;             /* GPS_FLAG_* (backward), as GpsLayerArgs.flags                   */
  int32_t variant;           /* 0: SANLayer; 1: SAN2Layer (softmax attention, learned gamma)   */
  uint64_t seed;             /* Philox key of this call's dropout masks                       */
  uint64_t offset;           /* Philox counter base                                            */
  const uint64_t* offset_dev;/* optional device-resident addend to offset (CUDA-graph replays); NULL = none */
  GpsGraph graph;
  int64_t nmax;              /* largest graph of the batch                                     */
  const float* x;            /* [N, d] batch.x                                                 */
  const float* edge_attr;    /* [E, d] batch.edge_attr (non-NULL when E > 0)                   */
  float* x_out;              /* [N, d] new batch.x (forward)                                   */
  const float* grad_x_out;   /* [N, d] (backward)                                              */
  float* grad_x;             /* [N, d] (backward)                                              */
  float* grad_edge_attr;     /* [E, d] (backward, NULL = not needed)                           */
  void* saved; int64_t saved_bytes;         /* written by forward, read by backward            */
  void* workspace; int64_t workspace_bytes; /* transient                                       */
  GpsLinear Q, K, V, Q2, K2, E, E2, O_h, ffn1, ffn2;
  GpsBatchNorm bn1, bn2;
  const float* fake_edge_emb;
  float* grad_fake_edge_emb;
  const double* gamma_param; /* variant 1: attention.gamma, one float64 on the device, read by the kernels */
  double* grad_gamma;        /* variant 1 (backward): its gradient, one float64 (NULL = not needed)       */
} GpsSanArgs;

typedef struct {
  int64_t saved_bytes;
  int64_t fwd_workspace_bytes;
  int64_t bwd_workspace_bytes;
} GpsSanPlan;

/* Sizes for the configuration and graph of args (only d, heads, precision, training, dropout, gamma, variant, nmax
 * and graph.N / graph.E / graph.B are read). */
int gps_san_plan(const GpsSanArgs* args, GpsSanPlan* plan);
int gps_san_forward(const GpsSanArgs* args, void* stream);
int gps_san_backward(const GpsSanArgs* args, void* stream);

/* ------------------------------------------------------------------------------------------
 * The message-passing layers of CustomGNN (graphgps/network/custom_gnn.py:31-37), standalone as the LRGB GatedGCN and
 * GINE configs stack them, in_dim == out_dim == d:
 *   GPS_CUSTOM_GATEDGCN  GatedGCNLayer (gatedgcn_layer.py:11-136, no EquivStableLapPE gate):
 *       [Ax|Bx|Dx|Ex] = x W^T + b, Ce = edge_attr C^T + bC, e_ij = Dx_i + Ex_j + Ce, sigma = sigmoid(e_ij),
 *       xt = Ax + sum sigma Bx_j / (sum sigma + 1e-6)
 *       x_out = [x +] drop_15(act(bn_node_x(xt))),  edge_out = [edge_attr +] drop_4095(act(bn_edge_e(e_ij)))
 *   GPS_CUSTOM_GINE      GINEConvLayer (gine_conv_layer.py:90-116), GINEConv(nn.0, ReLU, nn.2) with eps = gine_eps:
 *       x_out = [x +] drop_15(relu(nn.2(relu(nn.0((1 + eps) x + sum_j relu(x_j + e_ij))))))
 * [..] only with residual != 0; dropout sites 15 and 4095.  Any 1 <= d <= 4096 (else GPS_ERR_UNSUPPORTED): at
 * d % 8 != 0 every intermediate runs at the pitch dp = round_up(d, 8) with zero pad columns, and the inputs, outputs,
 * running statistics and gradients cross the call at pitch d.  Parameters (all non-NULL, else GPS_ERR_ARG): GatedGCN
 * A..E [d, d] with biases, bn_node_x / bn_edge_e with running statistics (updated in training mode as
 * torch.nn.BatchNorm1d, momentum 0.1); GINE nn0 = model.nn.0, nn2 = model.nn.2 [d, d] with biases.  wplanes: a
 * caller-owned buffer (GpsCustomGnnPlan.wplanes_bytes) for the padded weight planes, biases and BatchNorm affine
 * parameters; wplanes_valid != 0: it already holds them for the current parameters (packed once per optimiser step);
 * the backward always reads it as the forward left it.  Backward writes grad_x, grad_edge_attr (NULL = not needed) and
 * every non-NULL parameter gradient; grad_edge_out NULL = zero (GatedGCN).  The weight products run on a side stream
 * that joins the caller's stream before the call returns.  Every width runs the same kernels at a pitch that is a
 * multiple of 8, where the weight products take the deterministic split-K path: two runs give the same bits.
 * ---------------------------------------------------------------------------------------- */
enum { GPS_CUSTOM_GATEDGCN = 0, GPS_CUSTOM_GINE = 1 };
typedef struct {
  int64_t d;                 /* in_dim == out_dim                                              */
  int32_t kind;              /* GPS_CUSTOM_*                                                   */
  int32_t act;               /* GatedGCN: GPS_ACT_RELU / GPS_ACT_GELU; GINE: ReLU, not read     */
  int32_t training;          /* 1: batch statistics and dropout; 0: running statistics         */
  int32_t precision;         /* GPS_PREC_*                                                     */
  int32_t residual;          /* 1: add the layer's input to its output(s)                      */
  int32_t flags;             /* reserved, 0                                                    */
  float dropout;             /* sites 15 (node output) and 4095 (GatedGCN edge output)         */
  float gine_eps;            /* model.eps buffer value (GINE)                                  */
  uint64_t seed;             /* Philox key of this call's dropout masks                       */
  uint64_t offset;           /* Philox counter base                                            */
  const uint64_t* offset_dev;/* optional device-resident addend to offset (CUDA-graph replays); NULL = none */
  GpsGraph graph;
  const float* x;            /* [N, d] batch.x                                                 */
  const float* edge_attr;    /* [E, d] batch.edge_attr (non-NULL when E > 0)                   */
  float* x_out;              /* [N, d] new batch.x (forward)                                   */
  float* edge_out;           /* [E, d] new batch.edge_attr (forward, GatedGCN)                 */
  const float* grad_x_out;   /* [N, d] (backward)                                              */
  const float* grad_edge_out;/* [E, d] (backward, GatedGCN; NULL = zero)                       */
  float* grad_x;             /* [N, d] (backward)                                              */
  float* grad_edge_attr;     /* [E, d] (backward, NULL = not needed)                           */
  void* saved; int64_t saved_bytes;         /* written by forward, read by backward            */
  void* workspace; int64_t workspace_bytes; /* transient                                       */
  void* wplanes; int64_t wplanes_bytes; int32_t wplanes_valid; int32_t reserved;
  GpsLinear A, B, C, D, E;   /* GatedGCN                                                        */
  GpsBatchNorm bn_node_x, bn_edge_e;
  GpsLinear nn0, nn2;        /* GINE                                                            */
} GpsCustomGnnArgs;

typedef struct {
  int64_t saved_bytes;
  int64_t fwd_workspace_bytes;
  int64_t bwd_workspace_bytes;
  int64_t wplanes_bytes;
} GpsCustomGnnPlan;

/* Sizes for the configuration and graph of args (only d, kind, act, precision, training, residual, dropout, flags and
 * graph.N / graph.E / graph.B are read). */
int gps_custom_gnn_plan(const GpsCustomGnnArgs* args, GpsCustomGnnPlan* plan);
int gps_custom_gnn_forward(const GpsCustomGnnArgs* args, void* stream);
int gps_custom_gnn_backward(const GpsCustomGnnArgs* args, void* stream);

/* SAN attention stage (the kernels the layer calls).  Y [N, ld] holds the column blocks Q | K | V | Q2 | K2 (each
 * heads * hd wide, ld >= 5 heads hd); E [E, heads * hd] the edge projection in edge-id order; E2 [heads * hd] the
 * projected fake-edge embedding.  Forward: O [N, ldo] = the attention output, rz [N, heads] = 1 / (Z + 1e-6).
 * Backward from dO: dY [N, ldg] = the gradients of the five blocks (dQ2 with respect to Q2 itself), dE [E, heads * hd]
 * and dE2 [heads * hd], all written.  workspace: gps_san_attention_workspace_bytes.  Bad arguments are GPS_ERR_ARG (or
 * GPS_ERR_UNSUPPORTED for the shape limits of the layer) before any CUDA call. */
int64_t gps_san_attention_workspace_bytes(int64_t N, int64_t d, int64_t heads, int64_t nmax);
int gps_san_attention_forward(const GpsGraph* g, int64_t heads, int64_t hd, const float* Y, int64_t ld, const float* E,
                              const float* E2, float gamma, int64_t nmax, void* workspace, int64_t workspace_bytes,
                              float* O, int64_t ldo, float* rz, void* stream);
int gps_san_attention_backward(const GpsGraph* g, int64_t heads, int64_t hd, const float* Y, int64_t ld,
                               const float* E, const float* E2, float gamma, int64_t nmax, void* workspace,
                               int64_t workspace_bytes, const float* O, const float* dO, int64_t ldo, const float* rz,
                               float* dY, int64_t ldg, float* dE, float* dE2, void* stream);

/* SAN2 attention stage (variant 1 of the layer), arguments as the SAN stage but with gamma one float64 on the device.
 * Forward: O [N, ldo] = the attention output, R and F [N, heads * hd] = the unscaled real-edge and fake-pair softmax
 * outputs (sum alpha V, sum beta V), lse [2, N, heads] = their log-sum-exps (real, then fake).  Backward from dO and
 * the forward's R, F and lse: dY, dE, dE2 as the SAN stage, and *dgamma (float64), all written. */
int64_t gps_san2_attention_workspace_bytes(int64_t N, int64_t d, int64_t heads, int64_t nmax);
int gps_san2_attention_forward(const GpsGraph* g, int64_t heads, int64_t hd, const float* Y, int64_t ld,
                               const float* E, const float* E2, const double* gamma, int64_t nmax, void* workspace,
                               int64_t workspace_bytes, float* O, int64_t ldo, float* R, float* F, float* lse,
                               void* stream);
int gps_san2_attention_backward(const GpsGraph* g, int64_t heads, int64_t hd, const float* Y, int64_t ld,
                                const float* E, const float* E2, const double* gamma, int64_t nmax, void* workspace,
                                int64_t workspace_bytes, const float* R, const float* F, const float* lse,
                                const float* dO, int64_t ldo, float* dY, int64_t ldg, float* dE, float* dE2,
                                double* dgamma, void* stream);

/* ------------------------------------------------------------------------------------------
 * Stage-level entry points (the same kernels the layer calls; exported so the parity tests can
 * pin each stage against the oracle separately).
 * ---------------------------------------------------------------------------------------- */

/* C[M,N] = A[M,K] · W[N,K]ᵀ + bias  — replaces pyg_nn.Linear / nn.Linear (gatedgcn_layer.py:57-61,
 * gps_layer.py:253-257).  precision selects the tensor-core path (GPS_PREC_*). */
int gps_linear_forward(const float* A, int64_t lda, const float* W, int64_t ldw, const float* bias,
                       float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, int32_t act,
                       int32_t precision, void* stream);

/* General dense product used for the data / weight gradients of every Linear:
 *   C[M,N] (+)= Aop[M,K] * Bop[K,N];  ta==0: Aop[m,k]=A[m*lda+k], ta==1: Aop[m,k]=A[k*lda+m];
 *   tb==0: Bop[k,n]=B[n*ldb+k] (an nn.Linear weight), tb==1: Bop[k,n]=B[k*ldb+n].
 * splitk > 1 accumulates into a pre-zeroed C (one adder per element: the same result in every run).  impl: 0 = dispatcher (tensor cores when the
 * shape qualifies), 1 = exact CUDA-core kernel, 2 = tensor-core kernel (GPS_ERR_UNSUPPORTED if it does
 * not take the shape). */
int gps_gemm(const float* A, int64_t lda, int32_t ta, const float* B, int64_t ldb, int32_t tb, float* C,
             int64_t ldc, int64_t M, int64_t N, int64_t K, int32_t splitk, int32_t precision, int32_t impl,
             void* stream);

/* GatedGCN message+aggregate+update (gatedgcn_layer.py:90-136) given the five projections.
 * Y holds [Ax | Bx | Dx | Ex] columns at the given offsets with row stride ldy; Ce [E,d] is
 * overwritten with e_ij (pre-activation edge output, :106,:134); xt [N,d] = Ax + num/(den+1e-6).
 * stats_x/stats_e: optional double [2][d] column sum / sum of squares accumulators (BatchNorm). */
int gps_gatedgcn_aggregate_forward(const GpsGraph* g, int64_t d, const float* Ax, const float* Bx,
                                   const float* Dx, const float* Ex, int64_t ldy, float* Ce,
                                   float* xt, double* stats_x, double* stats_e, void* stream);

/* GINE aggregate: out_i = (1+eps)·x_i + Σ_{j→i} relu(x_j + e_ij)  (gine_conv_layer.py:56-84) */
int gps_gine_aggregate_forward(const GpsGraph* g, int64_t d, const float* x, const float* e,
                               float eps, float* out, void* stream);

/* The stage entry points below take d > 0, d % 4 == 0, d <= 4096 (else GPS_ERR_UNSUPPORTED) and validate every pointer
 * they read or write before any CUDA call (GPS_ERR_ARG); pointers that only edges use may be NULL when E == 0. */
/* as gps_gatedgcn_aggregate_forward, plus rho [E] (NULL = no gate): sigma_ij = sigmoid(e_ij) * rho_e
 * (EquivStableLapPE, gatedgcn_layer.py:101-104) */
int gps_gatedgcn_aggregate_forward_gated(const GpsGraph* g, int64_t d, const float* Ax, const float* Bx,
                                         const float* Dx, const float* Ex, int64_t ldy, float* Ce, float* xt,
                                         double* stats_x, double* stats_e, const float* rho, void* stream);
/* backward of the above: the dst-ordered pass, then the src-ordered pass.  gY [N, ldg] holds the column blocks
 * [g_Ax | g_Bx | g_Dx | g_Ex]: block 0 holds g_xt on entry and is only read; blocks 1..3 are written.  g_e [E,d] holds
 * the BN_e-path gradient on entry and the total gradient of e_ij on exit.  g_num [N,d] is written; g_den [N,d] is written
 * when rho != NULL.  gY_planes (4d columns) / g_e_planes: optional bf16 hi/lo images of gY blocks 1..3 / g_e (hi NULL
 * = none). */
int gps_gatedgcn_aggregate_backward(const GpsGraph* g, int64_t d, const float* ehat, const float* Bx, int64_t ldy,
                                    const float* rho, float* gY, int64_t ldg, float* g_e, float* g_num, float* g_den,
                                    const GpsPlanes* gY_planes, const GpsPlanes* g_e_planes, void* stream);
/* EquivStableLapPE gate (gatedgcn_layer.py:29-35,101-104): r [E] = |pe_i - pe_j|^2, rho [E] = mlp_r_ij(r); pe [N,k],
 * w1 = mlp_r_ij.0.weight [d,1], b1 [d], w2 = mlp_r_ij.2.weight [1,d], b2 [1]; act GPS_ACT_* */
int gps_eslap_forward(const GpsGraph* g, const float* pe, int64_t k, int64_t d, int32_t act, const float* w1,
                      const float* b1, const float* w2, const float* b2, float* r, float* rho, void* stream);
/* bytes of scratch gps_eslap_backward needs */
int64_t gps_eslap_workspace_bytes(int64_t E, int64_t d);
/* its backward, after gps_gatedgcn_aggregate_backward with rho: grad_pe [N,k] (NULL = not needed) and the mlp_r_ij
 * gradients (each NULL = not needed), written, or added to when accumulate != 0 */
int gps_eslap_backward(const GpsGraph* g, const float* pe, int64_t k, int64_t d, int32_t act, const float* g_num,
                       const float* g_den, const float* Bx, int64_t ldy, const float* ehat, const float* r,
                       const float* rho, const float* w1, const float* b1, const float* w2, void* workspace,
                       int64_t workspace_bytes, float* grad_pe, float* gw1, float* gb1, float* gw2, float* gb2,
                       int32_t accumulate, void* stream);
/* backward of gps_gine_aggregate_forward: g_e [E,d] = g_out[dst] * [x_src + e > 0],
 * g_x [N,d] = (1+eps) g_out + sum over out-edges of g_e (+ add [N,d], NULL = none) */
int gps_gine_aggregate_backward(const GpsGraph* g, int64_t d, const float* x, const float* e, const float* g_out,
                                float eps, const float* add, float* g_e, float* g_x, void* stream);
/* GCN aggregation (gps_layer.py:49-51): dinv [N] = (1 + #non-self in-edges)^-1/2, then
 * xloc = x + dropout(bias + A_hat Y) with the layer's local dropout site and (seed, offset) (gps_dropout_mask site 3);
 * stats: optional double [2][d] column sums of xloc.  Y [N, ldy]. */
int gps_gcn_aggregate_forward(const GpsGraph* g, int64_t d, const float* Y, int64_t ldy, const float* bias,
                              const float* x, float* dinv, float* xloc, float p_drop, uint64_t seed, uint64_t offset,
                              double* stats, void* stream);
/* its backward: gY [N, ldg] = A_hat^T g_h (+ optional bf16 hi/lo planes of it) */
int gps_gcn_aggregate_backward(const GpsGraph* g, int64_t d, const float* g_h, const float* dinv, float* gY,
                               int64_t ldg, const GpsPlanes* gY_planes, void* stream);

/* GAT stage entry points (the functions the GAT layer calls).  H > 0 with d % H == 0 and d % 4 == 0, d <= 4096 (else
 * GPS_ERR_UNSUPPORTED; d % H != 0 is GPS_ERR_ARG); NULL pointers are GPS_ERR_ARG; both before any CUDA call.  C = d / H.
 * fold: v [H, d] = W_edge[hC:(h+1)C, :]^T att_edge[h] (W_edge = lin_edge.weight [d,d], att_edge [H*C]); its backward
 * writes (accumulate != 0: adds) g_W_edge [d,d] and g_att_edge [H*C] from g_v [H, d] (either output may be NULL). */
int gps_gat_fold_forward(const float* W_edge, const float* att_edge, int64_t d, int64_t H, float* v, void* stream);
int gps_gat_fold_backward(const float* W_edge, const float* att_edge, const float* g_v, int64_t d, int64_t H,
                          float* g_W_edge, float* g_att_edge, int32_t accumulate, void* stream);
/* xloc [N,d] = x + dropout(GATConv aggregation of Y + bias) with the local dropout site (gps_dropout_mask site 3);
 * Y [N, ldy] (ldy % 4 == 0) = x lin_src^T; edge_attr [E,d]; v from the fold; stats: optional double [2][d] column sums
 * of xloc.  scores: (4N + E) H floats written: a_src, a_dst, a_self (the added loop's edge score), lse (log-sum-exp of
 * each (node, head) softmax), each [N, H], then a_edge [E, H] in edge-id order. */
int gps_gat_forward(const GpsGraph* g, int64_t d, int64_t H, const float* Y, int64_t ldy, const float* edge_attr,
                    const float* v, const float* att_src, const float* att_dst, const float* bias, const float* x,
                    float* scores, float* xloc, float p_drop, uint64_t seed, uint64_t offset, double* stats,
                    void* stream);
/* bytes of scratch gps_gat_backward needs */
int64_t gps_gat_workspace_bytes(int64_t N, int64_t E, int64_t H, int64_t d);
/* its backward from g_h [N,d] (the gradient of the aggregation output, i.e. of GATConv's output): gY [N, ldg]
 * (+ optional bf16 planes), grad_edge_attr [E,d] (NULL = not needed), g_v [H,d], all written; g_att_src / g_att_dst /
 * g_bias [d] written, or added when accumulate != 0 (each NULL = not needed). */
int gps_gat_backward(const GpsGraph* g, int64_t d, int64_t H, const float* Y, int64_t ldy, const float* edge_attr,
                     const float* v, const float* att_src, const float* att_dst, const float* scores, const float* g_h,
                     void* workspace, int64_t workspace_bytes, float* gY, int64_t ldg, const GpsPlanes* gY_planes,
                     float* grad_edge_attr, float* g_v, float* g_att_src, float* g_att_dst, float* g_bias,
                     int32_t accumulate, void* stream);

/* GENConv stage entry points (the kernels the GENConv layer calls around its MLP).  x, e [E,d] (NULL when E == 0).
 * Forward: agg [N,d] = the softmax aggregation of the messages relu(x_src + e) + 1e-7, lse [N,d] = each (node, channel)
 * segment's log-sum-exp (0 for a node without in-edges), u [N,d] = agg + x.
 * Backward from g_u [N,d] (the gradient of u): g_e [E,d] = g_u[dst] alpha (1 + m - agg[dst]) [x_src + e > 0] (NULL
 * when E == 0), g_x [N,d] = g_u + sum over out-edges of g_e (+ add [N,d], NULL = none). */
int gps_genconv_aggregate_forward(const GpsGraph* g, int64_t d, const float* x, const float* e, float* agg, float* lse,
                                  float* u, void* stream);
int gps_genconv_aggregate_backward(const GpsGraph* g, int64_t d, const float* x, const float* e, const float* agg,
                                   const float* lse, const float* g_u, const float* add, float* g_e, float* g_x,
                                   void* stream);

/* PNA stage entry points (the kernels the PNA layer calls between its dense products).  W_e is the column block
 * 2d..3d of pre_w [d, 3d]; de = edge_dim (0 < de <= d, de % 4 == 0, else GPS_ERR_UNSUPPORTED).
 * Fold: F [d, de] = W_e enc_w, c [d] = W_e enc_b + pre_b, so that pre's edge term is e F^T + c.
 * Fold backward from g_F [d, de] and g_c [d]: the gradients of pre_w's block 2d..3d (the other blocks are not
 * touched), pre_b, enc_w [d, de] and enc_b, written, or added when accumulate != 0 (each NULL = not needed).
 * Aggregate forward: m_k = Y[i, 0:d] + Y[j, d:2d] + q[k] for edge k from j to i (Y [N, ldy], q [E, d], NULL when
 * E == 0); Z [N, 4d] = [x | mean | max | sum] of m over each node's in-edges (0 without any), arg [N, d] int32 = edge
 * id of the first maximiser (-1 without in-edges).
 * Aggregate backward from g_Z [N, 4d]: g_q [E, d] (g_m of every edge), gY[:, 0:d] = the sum of g_m over in-edges,
 * gY[:, d:2d] = the sum of g_m over out-edges (gY [N, ldg], ldg >= 2d), g_x [N, d] = g_Z[:, 0:d] (+ add, NULL =
 * none). */
int gps_pna_fold_forward(const float* pre_w, const float* pre_b, const float* enc_w, const float* enc_b, int64_t d,
                         int64_t de, float* F, float* c, void* stream);
int gps_pna_fold_backward(const float* pre_w, const float* enc_w, const float* enc_b, const float* g_F,
                          const float* g_c, int64_t d, int64_t de, float* grad_pre_w, float* grad_pre_b,
                          float* grad_enc_w, float* grad_enc_b, int32_t accumulate, void* stream);
int gps_pna_aggregate_forward(const GpsGraph* g, int64_t d, const float* x, const float* Y, int64_t ldy,
                              const float* q, float* Z, int32_t* arg, void* stream);
int gps_pna_aggregate_backward(const GpsGraph* g, int64_t d, const float* g_Z, const int32_t* arg, const float* add,
                               float* g_q, float* gY, int64_t ldg, float* g_x, void* stream);

/* Performer stage entry points (FAVOR+, performer_layer.py:119-144,200-205), the calls one layer makes, in order.
 * They take dim_head == 64 and 256 < m <= 272 features (else GPS_ERR_UNSUPPORTED), H > 0 and N * H * 272 < 2^31 (else
 * GPS_ERR_UNSUPPORTED), and reject NULL pointers with GPS_ERR_ARG, before any CUDA call.  Layout: a (node, head) row
 * r = n * H + h; Q, K, V, O [N*H, 64]; feature maps [N*H, 272] with columns m..271 zero; gmax, ggmax, argk [B*H];
 * argq, den, gden, gmrow [N*H].  form: 0 = per-graph context, 1 = pairwise; either runs on any batch. */
/* P [m, 64] -> Pn [272, 64] = 64^-1/4 P padded with zero rows; nmax [1] = max graph size; gmax = 0 for graphs with
 * padded rows of the dense batch (n < nmax), else -inf; argk = INT_MAX */
int gps_performer_prep(const GpsGraph* g, int64_t H, int64_t dim_head, int64_t m, const float* P, float* Pn, int* nmax,
                       float* gmax, int* argk, void* stream);
/* fq / fk hold dd = x Pn^T on entry (only columns < m are read) and the feature maps q', k' on exit; gmax: key max
 * per (graph, head) (prep's value on entry); argq: per-row arg-max feature; argk: flat arg-max r * 272 + j, INT_MAX
 * when the max is a padded row's 0.  Ties go to the lowest index. */
int gps_performer_features_forward(const GpsGraph* g, int64_t H, int64_t dim_head, int64_t m, float* fq, float* fk,
                                   const float* Q, const float* K, float* gmax, int* argq, int* argk, void* stream);
/* O = (q' . sum k'^T v) / den, den = q' . (sum k' + (nmax - n) k'_pad); den written by the pairwise form only */
int gps_performer_attention_forward(const GpsGraph* g, int64_t H, int64_t dim_head, int64_t m, int32_t form,
                                    const int* nmax, const float* qf, const float* kf, const float* V,
                                    const float* gmax, float* O, float* den, void* stream);
/* its backward from gO: g_qf, g_kf (all 272 columns), gV, and the gradient of gmax through k'_pad: the context form
 * writes it per (graph, head) to ggmax; the pairwise form writes each query row's share to gmrow (and gden; O, den from
 * its forward) */
int gps_performer_attention_backward(const GpsGraph* g, int64_t H, int64_t dim_head, int64_t m, int32_t form,
                                     const int* nmax, const float* qf, const float* kf, const float* V,
                                     const float* gmax, const float* O, const float* den, const float* gO, float* gden,
                                     float* g_qf, float* g_kf, float* gV, float* ggmax, float* gmrow, void* stream);
/* backward of gps_performer_features_forward: g_fq / g_fk hold the feature-map gradients on entry (columns < m read)
 * and the gradients of dd on exit; gQ / gK [N*H, 64] = the gradients through diag (written).  The upstream gradient
 * of gmax is ggmax (form 0) or the per-(graph, head) sum of gmrow (form 1); gmrow is overwritten. */
int gps_performer_features_backward(const GpsGraph* g, int64_t H, int64_t dim_head, int64_t m, int32_t form,
                                    float* g_fq, float* g_fk, const float* fq, const float* fk, const float* Q,
                                    const float* K, float* gQ, float* gK, const int* argq, const int* argk,
                                    const float* ggmax, float* gmrow, void* stream);

/* Dense softmax attention over each graph's own nodes — replaces to_dense_batch +
 * nn.MultiheadAttention core + [mask] (gps_layer.py:199-201,234-241) without padding.
 * Q,K,V: [N, heads*hd] slices with row stride ld; O [N, heads*hd] (row stride ldo); lse [N,heads].  Any head dim
 * 1 <= hd <= 192 (else GPS_ERR_UNSUPPORTED); float4 kernels when hd and the leading dimensions are multiples of 4. */
int gps_attention_forward(const GpsGraph* g, int64_t heads, int64_t hd, const float* Q,
                          const float* K, const float* V, int64_t ld, float* O, int64_t ldo,
                          float* lse, float p_drop, uint64_t seed, uint64_t offset, void* stream);
/* The same forward on the tensor cores (csrc/attention_tc.cu: wgmma S = QK^T and O += PV, TMA-staged tiles,
 * block-diagonal graph mask applied in-kernel).  qkv_hi/qkv_lo: bf16 hi/lo planes [N, ld] holding Q | K | V per head in
 * the padded layout column (which * heads + h) * hd_pad + k with hd_pad = round_up(hd, 16) and zero pad columns
 * (qkv_lo NULL for GPS_PREC_BF16).  Same O / lse conventions as gps_attention_forward, so either backward applies. */
int gps_attention_forward_tc(const GpsGraph* g, int64_t heads, int64_t hd, const void* qkv_hi, const void* qkv_lo,
                             int64_t ld, float* O, int64_t ldo, float* lse, float p_drop, uint64_t seed,
                             uint64_t offset, int32_t precision, void* stream);
/* (the layer-level calls additionally honour GpsLayerArgs.offset_dev) */
int gps_attention_backward(const GpsGraph* g, int64_t heads, int64_t hd, const float* Q,
                           const float* K, const float* V, int64_t ld, const float* O,
                           const float* dO, int64_t ldo, const float* lse, float* delta,
                           float* dQ, float* dK, float* dV, int64_t ldg, float p_drop,
                           uint64_t seed, uint64_t offset, void* stream);
/* The three attention stages with a GpsAttnBias (non-NULL, nmax >= 1, bias->bias != NULL, else GPS_ERR_ARG); the
 * backward writes bias->grad_bias when it is not NULL.  Other arguments as above. */
int gps_attention_forward_biased(const GpsGraph* g, int64_t heads, int64_t hd, const float* Q, const float* K,
                                 const float* V, int64_t ld, float* O, int64_t ldo, float* lse, float p_drop,
                                 uint64_t seed, uint64_t offset, const GpsAttnBias* bias, void* stream);
int gps_attention_forward_tc_biased(const GpsGraph* g, int64_t heads, int64_t hd, const void* qkv_hi,
                                    const void* qkv_lo, int64_t ld, float* O, int64_t ldo, float* lse, float p_drop,
                                    uint64_t seed, uint64_t offset, int32_t precision, const GpsAttnBias* bias,
                                    void* stream);
int gps_attention_backward_biased(const GpsGraph* g, int64_t heads, int64_t hd, const float* Q, const float* K,
                                  const float* V, int64_t ld, const float* O, const float* dO, int64_t ldo,
                                  const float* lse, float* delta, float* dQ, float* dK, float* dV, int64_t ldg,
                                  float p_drop, uint64_t seed, uint64_t offset, const GpsAttnBias* bias, void* stream);
/* One softmax-attention stage with every field the layers pass, so each can be tested alone.  The six entry points
 * above are this call with the fields they do not take left zero; all seven share one argument contract.
 *   FWD     CUDA-core forward: O, lse from Q, K, V (pitch ld) [+ O_planes]
 *   FWD_TC  wgmma forward: O, lse from the qkv planes in the per-head padded layout (gps_attention_forward_tc)
 *           [+ O_planes]; precision GPS_PREC_FP32 reads qkv.lo, GPS_PREC_BF16 ignores it
 *   BWD     delta, dQ, dK, dV (pitch ldg) [+ their planes] from Q, K, V, O, dO (pitch ldo), lse; bias->grad_bias
 *           written whole when given
 * bias NULL = unbiased.  Dropout on the probabilities draws Philox site 16 + head at offset + *offset_dev (offset_dev
 * NULL: + 0).  GPS_ERR_ARG, before any CUDA call: NULL args, an unknown op, a negative N or B, N > 0 with B < 1 or no
 * graph_ptr, heads < 1, a NULL tensor the op reads or writes, ld / ldo / ldg below heads * hd (the op's pitches), an
 * output plane pitch below heads * hd or a qkv plane pitch below 3 * heads * hd_pad, lo planes without hi, precision
 * other than GPS_PREC_FP32 / GPS_PREC_BF16, p_drop outside [0, 1) or NaN, a bias with bias->bias NULL or nmax < 1.
 * GPS_ERR_UNSUPPORTED: hd outside 1..192 (FWD_TC: not a multiple of 4 or above 128), a plane pitch that is not a
 * multiple of 8, and FWD_TC in GPS_PREC_FP32 without qkv.lo. */
enum { GPS_ATTN_FWD = 0, GPS_ATTN_FWD_TC = 1, GPS_ATTN_BWD = 2 };
typedef struct {
  GpsGraph graph;
  int64_t heads, hd;
  const float* Q; const float* K; const float* V; int64_t ld;
  GpsPlanes qkv; int32_t precision, reserved;
  float* O; int64_t ldo;
  GpsPlanes O_planes;
  float* lse;
  const float* dO; float* delta;
  float* dQ; float* dK; float* dV; int64_t ldg;
  GpsPlanes dQ_planes, dK_planes, dV_planes;
  const GpsAttnBias* bias;
  float p_drop; int32_t reserved2;
  uint64_t seed, offset;
  const unsigned long long* offset_dev;
} GpsAttnStageArgs;
int gps_attention_stage(const GpsAttnStageArgs* a, int32_t op, void* stream);

/* Operand "planes" of the TMA-fed wgmma GEMM (csrc/gemm_tma.cu).  A plane pair is the bf16 image of an
 * fp32 matrix: hi = bf16(v), lo = bf16(v - hi), both plain row-major with pitch ldp (elements, multiple of 8); lo may
 * be NULL for GPS_PREC_BF16.  gps_to_planes converts; gps_gemm_planes multiplies plane operands stored as
 * A: [M,K] (ta = 0) or [K,M] (ta = 1), B: [N,K] (tb = 0, an nn.Linear weight) or [K,N] (tb = 1), writes fp32 C
 * (may be NULL) and/or the planes of C, optionally adds the row sums of Aop into colsum_a[M] (ta = 1: the bias
 * gradient of dW = G^T X).  splitk > 1 splits K over a cluster of at most 8 CTAs whose partial tiles are summed in
 * rank order, then added into a pre-zeroed fp32 C by one CTA per element: the same result in every run. */
int gps_to_planes(const float* src, int64_t ld, int64_t rows, int64_t cols, void* hi, void* lo, int64_t ldp,
                  void* stream);
int gps_gemm_planes(const void* A_hi, const void* A_lo, int64_t lda, int32_t ta, const void* B_hi, const void* B_lo,
                    int64_t ldb, int32_t tb, float* C, int64_t ldc, void* C_hi, void* C_lo, int64_t ldcp, int64_t M,
                    int64_t N, int64_t K, int32_t splitk, int32_t precision, float* colsum_a, void* stream);
/* One dense product with the fused epilogue every Linear of the layers runs (the arguments of gps_gemm_planes plus
 * the epilogue fields), so the epilogue can be tested step by step.  In this order, per output element:
 *   v = Aop Bop + bias[n]; C_pre = v; v = act(v); v *= act'(mask_src) (mask_is_post, relu only: [mask_src > 0]);
 *   v *= drop(p_drop2, site2); v *= drop(p_drop, site); v += R1 + R2; C = v; Cp = bf16 hi/lo planes of v;
 *   stats[0][n] += v, stats[1][n] += v^2 (float64, pre-zeroed by the caller).
 * act / mask_act: -1 none, GPS_ACT_*.  Dropout (p > 0, N % 4 == 0) draws gps_dropout_mask(M, N, p, seed,
 * offset + *offset_dev (offset_dev NULL: + 0), site): the index is over a dense [M, N] grid whatever ldc is.
 * cp_hd > 0 writes Cp in the per-head padded layout of the wgmma attention: column c lands at
 * (c / cp_hd) * cp_hd_pad + c % cp_hd, and the cp_hd_pad - cp_hd pad columns of every head are zeros.
 * splitk > 1 adds Aop Bop (+ R1 + R2) into a pre-zeroed C and takes no other epilogue field (GPS_ERR_ARG).
 * colsum_a (ta = 1 only, else GPS_ERR_ARG) adds the row sums of Aop.
 * impl: 0 = the dispatcher the layers call (planes when both are given, else or on rejection the fp32 kernels),
 * 1 = exact CUDA-core kernel, 2 = register-staged tensor-core kernel, 3 = TMA-fed tensor-core kernel.  1 and 2 read the
 * fp32 A and B and never write planes: Cp, or a NULL A or B, with impl 1 or 2 is GPS_ERR_ARG, as are a NULL args, sizes
 * outside [0, 2^31), an impl outside 0..3 and neither C nor Cp given, all before any CUDA call.  A kernel that does not take the shape,
 * layout or alignment returns GPS_ERR_UNSUPPORTED; so does the dispatcher when the TMA kernel rejects a product whose
 * planes need the per-head layout (the fp32 fallback writes the identity layout only). */
typedef struct {
  int64_t M, N, K;
  const float* A; int64_t lda;
  const float* B; int64_t ldb;
  int32_t ta, tb;
  GpsPlanes Ap, Bp, Cp;
  float* C; int64_t ldc;
  int32_t cp_hd, cp_hd_pad;
  const float* bias;
  float* C_pre; int64_t ldpre;
  const float* mask_src; int64_t ldmask;
  int32_t act, mask_act, mask_is_post;
  float p_drop; int32_t site;
  float p_drop2; int32_t site2;
  int32_t splitk;
  uint64_t seed, offset;
  const unsigned long long* offset_dev;
  const float* R1; int64_t ldr1;
  const float* R2; int64_t ldr2;
  double* stats;
  float* colsum_a;
  int32_t precision, reserved;
} GpsGemmArgs;
int gps_gemm_epilogue(const GpsGemmArgs* a, int32_t impl, void* stream);

/* One row-wise stage of the layers (csrc/elementwise.cu, and the dropout-only pass of layer.cu), called exactly as the
 * layers call it, so the BatchNorm apply, statistics finalisation, backward, dropout-gradient and bias-gradient passes
 * can be tested alone.  Per op, on rows x d (pitch ldx / ldg / ldo where the op reads it, else d; an ld of 0 means d):
 *   BN_ACT_RESIDUAL   out = R + drop(p, site)(act(BN0(x)))  [+ out's planes]  [stats[0][c] += out, stats[1][c] += out^2]
 *   BN_ACT_RESIDUAL2  the GatedGCN outputs: out = R + drop(p, site)(act(BN0(x))) over rows with column sums into stats,
 *                     and out2 = R2 + drop(p, site2)(act(BN1(x2))) over E rows [+ out2's planes], one launch; stats
 *                     NULL runs the two-launch form (eval mode), as does rows == 0 or E == 0
 *   BN_COMBINE        out = BN0(x) [+ BN1(x2)]  [+ out's planes]
 *   BN_BWD_REDUCE     g' = drop(p, site)(g) * act'(BN0(x)) (act -1: none); bn[0].sums [2][d] += (sum g', sum g' xhat)
 *   BN_BWD_APPLY      out = gamma invstd (g' - S1/n - xhat S2/n) in training, gamma invstd g' in eval, from
 *                     bn[0].sums = (S1, S2) [+ out's planes]; grad_weight = S2 and grad_bias = S1 (each NULL = not
 *                     wanted; added with accumulate), zeroed for rows == 0 unless accumulating
 *   DROPMUL           out = x * drop(p, site) * drop(p2, site2) [+ out's planes]  (each p 0 = none)
 *   COLSUM            out[c] += sum_r x[r, c]  (float32, the same bits in every run)
 * A BatchNorm is a GpsRowwiseBn: the module (weight, bias, running statistics, num_batches_tracked, gradients), its
 * mode (train), its saved [mean | invstd] (2d floats) and its float64 sums [2][d].  A forward op in training mode
 * finalises mean / invstd from sums (the producer's column sums over its rows), writes them to saved and updates the
 * running statistics (momentum 0.1, unbiased variance) and num_batches_tracked; in eval mode it reads the running
 * statistics.  A backward op reads saved in training mode and the running statistics in eval mode.  Dropout draws
 * gps_dropout_mask(rows, d, p, seed, offset + *offset_dev (offset_dev NULL: + 0), site).  R and R2 may be NULL.
 * NULL args, an unknown op, a negative size, an ld below d or above it and not a multiple of 4, an ld other than d
 * where the op takes pitch d, and a NULL pointer the op needs (a tensor over rows, or E, may be NULL when there are
 * none) are GPS_ERR_ARG, before any CUDA call; d outside the
 * row-wise stages' range (d % 4 != 0 or d > 4096; DROPMUL and COLSUM: d % 4 != 0) is GPS_ERR_UNSUPPORTED. */
enum {
  GPS_ROWWISE_BN_ACT_RESIDUAL = 0, GPS_ROWWISE_BN_ACT_RESIDUAL2 = 1, GPS_ROWWISE_BN_COMBINE = 2,
  GPS_ROWWISE_BN_BWD_REDUCE = 3, GPS_ROWWISE_BN_BWD_APPLY = 4, GPS_ROWWISE_DROPMUL = 5, GPS_ROWWISE_COLSUM = 6
};
typedef struct {
  GpsBatchNorm bn;
  float* saved;
  double* sums;
  int32_t train, reserved;
} GpsRowwiseBn;
typedef struct {
  int64_t rows, E, d;
  const float* x; int64_t ldx;
  const float* x2;
  const float* g; int64_t ldg;
  const float* R;
  const float* R2;
  float* out; int64_t ldo;
  float* out2;
  GpsPlanes planes;
  GpsRowwiseBn bn[2];
  int32_t act;
  float p; int32_t site;
  float p2; int32_t site2;
  int32_t accumulate;
  uint64_t seed, offset;
  const unsigned long long* offset_dev;
  double* stats;
} GpsRowwiseArgs;
int gps_rowwise_stage(const GpsRowwiseArgs* a, int32_t op, void* stream);

/* number of dense products that fell back from the tensor-core kernels to the exact CUDA-core kernel
 * (unaligned / odd shapes) in this process; with GPS_B200_STRICT=1 in the environment such a fallback is an error */
unsigned long long gps_fallback_count(void);

/* Dropout keep-mask generator used by every dropout site (tests replay it): writes 1/0 floats. */
int gps_dropout_mask(float* mask, int64_t rows, int64_t cols, float p, uint64_t seed,
                     uint64_t offset, int32_t site, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GPS_B200_H_ */
