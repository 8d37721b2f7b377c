"""ctypes binding of libgps_b200.so (the C ABI declared in include/gps_b200.h).

The library is the product: there is no CPU or eager-PyTorch fallback.  If the shared object is
missing or fails to load, importing a function from here raises immediately.
"""
from __future__ import annotations

import ctypes as C
import os

import torch  # noqa: F401  (loads libcudart.so.12 into the process before our library resolves it)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgps_b200.so")

GPS_OK, GPS_ERR_ARG, GPS_ERR_UNSUPPORTED, GPS_ERR_CUDA = 0, -1, -2, -3
LOCAL = {"None": 0, "CustomGatedGCN": 1, "GINE": 2, "GCN": 3, "GAT": 4, "GENConv": 5, "PNA": 6}
GLOBAL = {"None": 0, "Transformer": 1, "Performer": 2, "BigBird": 3}
GLOBAL_BIGBIRD = GLOBAL["BigBird"]   # the name existing binders import; the same value
BIGBIRD_ACT = {"relu": 0, "sigmoid": 1}   # GpsBigBird.hidden_act
ACT = {"relu": 0, "gelu": 1}
PRECISION = {"fp32": 0, "bf16": 1}
NORM = {"batch": 0, "none": 1}
# GpsLayerArgs.flags (backward), also GpsGraphormerArgs.flags and GpsSanArgs.flags
FLAG_GRADS_ZEROED, FLAG_GRADS_ACCUMULATE = 1, 2

_fp = C.c_void_p  # device pointers travel as void*


class GpsGraph(C.Structure):
    _fields_ = [("N", C.c_int64), ("E", C.c_int64), ("B", C.c_int64),
                ("dst_ptr", _fp), ("dst_src", _fp), ("dst_eid", _fp),
                ("src_ptr", _fp), ("src_dst", _fp), ("src_eid", _fp), ("graph_ptr", _fp)]


class GpsBatchNorm(C.Structure):
    _fields_ = [("weight", _fp), ("bias", _fp), ("running_mean", _fp), ("running_var", _fp),
                ("num_batches_tracked", _fp), ("grad_weight", _fp), ("grad_bias", _fp)]


class GpsLinear(C.Structure):
    _fields_ = [("weight", _fp), ("bias", _fp), ("grad_weight", _fp), ("grad_bias", _fp)]


class GpsPlanes(C.Structure):
    _fields_ = [("hi", _fp), ("lo", _fp), ("ld", C.c_int64)]


class GpsAttnBias(C.Structure):
    """Attention bias of the BiasedTransformer: bias / grad_bias [B*heads, nmax, nmax] float32."""
    _fields_ = [("bias", _fp), ("nmax", C.c_int64), ("grad_bias", _fp)]


class GpsGat(C.Structure):
    """GAT local model: lin_src (weight = local_model.lin_src.weight, bias = local_model.bias), lin_edge, att_* [H*C]."""
    _fields_ = [("lin_src", GpsLinear), ("lin_edge", GpsLinear), ("att_src", _fp), ("att_dst", _fp), ("att_edge", _fp),
                ("grad_att_src", _fp), ("grad_att_dst", _fp), ("grad_att_edge", _fp)]


class GpsGenConv(C.Structure):
    """GENConv local model: lin0 = local_model.mlp.0, bn = local_model.mlp.1 [2d], lin1 = local_model.mlp.4 (no biases)."""
    _fields_ = [("lin0", GpsLinear), ("bn", GpsBatchNorm), ("lin1", GpsLinear)]


class GpsPna(C.Structure):
    """PNA local model: edge_encoder [d, edge_dim], pre = pre_nns.0.0 [d, 3d], post = post_nns.0.0 [d, 4d], lin [d, d]."""
    _fields_ = [("edge_encoder", GpsLinear), ("pre", GpsLinear), ("post", GpsLinear), ("lin", GpsLinear),
                ("edge_dim", C.c_int64)]


class GpsBigBird(C.Structure):
    """BigBird global model: block geometry, the per-head block lists (device int32) and the eight parameters of
    self_attn.encoder.layers.0 (query, key, value, attention.output.dense / .LayerNorm, intermediate.dense,
    output.dense / .LayerNorm)."""
    _fields_ = [("block_size", C.c_int64), ("num_blocks", C.c_int64), ("hidden_act", C.c_int32), ("ln_eps", C.c_float),
                ("key_ptr", _fp), ("key_idx", _fp), ("query_ptr", _fp), ("query_idx", _fp),
                ("query", GpsLinear), ("key", GpsLinear), ("value", GpsLinear), ("self_out", GpsLinear),
                ("ln1", GpsLinear), ("intermediate", GpsLinear), ("output", GpsLinear), ("ln2", GpsLinear)]


class GpsLayerArgs(C.Structure):
    _fields_ = [
        ("d", C.c_int64), ("heads", C.c_int64),
        ("local_type", C.c_int32), ("global_type", C.c_int32), ("act", C.c_int32),
        ("training", C.c_int32), ("precision", C.c_int32), ("flags", C.c_int32),
        ("dropout", C.c_float), ("attn_dropout", C.c_float),
        ("seed", C.c_uint64), ("offset", C.c_uint64),
        ("gine_eps", C.c_float), ("norm_type", C.c_int32),
        ("graph", GpsGraph),
        ("x", _fp), ("edge_attr", _fp), ("x_out", _fp), ("edge_out", _fp),
        ("gcn_A", GpsLinear), ("gcn_B", GpsLinear), ("gcn_C", GpsLinear), ("gcn_D", GpsLinear),
        ("gcn_E", GpsLinear),
        ("bn_node_x", GpsBatchNorm), ("bn_edge_e", GpsBatchNorm),
        ("gine_lin0", GpsLinear), ("gine_lin1", GpsLinear),
        ("attn_in", GpsLinear), ("attn_out", GpsLinear),
        ("perf_q", GpsLinear), ("perf_k", GpsLinear), ("perf_v", GpsLinear),
        ("perf_proj", _fp), ("perf_features", C.c_int64), ("perf_dim_head", C.c_int64),
        ("norm1_local", GpsBatchNorm), ("norm1_attn", GpsBatchNorm), ("norm2", GpsBatchNorm),
        ("ff1", GpsLinear), ("ff2", GpsLinear),
        ("grad_x_out", _fp), ("grad_edge_out", _fp), ("grad_x", _fp), ("grad_edge_attr", _fp),
        ("saved", _fp), ("saved_bytes", C.c_int64),
        ("workspace", _fp), ("workspace_bytes", C.c_int64),
        ("offset_dev", _fp),
        ("gcn_conv", GpsLinear),
        ("ev_grads_early", _fp),
        ("x_planes_in", GpsPlanes), ("e_planes_in", GpsPlanes), ("x_planes_out", GpsPlanes), ("e_planes_out", GpsPlanes),
        ("wplanes", _fp), ("wplanes_bytes", C.c_int64), ("wplanes_valid", C.c_int32), ("reserved2", C.c_int32),
        ("ev_grads_mid", _fp), ("ev_grads_done", _fp),
        ("pe", _fp), ("pe_dim", C.c_int64), ("grad_pe", _fp), ("pe_mlp0", GpsLinear), ("pe_mlp1", GpsLinear),
        ("attn_bias", GpsAttnBias), ("gat", GpsGat), ("genconv", GpsGenConv), ("pna", GpsPna), ("bigbird", GpsBigBird),
    ]


class GpsGraphormerArgs(C.Structure):
    """Graphormer layer (graphormer_layer.py): config, dropout stream, graph, tensors, scratch and the six parameters
    input_norm, attention.in_proj, attention.out_proj, mlp.0, mlp.1, mlp.4."""
    _fields_ = [("d", C.c_int64), ("heads", C.c_int64), ("training", C.c_int32), ("precision", C.c_int32),
                ("dropout", C.c_float), ("attn_dropout", C.c_float), ("mlp_dropout", C.c_float), ("flags", C.c_int32),
                ("seed", C.c_uint64), ("offset", C.c_uint64), ("offset_dev", _fp),
                ("graph", GpsGraph),
                ("x", _fp), ("x_out", _fp), ("grad_x_out", _fp), ("grad_x", _fp),
                ("saved", _fp), ("saved_bytes", C.c_int64), ("workspace", _fp), ("workspace_bytes", C.c_int64),
                ("input_norm", GpsLinear), ("attn_in", GpsLinear), ("attn_out", GpsLinear), ("mlp_norm", GpsLinear),
                ("mlp_lin1", GpsLinear), ("mlp_lin2", GpsLinear)]


class GpsGraphormerPlan(C.Structure):
    _fields_ = [("saved_bytes", C.c_int64), ("fwd_workspace_bytes", C.c_int64), ("bwd_workspace_bytes", C.c_int64)]


class GpsGraphormerBiasArgs(C.Structure):
    """Graphormer's BiasEncoder (graphormer_encoder.py:103-183): sizes, the collated pair attributes (int64), the four
    parameters, attn_bias / grad_attn_bias [B*H, N', N'], the parameter gradients and the backward's scratch."""
    _fields_ = [("num_pairs", C.c_int64), ("num_graphs", C.c_int64), ("nmax", C.c_int64), ("heads", C.c_int64),
                ("num_spatial_types", C.c_int64), ("num_edge_types", C.c_int64), ("use_graph_token", C.c_int32),
                ("reserved", C.c_int32),
                ("spatial_types", _fp), ("graph_index", _fp), ("shortest_path_types", _fp), ("node_ptr", _fp),
                ("spatial_weight", _fp), ("edge_dis_weight", _fp), ("edge_weight", _fp), ("graph_token", _fp),
                ("attn_bias", _fp), ("grad_attn_bias", _fp),
                ("grad_spatial_weight", _fp), ("grad_edge_dis_weight", _fp), ("grad_edge_weight", _fp),
                ("grad_graph_token", _fp),
                ("workspace", _fp), ("workspace_bytes", C.c_int64)]


class GpsGraphormerBiasPlan(C.Structure):
    _fields_ = [("fwd_workspace_bytes", C.c_int64), ("bwd_workspace_bytes", C.c_int64)]


class GpsLinkHeadArgs(C.Structure):
    """Inductive link-prediction head (inductive_edge.py, dot decoding, layers_post_mp 1): config, the labeled-pair
    graph, edge_index_labeled / edge_label, x, layer_post_mp.model.0.model, outputs, gradients and scratch."""
    _fields_ = [("d", C.c_int64), ("training", C.c_int32), ("precision", C.c_int32), ("flags", C.c_int32),
                ("label_bytes", C.c_int32), ("seed", C.c_uint64),
                ("pairs", GpsGraph), ("edge_index_labeled", _fp), ("edge_label", _fp), ("x", _fp),
                ("lin", GpsLinear), ("y", _fp), ("pred", _fp), ("stats", _fp),
                ("grad_y", _fp), ("grad_pred", _fp), ("grad_x", _fp),
                ("saved", _fp), ("saved_bytes", C.c_int64), ("workspace", _fp), ("workspace_bytes", C.c_int64)]


class GpsLinkHeadPlan(C.Structure):
    _fields_ = [("saved_bytes", C.c_int64), ("fwd_workspace_bytes", C.c_int64), ("bwd_workspace_bytes", C.c_int64)]


GRAPH_HEAD = {"san_graph": 0, "graphormer_graph": 1}
POOLING = {"mean": 0, "add": 1, "graph_token": 2}
GRAPH_HEAD_MAX_L = 12


class GpsGraphHeadArgs(C.Structure):
    """Graph-prediction head (san_graph.py's SANGraphHead or graphormer_graph.py's GraphormerHead): config, the batch's
    graph, x, pred and their gradients, ln (GraphormerHead) and fc[l] = FC_layers.l / layers.0, and scratch."""
    _fields_ = [("kind", C.c_int32), ("pooling", C.c_int32), ("act", C.c_int32), ("L", C.c_int32),
                ("dim_in", C.c_int64), ("dim_out", C.c_int64),
                ("training", C.c_int32), ("precision", C.c_int32), ("flags", C.c_int32), ("reserved", C.c_int32),
                ("seed", C.c_uint64), ("graph", GpsGraph),
                ("x", _fp), ("pred", _fp), ("grad_pred", _fp), ("grad_x", _fp),
                ("ln", GpsLinear), ("fc", GpsLinear * (GRAPH_HEAD_MAX_L + 1)),
                ("saved", _fp), ("saved_bytes", C.c_int64), ("workspace", _fp), ("workspace_bytes", C.c_int64)]


class GpsGraphHeadPlan(C.Structure):
    _fields_ = [("saved_bytes", C.c_int64), ("fwd_workspace_bytes", C.c_int64), ("bwd_workspace_bytes", C.c_int64)]


NODE_HEAD_MAX_L, NODE_LOSS_MAX_C = 8, 4096


class GpsNodeHeadArgs(C.Structure):
    """Node-prediction head (GraphGym's MLP under inductive_node.py's GNNInductiveNodeHead or GNNNodeHead): L and the
    widths, x, the optional row selection, y / pred and their gradients, fc[l] = the MLP's Linears in order, scratch."""
    _fields_ = [("L", C.c_int32), ("precision", C.c_int32), ("flags", C.c_int32), ("training", C.c_int32),
                ("seed", C.c_uint64), ("dim_in", C.c_int64), ("dim_inner", C.c_int64), ("dim_out", C.c_int64), ("N", C.c_int64),
                ("M", C.c_int64), ("x", _fp), ("rows", _fp), ("y", _fp), ("pred", _fp), ("grad_y", _fp),
                ("grad_pred", _fp), ("grad_x", _fp), ("fc", GpsLinear * NODE_HEAD_MAX_L),
                ("saved", _fp), ("saved_bytes", C.c_int64), ("workspace", _fp), ("workspace_bytes", C.c_int64)]


class GpsNodeHeadPlan(C.Structure):
    _fields_ = [("saved_bytes", C.c_int64), ("fwd_workspace_bytes", C.c_int64), ("bwd_workspace_bytes", C.c_int64)]


class GpsNodeLossArgs(C.Structure):
    """Node loss (weighted_cross_entropy.py or GraphGym's cross_entropy): sizes, mode, pred / label, the device loss,
    pred_score, their gradients and scratch."""
    _fields_ = [("M", C.c_int64), ("C", C.c_int64), ("weighted", C.c_int32), ("flags", C.c_int32),
                ("pred", _fp), ("label", _fp), ("loss", _fp), ("pred_score", _fp), ("grad_loss", _fp),
                ("grad_score", _fp), ("grad_pred", _fp),
                ("saved", _fp), ("saved_bytes", C.c_int64), ("workspace", _fp), ("workspace_bytes", C.c_int64)]


class GpsNodeLossPlan(C.Structure):
    _fields_ = [("saved_bytes", C.c_int64), ("fwd_workspace_bytes", C.c_int64), ("bwd_workspace_bytes", C.c_int64)]


RWSE_MAX_COLS, RWSE_MAX_STEPS = 64, 256


class GpsKernelPeArgs(C.Structure):
    """KernelPENodeEncoder (kernel_pos_encoder.py, model "linear"): sizes and modes, pestat, x, out and their gradients,
    linear_x, pe_encoder and raw_norm, and scratch."""
    _fields_ = [("N", C.c_int64), ("K", C.c_int64), ("dim_in", C.c_int64), ("dim_emb", C.c_int64),
                ("dim_pe", C.c_int64), ("expand_x", C.c_int32), ("batch_norm", C.c_int32), ("training", C.c_int32),
                ("flags", C.c_int32), ("pestat", _fp), ("x", _fp), ("out", _fp), ("grad_out", _fp), ("grad_x", _fp),
                ("linear_x", GpsLinear), ("pe_encoder", GpsLinear), ("raw_norm", GpsBatchNorm),
                ("saved", _fp), ("saved_bytes", C.c_int64), ("workspace", _fp), ("workspace_bytes", C.c_int64)]


class GpsKernelPePlan(C.Structure):
    _fields_ = [("saved_bytes", C.c_int64), ("fwd_workspace_bytes", C.c_int64), ("bwd_workspace_bytes", C.c_int64)]


class GpsSanArgs(C.Structure):
    """SAN layer (san_layer.py, variant 0) or SAN2 layer (san2_layer.py, variant 1): config, dropout stream, graph and
    nmax, tensors, scratch, the ten Linears attention.{Q,K,V,Q_2,K_2,E,E_2}, O_h, FFN_h_layer1, FFN_h_layer2,
    batch_norm{1,2}_h, attention.fake_edge_emb and (variant 1) the float64 attention.gamma and its gradient."""
    _fields_ = [("d", C.c_int64), ("heads", C.c_int64), ("training", C.c_int32), ("precision", C.c_int32),
                ("gamma", C.c_float), ("dropout", C.c_float), ("flags", C.c_int32), ("variant", C.c_int32),
                ("seed", C.c_uint64), ("offset", C.c_uint64), ("offset_dev", _fp),
                ("graph", GpsGraph), ("nmax", C.c_int64),
                ("x", _fp), ("edge_attr", _fp), ("x_out", _fp), ("grad_x_out", _fp), ("grad_x", _fp),
                ("grad_edge_attr", _fp),
                ("saved", _fp), ("saved_bytes", C.c_int64), ("workspace", _fp), ("workspace_bytes", C.c_int64),
                ("Q", GpsLinear), ("K", GpsLinear), ("V", GpsLinear), ("Q2", GpsLinear), ("K2", GpsLinear),
                ("E", GpsLinear), ("E2", GpsLinear), ("O_h", GpsLinear), ("ffn1", GpsLinear), ("ffn2", GpsLinear),
                ("bn1", GpsBatchNorm), ("bn2", GpsBatchNorm),
                ("fake_edge_emb", _fp), ("grad_fake_edge_emb", _fp), ("gamma_param", _fp), ("grad_gamma", _fp)]


class GpsSanPlan(C.Structure):
    _fields_ = [("saved_bytes", C.c_int64), ("fwd_workspace_bytes", C.c_int64), ("bwd_workspace_bytes", C.c_int64)]


class GpsCustomGnnArgs(C.Structure):
    """CustomGNN's GatedGCNLayer / GINEConvLayer (custom_gnn.py): config, dropout stream, graph, tensors, scratch, the
    persistent weight buffer, GatedGCN's A..E and two BatchNorms, GINE's model.nn.0 / model.nn.2."""
    _fields_ = [("d", C.c_int64), ("kind", C.c_int32), ("act", C.c_int32), ("training", C.c_int32),
                ("precision", C.c_int32), ("residual", C.c_int32), ("flags", C.c_int32), ("dropout", C.c_float),
                ("gine_eps", C.c_float), ("seed", C.c_uint64), ("offset", C.c_uint64), ("offset_dev", _fp),
                ("graph", GpsGraph),
                ("x", _fp), ("edge_attr", _fp), ("x_out", _fp), ("edge_out", _fp), ("grad_x_out", _fp),
                ("grad_edge_out", _fp), ("grad_x", _fp), ("grad_edge_attr", _fp),
                ("saved", _fp), ("saved_bytes", C.c_int64), ("workspace", _fp), ("workspace_bytes", C.c_int64),
                ("wplanes", _fp), ("wplanes_bytes", C.c_int64), ("wplanes_valid", C.c_int32), ("reserved", C.c_int32),
                ("A", GpsLinear), ("B", GpsLinear), ("C", GpsLinear), ("D", GpsLinear), ("E", GpsLinear),
                ("bn_node_x", GpsBatchNorm), ("bn_edge_e", GpsBatchNorm), ("nn0", GpsLinear), ("nn2", GpsLinear)]


class GpsCustomGnnPlan(C.Structure):
    _fields_ = [("saved_bytes", C.c_int64), ("fwd_workspace_bytes", C.c_int64), ("bwd_workspace_bytes", C.c_int64),
                ("wplanes_bytes", C.c_int64)]


CUSTOM_GATEDGCN, CUSTOM_GINE = 0, 1


class GpsGemmArgs(C.Structure):
    """One dense product with its fused epilogue (gps_gemm_epilogue): sizes, fp32 operands, operand / output planes,
    the epilogue fields in the order they apply, and the arithmetic."""
    _fields_ = [("M", C.c_int64), ("N", C.c_int64), ("K", C.c_int64),
                ("A", _fp), ("lda", C.c_int64), ("B", _fp), ("ldb", C.c_int64), ("ta", C.c_int32), ("tb", C.c_int32),
                ("Ap", GpsPlanes), ("Bp", GpsPlanes), ("Cp", GpsPlanes),
                ("C", _fp), ("ldc", C.c_int64), ("cp_hd", C.c_int32), ("cp_hd_pad", C.c_int32),
                ("bias", _fp), ("C_pre", _fp), ("ldpre", C.c_int64), ("mask_src", _fp), ("ldmask", C.c_int64),
                ("act", C.c_int32), ("mask_act", C.c_int32), ("mask_is_post", C.c_int32),
                ("p_drop", C.c_float), ("site", C.c_int32), ("p_drop2", C.c_float), ("site2", C.c_int32),
                ("splitk", C.c_int32), ("seed", C.c_uint64), ("offset", C.c_uint64), ("offset_dev", _fp),
                ("R1", _fp), ("ldr1", C.c_int64), ("R2", _fp), ("ldr2", C.c_int64),
                ("stats", _fp), ("colsum_a", _fp), ("precision", C.c_int32), ("reserved", C.c_int32)]


# gps_rowwise_stage ops
ROWWISE = {"bn_act_residual": 0, "bn_act_residual2": 1, "bn_combine": 2, "bn_bwd_reduce": 3, "bn_bwd_apply": 4,
           "dropmul": 5, "colsum": 6}


class GpsRowwiseBn(C.Structure):
    """A BatchNorm as a row-wise stage reads it: the module, its mode, saved [mean | invstd] (2d floats) and its
    float64 sums [2][d]."""
    _fields_ = [("bn", GpsBatchNorm), ("saved", _fp), ("sums", _fp), ("train", C.c_int32), ("reserved", C.c_int32)]


class GpsRowwiseArgs(C.Structure):
    """One row-wise stage (gps_rowwise_stage): sizes, tensors with their pitches, output planes, up to two BatchNorms,
    the activation, the dropout sites, the accumulate flag and the column statistics output."""
    _fields_ = [("rows", C.c_int64), ("E", C.c_int64), ("d", C.c_int64),
                ("x", _fp), ("ldx", C.c_int64), ("x2", _fp), ("g", _fp), ("ldg", C.c_int64), ("R", _fp), ("R2", _fp),
                ("out", _fp), ("ldo", C.c_int64), ("out2", _fp), ("planes", GpsPlanes), ("bn", GpsRowwiseBn * 2),
                ("act", C.c_int32), ("p", C.c_float), ("site", C.c_int32), ("p2", C.c_float), ("site2", C.c_int32),
                ("accumulate", C.c_int32), ("seed", C.c_uint64), ("offset", C.c_uint64), ("offset_dev", _fp),
                ("stats", _fp)]


# gps_attention_stage ops
ATTN = {"fwd": 0, "fwd_tc": 1, "bwd": 2}


class GpsAttnStageArgs(C.Structure):
    """One softmax-attention stage (gps_attention_stage): graph, heads, head dim, Q / K / V or the qkv planes, O with its
    planes and lse, the backward's dO, delta, dQ / dK / dV with their planes, the bias and the dropout stream."""
    _fields_ = [("graph", GpsGraph), ("heads", C.c_int64), ("hd", C.c_int64),
                ("Q", _fp), ("K", _fp), ("V", _fp), ("ld", C.c_int64),
                ("qkv", GpsPlanes), ("precision", C.c_int32), ("reserved", C.c_int32),
                ("O", _fp), ("ldo", C.c_int64), ("O_planes", GpsPlanes), ("lse", _fp),
                ("dO", _fp), ("delta", _fp), ("dQ", _fp), ("dK", _fp), ("dV", _fp), ("ldg", C.c_int64),
                ("dQ_planes", GpsPlanes), ("dK_planes", GpsPlanes), ("dV_planes", GpsPlanes),
                ("bias", C.POINTER(GpsAttnBias)),
                ("p_drop", C.c_float), ("reserved2", C.c_int32), ("seed", C.c_uint64), ("offset", C.c_uint64),
                ("offset_dev", _fp)]


class GpsLayerPlan(C.Structure):
    _fields_ = [("saved_bytes", C.c_int64), ("fwd_workspace_bytes", C.c_int64),
                ("bwd_workspace_bytes", C.c_int64), ("wplanes_bytes", C.c_int64)]


# every symbol include/gps_b200.h declares: name -> (restype, argtypes)
_i64, _i32, _f32, _u64 = C.c_int64, C.c_int32, C.c_float, C.c_uint64
SYMBOLS = {
    "gps_last_error": (C.c_char_p, []),
    "gps_abi_version": (C.c_int, []),
    "gps_build_arch": (C.c_char_p, []),
    "gps_graph_bytes": (_i64, [_i64, _i64, _i64]),
    "gps_graph_build": (C.c_int, [_fp, _fp, _i64, _i64, _i64, _fp, _i64, C.POINTER(GpsGraph), _fp]),
    "gps_layer_plan": (C.c_int, [C.POINTER(GpsLayerArgs), C.POINTER(GpsLayerPlan)]),
    "gps_layer_forward": (C.c_int, [C.POINTER(GpsLayerArgs), _fp]),
    "gps_layer_backward": (C.c_int, [C.POINTER(GpsLayerArgs), _fp]),
    "gps_bigbird_attention_forward": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, C.POINTER(GpsBigBird), _fp, _fp, _fp,
                                                _i64, _fp, _i64, _fp, _fp]),
    "gps_bigbird_attention_backward": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, C.POINTER(GpsBigBird), _fp, _fp, _fp,
                                                 _i64, _fp, _fp, _i64, _fp, _fp, _fp, _fp, _fp, _i64, _fp]),
    "gps_graphormer_plan": (C.c_int, [C.POINTER(GpsGraphormerArgs), C.POINTER(GpsGraphormerPlan)]),
    "gps_graphormer_forward": (C.c_int, [C.POINTER(GpsGraphormerArgs), C.POINTER(GpsAttnBias), _fp]),
    "gps_graphormer_backward": (C.c_int, [C.POINTER(GpsGraphormerArgs), C.POINTER(GpsAttnBias), _fp]),
    "gps_graphormer_bias_plan": (C.c_int, [C.POINTER(GpsGraphormerBiasArgs), C.POINTER(GpsGraphormerBiasPlan)]),
    "gps_graphormer_bias_forward": (C.c_int, [C.POINTER(GpsGraphormerBiasArgs), _fp]),
    "gps_graphormer_bias_backward": (C.c_int, [C.POINTER(GpsGraphormerBiasArgs), _fp]),
    "gps_link_head_plan": (C.c_int, [C.POINTER(GpsLinkHeadArgs), C.POINTER(GpsLinkHeadPlan)]),
    "gps_link_head_forward": (C.c_int, [C.POINTER(GpsLinkHeadArgs), _fp]),
    "gps_link_head_backward": (C.c_int, [C.POINTER(GpsLinkHeadArgs), _fp]),
    "gps_link_rank_metrics": (C.c_int, [C.POINTER(GpsGraph), _fp, _i64, _i64, _fp, _i32, _fp, _fp, _i64, _fp]),
    "gps_graph_head_plan": (C.c_int, [C.POINTER(GpsGraphHeadArgs), C.POINTER(GpsGraphHeadPlan)]),
    "gps_graph_head_forward": (C.c_int, [C.POINTER(GpsGraphHeadArgs), _fp]),
    "gps_graph_head_backward": (C.c_int, [C.POINTER(GpsGraphHeadArgs), _fp]),
    "gps_node_head_plan": (C.c_int, [C.POINTER(GpsNodeHeadArgs), C.POINTER(GpsNodeHeadPlan)]),
    "gps_node_head_forward": (C.c_int, [C.POINTER(GpsNodeHeadArgs), _fp]),
    "gps_node_head_backward": (C.c_int, [C.POINTER(GpsNodeHeadArgs), _fp]),
    "gps_row_l2norm_forward": (C.c_int, [_fp, _i64, _i64, _i64, _fp, _fp, _fp]),
    "gps_row_l2norm_backward": (C.c_int, [_fp, _fp, _fp, _i64, _i64, _i64, _fp, _fp]),
    "gps_node_loss_plan": (C.c_int, [C.POINTER(GpsNodeLossArgs), C.POINTER(GpsNodeLossPlan)]),
    "gps_node_loss_forward": (C.c_int, [C.POINTER(GpsNodeLossArgs), _fp]),
    "gps_node_loss_backward": (C.c_int, [C.POINTER(GpsNodeLossArgs), _fp]),
    "gps_rwse_landing": (C.c_int, [C.POINTER(GpsGraph), C.POINTER(_i32), _i32, _i32, _fp, _fp, _i64, _fp]),
    "gps_kernel_pe_plan": (C.c_int, [C.POINTER(GpsKernelPeArgs), C.POINTER(GpsKernelPePlan)]),
    "gps_kernel_pe_forward": (C.c_int, [C.POINTER(GpsKernelPeArgs), _fp]),
    "gps_kernel_pe_backward": (C.c_int, [C.POINTER(GpsKernelPeArgs), _fp]),
    "gps_graph_pool_forward": (C.c_int, [C.POINTER(GpsGraph), _i32, _fp, _i64, _fp, _i64, _fp, _i64, _fp]),
    "gps_graph_pool_backward": (C.c_int, [C.POINTER(GpsGraph), _i32, _fp, _i64, _i64, _fp, _fp]),
    "gps_san_plan": (C.c_int, [C.POINTER(GpsSanArgs), C.POINTER(GpsSanPlan)]),
    "gps_san_forward": (C.c_int, [C.POINTER(GpsSanArgs), _fp]),
    "gps_san_backward": (C.c_int, [C.POINTER(GpsSanArgs), _fp]),
    "gps_custom_gnn_plan": (C.c_int, [C.POINTER(GpsCustomGnnArgs), C.POINTER(GpsCustomGnnPlan)]),
    "gps_custom_gnn_forward": (C.c_int, [C.POINTER(GpsCustomGnnArgs), _fp]),
    "gps_custom_gnn_backward": (C.c_int, [C.POINTER(GpsCustomGnnArgs), _fp]),
    "gps_san_attention_workspace_bytes": (_i64, [_i64, _i64, _i64, _i64]),
    "gps_san_attention_forward": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _fp, _i64, _fp, _fp, _f32, _i64, _fp, _i64,
                                            _fp, _i64, _fp, _fp]),
    "gps_san_attention_backward": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _fp, _i64, _fp, _fp, _f32, _i64, _fp,
                                             _i64, _fp, _fp, _i64, _fp, _fp, _i64, _fp, _fp, _fp]),
    "gps_san2_attention_workspace_bytes": (_i64, [_i64, _i64, _i64, _i64]),
    "gps_san2_attention_forward": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _fp, _i64, _fp, _fp, _fp, _i64, _fp,
                                             _i64, _fp, _i64, _fp, _fp, _fp, _fp]),
    "gps_san2_attention_backward": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _fp, _i64, _fp, _fp, _fp, _i64, _fp,
                                              _i64, _fp, _fp, _fp, _fp, _i64, _fp, _i64, _fp, _fp, _fp, _fp]),
    "gps_layernorm_forward": (C.c_int, [_fp, _i64, _i64, _fp, _fp, _f32, _fp, _fp, _fp, _fp]),
    "gps_layernorm_backward": (C.c_int, [_fp, _fp, _i64, _i64, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _i32, _fp]),
    "gps_linear_forward": (C.c_int, [_fp, _i64, _fp, _i64, _fp, _fp, _i64, _i64, _i64, _i64, _i32, _i32, _fp]),
    "gps_gemm": (C.c_int, [_fp, _i64, _i32, _fp, _i64, _i32, _fp, _i64, _i64, _i64, _i64, _i32, _i32, _i32, _fp]),
    "gps_gatedgcn_aggregate_forward": (C.c_int, [C.POINTER(GpsGraph), _i64, _fp, _fp, _fp, _fp, _i64, _fp, _fp,
                                                 _fp, _fp, _fp]),
    "gps_gine_aggregate_forward": (C.c_int, [C.POINTER(GpsGraph), _i64, _fp, _fp, _f32, _fp, _fp]),
    "gps_gatedgcn_aggregate_forward_gated": (C.c_int, [C.POINTER(GpsGraph), _i64, _fp, _fp, _fp, _fp, _i64, _fp, _fp,
                                                       _fp, _fp, _fp, _fp]),
    "gps_gatedgcn_aggregate_backward": (C.c_int, [C.POINTER(GpsGraph), _i64, _fp, _fp, _i64, _fp, _fp, _i64, _fp, _fp,
                                                  _fp, C.POINTER(GpsPlanes), C.POINTER(GpsPlanes), _fp]),
    "gps_eslap_forward": (C.c_int, [C.POINTER(GpsGraph), _fp, _i64, _i64, _i32, _fp, _fp, _fp, _fp, _fp, _fp, _fp]),
    "gps_eslap_workspace_bytes": (_i64, [_i64, _i64]),
    "gps_eslap_backward": (C.c_int, [C.POINTER(GpsGraph), _fp, _i64, _i64, _i32, _fp, _fp, _fp, _i64, _fp, _fp, _fp,
                                     _fp, _fp, _fp, _fp, _i64, _fp, _fp, _fp, _fp, _fp, _i32, _fp]),
    "gps_gine_aggregate_backward": (C.c_int, [C.POINTER(GpsGraph), _i64, _fp, _fp, _fp, _f32, _fp, _fp, _fp, _fp]),
    "gps_gcn_aggregate_forward": (C.c_int, [C.POINTER(GpsGraph), _i64, _fp, _i64, _fp, _fp, _fp, _fp, _f32, _u64, _u64,
                                            _fp, _fp]),
    "gps_gcn_aggregate_backward": (C.c_int, [C.POINTER(GpsGraph), _i64, _fp, _fp, _fp, _i64, C.POINTER(GpsPlanes), _fp]),
    "gps_gat_fold_forward": (C.c_int, [_fp, _fp, _i64, _i64, _fp, _fp]),
    "gps_gat_fold_backward": (C.c_int, [_fp, _fp, _fp, _i64, _i64, _fp, _fp, _i32, _fp]),
    "gps_gat_forward": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _fp, _i64, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp,
                                  _f32, _u64, _u64, _fp, _fp]),
    "gps_gat_workspace_bytes": (_i64, [_i64, _i64, _i64, _i64]),
    "gps_gat_backward": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _fp, _i64, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _i64,
                                   _fp, _i64, C.POINTER(GpsPlanes), _fp, _fp, _fp, _fp, _fp, _i32, _fp]),
    "gps_genconv_aggregate_forward": (C.c_int, [C.POINTER(GpsGraph), _i64, _fp, _fp, _fp, _fp, _fp, _fp]),
    "gps_genconv_aggregate_backward": (C.c_int, [C.POINTER(GpsGraph), _i64, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp,
                                                 _fp]),
    "gps_pna_fold_forward": (C.c_int, [_fp, _fp, _fp, _fp, _i64, _i64, _fp, _fp, _fp]),
    "gps_pna_fold_backward": (C.c_int, [_fp, _fp, _fp, _fp, _fp, _i64, _i64, _fp, _fp, _fp, _fp, _i32, _fp]),
    "gps_pna_aggregate_forward": (C.c_int, [C.POINTER(GpsGraph), _i64, _fp, _fp, _i64, _fp, _fp, _fp, _fp]),
    "gps_pna_aggregate_backward": (C.c_int, [C.POINTER(GpsGraph), _i64, _fp, _fp, _fp, _fp, _fp, _i64, _fp, _fp]),
    "gps_performer_prep": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _i64, _fp, _fp, _fp, _fp, _fp, _fp]),
    "gps_performer_features_forward": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _i64, _fp, _fp, _fp, _fp, _fp, _fp,
                                                 _fp, _fp]),
    "gps_performer_attention_forward": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _i64, _i32, _fp, _fp, _fp, _fp, _fp,
                                                  _fp, _fp, _fp]),
    "gps_performer_attention_backward": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _i64, _i32, _fp, _fp, _fp, _fp,
                                                   _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp]),
    "gps_performer_features_backward": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _i64, _i32, _fp, _fp, _fp, _fp, _fp,
                                                  _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp]),
    "gps_attention_forward": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _fp, _fp, _fp, _i64, _fp, _i64, _fp,
                                        _f32, _u64, _u64, _fp]),
    "gps_attention_backward": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _fp, _fp, _fp, _i64, _fp, _fp, _i64,
                                         _fp, _fp, _fp, _fp, _fp, _i64, _f32, _u64, _u64, _fp]),
    "gps_attention_forward_tc": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _fp, _fp, _i64, _fp, _i64, _fp, _f32, _u64, _u64,
                                           _i32, _fp]),
    "gps_attention_forward_biased": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _fp, _fp, _fp, _i64, _fp, _i64, _fp,
                                               _f32, _u64, _u64, C.POINTER(GpsAttnBias), _fp]),
    "gps_attention_forward_tc_biased": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _fp, _fp, _i64, _fp, _i64, _fp, _f32,
                                                  _u64, _u64, _i32, C.POINTER(GpsAttnBias), _fp]),
    "gps_attention_backward_biased": (C.c_int, [C.POINTER(GpsGraph), _i64, _i64, _fp, _fp, _fp, _i64, _fp, _fp, _i64,
                                                _fp, _fp, _fp, _fp, _fp, _i64, _f32, _u64, _u64, C.POINTER(GpsAttnBias),
                                                _fp]),
    "gps_attention_stage": (C.c_int, [C.POINTER(GpsAttnStageArgs), _i32, _fp]),
    "gps_dropout_mask": (C.c_int, [_fp, _i64, _i64, _f32, _u64, _u64, _i32, _fp]),
    "gps_to_planes": (C.c_int, [_fp, _i64, _i64, _i64, _fp, _fp, _i64, _fp]),
    "gps_gemm_planes": (C.c_int, [_fp, _fp, _i64, _i32, _fp, _fp, _i64, _i32, _fp, _i64, _fp, _fp, _i64, _i64, _i64, _i64,
                                  _i32, _i32, _fp, _fp]),
    "gps_gemm_epilogue": (C.c_int, [C.POINTER(GpsGemmArgs), _i32, _fp]),
    "gps_rowwise_stage": (C.c_int, [C.POINTER(GpsRowwiseArgs), _i32, _fp]),
    "gps_fallback_count": (C.c_ulonglong, []),
    # not in the header's stage list but part of the ABI: launch counter for bench.py
    "gps_launch_count": (C.c_ulonglong, []),
    "gps_debug_set": (None, [C.c_int]),
    "gps_debug_tma": (None, [C.c_int, _fp]),
    "gps_debug_tma_splits": (None, [C.c_int]),
    "gps_debug_attn": (None, [_fp]),
}

_lib = None


def load():
    """Loads libgps_b200.so (once).  Raises if it is missing: there is no fallback path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -m graphgps_b200.build` "
            "(nvcc, sm_90a). graphgps_b200 has no CPU/eager fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    if lib.gps_abi_version() != 4:
        raise RuntimeError("libgps_b200.so ABI version mismatch")
    _lib = lib
    return lib


class GpsError(RuntimeError):
    pass


def check(rc: int, what: str):
    if rc == GPS_OK:
        return
    msg = load().gps_last_error().decode("utf-8", "replace")
    if rc == GPS_ERR_UNSUPPORTED:
        raise NotImplementedError(f"{what}: {msg}")
    if rc == GPS_ERR_ARG:
        raise ValueError(f"{what}: {msg}")
    raise GpsError(f"{what}: {msg}")


def ptr(t):
    """Device (or host) address of a tensor, 0 for None."""
    return 0 if t is None else t.data_ptr()
