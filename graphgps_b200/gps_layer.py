"""H100-native drop-in for `graphgps.layer.gps_layer.GPSLayer`.

Same constructor signature, `forward(batch) -> batch` contract and `state_dict` layout as the
reference module (graphgps/layer/gps_layer.py:16-264; parameter names per SURVEY.md section 8b), so
`graphgps/network/gps_model.py:85-99` can instantiate it unchanged and reference checkpoints load
with `load_state_dict`.  All arithmetic of the layer — the five GatedGCN projections, the
CSR/CSC segmented gather-reduce, softmax attention over each graph's node set, residual/BatchNorm/FFN
and the whole backward pass — runs in hand-written CUDA (libgps_b200.so, sm_90a) reached through
one C-ABI call per direction; PyTorch only owns memory, streams and the autograd graph edge.
There is NO fallback: CPU tensors or a missing library raise.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from . import _lib
from .bigbird import BigBirdConfig, BigBirdParams, device_lists, gps_bigbird, padded_length
from ._call import _drop_counters  # noqa: F401  (the dropout counters, reachable here as before)
from ._call import (LayerFn, PlanCache, check_params, linear, read_attn_bias, read_x, weight_planes,
                    zeroed_grads)
from .graph import _cache_get, _cache_put, graph_of

_SUPPORTED_LOCAL = ("None", "CustomGatedGCN", "GINE", "GCN", "GAT", "GENConv", "PNA")
# local models that read batch.edge_attr (gps_layer.py:44-90)
_EDGE_LOCAL = ("CustomGatedGCN", "GINE", "GAT", "GENConv", "PNA")
_KNOWN_LOCAL = _SUPPORTED_LOCAL + ("GIN",)
_SUPPORTED_GLOBAL = ("None", "Transformer", "BiasedTransformer", "Performer", "BigBird")
_KNOWN_GLOBAL = _SUPPORTED_GLOBAL
_MHA_GLOBAL = ("Transformer", "BiasedTransformer")   # torch's MultiheadAttention (gps_layer.py:104-106)
# the library's global model: BiasedTransformer is the Transformer with GpsLayerArgs.attn_bias set
_GLOBAL_ABI = dict(_lib.GLOBAL, BiasedTransformer=_lib.GLOBAL["Transformer"])
_ACT_MODULES = {"relu": nn.ReLU, "gelu": nn.GELU}

_PLANES_ATTR = "_gps_b200_planes"


class _GatedGCNParams(nn.Module):
    """Parameter container with the names of graphgps/layer/gatedgcn_layer.py:21-38."""

    def __init__(self, dim, act="relu", equivstable_pe=False):
        super().__init__()
        self.A = nn.Linear(dim, dim, bias=True)
        self.B = nn.Linear(dim, dim, bias=True)
        self.C = nn.Linear(dim, dim, bias=True)
        self.D = nn.Linear(dim, dim, bias=True)
        self.E = nn.Linear(dim, dim, bias=True)
        if equivstable_pe:   # EquivStableLapPE edge gate, gatedgcn_layer.py:29-35
            self.mlp_r_ij = nn.Sequential(nn.Linear(1, dim), _ACT_MODULES[act](), nn.Linear(dim, 1), nn.Sigmoid())
        self.bn_node_x = nn.BatchNorm1d(dim)
        self.bn_edge_e = nn.BatchNorm1d(dim)


class _GINEParams(nn.Module):
    """Names of PyG GINEConv(gin_nn) as built at gps_layer.py:62-69: nn.0, nn.2, eps buffer."""

    def __init__(self, dim, act):
        super().__init__()
        self.nn = nn.Sequential(nn.Linear(dim, dim), _ACT_MODULES[act](), nn.Linear(dim, dim))
        self.register_buffer("eps", torch.Tensor([0.0]))


class _GCNConvParams(nn.Module):
    """Names of PyG 2.2 GCNConv(dim_h, dim_h) as built at gps_layer.py:49-51: lin.weight (no bias, glorot), bias (zeros)."""

    def __init__(self, dim):
        super().__init__()
        self.lin = nn.Linear(dim, dim, bias=False)
        nn.init.xavier_uniform_(self.lin.weight)       # PyG Linear(weight_initializer='glorot')
        self.bias = nn.Parameter(torch.zeros(dim))


def _glorot_(t):
    """PyG inits.glorot: U(-a, a), a = sqrt(6 / (size(-2) + size(-1)))."""
    a = math.sqrt(6.0 / (t.size(-2) + t.size(-1)))
    with torch.no_grad():
        t.uniform_(-a, a)
    return t


class _GATConvParams(nn.Module):
    """Names of PyG 2.2 GATConv(dim_h, dim_h // heads, heads=heads, edge_dim=dim_h) as built at gps_layer.py:70-74:
    lin_src.weight [d,d] and lin_edge.weight [d,d] (no bias, glorot), att_src / att_dst / att_edge [1,H,C] (glorot over
    (H, C)), bias [d] (zeros).  lin_dst is the same module as lin_src, so state_dict() holds both lin_src.weight and
    lin_dst.weight while named_parameters() yields lin_src.weight only."""

    def __init__(self, dim, heads):
        super().__init__()
        C = dim // heads
        self.lin_src = nn.Linear(dim, heads * C, bias=False)
        self.lin_dst = self.lin_src
        self.att_src = nn.Parameter(torch.empty(1, heads, C))
        self.att_dst = nn.Parameter(torch.empty(1, heads, C))
        self.lin_edge = nn.Linear(dim, heads * C, bias=False)
        self.att_edge = nn.Parameter(torch.empty(1, heads, C))
        self.bias = nn.Parameter(torch.zeros(heads * C))
        for t in (self.lin_src.weight, self.lin_edge.weight, self.att_src, self.att_dst, self.att_edge):
            _glorot_(t)


class _GENConvParams(nn.Module):
    """Names of PyG 2.2 GENConv(dim_h, dim_h) as built at gps_layer.py:60-61 (softmax aggregation with t = 1 as a Python
    float, so no parameters of its own; no lin_src / lin_dst / lin_edge / lin_aggr_out since in == out and edge_dim is
    None): mlp = Linear(d, 2d, bias=False), BatchNorm1d(2d), ReLU, Dropout(0), Linear(2d, d, bias=False), i.e. the keys
    mlp.0.weight, mlp.1.{weight, bias, running_mean, running_var, num_batches_tracked}, mlp.4.weight.  The MLP's
    activation is ReLU whatever gnn.act is."""

    def __init__(self, dim):
        super().__init__()
        self.mlp = nn.Sequential(nn.Linear(dim, 2 * dim, bias=False), nn.BatchNorm1d(2 * dim), nn.ReLU(),
                                 nn.Dropout(0.0), nn.Linear(2 * dim, dim, bias=False))


class _PNAConvParams(nn.Module):
    """Names of PyG 2.2 PNAConv(dim_h, dim_h, aggregators=['mean', 'max', 'sum'], scalers=['identity'], deg,
    edge_dim=min(128, dim_h), towers=1, pre_layers=1, post_layers=1, divide_input=False) as built at gps_layer.py:75-90:
    edge_encoder [d, de], pre_nns.0.0 [d, 3d], post_nns.0.0 [d, 4d] and lin [d, d], all with bias and torch's default
    Linear initialisation (PyG's Linear without initialisers).  DegreeScalerAggregation keeps the average degrees as a
    Python dict, so there are no buffers; with the identity scaler the histogram does not enter the arithmetic."""

    def __init__(self, dim, pna_degrees):
        super().__init__()
        self.edge_dim = min(128, dim)
        self.deg = [int(v) for v in pna_degrees]
        self.edge_encoder = nn.Linear(self.edge_dim, dim)
        self.pre_nns = nn.ModuleList([nn.Sequential(nn.Linear(3 * dim, dim))])
        self.post_nns = nn.ModuleList([nn.Sequential(nn.Linear(4 * dim, dim))])
        self.lin = nn.Linear(dim, dim)


def _pna_histogram(pna_degrees):
    """cfg.gt.pna_degrees as a list of counts; NotImplementedError where the reference cannot build PNAConv."""
    if pna_degrees is None:
        raise NotImplementedError(
            "PNA needs pna_degrees (cfg.gt.pna_degrees, the in-degree histogram): the reference fails to construct "
            "the layer without it (torch.from_numpy(np.array(None)) raises TypeError, gps_layer.py:80)")
    deg = torch.as_tensor(pna_degrees).flatten()
    if deg.numel() == 0 or bool((deg < 0).any()) or float(deg.sum()) == 0:
        raise NotImplementedError(
            "PNA needs a non-empty in-degree histogram with non-negative counts and a positive total: PNAConv divides "
            f"by the number of nodes it counts when it builds its average degrees (got {deg.tolist()})")
    return deg.tolist()


def _orthogonal_gaussian_matrix(nb_rows, nb_cols):
    """Random-feature projection drawn once at construction (performer_layer.py:163-195, scaling=0)."""
    blocks = []
    full = nb_rows // nb_cols
    for _ in range(full):
        q, _r = torch.linalg.qr(torch.randn(nb_cols, nb_cols), mode="reduced")
        blocks.append(q.t())
    rem = nb_rows - full * nb_cols
    if rem > 0:
        q, _r = torch.linalg.qr(torch.randn(nb_cols, nb_cols), mode="reduced")
        blocks.append(q.t()[:rem])
    final = torch.cat(blocks)
    mult = torch.randn(nb_rows, nb_cols).norm(dim=1)
    return torch.diag(mult) @ final


class _FastAttentionParams(nn.Module):
    def __init__(self, dim_head):
        super().__init__()
        nb = int(dim_head * math.log(dim_head))  # performer_layer.py:261
        self.register_buffer("projection_matrix", _orthogonal_gaussian_matrix(nb, dim_head))


class _PerformerParams(nn.Module):
    """Names of performer_pytorch.SelfAttention as built at gps_layer.py:111-114
    (dim_head=64, qkv_bias=False, attn_out_bias=True; performer_layer.py:421-474)."""

    def __init__(self, dim, heads, dim_head=64):
        super().__init__()
        inner = dim_head * heads
        self.heads, self.dim_head = heads, dim_head
        self.fast_attention = _FastAttentionParams(dim_head)
        self.to_q = nn.Linear(dim, inner, bias=False)
        self.to_k = nn.Linear(dim, inner, bias=False)
        self.to_v = nn.Linear(dim, inner, bias=False)
        self.to_out = nn.Linear(inner, dim, bias=True)


class GPSLayer(nn.Module):
    """Local MPNN + full graph attention x-former layer (reference: gps_layer.py:16-264)."""

    def __init__(self, dim_h, local_gnn_type, global_model_type, num_heads, act="relu",
                 pna_degrees=None, equivstable_pe=False, dropout=0.0, attn_dropout=0.0,
                 layer_norm=False, batch_norm=True, bigbird_cfg=None, log_attn_weights=False,
                 precision="fp32"):
        super().__init__()
        self.dim_h = dim_h
        self.num_heads = num_heads
        self.attn_dropout = attn_dropout
        self.dropout = dropout
        self.layer_norm = layer_norm
        self.batch_norm = batch_norm
        self.equivstable_pe = equivstable_pe
        self.act = act
        self.precision = precision
        if act not in _ACT_MODULES:
            raise NotImplementedError(f"activation '{act}' is not built in graphgps_b200 (relu, gelu)")
        self.activation = _ACT_MODULES[act]
        self.log_attn_weights = log_attn_weights
        if log_attn_weights and global_model_type not in ["Transformer", "BiasedTransformer"]:
            raise NotImplementedError(                                    # gps_layer.py:36-41
                f"Logging of attention weights is not supported "
                f"for '{global_model_type}' global attention model.")
        if log_attn_weights:
            raise NotImplementedError("log_attn_weights is not built in graphgps_b200")

        # ---- local message-passing model (gps_layer.py:44-99)
        self.local_gnn_with_edge_attr = True
        if local_gnn_type not in _KNOWN_LOCAL:
            raise ValueError(f"Unsupported local GNN model: {local_gnn_type}")
        if local_gnn_type not in _SUPPORTED_LOCAL:
            raise NotImplementedError(f"local GNN '{local_gnn_type}' is not built in graphgps_b200 "
                                      f"(available: {_SUPPORTED_LOCAL}); there is no fallback path")
        if equivstable_pe and local_gnn_type == "GINE":
            raise NotImplementedError(
                "GINE with equivstable_pe=True is not built in graphgps_b200: the reference itself fails to construct "
                "it (GINEConvESLapPE.__init__ calls reset_parameters(), which reads self.mlp_r_ij before it is defined: "
                "gine_conv_layer.py:35,44 raise AttributeError)")
        if equivstable_pe and local_gnn_type == "GENConv":
            raise NotImplementedError(
                "GENConv with equivstable_pe=True is not built in graphgps_b200: the reference passes "
                "batch.pe_EquivStableLapPE as GENConv.forward's fourth positional parameter, which is `size` "
                "(gps_layer.py:176-181), so there is no defined behaviour to match")
        if equivstable_pe and local_gnn_type == "PNA":
            raise NotImplementedError(
                "PNA with equivstable_pe=True is not built in graphgps_b200: the reference passes "
                "batch.pe_EquivStableLapPE as a fourth positional argument to PNAConv.forward(x, edge_index, edge_attr), "
                "which fails (gps_layer.py:176-181)")
        # EquivStableLapPE gate: read by GatedGCN only; GCN and None ignore the flag (gps_layer.py:176-187)
        self._eslap = bool(equivstable_pe) and local_gnn_type == "CustomGatedGCN"
        if local_gnn_type == "None":
            self.local_model = None
        elif local_gnn_type == "GINE":
            self.local_model = _GINEParams(dim_h, act)
        elif local_gnn_type == "GCN":
            self.local_gnn_with_edge_attr = False
            self.local_model = _GCNConvParams(dim_h)
        elif local_gnn_type == "GAT":
            # the reference builds GATConv(out_channels=dim_h // num_heads) and only fails at the residual add
            if num_heads < 1 or dim_h % num_heads != 0:
                raise ValueError(f"GAT needs dim_h ({dim_h}) divisible by num_heads ({num_heads})")
            self.local_model = _GATConvParams(dim_h, num_heads)
        elif local_gnn_type == "GENConv":
            self.local_model = _GENConvParams(dim_h)
        elif local_gnn_type == "PNA":
            self.local_model = _PNAConvParams(dim_h, _pna_histogram(pna_degrees))
        else:
            self.local_model = _GatedGCNParams(dim_h, act, self._eslap)
        self.local_gnn_type = local_gnn_type

        # ---- global attention model (gps_layer.py:101-122)
        if global_model_type not in _KNOWN_GLOBAL:
            raise ValueError(f"Unsupported global x-former model: {global_model_type}")
        if global_model_type not in _SUPPORTED_GLOBAL:
            raise NotImplementedError(f"global model '{global_model_type}' is not built in graphgps_b200")
        if global_model_type == "None":
            self.self_attn = None
        elif global_model_type == "BigBird":
            if bigbird_cfg is None:
                raise NotImplementedError(
                    "GPSLayer('BigBird') needs bigbird_cfg (cfg.gt.bigbird): the reference writes dim_hidden, n_heads "
                    "and dropout into it (gps_layer.py:116-118) and fails with AttributeError on None")
            # the reference's own mutation of the caller's config (gps_layer.py:116-118)
            bigbird_cfg.dim_hidden = dim_h
            bigbird_cfg.n_heads = num_heads
            bigbird_cfg.dropout = dropout
            bb_cfg = BigBirdConfig(bigbird_cfg)
            bb_cfg.check()
            if num_heads < 1 or dim_h % num_heads != 0:
                raise ValueError(f"BigBird needs dim_h ({dim_h}) divisible by num_heads ({num_heads})")
            # attn_dropout is accepted and not read, as in the reference (BigBird attention has no dropout)
            self.self_attn = BigBirdParams(dim_h, num_heads, bb_cfg)
        elif global_model_type in _MHA_GLOBAL:
            if dim_h % num_heads != 0:
                raise ValueError("embed_dim must be divisible by num_heads")
            # torch's own module is the parameter container (same init, same state_dict keys);
            # its forward is never called.
            self.self_attn = nn.MultiheadAttention(dim_h, num_heads, dropout=attn_dropout, batch_first=True)
        else:
            self.self_attn = _PerformerParams(dim_h, num_heads)
        self.global_model_type = global_model_type

        if self.layer_norm and self.batch_norm:
            raise ValueError("Cannot apply two types of normalization together")   # gps_layer.py:125-126
        if self.layer_norm:
            raise NotImplementedError("graphgps_b200 does not build PyG graph LayerNorm (layer_norm=True); "
                                      "batch_norm=True and batch_norm=False are built")
        if self.local_model is None and self.self_attn is None:
            raise ValueError("GPSLayer needs a local model or a global model")
        # batch_norm=False: norm1_local / norm1_attn / norm2 do not exist, as in the reference (gps_layer.py:128-151)
        if self.batch_norm:
            self.norm1_local = nn.BatchNorm1d(dim_h)
            self.norm1_attn = nn.BatchNorm1d(dim_h)
        self.ff_linear1 = nn.Linear(dim_h, dim_h * 2)
        self.ff_linear2 = nn.Linear(dim_h * 2, dim_h)
        if self.batch_norm:
            self.norm2 = nn.BatchNorm1d(dim_h)
        self._param_names = [n for n, _ in self.named_parameters()]
        self._grad_shapes = [tuple(p.shape) for _, p in self.named_parameters()]
        self._grad_sizes = [p.numel() for _, p in self.named_parameters()]
        self._grad_numel = sum(self._grad_sizes)
        self._plans = PlanCache(self._entry, _lib.GpsLayerPlan)

    # ------------------------------------------------------------------ hooks of _call.LayerFn
    _entry = "gps_layer"
    _check_params = check_params

    def _dropout_live(self):
        return self.dropout > 0 or self.attn_dropout > 0

    def _args(self, call, inputs, named, grads=None):
        """GpsLayerArgs with configuration, graph, parameter (+gradient) and per-batch pointers filled in.

        The forward-direction struct (no gradient pointers) only depends on the parameter addresses and the
        module flags, so it is cached and copied; building ~30 nested ctypes structs per call costs more host
        time than the GPU needs for the whole layer at the ZINC shape.  The per-batch fields never enter the cache:
        the EquivStableLapPE pointer, the BiasedTransformer's attention bias and BigBird's block count and lists."""
        x, e, pe, bias = inputs
        pe_k = pe.shape[1] if self._eslap else 0
        if grads is None:
            key = (tuple(t.data_ptr() for t in named.values()), self.training, self.precision,
                   float(self.dropout), float(self.attn_dropout), pe_k > 0, pe_k)
            cached = self.__dict__.get("_args_cache")
            if cached is None or cached[0] != key:
                self._check_params(named)
                cached = (key, self._build_args(named, None, pe_k))
                self.__dict__["_args_cache"] = cached
            a = _lib.GpsLayerArgs.from_buffer_copy(cached[1])
        else:
            a = self._build_args(named, grads, pe_k)
        a.graph = call["gs"].desc
        if self._eslap:
            a.pe = pe.data_ptr()
        if call["nmax"]:
            a.attn_bias = _lib.GpsAttnBias(bias.data_ptr(), call["nmax"], 0)
        if call["bb"] is not None:
            lists, nb = call["bb"]
            b = a.bigbird   # a view into a
            b.num_blocks = nb
            b.key_ptr, b.key_idx, b.query_ptr, b.query_idx = (t.data_ptr() for t in lists)
        return a

    def _plan(self, args, call):
        """gps_layer_plan is pure in (config, N, E, B, training, precision, PE width)."""
        gs = call["gs"]
        return self._plans((gs.N, gs.E, gs.B, bool(self.training), self.precision, float(self.dropout),
                            float(self.attn_dropout), bool(args.pe), int(args.pe_dim)), args)

    def _bind_forward(self, args, call, inputs, plan, params):
        x, e = inputs[:2]
        x_out = torch.empty_like(x)
        e_out = torch.empty_like(e) if self.local_gnn_type == "CustomGatedGCN" else None
        args.x, args.edge_attr = x.data_ptr(), _lib.ptr(e)
        args.x_out, args.edge_out = x_out.data_ptr(), _lib.ptr(e_out)
        hand = self._handoff_args(args, plan, params, call, x, e, x_out, e_out)
        return ((x_out,) if e_out is None else (x_out, e_out)), (), hand

    def _grads(self, named):
        bucket = self._bucket_grads(named)
        if bucket is not None:
            # static gradient bucket (graphgps_b200.dp.GradBucket): the library ADDS this call's gradients to the
            # parameters' .grad views in place (torch's accumulation semantics), so CUDA-graph replays and the
            # gradient all-reduce see the same memory
            return bucket, _lib.FLAG_GRADS_ACCUMULATE, (None,) * len(self._param_names)
        grads = zeroed_grads(named)
        # parameters the configuration never reads get no gradient (as under autograd in the reference)
        unused = []
        if self.local_gnn_type == "None":
            unused.append("norm1_local.")
        if self.global_model_type == "None":
            unused.append("norm1_attn.")
        pg = tuple(None if any(n.startswith(u) for u in unused) else grads[n] for n in self._param_names)
        return grads, _lib.FLAG_GRADS_ZEROED, pg

    def _bind_backward(self, args, call, inputs, g_outs, needs, hand):
        x, e, pe, bias = inputs
        g_pe = torch.empty_like(pe) if self._eslap and needs[2] else None
        g_bias = torch.empty_like(bias) if call["nmax"] and needs[3] else None
        g_x = torch.empty_like(x)
        g_e = torch.empty_like(e) if self.local_gnn_type in _EDGE_LOCAL else None
        args.grad_pe = _lib.ptr(g_pe)
        args.attn_bias.grad_bias = _lib.ptr(g_bias)
        args.x, args.edge_attr = x.data_ptr(), _lib.ptr(e)
        args.grad_x_out = g_outs[0].data_ptr()
        args.grad_edge_out = _lib.ptr(g_outs[1]) if self.local_gnn_type == "CustomGatedGCN" else 0
        args.grad_x, args.grad_edge_attr = g_x.data_ptr(), _lib.ptr(g_e)
        if hand is not None:
            args.x_planes_in, args.e_planes_in, args.wplanes, args.wplanes_bytes = hand[:4]
            args.wplanes_valid = 1
        evs = self.__dict__.get("grad_events")
        if evs is not None:
            args.ev_grads_early, args.ev_grads_mid, args.ev_grads_done = (ev.cuda_event for ev in evs)
        return (g_x, g_e, g_pe, g_bias), ()

    # ------------------------------------------------------------------ operand planes across layers / steps
    def _handoff_args(self, args, plan, params, call, x, e, x_out, e_out):
        """Fills the plane fields: (i) the bf16 hi/lo planes of x / edge_attr that the previous GPSLayer of the
        model wrote next to its outputs (gps_model.py:100,105-108 chains the layers on one batch object), so this layer
        skips converting its inputs; (ii) plane buffers for this layer's own outputs; (iii) the persistent weight-plane
        buffer (_call.weight_planes).  Returns what backward needs to see again, and keeps the buffers alive through
        the autograd node."""
        src = call.pop("planes_in") or {}
        if plan[2] <= 0 or not self.__dict__.get("plane_handoff", True):
            return None
        dev = x.device
        lo = self.precision == "fp32"

        def planes_of(t):
            buf = torch.empty((2 if lo else 1, t.shape[0], (t.shape[1] + 7) // 8 * 8), dtype=torch.bfloat16, device=dev)
            return buf, _lib.GpsPlanes(buf[0].data_ptr(), buf[1].data_ptr() if lo else 0, buf.shape[2])

        keep = []
        zero = _lib.GpsPlanes(0, 0, 0)
        xin, ein = zero, zero
        for name, t in (("x", x), ("e", e)):
            h = src.get(name)
            if h is not None and h[0] == (t.data_ptr(), t._version, tuple(t.shape), lo):
                keep.append(h[1])
                pl = _lib.GpsPlanes(h[1][0].data_ptr(), h[1][1].data_ptr() if lo else 0, h[1].shape[2])
                if name == "x":
                    xin = pl
                else:
                    ein = pl
        args.x_planes_in, args.e_planes_in = xin, ein
        out = {}
        xb, args.x_planes_out = planes_of(x_out)
        out["x"] = (x_out, xb)
        if e_out is not None:
            eb, args.e_planes_out = planes_of(e_out)
            out["e"] = (e_out, eb)
        call["planes_out"] = out
        keep.append(weight_planes(self, args, plan[2], params, dev))
        return (xin, ein, args.wplanes, args.wplanes_bytes, keep)

    def _bucket_grads(self, named):
        """{name: .grad view} when every parameter's .grad is a view of this layer's static bucket, else None."""
        b = self.__dict__.get("_grad_bucket")
        if b is None:
            return None
        lo, hi = b
        out = {}
        for n, p in self.named_parameters():
            g = p.grad
            if g is None or not (lo <= g.data_ptr() < hi) or not g.is_contiguous():
                return None
            out[n] = g
        return out

    # ------------------------------------------------------------------------------------
    def _build_args(self, named, grads, pe_k=0):
        g = grads or {}
        a = _lib.GpsLayerArgs()
        a.d, a.heads = self.dim_h, self.num_heads
        a.local_type = _lib.LOCAL[self.local_gnn_type]
        a.global_type = _GLOBAL_ABI[self.global_model_type]
        a.act = _lib.ACT[self.act]
        a.training = 1 if self.training else 0
        a.precision = _lib.PRECISION[self.precision]
        a.dropout, a.attn_dropout = float(self.dropout), float(self.attn_dropout)
        a.norm_type = _lib.NORM["batch" if self.batch_norm else "none"]

        def lin(prefix, bias=True):
            return linear(named[prefix + ".weight"], named.get(prefix + ".bias") if bias else None,
                        g.get(prefix + ".weight"), g.get(prefix + ".bias") if bias else None)

        def bn(prefix, mod):
            return _lib.GpsBatchNorm(_lib.ptr(named[prefix + ".weight"]), _lib.ptr(named[prefix + ".bias"]),
                                     _lib.ptr(mod.running_mean), _lib.ptr(mod.running_var),
                                     _lib.ptr(mod.num_batches_tracked),
                                     _lib.ptr(g.get(prefix + ".weight")), _lib.ptr(g.get(prefix + ".bias")))

        if self.local_gnn_type == "CustomGatedGCN":
            a.gcn_A, a.gcn_B, a.gcn_C = lin("local_model.A"), lin("local_model.B"), lin("local_model.C")
            a.gcn_D, a.gcn_E = lin("local_model.D"), lin("local_model.E")
            a.bn_node_x = bn("local_model.bn_node_x", self.local_model.bn_node_x)
            a.bn_edge_e = bn("local_model.bn_edge_e", self.local_model.bn_edge_e)
            if self._eslap:   # the PE pointer itself is set per call
                a.pe_dim = pe_k
                a.pe_mlp0, a.pe_mlp1 = lin("local_model.mlp_r_ij.0"), lin("local_model.mlp_r_ij.2")
        elif self.local_gnn_type == "GINE":
            a.gine_lin0, a.gine_lin1 = lin("local_model.nn.0"), lin("local_model.nn.2")
            a.gine_eps = float(self._gine_eps_host)
        elif self.local_gnn_type == "GCN":
            a.gcn_conv = linear(named["local_model.lin.weight"], named["local_model.bias"],
                              g.get("local_model.lin.weight"), g.get("local_model.bias"))
        elif self.local_gnn_type == "GAT":   # lin_src carries GATConv.bias, as GCNConv's lin / bias pair
            p = "local_model."
            a.gat = _lib.GpsGat(
                linear(named[p + "lin_src.weight"], named[p + "bias"], g.get(p + "lin_src.weight"), g.get(p + "bias")),
                lin(p + "lin_edge", False),
                *(_lib.ptr(named[p + n]) for n in ("att_src", "att_dst", "att_edge")),
                *(_lib.ptr(g.get(p + n)) for n in ("att_src", "att_dst", "att_edge")))
        elif self.local_gnn_type == "GENConv":
            a.genconv = _lib.GpsGenConv(lin("local_model.mlp.0", False), bn("local_model.mlp.1", self.local_model.mlp[1]),
                                        lin("local_model.mlp.4", False))
        elif self.local_gnn_type == "PNA":
            a.pna = _lib.GpsPna(lin("local_model.edge_encoder"), lin("local_model.pre_nns.0.0"),
                                lin("local_model.post_nns.0.0"), lin("local_model.lin"), self.local_model.edge_dim)
        if self.global_model_type in _MHA_GLOBAL:
            a.attn_in = linear(named["self_attn.in_proj_weight"], named["self_attn.in_proj_bias"],
                             g.get("self_attn.in_proj_weight"), g.get("self_attn.in_proj_bias"))
            a.attn_out = lin("self_attn.out_proj")
        elif self.global_model_type == "Performer":
            a.perf_q, a.perf_k, a.perf_v = (lin("self_attn.to_q", False), lin("self_attn.to_k", False),
                                            lin("self_attn.to_v", False))
            a.attn_out = lin("self_attn.to_out")
            pm = self.self_attn.fast_attention.projection_matrix
            a.perf_proj, a.perf_features, a.perf_dim_head = pm.data_ptr(), pm.shape[0], pm.shape[1]
        elif self.global_model_type == "BigBird":   # num_blocks and the block lists are set per batch
            a.bigbird = gps_bigbird(self.self_attn, named, grads, "self_attn.")
        if self.batch_norm:   # else the three structs stay zero: the library does not read them
            a.norm1_local = bn("norm1_local", self.norm1_local)
            a.norm1_attn = bn("norm1_attn", self.norm1_attn)
            a.norm2 = bn("norm2", self.norm2)
        a.ff1, a.ff2 = lin("ff_linear1"), lin("ff_linear2")
        return a

    def _bigbird_lists(self, x, gs):
        """(block lists, nb) of this batch: nb from Nmax padded to the block size; NotImplementedError (before any
        launch) for a batch the reference cannot run."""
        cfg = self.self_attn.cfg
        nb = padded_length(gs.nmax, cfg.block_size) // cfg.block_size
        lists = device_lists(x.device, nb, self.num_heads, cfg.block_size, cfg.num_random_blocks,
                             cfg.max_position_embeddings)
        return lists, nb

    @property
    def _gine_eps_host(self):
        # eps is a constant buffer (train_eps=False); read once, no per-step sync
        v = self.__dict__.get("_gine_eps_cache")
        if v is None:
            v = float(self.local_model.eps.item())
            self.__dict__["_gine_eps_cache"] = v
        return v

    def forward(self, batch):
        x = read_x(batch, self)
        e = getattr(batch, "edge_attr", None)
        if self.local_gnn_type == "PNA":   # PNAConv(edge_dim=min(128, dim_h)): the edge encoder's input width
            if e is None or e.dim() != 2 or e.shape[-1] != self.local_model.edge_dim:
                raise ValueError(f"PNA reads batch.edge_attr of width min(128, dim_h) = {self.local_model.edge_dim} "
                                 f"(got {None if e is None else tuple(e.shape)})")
        elif self.local_gnn_type in _EDGE_LOCAL:
            if e is None or e.shape[-1] != self.dim_h:
                raise ValueError("Node and edge feature dimensionalities do not match")
        if self.local_gnn_type in _EDGE_LOCAL:
            if e.dtype != torch.float32 or e.device != x.device:
                raise TypeError("batch.edge_attr must be float32 on the device of batch.x")
            e = e.contiguous()
        else:
            e = None
        pe = self._read_pe(batch, x) if self._eslap else None
        gs = graph_of(batch)
        # batch.attn_bias (gps_layer.py:202-204): missing is an AttributeError, as in the reference
        bias = read_attn_bias(batch, x, gs, self, True) if self.global_model_type == "BiasedTransformer" else None
        call = {"gs": gs, "nmax": gs.nmax if bias is not None else 0,
                "bb": self._bigbird_lists(x, gs) if self.global_model_type == "BigBird" else None,
                "planes_in": _cache_get(batch, _PLANES_ATTR, dict)}
        params = [p for _, p in self.named_parameters()]
        empty = x.new_empty(0)
        out = LayerFn.apply(self, call, x, empty if e is None else e, empty if pe is None else pe,
                            empty if bias is None else bias, *params)
        if self.local_gnn_type == "CustomGatedGCN":
            batch.x, batch.edge_attr = out           # gps_layer.py:173-174, :231
        else:
            batch.x = out
        # the operand planes this layer wrote next to its outputs, keyed by the identity (address, version, shape) of
        # the tensors they mirror: the next GPSLayer uses them only if batch.x / batch.edge_attr are still those tensors
        lo = self.precision == "fp32"
        _cache_put(batch, {name: ((t.data_ptr(), t._version, tuple(t.shape), lo), buf)
                           for name, (t, buf) in call.pop("planes_out", {}).items()}, _PLANES_ATTR)
        return batch

    @staticmethod
    def _read_pe(batch, x):
        """batch.pe_EquivStableLapPE [N, k] (gps_layer.py:165-166): float32, on the device of x, one row per node."""
        pe = getattr(batch, "pe_EquivStableLapPE", None)
        if pe is None:
            raise AttributeError("GPSLayer(equivstable_pe=True) reads batch.pe_EquivStableLapPE [num_nodes, k], which "
                                 "this batch does not have (posenc_EquivStableLapPE's node encoder writes it)")
        if not torch.is_tensor(pe) or pe.dtype != torch.float32 or pe.device != x.device:
            raise TypeError("batch.pe_EquivStableLapPE must be a float32 tensor on the device of batch.x (got "
                            f"{getattr(pe, 'dtype', type(pe))} on {getattr(pe, 'device', None)})")
        if pe.dim() != 2 or pe.shape[0] != x.shape[0] or pe.shape[1] < 1:
            raise ValueError(f"batch.pe_EquivStableLapPE must have shape [num_nodes={x.shape[0]}, k >= 1] "
                             f"(got {tuple(pe.shape)})")
        return pe.contiguous()

    def extra_repr(self):
        return (f"summary: dim_h={self.dim_h}, local_gnn_type={self.local_gnn_type}, "
                f"global_model_type={self.global_model_type}, heads={self.num_heads}, "
                f"backend=libgps_b200(sm_90a), precision={self.precision}")
