"""H100-native drop-in for Graphormer's attention-bias encoder, `graphgps.encoder.graphormer_encoder.BiasEncoder`
(graphormer_encoder.py:103-183).

Same constructor, parameter names, shapes and initialisation as the reference, and the same `forward(data) -> data`
contract: it reads graphormer_pre_processing's collated attributes (`spatial_types`, `graph_index`, and
`shortest_path_types` when the dataset has edge attributes) and sets

    data.attn_bias [B * H, N', N'] float32, row b * H + h,   N' = Nmax (+ 1 with the graph token)

the layout GraphormerLayer and GPSLayer's BiasedTransformer read.  One C call per direction (libgps_b200.so, sm_90a);
there is no CPU fallback.  The batch's Nmax and graph count are read from the device once per batch object, together
with the range checks of the index tensors, and cached on it, so a step can be captured in a CUDA graph after that
first call.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from ._call import workspace
from .graph import _cache_get, _cache_put

_META_ATTR = "_gps_b200_bias_meta"


class _BatchMeta:
    """What the encoder reads from the device once per batch: node offsets, graph count, Nmax and index ranges."""

    def __init__(self, key, ptr, nmax, num_graphs, bad_pairs, spatial_range, path_range):
        self.key, self.ptr, self.nmax, self.num_graphs = key, ptr, nmax, num_graphs
        self.bad_pairs, self.spatial_range, self.path_range = bad_pairs, spatial_range, path_range


def _key(*ts):
    return tuple(None if t is None else (t.data_ptr(), t._version, tuple(t.shape)) for t in ts)


def _batch_meta(data, st, gi, spt):
    """Node offsets [>= B+1] on the device and, from one host read, Nmax, B = batch.max() + 1 (to_dense_adj's batch
    size), the number of pairs whose nodes are not both in one graph, and the ranges of the type tensors."""
    bvec = data.batch
    ptr_attr = getattr(data, "ptr", None)
    key = _key(st, gi, spt, bvec, ptr_attr)
    hit = _cache_get(data, _META_ATTR, _BatchMeta)
    if hit is not None and hit.key == key:
        return hit
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError("graphgps_b200.BiasEncoder reads Nmax from the device once per batch and cannot do so inside "
                           "a CUDA-graph capture: run the encoder on this batch once before capturing")
    dev = st.device
    if ptr_attr is not None:
        if ptr_attr.dtype != torch.int64:
            raise TypeError(f"batch.ptr must be int64 (got {ptr_attr.dtype})")
        ptr = ptr_attr.to(dev).contiguous()
    else:
        if bvec.dtype != torch.int64:
            raise TypeError(f"batch.batch must be int64 (got {bvec.dtype})")
        # batch is sorted (PyG collation): ptr[b] = number of nodes of graphs < b, for b = 0 .. N
        ptr = torch.searchsorted(bvec.to(dev).contiguous(), torch.arange(bvec.numel() + 1, device=dev))
    n_nodes = ptr[-1]
    zero = torch.zeros((), dtype=torch.int64, device=dev)
    num_graphs = (ptr[:-1] < n_nodes).sum()
    sizes = ptr[1:] - ptr[:-1]
    stats = [sizes.max() if sizes.numel() else zero, num_graphs]
    P = st.numel()
    if P:
        i, j = gi[0], gi[1]
        g = (torch.searchsorted(ptr, i, right=True) - 1).clamp_(0, ptr.numel() - 2)
        ok = (i >= ptr[0]) & (i < n_nodes) & (j >= ptr[g]) & (j < ptr[g + 1])
        stats += [(~ok).sum(), st.min(), st.max()]
        if spt is not None and spt.numel():
            stats += [spt.min(), spt.max()]
    vals = torch.stack(stats).tolist()   # the one host read per batch
    meta = _BatchMeta(key, ptr, int(vals[0]), int(vals[1]), int(vals[2]) if P else 0,
                      (vals[3], vals[4]) if P else None, (vals[5], vals[6]) if len(vals) > 5 else None)
    _cache_put(data, meta, _META_ATTR)
    return meta


class _BiasFn(torch.autograd.Function):
    """One autograd node: forward = gps_graphormer_bias_forward, backward = gps_graphormer_bias_backward."""

    @staticmethod
    def forward(ctx, enc, meta, st, gi, spt, spatial_w, dis_w, edge_w, token):
        lib = _lib.load()
        npad = meta.nmax + (1 if enc.use_graph_token else 0)
        out = torch.empty(meta.num_graphs * enc.num_heads, npad, npad, dtype=torch.float32, device=st.device)
        args = enc._args(meta, st, gi, spt, spatial_w, dis_w, edge_w, token)
        args.attn_bias = out.data_ptr()
        stream = torch.cuda.current_stream(st.device).cuda_stream
        _lib.check(lib.gps_graphormer_bias_forward(C.byref(args), stream), "gps_graphormer_bias_forward")
        ctx.enc, ctx.meta = enc, meta
        ctx.save_for_backward(st, gi, spt, spatial_w, dis_w, edge_w, token)
        return out

    @staticmethod
    def backward(ctx, g_out):
        lib = _lib.load()
        enc, meta = ctx.enc, ctx.meta
        st, gi, spt, spatial_w, dis_w, edge_w, token = ctx.saved_tensors
        need = ctx.needs_input_grad
        g_out = g_out.contiguous()
        edges = spt is not None
        g_sp = torch.empty_like(spatial_w) if need[5] else None
        g_dis = torch.empty_like(dis_w) if edges and need[6] else None
        g_ew = torch.empty_like(edge_w) if edges and need[7] else None
        g_tok = torch.empty_like(token) if token is not None and need[8] else None
        args = enc._args(meta, st, gi, spt, spatial_w, dis_w, edge_w, token)
        args.grad_attn_bias = g_out.data_ptr()
        args.grad_spatial_weight, args.grad_edge_dis_weight = _lib.ptr(g_sp), _lib.ptr(g_dis)
        args.grad_edge_weight, args.grad_graph_token = _lib.ptr(g_ew), _lib.ptr(g_tok)
        plan = _lib.GpsGraphormerBiasPlan()
        _lib.check(lib.gps_graphormer_bias_plan(C.byref(args), C.byref(plan)), "gps_graphormer_bias_plan")
        ws = workspace(st.device, plan.bwd_workspace_bytes)
        args.workspace, args.workspace_bytes = ws.data_ptr(), ws.numel()
        stream = torch.cuda.current_stream(st.device).cuda_stream
        _lib.check(lib.gps_graphormer_bias_backward(C.byref(args), stream), "gps_graphormer_bias_backward")
        return None, None, None, None, None, g_sp, g_dis, g_ew, g_tok


class BiasEncoder(nn.Module):
    """Graphormer's attention-bias encoder (reference: graphgps/encoder/graphormer_encoder.py:103-183)."""

    def __init__(self, num_heads: int, num_spatial_types: int, num_edge_types: int, use_graph_token: bool = True):
        super().__init__()
        self.num_heads = num_heads
        self.num_spatial_types, self.num_edge_types = num_spatial_types, num_edge_types
        # the reference's modules in its order: same state_dict keys, same draws from the same seed
        self.spatial_encoder = nn.Embedding(num_spatial_types + 1, num_heads)
        self.edge_dis_encoder = nn.Embedding(num_spatial_types * num_heads * num_heads, 1)
        self.edge_encoder = nn.Embedding(num_edge_types, num_heads)
        self.use_graph_token = use_graph_token
        if self.use_graph_token:
            self.graph_token = nn.Parameter(torch.zeros(1, num_heads, 1))
        self.reset_parameters()

    def reset_parameters(self):
        self.spatial_encoder.weight.data.normal_(std=0.02)
        self.edge_encoder.weight.data.normal_(std=0.02)
        self.edge_dis_encoder.weight.data.normal_(std=0.02)
        if self.use_graph_token:
            self.graph_token.data.normal_(std=0.02)

    def _args(self, meta, st, gi, spt, spatial_w, dis_w, edge_w, token):
        a = _lib.GpsGraphormerBiasArgs()
        a.num_pairs, a.num_graphs, a.nmax = st.numel(), meta.num_graphs, meta.nmax
        a.heads, a.num_spatial_types, a.num_edge_types = self.num_heads, self.num_spatial_types, self.num_edge_types
        a.use_graph_token = 1 if self.use_graph_token else 0
        a.spatial_types, a.graph_index, a.node_ptr = st.data_ptr(), gi.data_ptr(), meta.ptr.data_ptr()
        a.shortest_path_types = _lib.ptr(spt)
        a.spatial_weight, a.edge_dis_weight = spatial_w.data_ptr(), dis_w.data_ptr()
        a.edge_weight, a.graph_token = edge_w.data_ptr(), _lib.ptr(token)
        return a

    @staticmethod
    def _index(data, name, required):
        t = getattr(data, name) if required else getattr(data, name, None)   # AttributeError as in the reference
        if t is None:
            return None
        if not torch.is_tensor(t) or not t.is_cuda:
            raise RuntimeError(f"graphgps_b200.BiasEncoder runs on CUDA tensors only; there is no CPU fallback "
                               f"(batch.{name} is on {getattr(t, 'device', type(t))})")
        if t.dtype != torch.int64:
            raise TypeError(f"batch.{name} must be int64 (got {t.dtype})")
        return t.contiguous()

    def forward(self, data):
        st = self._index(data, "spatial_types", True)
        gi = self._index(data, "graph_index", True)
        # the reference tests hasattr(data, "shortest_path_types") (graphormer_encoder.py:156)
        spt = self._index(data, "shortest_path_types", False) if hasattr(data, "shortest_path_types") else None
        params = [self.spatial_encoder.weight, self.edge_dis_encoder.weight, self.edge_encoder.weight]
        if self.use_graph_token:
            params.append(self.graph_token)
        for p in params:
            if not p.is_cuda or p.device != st.device or p.dtype != torch.float32:
                raise RuntimeError(f"graphgps_b200.BiasEncoder: parameters must be float32 on {st.device} (got "
                                   f"{p.dtype} on {p.device}); there is no CPU fallback")
        P, S, T = st.numel(), self.num_spatial_types, self.num_edge_types
        if st.dim() != 1 or tuple(gi.shape) != (2, P):
            raise ValueError(f"spatial_types must be [P] and graph_index [2, P] (got {list(st.shape)} and "
                             f"{list(gi.shape)})")
        if spt is not None and tuple(spt.shape) != (P, S):
            raise ValueError(f"shortest_path_types must be [P, num_spatial_types] = {[P, S]} (got {list(spt.shape)})")
        meta = _batch_meta(data, st, gi, spt)
        if meta.bad_pairs:
            raise IndexError(f"graph_index: {meta.bad_pairs} pairs do not lie within one graph of the batch")
        if meta.spatial_range is not None and (meta.spatial_range[0] < 0 or meta.spatial_range[1] > S):
            raise IndexError(f"spatial_types values {list(meta.spatial_range)} out of range for {S + 1} spatial types")
        if meta.path_range is not None and (meta.path_range[0] < 0 or meta.path_range[1] >= T):
            raise IndexError(f"shortest_path_types values {list(meta.path_range)} out of range for {T} edge types")
        token = self.graph_token if self.use_graph_token else None
        data.attn_bias = _BiasFn.apply(self, meta, st, gi, spt, self.spatial_encoder.weight.contiguous(),
                                       self.edge_dis_encoder.weight.contiguous(), self.edge_encoder.weight.contiguous(),
                                       token)
        return data

    def extra_repr(self):
        return (f"num_heads={self.num_heads}, num_spatial_types={self.num_spatial_types}, "
                f"num_edge_types={self.num_edge_types}, use_graph_token={self.use_graph_token}, "
                "backend=libgps_b200(sm_90a)")
