"""H100-native drop-in for the inductive link-prediction head of the PCQM-Contact configs,
`graphgps.head.inductive_edge.GNNInductiveEdgeHead` with `edge_decoding: dot` and `layers_post_mp: 1`.

Same `forward(batch)` contract as the reference:

    batch.x = y = x W^T + b                           (layer_post_mp, GraphGym's one-layer MLP)
    pred[k] = <y[s_k], y[t_k]>                        (s_k, t_k) = batch.edge_index_labeled[:, k]
    training: returns (pred, batch.edge_label)
    eval:     returns (pred, batch.edge_label, {'hits@1', 'hits@3', 'hits@10', 'mrr'})

The eval statistics are computed on the device and read with one device-to-host copy per batch.  For a positive pair
(i, j) (edge_label == 1) of a graph, the candidates are every node k != j of that graph, and
rank = 1 + #{k : <y_i, y_k> > <y_i, y_j>}: the rank a stable descending sort gives, so a tie counts in the positive's
favour (the reference's unstable argsort leaves ties implementation-defined; tie-free inputs agree exactly).  A graph's
four values are the means over its positives of rank <= 1, <= 3, <= 10 and 1 / rank, 0 for a graph without positives,
and the batch's are the means over its graphs.

One C call per direction (libgps_b200.so, sm_90a); there is no CPU fallback.  The labeled pairs are checked and built
into a CSR / CSC once per batch object with one host read, and cached on it, so a training step can be captured in a
CUDA graph after that first call.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _lib
from ._call import LayerFn, PlanCache, check_params, linear, read_x
from .graph import GraphStructure, _cache_get, _cache_put, _num_graphs

_META_ATTR = "_gps_b200_link_pairs"
_STATS = ("hits@1", "hits@3", "hits@10", "mrr")


class _PairMeta:
    """The labeled pairs of one batch: their CSR / CSC and graph offsets (None when out of range), the number of
    out-of-range pairs and the number of positives whose nodes lie in different graphs."""

    def __init__(self, key, gs, bad, cross):
        self.key, self.gs, self.bad, self.cross = key, gs, bad, cross


def _key(*ts):
    return tuple((t.data_ptr(), t._version, tuple(t.shape)) for t in ts)


def _pair_meta(batch, eli, label, bvec, N):
    key = _key(eli, label, bvec)
    hit = _cache_get(batch, _META_ATTR, _PairMeta)
    if hit is not None and hit.key == key:
        return hit
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError("graphgps_b200.InductiveEdgeHead checks the labeled pairs on the host once per batch and "
                           "cannot do so inside a CUDA-graph capture: run the head on this batch once before capturing")
    K = eli.shape[1]
    bad = cross = 0
    if K and N == 0:
        bad = K
    elif K:
        out = ((eli < 0) | (eli >= N)).any(0)
        s, t = eli[0].clamp(0, N - 1), eli[1].clamp(0, N - 1)
        pos_cross = (label == 1) & (bvec[s] != bvec[t]) & ~out
        bad, cross = torch.stack([out.sum(), pos_cross.sum()]).tolist()   # the one host read per batch
    gs = None if bad else GraphStructure(eli, bvec, _num_graphs(batch))
    meta = _PairMeta(key, gs, int(bad), int(cross))
    _cache_put(batch, meta, _META_ATTR)
    return meta


class _GymLinear(nn.Module):
    """torch_geometric.graphgym.models.layer.Linear: the parameters live in its `model` (torch_geometric.nn.Linear)."""

    def __init__(self, dim):
        super().__init__()
        self.model = nn.Linear(dim, dim, bias=True)


class _GymMLP(nn.Module):
    """torch_geometric.graphgym.models.layer.MLP with one layer: `model` is a Sequential holding that Linear."""

    def __init__(self, dim):
        super().__init__()
        self.model = nn.Sequential(_GymLinear(dim))


class _Call:
    """Per-call state of LayerFn: the batch's pair structure and the index tensors."""

    def __init__(self, meta, eli, label):
        self.meta, self.eli, self.label = meta, eli, label


class InductiveEdgeHead(nn.Module):
    """Inductive link-prediction head (reference: graphgps/head/inductive_edge.py, GNNInductiveEdgeHead)."""

    _entry = "gps_link_head"

    def __init__(self, dim_in, dim_out, edge_decoding="dot", layers_post_mp=1, precision="fp32"):
        super().__init__()
        # the reference's checks in its order (inductive_edge.py:22-44)
        if edge_decoding == "concat":
            raise NotImplementedError("graphgps_b200.InductiveEdgeHead: edge_decoding 'concat' is not built (dot is)")
        if dim_out > 1:
            raise ValueError(f"Binary edge decoding ({edge_decoding})is used for multi-class edge/link prediction.")
        if edge_decoding == "cosine_similarity":
            raise NotImplementedError("graphgps_b200.InductiveEdgeHead: edge_decoding 'cosine_similarity' is not built "
                                      "(dot is; the reference's compute_mrr refuses it as well)")
        if edge_decoding != "dot":
            raise ValueError(f"Unknown edge decoding {edge_decoding}.")
        if layers_post_mp != 1:
            raise NotImplementedError(f"graphgps_b200.InductiveEdgeHead: layers_post_mp={layers_post_mp} is not built "
                                      "(1 is, as every PCQM-Contact config sets)")
        if precision not in _lib.PRECISION:
            raise ValueError(f"precision must be one of {tuple(_lib.PRECISION)} (got {precision!r})")
        if not 1 <= int(dim_in) <= 4096:
            raise NotImplementedError(f"graphgps_b200.InductiveEdgeHead: needs 1 <= dim_in <= 4096 (got {dim_in})")
        self.dim_in, self.dim_out = int(dim_in), int(dim_out)
        self.edge_decoding, self.precision = edge_decoding, precision
        self.layer_post_mp = _GymMLP(self.dim_in)
        self._param_names = [n for n, _ in self.named_parameters()]
        self._plans = PlanCache(self._entry, _lib.GpsLinkHeadPlan)

    # ------------------------------------------------------------------ hooks of _call.LayerFn
    def _dropout_live(self):
        return False

    def _args(self, call, inputs, named, grads=None):
        g = grads or {}
        check_params(self, named)
        w, b = self._param_names
        a = _lib.GpsLinkHeadArgs()
        a.d = self.dim_in
        a.training = 1 if self.training else 0
        a.precision = _lib.PRECISION[self.precision]
        a.label_bytes = call.label.element_size()
        a.pairs = call.meta.gs.desc
        a.edge_index_labeled, a.edge_label = call.eli.data_ptr(), call.label.data_ptr()
        a.x = inputs[0].data_ptr()
        a.lin = linear(named[w], named[b], g.get(w), g.get(b))
        return a

    def _plan(self, args, call):
        gs = call.meta.gs
        return self._plans((gs.N, gs.E, gs.B, self.precision, bool(args.training)), args)

    def _bind_forward(self, args, call, inputs, plan, params):
        x = inputs[0]
        y = torch.empty_like(x)
        pred = torch.empty(call.eli.shape[1], dtype=torch.float32, device=x.device)
        args.y, args.pred = y.data_ptr(), pred.data_ptr()
        if args.training:
            return (y, pred), (), None
        stats = torch.empty(4, dtype=torch.float64, device=x.device)
        args.stats = stats.data_ptr()
        return (y, pred, stats), (), None

    def _grads(self, named):
        grads = {n: torch.empty_like(p) for n, p in named.items()}   # the library writes both gradients whole
        return grads, 0, tuple(grads[n] for n in self._param_names)

    def _bind_backward(self, args, call, inputs, g_outs, needs, keep):
        g_x = torch.empty_like(inputs[0])
        args.grad_y, args.grad_pred = _lib.ptr(g_outs[0]), _lib.ptr(g_outs[1])
        args.grad_x = g_x.data_ptr()
        return (g_x,), ()

    # ------------------------------------------------------------------ forward
    def forward(self, batch):
        x = read_x(batch, self, self.dim_in)
        eli, label = batch.edge_index_labeled, batch.edge_label
        for name, t in (("edge_index_labeled", eli), ("edge_label", label)):
            if not torch.is_tensor(t) or t.device != x.device:
                raise RuntimeError(f"graphgps_b200.InductiveEdgeHead: batch.{name} must be a tensor on {x.device}; "
                                   "there is no CPU fallback")
        if eli.dtype != torch.int64:
            raise IndexError(f"batch.edge_index_labeled must be int64 (got {eli.dtype})")
        if eli.dim() != 2 or eli.shape[0] != 2:
            raise IndexError(f"batch.edge_index_labeled must have shape [2, K] (got {list(eli.shape)})")
        K = eli.shape[1]
        if label.dtype not in (torch.int32, torch.int64):
            raise TypeError(f"batch.edge_label must be int32 or int64 (got {label.dtype})")
        if tuple(label.shape) != (K,):
            raise ValueError(f"batch.edge_label must have shape [K] = [{K}] (got {list(label.shape)})")
        bvec = batch.batch
        N = x.shape[0]
        if bvec.dtype != torch.int64 or tuple(bvec.shape) != (N,) or bvec.device != x.device:
            raise ValueError(f"batch.batch must be int64 [num_nodes] = [{N}] on {x.device}")
        eli, label = eli.contiguous(), label.contiguous()
        meta = _pair_meta(batch, eli, label, bvec.contiguous(), N)
        if meta.bad:
            raise IndexError(f"edge_index_labeled: {meta.bad} pairs have a node outside [0, {N})")
        if not self.training and meta.cross:
            raise ValueError(f"edge_index_labeled: {meta.cross} positive pairs join nodes of different graphs; the "
                             "ranking metrics rank each positive among the nodes of its own graph")
        params = [p for _, p in self.named_parameters()]
        out = LayerFn.apply(self, _Call(meta, eli, label), x, *params)
        batch.x = out[0]
        if self.training:
            return out[1], batch.edge_label
        stats = out[2].tolist()   # the one device-to-host copy of an eval batch
        return out[1], batch.edge_label, dict(zip(_STATS, stats))

    def extra_repr(self):
        return (f"dim_in={self.dim_in}, dim_out={self.dim_out}, edge_decoding={self.edge_decoding}, "
                f"backend=libgps_b200(sm_90a), precision={self.precision}")
