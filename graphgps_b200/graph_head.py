"""H100-native drop-ins for the graph-prediction heads of the graph-level configs:
`graphgps.head.san_graph.SANGraphHead` (`gnn.head: san_graph`) and `graphgps.head.graphormer_graph.GraphormerHead`
(`gnn.head: graphormer_graph`).

Same `forward(batch)` contract as the reference:

    SANGraphHead     h = pool(batch.x, batch.batch); h = act(FC_l(h)) for l < L; pred = FC_L(h)
    GraphormerHead   pred = layers(pool(ln(batch.x), batch.batch))
    both             batch.graph_feature = pred; return (pred, batch.y)

Pooling: mean (per-graph sum / max(count, 1)), add (per-graph sum), graph_token (each graph's first row, as
`to_dense_batch(x, batch)[:, 0, :]`); an empty graph gives a zero row.  The output has `num_graphs` rows, the count
`graph_of(batch)` reads (PyG's `batch.num_graphs`), which equals the reference's `batch.max() + 1` whenever the last
graph has nodes.  The rows of batch.batch are sorted by graph, as PyG collates them.  LayerNorm is row-wise, so under
graph_token GraphormerHead pools first and normalises the B token rows only; its grad_x is zero off the token rows,
and an empty graph's row is zero after the LayerNorm too, as in the reference (its pred is the bias).

One C call per direction (libgps_b200.so, sm_90a); there is no CPU fallback.  The graph offsets come from the batch's
cached graph structure, so a batch the layers already ran on costs no host read and the head can be captured in the
same CUDA graph as they are.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _lib
from ._call import LayerFn, PlanCache, check_params, linear, read_x
from .graph import graph_of


class _GraphHead(nn.Module):
    """The LayerFn hooks both heads share; subclasses set _kind, _pool, _act, L and their parameters."""

    _entry = "gps_graph_head"

    def _init_common(self, dim_in, dim_out, graph_pooling, precision, pools):
        if graph_pooling not in pools:
            raise NotImplementedError(f"graphgps_b200.{type(self).__name__}: graph_pooling {graph_pooling!r} is not "
                                      f"built ({', '.join(pools)} {'is' if len(pools) == 1 else 'are'})")
        if precision not in _lib.PRECISION:
            raise ValueError(f"precision must be one of {tuple(_lib.PRECISION)} (got {precision!r})")
        if not (1 <= int(dim_in) <= 4096 and 1 <= int(dim_out) <= 4096):
            raise NotImplementedError(f"graphgps_b200.{type(self).__name__}: needs 1 <= dim_in, dim_out <= 4096 "
                                      f"(got {dim_in}, {dim_out})")
        self.dim_in, self.dim_out = int(dim_in), int(dim_out)
        self.graph_pooling, self.precision = graph_pooling, precision

    def _finish_init(self):
        self._param_names = [n for n, _ in self.named_parameters()]
        self._plans = PlanCache(self._entry, _lib.GpsGraphHeadPlan)

    # ------------------------------------------------------------------ hooks of _call.LayerFn
    def _dropout_live(self):
        return False

    def _args(self, gs, inputs, named, grads=None):
        g = grads or {}
        check_params(self, named)
        a = _lib.GpsGraphHeadArgs()
        a.kind, a.pooling, a.act, a.L = self._kind, _lib.POOLING[self.graph_pooling], self._act, self.L
        a.dim_in, a.dim_out = self.dim_in, self.dim_out
        a.training = 1 if self.training else 0
        a.precision = _lib.PRECISION[self.precision]
        a.graph = gs.desc
        a.x = inputs[0].data_ptr()
        for i, (w, b) in enumerate(self._linears()):
            a.fc[i] = linear(named[w], named[b], g.get(w), g.get(b))
        if self._kind == _lib.GRAPH_HEAD["graphormer_graph"]:
            a.ln = linear(named["ln.weight"], named["ln.bias"], g.get("ln.weight"), g.get("ln.bias"))
        return a

    def _plan(self, args, gs):
        return self._plans((gs.N, gs.B, self.precision), args)

    def _bind_forward(self, args, gs, inputs, plan, params):
        pred = torch.empty(gs.B, self.dim_out, dtype=torch.float32, device=inputs[0].device)
        args.pred = pred.data_ptr()
        return (pred,), (), None

    def _grads(self, named):
        grads = {n: torch.empty_like(p) for n, p in named.items()}   # the library writes every gradient whole
        return grads, 0, tuple(grads[n] for n in self._param_names)

    def _bind_backward(self, args, gs, inputs, g_outs, needs, keep):
        g_x = torch.empty_like(inputs[0])
        args.grad_pred, args.grad_x = _lib.ptr(g_outs[0]), g_x.data_ptr()
        return (g_x,), ()

    # ------------------------------------------------------------------ forward
    def forward(self, batch):
        x = read_x(batch, self, self.dim_in)
        bvec = batch.batch
        N = x.shape[0]
        if not torch.is_tensor(bvec) or bvec.dtype != torch.int64 or tuple(bvec.shape) != (N,) or \
                bvec.device != x.device:
            raise ValueError(f"batch.batch must be int64 [num_nodes] = [{N}] on {x.device}")
        gs = graph_of(batch)
        params = [p for _, p in self.named_parameters()]
        pred = LayerFn.apply(self, gs, x, *params)
        batch.graph_feature = pred
        return pred, batch.y

    def extra_repr(self):
        return (f"dim_in={self.dim_in}, dim_out={self.dim_out}, graph_pooling={self.graph_pooling}, "
                f"backend=libgps_b200(sm_90a), precision={self.precision}")


class SANGraphHead(_GraphHead):
    """SAN prediction head for graph prediction tasks (reference: graphgps/head/san_graph.py): pooling, then L hidden
    Linears of widths dim_in // 2**(l+1) with the activation, then a Linear to dim_out."""

    _kind = _lib.GRAPH_HEAD["san_graph"]

    def __init__(self, dim_in, dim_out, L=2, graph_pooling="mean", act="relu", precision="fp32"):
        super().__init__()
        self._init_common(dim_in, dim_out, graph_pooling, precision, ("mean", "add", "graph_token"))
        if act not in _lib.ACT:
            raise NotImplementedError(f"graphgps_b200.SANGraphHead: act {act!r} is not built (relu and gelu are)")
        L = int(L)
        if L < 0 or L > _lib.GRAPH_HEAD_MAX_L or self.dim_in >> L < 1:
            raise NotImplementedError(f"graphgps_b200.SANGraphHead: L={L} leaves a zero width for dim_in "
                                      f"{self.dim_in} (needs dim_in // 2**L >= 1)")
        self.L, self.act, self._act = L, act, _lib.ACT[act]
        # the reference's modules in its order, so the same seed draws the same parameters (san_graph.py:22-28)
        fc = [nn.Linear(self.dim_in // 2 ** l, self.dim_in // 2 ** (l + 1), bias=True) for l in range(L)]
        fc.append(nn.Linear(self.dim_in // 2 ** L, self.dim_out, bias=True))
        self.FC_layers = nn.ModuleList(fc)
        self._finish_init()

    def _linears(self):
        return [(f"FC_layers.{l}.weight", f"FC_layers.{l}.bias") for l in range(self.L + 1)]

    def extra_repr(self):
        return f"L={self.L}, act={self.act}, " + super().extra_repr()


class GraphormerHead(_GraphHead):
    """Graphormer prediction head for graph prediction tasks (reference: graphgps/head/graphormer_graph.py):
    LayerNorm(dim_in), pooling, one Linear to dim_out."""

    _kind = _lib.GRAPH_HEAD["graphormer_graph"]
    _act = 0
    L = 0

    def __init__(self, dim_in, dim_out, graph_pooling="graph_token", precision="fp32"):
        super().__init__()
        self._init_common(dim_in, dim_out, graph_pooling, precision, ("graph_token",))
        if self.dim_in % 4:
            raise NotImplementedError(f"graphgps_b200.GraphormerHead: needs dim_in % 4 == 0 (got {self.dim_in}), as "
                                      "the Graphormer layer does")
        self.ln = nn.LayerNorm(self.dim_in)
        self.layers = nn.Sequential(nn.Linear(self.dim_in, self.dim_out))
        self._finish_init()

    def _linears(self):
        return [("layers.0.weight", "layers.0.bias")]
