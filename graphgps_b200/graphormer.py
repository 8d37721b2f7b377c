"""H100-native drop-in for `graphgps.layer.graphormer_layer.GraphormerLayer` (graphormer_layer.py:5-49).

Same constructor, `forward(batch) -> batch` contract and `state_dict` as the reference: the reference's own torch
modules (`attention`, `input_norm`, `dropout`, `mlp`) are built as parameter containers, so checkpoints load strictly and
the same seed gives the same initial values; their `forward` is never called.  The layer computes

    h   = input_norm(x)
    a   = MHA(h, h, h) over each graph's own nodes, + batch.attn_bias after scaling when the batch has one
    x1  = dropout(a) + x
    out = mlp(x1) + x1            mlp = LayerNorm, Linear, GELU, Dropout(mlp_dropout), Linear, Dropout(dropout)

in one C call per direction (libgps_b200.so, sm_90a).  There is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from ._call import LayerFn, PlanCache, check_params, linear, read_attn_bias, read_x, zeroed_grads
from .graph import graph_of


class GraphormerLayer(nn.Module):
    """Graphormer layer (reference: graphgps/layer/graphormer_layer.py:5-49)."""

    def __init__(self, embed_dim: int, num_heads: int, dropout: float, attention_dropout: float, mlp_dropout: float,
                 precision: str = "fp32"):
        super().__init__()
        if precision not in _lib.PRECISION:
            raise ValueError(f"precision must be one of {tuple(_lib.PRECISION)} (got {precision!r})")
        if num_heads < 1 or embed_dim % num_heads != 0:
            raise ValueError("embed_dim must be divisible by num_heads")
        # the reference's modules, in its order (same state_dict keys, same draws from the same seed)
        self.attention = nn.MultiheadAttention(embed_dim, num_heads, attention_dropout, batch_first=True)
        self.input_norm = nn.LayerNorm(embed_dim)
        self.dropout = nn.Dropout(dropout)
        self.mlp = nn.Sequential(
            nn.LayerNorm(embed_dim),
            nn.Linear(embed_dim, embed_dim),
            nn.GELU(),
            nn.Dropout(mlp_dropout),
            nn.Linear(embed_dim, embed_dim),
            nn.Dropout(dropout),
        )
        self.embed_dim, self.num_heads = embed_dim, num_heads
        self.p_dropout, self.p_attn, self.p_mlp = float(dropout), float(attention_dropout), float(mlp_dropout)
        self.precision = precision
        self._param_names = [n for n, _ in self.named_parameters()]
        self._plans = PlanCache(self._entry, _lib.GpsGraphormerPlan)

    # ------------------------------------------------------------------ hooks of _call.LayerFn; call = the graph
    _entry = "gps_graphormer"

    def _dropout_live(self):
        return self.p_dropout > 0 or self.p_attn > 0 or self.p_mlp > 0

    def _args(self, gs, inputs, named, grads=None):
        g = grads or {}
        check_params(self, named)
        a = _lib.GpsGraphormerArgs()
        a.d, a.heads = self.embed_dim, self.num_heads
        a.training = 1 if self.training else 0
        a.precision = _lib.PRECISION[self.precision]
        a.dropout, a.attn_dropout, a.mlp_dropout = self.p_dropout, self.p_attn, self.p_mlp

        def lin(w, b):
            return linear(named[w], named[b], g.get(w), g.get(b))

        a.input_norm = lin("input_norm.weight", "input_norm.bias")
        a.attn_in = lin("attention.in_proj_weight", "attention.in_proj_bias")
        a.attn_out = lin("attention.out_proj.weight", "attention.out_proj.bias")
        a.mlp_norm = lin("mlp.0.weight", "mlp.0.bias")
        a.mlp_lin1 = lin("mlp.1.weight", "mlp.1.bias")
        a.mlp_lin2 = lin("mlp.4.weight", "mlp.4.bias")
        a.graph = gs.desc
        return a

    def _plan(self, args, gs):
        """gps_graphormer_plan is pure in (d, heads, precision, N, B)."""
        return self._plans((gs.N, gs.B, self.precision), args)

    @staticmethod
    def _attn_bias(bias, g_bias):
        """The library's second argument: the bias of a batch that has one, else NULL."""
        return C.byref(_lib.GpsAttnBias(bias.data_ptr(), bias.shape[-1], _lib.ptr(g_bias))) if bias.numel() else None

    def _bind_forward(self, args, gs, inputs, plan, params):
        x, bias = inputs
        x_out = torch.empty_like(x)
        args.x, args.x_out = x.data_ptr(), x_out.data_ptr()
        return (x_out,), (self._attn_bias(bias, None),), None

    def _grads(self, named):
        grads = zeroed_grads(named)
        return grads, _lib.FLAG_GRADS_ZEROED, tuple(grads[n] for n in self._param_names)

    def _bind_backward(self, args, gs, inputs, g_outs, needs, keep):
        x, bias = inputs
        g_x = torch.empty_like(x)
        g_bias = torch.empty_like(bias) if bias.numel() and needs[1] else None
        args.x, args.grad_x_out, args.grad_x = x.data_ptr(), g_outs[0].data_ptr(), g_x.data_ptr()
        return (g_x, g_bias), (self._attn_bias(bias, g_bias),)

    def forward(self, batch):
        x = read_x(batch, self, self.embed_dim)
        gs = graph_of(batch)
        # the reference's hasattr test (graphormer_layer.py:43-46): no attribute or None = no bias
        bias = read_attn_bias(batch, x, gs, self, False)
        params = [p for _, p in self.named_parameters()]
        batch.x = LayerFn.apply(self, gs, x, x.new_empty(0) if bias is None else bias, *params)
        return batch

    def extra_repr(self):
        return (f"embed_dim={self.embed_dim}, num_heads={self.num_heads}, backend=libgps_b200(sm_90a), "
                f"precision={self.precision}")
