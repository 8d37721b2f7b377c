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
from .gps_layer import _lin, _next_dropout_offset, _workspace
from .graph import graph_of

_dropout_calls = [0]


class _GraphormerFn(torch.autograd.Function):
    """One autograd node for the layer: forward = gps_graphormer_forward, backward = gps_graphormer_backward."""

    @staticmethod
    def forward(ctx, layer, gs, x, bias, *params):
        lib = _lib.load()
        dev = x.device
        named = dict(zip(layer._param_names, params))
        args = layer._args(gs, named)
        plan = layer._plan(args, gs)
        x_out = torch.empty_like(x)
        saved = torch.empty(max(plan[0], 256), dtype=torch.uint8, device=dev)
        ws = _workspace(dev, plan[1])
        args.x, args.x_out = x.data_ptr(), x_out.data_ptr()
        args.saved, args.saved_bytes = saved.data_ptr(), saved.numel()
        args.workspace, args.workspace_bytes = ws.data_ptr(), ws.numel()
        snap = None
        if layer.training and layer._any_dropout:
            snap = _next_dropout_offset(dev)
            args.offset, args.offset_dev = 0, snap.data_ptr()
        ctx.nmax = bias.shape[-1] if bias.numel() else 0
        ab = C.byref(_lib.GpsAttnBias(bias.data_ptr(), ctx.nmax, 0)) if ctx.nmax else None
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.gps_graphormer_forward(C.byref(args), ab, stream), "gps_graphormer_forward")
        ctx.layer, ctx.gs, ctx.saved_buf, ctx.snap = layer, gs, saved, snap
        ctx.seed, ctx.offset, ctx.training = args.seed, args.offset, bool(args.training)
        ctx.save_for_backward(x, bias, *params)
        return x_out

    @staticmethod
    def backward(ctx, g_x_out):
        lib = _lib.load()
        layer, gs = ctx.layer, ctx.gs
        x, bias, *params = ctx.saved_tensors
        dev = x.device
        named = dict(zip(layer._param_names, params))
        grads = {n: torch.empty_like(p) for n, p in named.items()}
        torch._foreach_zero_(list(grads.values()))   # one multi-tensor fill; the library then skips its memsets
        args = layer._args(gs, named, grads)
        args.flags = _lib.FLAG_GRADS_ZEROED
        args.seed, args.offset, args.training = ctx.seed, ctx.offset, 1 if ctx.training else 0
        if ctx.snap is not None:
            args.offset_dev = ctx.snap.data_ptr()
        g_x_out = g_x_out.contiguous()
        g_x = torch.empty_like(x)
        plan = layer._plan(args, gs)
        ws = _workspace(dev, plan[1])
        args.x, args.grad_x_out, args.grad_x = x.data_ptr(), g_x_out.data_ptr(), g_x.data_ptr()
        args.saved, args.saved_bytes = ctx.saved_buf.data_ptr(), ctx.saved_buf.numel()
        args.workspace, args.workspace_bytes = ws.data_ptr(), ws.numel()
        g_bias = torch.empty_like(bias) if ctx.nmax and ctx.needs_input_grad[3] else None
        ab = C.byref(_lib.GpsAttnBias(bias.data_ptr(), ctx.nmax, _lib.ptr(g_bias))) if ctx.nmax else None
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.gps_graphormer_backward(C.byref(args), ab, stream), "gps_graphormer_backward")
        # (ctx.saved_buf stays alive with the autograd node: backward(retain_graph=True) may run again)
        return (None, None, g_x, g_bias) + tuple(grads[n] for n in layer._param_names)


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
        self._plan_cache = {}

    @property
    def _any_dropout(self):
        return self.p_dropout > 0 or self.p_attn > 0 or self.p_mlp > 0

    def _args(self, gs, named, grads=None):
        g = grads or {}
        for n, t in named.items():
            if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
                raise TypeError(f"graphgps_b200.GraphormerLayer: parameter '{n}' must be a contiguous float32 CUDA "
                                f"tensor (got {t.dtype} on {t.device})")
        a = _lib.GpsGraphormerArgs()
        a.d, a.heads = self.embed_dim, self.num_heads
        a.training = 1 if self.training else 0
        a.precision = _lib.PRECISION[self.precision]
        a.dropout, a.attn_dropout, a.mlp_dropout = self.p_dropout, self.p_attn, self.p_mlp

        def lin(w, b):
            return _lin(named[w], named[b], g.get(w), g.get(b))

        a.input_norm = lin("input_norm.weight", "input_norm.bias")
        a.attn_in = lin("attention.in_proj_weight", "attention.in_proj_bias")
        a.attn_out = lin("attention.out_proj.weight", "attention.out_proj.bias")
        a.mlp_norm = lin("mlp.0.weight", "mlp.0.bias")
        a.mlp_lin1 = lin("mlp.1.weight", "mlp.1.bias")
        a.mlp_lin2 = lin("mlp.4.weight", "mlp.4.bias")
        a.seed = int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF
        _dropout_calls[0] += 1
        a.offset = _dropout_calls[0] * 4096
        a.graph = gs.desc
        return a

    def _plan(self, args, gs):
        """(saved_bytes, workspace_bytes); gps_graphormer_plan is pure in (d, heads, precision, N, B)."""
        key = (gs.N, gs.B, self.precision)
        hit = self._plan_cache.get(key)
        if hit is None:
            plan = _lib.GpsGraphormerPlan()
            _lib.check(_lib.load().gps_graphormer_plan(C.byref(args), C.byref(plan)), "gps_graphormer_plan")
            hit = (int(plan.saved_bytes), int(max(plan.fwd_workspace_bytes, plan.bwd_workspace_bytes)))
            if len(self._plan_cache) > 64:
                self._plan_cache.clear()
            self._plan_cache[key] = hit
        return hit

    def _read_attn_bias(self, batch, x, gs):
        """The reference's hasattr test (graphormer_layer.py:43-46): no attribute or None = no bias, else
        batch.attn_bias [num_graphs * heads, Nmax, Nmax], row g * heads + h, float32 on the device of x."""
        ab = getattr(batch, "attn_bias", None)
        if ab is None:
            return None
        if not torch.is_tensor(ab) or ab.dtype != torch.float32 or ab.device != x.device:
            raise TypeError("batch.attn_bias must be a float32 tensor on the device of batch.x (got "
                            f"{getattr(ab, 'dtype', type(ab))} on {getattr(ab, 'device', None)})")
        want = (gs.B * self.num_heads, gs.nmax, gs.nmax)
        if tuple(ab.shape) != want:
            raise ValueError(f"batch.attn_bias must have shape [num_graphs * heads, Nmax, Nmax] = {list(want)} "
                             f"(got {list(ab.shape)})")
        if gs.nmax == 0:
            return None
        return ab.contiguous()

    def forward(self, batch):
        x = batch.x
        if not x.is_cuda:
            raise RuntimeError("graphgps_b200.GraphormerLayer runs on CUDA tensors only; there is no CPU fallback")
        if x.dtype != torch.float32:
            raise TypeError("batch.x must be float32")
        if x.dim() != 2 or x.shape[1] != self.embed_dim:
            raise ValueError(f"batch.x must have shape [num_nodes, {self.embed_dim}] (got {tuple(x.shape)})")
        x = x.contiguous()
        gs = graph_of(batch)
        bias = self._read_attn_bias(batch, x, gs)
        params = [p for _, p in self.named_parameters()]
        bias_arg = bias if bias is not None else x.new_empty(0)
        batch.x = _GraphormerFn.apply(self, gs, x, bias_arg, *params)
        return batch

    def extra_repr(self):
        return (f"embed_dim={self.embed_dim}, num_heads={self.num_heads}, backend=libgps_b200(sm_90a), "
                f"precision={self.precision}")
