"""H100-native drop-in for `graphgps.layer.san_layer.SANLayer` (san_layer.py:123-216), the layer of SANTransformer.

Same constructor, `forward(batch) -> batch` contract and `state_dict` as the reference: the reference's own torch
modules (`attention.{Q,K,E,Q_2,K_2,E_2,fake_edge_emb,V}`, `O_h`, `batch_norm1_h`, `FFN_h_layer1`, `FFN_h_layer2`,
`batch_norm2_h`) are built in its order as parameter containers, so checkpoints load strictly and the same seed gives
the same initial values; their `forward` is never called.  The `fake_edge_emb` module passed in is registered as
`attention.fake_edge_emb` itself, so the L layers of a SANTransformer share it and its gradient is their sum.  For
d = out_dim, H = num_heads, hd = d / H:

    attn = full-graph SAN attention over the real edges (scores modulated by E(edge_attr)) and the complement pairs
           of each graph (Q_2, K_2 and E_2(fake_edge_emb)), exp(clamp(., -5, 5)) scores weighted 1 : gamma
    h1   = batch_norm1_h(x + O_h(dropout(attn)))
    out  = batch_norm2_h(h1 + FFN_h_layer2(dropout(relu(FFN_h_layer1(h1)))))

in one C call per direction (libgps_b200.so, sm_90a).  There is no CPU fallback.  The reference's side effects on the
batch (Q_h, K_h, E, wV, Z, ...) are internals and are not reproduced; batch.edge_attr is left unchanged.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from .gps_layer import _bn, _lin, _next_dropout_offset, _workspace
from .graph import graph_of

_dropout_calls = [0]
# the five node projections, in the order of the fused product [Q | K | V | Q2 | K2]
_NODE = ("attention.Q.weight", "attention.K.weight", "attention.V.weight", "attention.Q_2.weight",
         "attention.K_2.weight")


class _SANFn(torch.autograd.Function):
    """One autograd node for the layer: forward = gps_san_forward, backward = gps_san_backward."""

    @staticmethod
    def forward(ctx, layer, gs, nmax, x, e, *params):
        lib = _lib.load()
        dev = x.device
        named = dict(zip(layer._param_names, params))
        args = layer._args(gs, nmax, named)
        plan = layer._plan(args, gs, nmax)
        x_out = torch.empty_like(x)
        saved = torch.empty(max(plan[0], 256), dtype=torch.uint8, device=dev)
        ws = _workspace(dev, plan[1])
        args.x, args.edge_attr, args.x_out = x.data_ptr(), e.data_ptr(), x_out.data_ptr()
        args.saved, args.saved_bytes = saved.data_ptr(), saved.numel()
        args.workspace, args.workspace_bytes = ws.data_ptr(), ws.numel()
        snap = None
        if layer.training and layer.p_dropout > 0:
            snap = _next_dropout_offset(dev)
            args.offset, args.offset_dev = 0, snap.data_ptr()
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.gps_san_forward(C.byref(args), stream), "gps_san_forward")
        ctx.layer, ctx.gs, ctx.nmax, ctx.saved_buf, ctx.snap = layer, gs, nmax, saved, snap
        ctx.seed, ctx.offset, ctx.training = args.seed, args.offset, bool(args.training)
        ctx.save_for_backward(x, e, *params)
        return x_out

    @staticmethod
    def backward(ctx, g_x_out):
        lib = _lib.load()
        layer, gs = ctx.layer, ctx.gs
        x, e, *params = ctx.saved_tensors
        dev = x.device
        named = dict(zip(layer._param_names, params))
        d = layer.out_channels
        # the five node-projection gradients as views of one [5d, d] buffer: one weight product in the library
        packed = torch.empty(5 * d, d, device=dev)
        grads = {n: packed[i * d:(i + 1) * d] for i, n in enumerate(_NODE)}
        for n, p in named.items():
            if n not in grads:
                grads[n] = torch.empty_like(p)
        torch._foreach_zero_([packed] + [g for n, g in grads.items() if n not in _NODE])
        args = layer._args(gs, ctx.nmax, named, grads)
        args.flags = _lib.FLAG_GRADS_ZEROED
        args.seed, args.offset, args.training = ctx.seed, ctx.offset, 1 if ctx.training else 0
        if ctx.snap is not None:
            args.offset_dev = ctx.snap.data_ptr()
        g_x_out = g_x_out.contiguous()
        g_x = torch.empty_like(x)
        g_e = torch.empty_like(e) if ctx.needs_input_grad[4] else None
        plan = layer._plan(args, gs, ctx.nmax)
        ws = _workspace(dev, plan[1])
        args.x, args.edge_attr = x.data_ptr(), e.data_ptr()
        args.grad_x_out, args.grad_x, args.grad_edge_attr = g_x_out.data_ptr(), g_x.data_ptr(), _lib.ptr(g_e)
        args.saved, args.saved_bytes = ctx.saved_buf.data_ptr(), ctx.saved_buf.numel()
        args.workspace, args.workspace_bytes = ws.data_ptr(), ws.numel()
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.gps_san_backward(C.byref(args), stream), "gps_san_backward")
        # (ctx.saved_buf stays alive with the autograd node: backward(retain_graph=True) may run again)
        return (None, None, None, g_x, g_e) + tuple(grads[n] for n in layer._param_names)


class _SANAttentionParams(nn.Module):
    """Parameter container with the names and construction order of MultiHeadAttentionLayer (san_layer.py:17-36) as
    SANLayer builds it: Q, K, E, Q_2, K_2, E_2 (no biases), the shared fake_edge_emb, V."""

    def __init__(self, in_dim, out_dim, num_heads, fake_edge_emb):
        super().__init__()
        self.Q = nn.Linear(in_dim, out_dim * num_heads, bias=False)
        self.K = nn.Linear(in_dim, out_dim * num_heads, bias=False)
        self.E = nn.Linear(in_dim, out_dim * num_heads, bias=False)
        self.Q_2 = nn.Linear(in_dim, out_dim * num_heads, bias=False)
        self.K_2 = nn.Linear(in_dim, out_dim * num_heads, bias=False)
        self.E_2 = nn.Linear(in_dim, out_dim * num_heads, bias=False)
        self.fake_edge_emb = fake_edge_emb
        self.V = nn.Linear(in_dim, out_dim * num_heads, bias=False)


class SANLayer(nn.Module):
    """SAN GraphTransformerLayer (reference: graphgps/layer/san_layer.py:123-216)."""

    def __init__(self, gamma, in_dim, out_dim, num_heads, full_graph, fake_edge_emb, dropout=0.0, layer_norm=False,
                 batch_norm=True, residual=True, use_bias=False, precision="fp32"):
        super().__init__()
        if precision not in _lib.PRECISION:
            raise ValueError(f"precision must be one of {tuple(_lib.PRECISION)} (got {precision!r})")
        for off, what in ((not full_graph, "full_graph=False"), (layer_norm, "layer_norm=True"),
                          (not batch_norm, "batch_norm=False"), (not residual, "residual=False"),
                          (use_bias, "use_bias=True")):
            if off:
                raise NotImplementedError(f"graphgps_b200.SANLayer: {what} is not built (no shipped SAN config uses "
                                          "it)")
        if in_dim != out_dim:
            raise NotImplementedError(f"graphgps_b200.SANLayer: in_dim != out_dim ({in_dim} != {out_dim}) is not built "
                                      "(SANTransformer always passes dim_hidden for both)")
        if num_heads < 1 or out_dim % num_heads != 0:
            raise ValueError(f"out_dim {out_dim} must be divisible by num_heads {num_heads} (the reference fails at "
                             "its view of the concatenated heads)")
        if out_dim % 4 != 0 or out_dim // num_heads > 192:
            raise NotImplementedError(f"graphgps_b200.SANLayer: needs out_dim % 4 == 0 and a head dim <= 192 (got "
                                      f"out_dim {out_dim}, {num_heads} heads)")
        if not isinstance(fake_edge_emb, nn.Embedding) or tuple(fake_edge_emb.weight.shape) != (1, out_dim):
            raise ValueError(f"fake_edge_emb must be an nn.Embedding(1, {out_dim})")
        self.in_channels = in_dim
        self.out_channels = out_dim
        self.num_heads = num_heads
        self.dropout = dropout
        self.residual = residual
        self.layer_norm = layer_norm
        self.batch_norm = batch_norm
        # the reference's modules, in its order (same state_dict keys, same draws from the same seed)
        self.attention = _SANAttentionParams(in_dim, out_dim // num_heads, num_heads, fake_edge_emb)
        self.O_h = nn.Linear(out_dim, out_dim)
        self.batch_norm1_h = nn.BatchNorm1d(out_dim)
        self.FFN_h_layer1 = nn.Linear(out_dim, out_dim * 2)
        self.FFN_h_layer2 = nn.Linear(out_dim * 2, out_dim)
        self.batch_norm2_h = nn.BatchNorm1d(out_dim)
        self.gamma = float(gamma)
        self.p_dropout = float(dropout)
        self.precision = precision
        self._param_names = [n for n, _ in self.named_parameters()]
        self._plan_cache = {}

    def _args(self, gs, nmax, named, grads=None):
        g = grads or {}
        for n, t in named.items():
            if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
                raise TypeError(f"graphgps_b200.SANLayer: parameter '{n}' must be a contiguous float32 CUDA tensor "
                                f"(got {t.dtype} on {t.device})")
        a = _lib.GpsSanArgs()
        a.d, a.heads = self.out_channels, self.num_heads
        a.training = 1 if self.training else 0
        a.precision = _lib.PRECISION[self.precision]
        a.gamma, a.dropout = self.gamma, self.p_dropout

        def lin(w, b=None):
            return _lin(named[w], named[b] if b else None, g.get(w), g.get(b) if b else None)

        a.Q, a.K, a.V = lin("attention.Q.weight"), lin("attention.K.weight"), lin("attention.V.weight")
        a.Q2, a.K2 = lin("attention.Q_2.weight"), lin("attention.K_2.weight")
        a.E, a.E2 = lin("attention.E.weight"), lin("attention.E_2.weight")
        a.O_h = lin("O_h.weight", "O_h.bias")
        a.ffn1 = lin("FFN_h_layer1.weight", "FFN_h_layer1.bias")
        a.ffn2 = lin("FFN_h_layer2.weight", "FFN_h_layer2.bias")
        a.bn1 = _bn(self.batch_norm1_h, g.get("batch_norm1_h.weight"), g.get("batch_norm1_h.bias"))
        a.bn2 = _bn(self.batch_norm2_h, g.get("batch_norm2_h.weight"), g.get("batch_norm2_h.bias"))
        a.fake_edge_emb = named["attention.fake_edge_emb.weight"].data_ptr()
        a.grad_fake_edge_emb = _lib.ptr(g.get("attention.fake_edge_emb.weight"))
        a.seed = int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF
        _dropout_calls[0] += 1
        a.offset = _dropout_calls[0] * 4096
        a.graph = gs.desc
        a.nmax = nmax
        return a

    def _plan(self, args, gs, nmax):
        """(saved_bytes, workspace_bytes); gps_san_plan is pure in its arguments' sizes and modes."""
        key = (gs.N, gs.E, gs.B, nmax, self.precision, bool(args.training), self.p_dropout > 0)
        hit = self._plan_cache.get(key)
        if hit is None:
            plan = _lib.GpsSanPlan()
            _lib.check(_lib.load().gps_san_plan(C.byref(args), C.byref(plan)), "gps_san_plan")
            hit = (int(plan.saved_bytes), int(max(plan.fwd_workspace_bytes, plan.bwd_workspace_bytes)))
            if len(self._plan_cache) > 64:
                self._plan_cache.clear()
            self._plan_cache[key] = hit
        return hit

    def forward(self, batch):
        x = batch.x
        if not x.is_cuda:
            raise RuntimeError("graphgps_b200.SANLayer runs on CUDA tensors only; there is no CPU fallback")
        if x.dtype != torch.float32:
            raise TypeError("batch.x must be float32")
        d = self.out_channels
        if x.dim() != 2 or x.shape[1] != d:
            raise ValueError(f"batch.x must have shape [num_nodes, {d}] (got {tuple(x.shape)})")
        e = getattr(batch, "edge_attr", None)
        if e is None:
            raise ValueError("graphgps_b200.SANLayer needs batch.edge_attr (the reference projects it with attention.E)")
        if not torch.is_tensor(e) or e.dtype != torch.float32 or e.device != x.device:
            raise TypeError("batch.edge_attr must be a float32 tensor on the device of batch.x")
        E = int(batch.edge_index.shape[1])
        if e.dim() != 2 or tuple(e.shape) != (E, d):
            raise ValueError(f"batch.edge_attr must have shape [num_edges, {d}] = [{E}, {d}] (got {tuple(e.shape)})")
        x, e = x.contiguous(), e.contiguous()
        gs = graph_of(batch)
        nmax = gs.nmax
        params = [p for _, p in self.named_parameters()]
        batch.x = _SANFn.apply(self, gs, nmax, x, e, *params)
        return batch

    def __repr__(self):
        return "{}(in_channels={}, out_channels={}, heads={}, residual={}, backend=libgps_b200(sm_90a), " \
               "precision={})".format(self.__class__.__name__, self.in_channels, self.out_channels, self.num_heads,
                                      self.residual, self.precision)
