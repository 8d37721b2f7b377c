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

`SAN2Layer` is the drop-in for `graphgps.layer.san2_layer.SAN2Layer`, SANTransformer's other layer: the same trunk and
modules, plus `attention.gamma` (float64, learned, first in the state_dict as the reference creates it), with

    attn = (softmax over the real in-edges . V + gamma softmax over the fake pairs . V) / (gamma + 1)

(pyg_softmax per set and head, no clamp).  The library reads gamma on the device, so an optimiser step or a replayed
CUDA graph uses its current value; the constructor's `gamma` argument is ignored, as in the reference.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _lib
from ._call import LayerFn, PlanCache, batch_norm, check_params, linear, read_edge_attr, read_x
from .graph import graph_of

# the five node projections, in the order of the fused product [Q | K | V | Q2 | K2]
_NODE = ("attention.Q.weight", "attention.K.weight", "attention.V.weight", "attention.Q_2.weight",
         "attention.K_2.weight")


class _SANAttentionParams(nn.Module):
    """Parameter container with the names and construction order of MultiHeadAttentionLayer (san_layer.py:17-36) as
    SANLayer builds it: Q, K, E, Q_2, K_2, E_2 (no biases), the shared fake_edge_emb, V.  With `learned_gamma`, that of
    MultiHeadAttention2Layer (san2_layer.py:43-63): the float64 gamma = 0.5 first."""

    def __init__(self, in_dim, out_dim, num_heads, fake_edge_emb, learned_gamma=False):
        super().__init__()
        if learned_gamma:
            self.gamma = nn.Parameter(torch.tensor(0.5, dtype=torch.float64), requires_grad=True)
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

    _variant = 0   # GpsSanArgs.variant

    def __init__(self, gamma, in_dim, out_dim, num_heads, full_graph, fake_edge_emb, dropout=0.0, layer_norm=False,
                 batch_norm=True, residual=True, use_bias=False, precision="fp32"):
        super().__init__()
        if precision not in _lib.PRECISION:
            raise ValueError(f"precision must be one of {tuple(_lib.PRECISION)} (got {precision!r})")
        for off, what in ((not full_graph, "full_graph=False"), (layer_norm, "layer_norm=True"),
                          (not batch_norm, "batch_norm=False"), (not residual, "residual=False"),
                          (use_bias, "use_bias=True")):
            if off:
                raise NotImplementedError(f"graphgps_b200.{type(self).__name__}: {what} is not built (no shipped SAN "
                                          "config uses it)")
        if in_dim != out_dim:
            raise NotImplementedError(f"graphgps_b200.{type(self).__name__}: in_dim != out_dim ({in_dim} != {out_dim}) is not built "
                                      "(SANTransformer always passes dim_hidden for both)")
        if num_heads < 1 or out_dim % num_heads != 0:
            raise ValueError(f"out_dim {out_dim} must be divisible by num_heads {num_heads} (the reference fails at "
                             "its view of the concatenated heads)")
        if out_dim % 4 != 0 or out_dim // num_heads > 192:
            raise NotImplementedError(f"graphgps_b200.{type(self).__name__}: needs out_dim % 4 == 0 and a head dim <= 192 (got "
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
        self.attention = _SANAttentionParams(in_dim, out_dim // num_heads, num_heads, fake_edge_emb,
                                             learned_gamma=self._variant == 1)
        self.O_h = nn.Linear(out_dim, out_dim)
        self.batch_norm1_h = nn.BatchNorm1d(out_dim)
        self.FFN_h_layer1 = nn.Linear(out_dim, out_dim * 2)
        self.FFN_h_layer2 = nn.Linear(out_dim * 2, out_dim)
        self.batch_norm2_h = nn.BatchNorm1d(out_dim)
        if self._variant == 0:
            self.gamma = float(gamma)
        self.p_dropout = float(dropout)
        self.precision = precision
        self._param_names = [n for n, _ in self.named_parameters()]
        self._plans = PlanCache(self._entry, _lib.GpsSanPlan)

    # ------------------------------------------------------------------ hooks of _call.LayerFn; call = the graph
    _entry = "gps_san"

    def _dropout_live(self):
        return self.p_dropout > 0

    def _args(self, gs, inputs, named, grads=None):
        g = grads or {}
        a = _lib.GpsSanArgs()
        if self._variant == 0:
            check_params(self, named)
            a.gamma = self.gamma
        else:   # attention.gamma is float64, checked by forward
            check_params(self, {n: t for n, t in named.items() if n != "attention.gamma"})
            a.variant = 1
            a.gamma_param = named["attention.gamma"].data_ptr()
            a.grad_gamma = _lib.ptr(g.get("attention.gamma"))
        a.d, a.heads = self.out_channels, self.num_heads
        a.training = 1 if self.training else 0
        a.precision = _lib.PRECISION[self.precision]
        a.dropout = self.p_dropout

        def lin(w, b=None):
            return linear(named[w], named[b] if b else None, g.get(w), g.get(b) if b else None)

        a.Q, a.K, a.V = lin("attention.Q.weight"), lin("attention.K.weight"), lin("attention.V.weight")
        a.Q2, a.K2 = lin("attention.Q_2.weight"), lin("attention.K_2.weight")
        a.E, a.E2 = lin("attention.E.weight"), lin("attention.E_2.weight")
        a.O_h = lin("O_h.weight", "O_h.bias")
        a.ffn1 = lin("FFN_h_layer1.weight", "FFN_h_layer1.bias")
        a.ffn2 = lin("FFN_h_layer2.weight", "FFN_h_layer2.bias")
        a.bn1 = batch_norm(self.batch_norm1_h, g.get("batch_norm1_h.weight"), g.get("batch_norm1_h.bias"))
        a.bn2 = batch_norm(self.batch_norm2_h, g.get("batch_norm2_h.weight"), g.get("batch_norm2_h.bias"))
        a.fake_edge_emb = named["attention.fake_edge_emb.weight"].data_ptr()
        a.grad_fake_edge_emb = _lib.ptr(g.get("attention.fake_edge_emb.weight"))
        a.graph = gs.desc
        a.nmax = gs.nmax
        return a

    def _plan(self, args, gs):
        """gps_san_plan is pure in its arguments' sizes and modes."""
        return self._plans((gs.N, gs.E, gs.B, gs.nmax, self.precision, bool(args.training), self.p_dropout > 0), args)

    def _bind_forward(self, args, gs, inputs, plan, params):
        x, e = inputs
        x_out = torch.empty_like(x)
        args.x, args.edge_attr, args.x_out = x.data_ptr(), e.data_ptr(), x_out.data_ptr()
        return (x_out,), (), None

    def _grads(self, named):
        d = self.out_channels
        # the five node-projection gradients as views of one [5d, d] buffer: one weight product in the library
        packed = torch.empty(5 * d, d, device=named[_NODE[0]].device)
        grads = {n: packed[i * d:(i + 1) * d] for i, n in enumerate(_NODE)}
        for n, p in named.items():
            if n not in grads:
                grads[n] = torch.empty_like(p)
        torch._foreach_zero_([packed] + [g for n, g in grads.items() if n not in _NODE])
        return grads, _lib.FLAG_GRADS_ZEROED, tuple(grads[n] for n in self._param_names)

    def _bind_backward(self, args, gs, inputs, g_outs, needs, keep):
        x, e = inputs
        g_x = torch.empty_like(x)
        g_e = torch.empty_like(e) if needs[1] else None
        args.x, args.edge_attr = x.data_ptr(), e.data_ptr()
        args.grad_x_out, args.grad_x, args.grad_edge_attr = g_outs[0].data_ptr(), g_x.data_ptr(), _lib.ptr(g_e)
        return (g_x, g_e), ()

    def forward(self, batch):
        if self._variant == 1:
            gamma = self.attention.gamma
            if gamma.dtype != torch.float64 or gamma.numel() != 1 or gamma.device != batch.x.device:
                raise TypeError(f"graphgps_b200.{type(self).__name__}: parameter 'attention.gamma' must be one float64 "
                                f"value on the device of batch.x (got {gamma.dtype} of shape {tuple(gamma.shape)} on "
                                f"{gamma.device})")
        x = read_x(batch, self, self.out_channels)
        e = read_edge_attr(batch, x, self, self.out_channels)
        gs = graph_of(batch)
        params = [p for _, p in self.named_parameters()]
        batch.x = LayerFn.apply(self, gs, x, e, *params)
        return batch

    def __repr__(self):
        return "{}(in_channels={}, out_channels={}, heads={}, residual={}, backend=libgps_b200(sm_90a), " \
               "precision={})".format(self.__class__.__name__, self.in_channels, self.out_channels, self.num_heads,
                                      self.residual, self.precision)


class SAN2Layer(SANLayer):
    """SAN2Layer (reference: graphgps/layer/san2_layer.py:145-238): SANLayer's trunk around softmax attention over the
    real edges and the fake pairs, mixed by the learned float64 `attention.gamma`.  `gamma` is accepted and ignored, as
    the reference ignores it."""

    _variant = 1
