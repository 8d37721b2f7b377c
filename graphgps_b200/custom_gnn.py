"""H100-native drop-ins for the two message-passing layers of CustomGNN (graphgps/network/custom_gnn.py), the model of
the LRGB GatedGCN and GINE configs:

    GatedGCNLayer   graphgps.layer.gatedgcn_layer.GatedGCNLayer (gatedgcn_layer.py:11-136)
    GINEConvLayer   graphgps.layer.gine_conv_layer.GINEConvLayer (gine_conv_layer.py:90-116)

Same constructors, `forward(batch) -> batch` contract and `state_dict` as the reference (A..E, bn_node_x, bn_edge_e;
model.nn.0, model.nn.2 and the model.eps buffer), built in the reference's order, so checkpoints load strictly and the
same seed gives the same initial values.  For d = out_dim:

    GatedGCN  batch.x         = [x +] dropout(act(bn_node_x(A x + sum_j sigma_ij B x_j / (sum_j sigma_ij + 1e-6))))
              batch.edge_attr = [e +] dropout(act(bn_edge_e(e_ij))),  e_ij = D x_i + E x_j + C e_ij,
                                sigma_ij = sigmoid(e_ij)
    GINE      batch.x         = [x +] dropout(relu(nn.2(relu(nn.0((1 + eps) x + sum_j relu(x_j + e_ij))))))

each in one C call per direction (libgps_b200.so, sm_90a), any d up to 4096: widths that are not a multiple of 8 (138
and 166 in the shipped configs, 108 as well) run at the next multiple of 8 with zero pad columns inside the library.
GINE leaves batch.edge_attr unchanged; it still receives its gradient.  There is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from .gps_layer import _bn, _lin, _next_dropout_offset, _workspace
from .graph import graph_of

_dropout_calls = [0]
_ACTS = ("relu", "gelu")


class _CustomGnnFn(torch.autograd.Function):
    """One autograd node for the layer: forward = gps_custom_gnn_forward, backward = gps_custom_gnn_backward."""

    @staticmethod
    def forward(ctx, layer, gs, x, e, *params):
        lib = _lib.load()
        dev = x.device
        named = dict(zip(layer._param_names, params))
        args = layer._args(gs, named)
        saved_bytes, ws_bytes, wp_bytes = layer._plan(args, gs)
        x_out = torch.empty_like(x)
        e_out = torch.empty_like(e) if layer._gated else None
        saved = torch.empty(max(saved_bytes, 256), dtype=torch.uint8, device=dev)
        ws = _workspace(dev, ws_bytes)
        wp = layer._weight_buffer(dev, wp_bytes, params, args)
        args.x, args.edge_attr, args.x_out, args.edge_out = x.data_ptr(), e.data_ptr(), x_out.data_ptr(), _lib.ptr(e_out)
        args.saved, args.saved_bytes = saved.data_ptr(), saved.numel()
        args.workspace, args.workspace_bytes = ws.data_ptr(), ws.numel()
        snap = None
        if layer.training and layer.dropout > 0:
            snap = _next_dropout_offset(dev)
            args.offset, args.offset_dev = 0, snap.data_ptr()
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.gps_custom_gnn_forward(C.byref(args), stream), "gps_custom_gnn_forward")
        ctx.layer, ctx.gs, ctx.saved_buf, ctx.wp, ctx.snap = layer, gs, saved, wp, snap
        ctx.seed, ctx.offset, ctx.training = args.seed, args.offset, bool(args.training)
        ctx.save_for_backward(x, e, *params)
        return (x_out, e_out) if layer._gated else x_out

    @staticmethod
    def backward(ctx, g_x_out, g_e_out=None):
        lib = _lib.load()
        layer, gs = ctx.layer, ctx.gs
        x, e, *params = ctx.saved_tensors
        dev = x.device
        named = dict(zip(layer._param_names, params))
        grads = {n: torch.empty_like(p) for n, p in named.items()}   # written whole by the library
        args = layer._args(gs, named, grads)
        args.seed, args.offset, args.training = ctx.seed, ctx.offset, 1 if ctx.training else 0
        if ctx.snap is not None:
            args.offset_dev = ctx.snap.data_ptr()
        g_x_out = g_x_out.contiguous()
        g_e_out = g_e_out.contiguous() if g_e_out is not None else None
        g_x = torch.empty_like(x)
        g_e = torch.empty_like(e) if ctx.needs_input_grad[3] else None
        _, ws_bytes, _ = layer._plan(args, gs)
        ws = _workspace(dev, ws_bytes)
        args.x, args.edge_attr = x.data_ptr(), e.data_ptr()
        args.grad_x_out, args.grad_edge_out = g_x_out.data_ptr(), _lib.ptr(g_e_out)
        args.grad_x, args.grad_edge_attr = g_x.data_ptr(), _lib.ptr(g_e)
        args.saved, args.saved_bytes = ctx.saved_buf.data_ptr(), ctx.saved_buf.numel()
        args.workspace, args.workspace_bytes = ws.data_ptr(), ws.numel()
        args.wplanes, args.wplanes_bytes, args.wplanes_valid = ctx.wp.data_ptr(), ctx.wp.numel(), 1
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.gps_custom_gnn_backward(C.byref(args), stream), "gps_custom_gnn_backward")
        # (ctx.saved_buf stays alive with the autograd node: backward(retain_graph=True) may run again)
        return (None, None, g_x, g_e) + tuple(grads[n] for n in layer._param_names)


class _CustomGnnBase(nn.Module):
    """What both layers share: argument block, plan cache, persistent weight buffer and forward."""

    _gated = False

    def _check_common(self, in_dim, out_dim, dropout, precision, name):
        if precision not in _lib.PRECISION:
            raise ValueError(f"precision must be one of {tuple(_lib.PRECISION)} (got {precision!r})")
        if not 0.0 <= float(dropout) < 1.0:
            raise ValueError(f"dropout must be in [0, 1) (got {dropout})")
        if in_dim != out_dim:
            raise NotImplementedError(f"graphgps_b200.{name}: in_dim != out_dim ({in_dim} != {out_dim}) is not built "
                                      "(CustomGNN always passes dim_inner for both)")
        if not 1 <= int(out_dim) <= 4096:
            raise NotImplementedError(f"graphgps_b200.{name}: needs 1 <= out_dim <= 4096 (got {out_dim})")

    def _args(self, gs, named, grads=None):
        g = grads or {}
        for n, t in named.items():
            if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
                raise TypeError(f"graphgps_b200.{type(self).__name__}: parameter '{n}' must be a contiguous float32 "
                                f"CUDA tensor (got {t.dtype} on {t.device})")
        a = _lib.GpsCustomGnnArgs()
        a.d = self.out_dim
        a.kind = _lib.CUSTOM_GATEDGCN if self._gated else _lib.CUSTOM_GINE
        a.act = _lib.ACT[self.act] if self._gated else 0
        a.training = 1 if self.training else 0
        a.precision = _lib.PRECISION[self.precision]
        a.residual = 1 if self.residual else 0
        a.dropout = float(self.dropout)
        a.seed = int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF
        _dropout_calls[0] += 1
        a.offset = _dropout_calls[0] * 4096
        a.graph = gs.desc

        def lin(prefix):
            w, b = prefix + ".weight", prefix + ".bias"
            return _lin(named[w], named[b], g.get(w), g.get(b))

        if self._gated:
            a.A, a.B, a.C, a.D, a.E = (lin(n) for n in "ABCDE")
            a.bn_node_x = _bn(self.bn_node_x, g.get("bn_node_x.weight"), g.get("bn_node_x.bias"))
            a.bn_edge_e = _bn(self.bn_edge_e, g.get("bn_edge_e.weight"), g.get("bn_edge_e.bias"))
        else:
            a.nn0, a.nn2 = lin("model.nn.0"), lin("model.nn.2")
            a.gine_eps = self._eps_host()
        return a

    def _plan(self, args, gs):
        """(saved_bytes, workspace_bytes, wplanes_bytes); gps_custom_gnn_plan is pure in its arguments' sizes and
        modes."""
        key = (gs.N, gs.E, self.precision, bool(args.training), self.dropout > 0)
        hit = self._plan_cache.get(key)
        if hit is None:
            plan = _lib.GpsCustomGnnPlan()
            _lib.check(_lib.load().gps_custom_gnn_plan(C.byref(args), C.byref(plan)), "gps_custom_gnn_plan")
            hit = (int(plan.saved_bytes), int(max(plan.fwd_workspace_bytes, plan.bwd_workspace_bytes)),
                   int(plan.wplanes_bytes))
            if len(self._plan_cache) > 64:
                self._plan_cache.clear()
            self._plan_cache[key] = hit
        return hit

    def _weight_buffer(self, dev, nbytes, params, args):
        """The padded weight planes this forward and its backward read (the autograd node holds the buffer).

        A packed buffer is never written again: while every parameter is the same tensor at the same version, forwards
        share the layer's current buffer without packing (once per optimiser step); otherwise the forward packs into a
        fresh one, so a backward still outstanding reads the weights its own forward used.  Under CUDA-graph capture
        each call packs into a buffer of its own from the graph's pool, which every replay re-packs."""
        def fresh():
            return torch.empty(max(nbytes, 256), dtype=torch.uint8, device=dev)

        valid = 0
        if torch.cuda.is_current_stream_capturing():
            buf = fresh()
        else:
            key = (tuple((p.data_ptr(), p._version) for p in params), self.precision, dev)
            cur = self.__dict__.get("_wplanes")
            if cur is not None and cur[1] == key and cur[0].numel() >= nbytes:
                buf, valid = cur[0], 1
            else:
                buf = fresh()
                self.__dict__["_wplanes"] = (buf, key)
        args.wplanes, args.wplanes_bytes, args.wplanes_valid = buf.data_ptr(), buf.numel(), valid
        return buf

    def forward(self, batch):
        x = batch.x
        name = type(self).__name__
        if not x.is_cuda:
            raise RuntimeError(f"graphgps_b200.{name} runs on CUDA tensors only; there is no CPU fallback")
        if x.dtype != torch.float32:
            raise TypeError("batch.x must be float32")
        d = self.out_dim
        if x.dim() != 2 or x.shape[1] != d:
            raise ValueError(f"batch.x must have shape [num_nodes, {d}] (got {tuple(x.shape)})")
        e = getattr(batch, "edge_attr", None)
        if e is None:
            raise ValueError(f"graphgps_b200.{name} needs batch.edge_attr")
        if not torch.is_tensor(e) or e.dtype != torch.float32 or e.device != x.device:
            raise TypeError("batch.edge_attr must be a float32 tensor on the device of batch.x")
        E = int(batch.edge_index.shape[1])
        if e.dim() != 2 or tuple(e.shape) != (E, d):
            raise ValueError(f"batch.edge_attr must have shape [num_edges, {d}] = [{E}, {d}] (got {tuple(e.shape)})")
        x, e = x.contiguous(), e.contiguous()
        gs = graph_of(batch)
        if self._gated and self.training:
            # a BatchNorm over no rows counts the batch and leaves its running statistics alone, as torch's does;
            # the library launches nothing for it
            with torch.no_grad():
                if gs.N == 0:
                    self.bn_node_x.num_batches_tracked.add_(1)
                if gs.E == 0:
                    self.bn_edge_e.num_batches_tracked.add_(1)
        params = [p for _, p in self.named_parameters()]
        out = _CustomGnnFn.apply(self, gs, x, e, *params)
        if self._gated:
            batch.x, batch.edge_attr = out
        else:
            batch.x = out
        return batch


class GatedGCNLayer(_CustomGnnBase):
    """GatedGCN layer (reference: graphgps/layer/gatedgcn_layer.py:11-136)."""

    _gated = True

    def __init__(self, in_dim, out_dim, dropout, residual, act="relu", equivstable_pe=False, precision="fp32",
                 **kwargs):
        super().__init__()
        self._check_common(in_dim, out_dim, dropout, precision, "GatedGCNLayer")
        if act not in _ACTS:
            raise NotImplementedError(f"graphgps_b200.GatedGCNLayer: act {act!r} is not built (relu and gelu are)")
        if equivstable_pe:
            raise NotImplementedError("graphgps_b200.GatedGCNLayer: equivstable_pe=True is not built (CustomGNN never "
                                      "passes it; GPSLayer's GatedGCN has it)")
        if kwargs:
            raise NotImplementedError(f"graphgps_b200.GatedGCNLayer: MessagePassing options {sorted(kwargs)} are not "
                                      "built")
        self.in_dim, self.out_dim = int(in_dim), int(out_dim)
        # the reference's modules, in its order (same state_dict keys, same draws from the same seed)
        self.A = nn.Linear(in_dim, out_dim, bias=True)
        self.B = nn.Linear(in_dim, out_dim, bias=True)
        self.C = nn.Linear(in_dim, out_dim, bias=True)
        self.D = nn.Linear(in_dim, out_dim, bias=True)
        self.E = nn.Linear(in_dim, out_dim, bias=True)
        self.bn_node_x = nn.BatchNorm1d(out_dim)
        self.bn_edge_e = nn.BatchNorm1d(out_dim)
        self.act = act
        self.dropout = float(dropout)
        self.residual = bool(residual)
        self.EquivStablePE = False
        self.precision = precision
        self._param_names = [n for n, _ in self.named_parameters()]
        self._plan_cache = {}

    def __repr__(self):
        return "{}({}, {}, residual={}, act={}, backend=libgps_b200(sm_90a), precision={})".format(
            self.__class__.__name__, self.in_dim, self.out_dim, self.residual, self.act, self.precision)


class _GINEConvParams(nn.Module):
    """Names of GINEConv(Sequential(Linear, ReLU, Linear)) as GINEConvLayer builds it: nn.0, nn.2 and the eps buffer
    (train_eps=False, no edge_dim)."""

    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.nn = nn.Sequential(nn.Linear(dim_in, dim_out), nn.ReLU(), nn.Linear(dim_out, dim_out))
        self.register_buffer("eps", torch.Tensor([0.0]))


class GINEConvLayer(_CustomGnnBase):
    """GINE layer (reference: graphgps/layer/gine_conv_layer.py:90-116)."""

    def __init__(self, dim_in, dim_out, dropout, residual, precision="fp32"):
        super().__init__()
        self._check_common(dim_in, dim_out, dropout, precision, "GINEConvLayer")
        self.dim_in, self.dim_out = int(dim_in), int(dim_out)
        self.out_dim = self.dim_out
        self.dropout = float(dropout)
        self.residual = bool(residual)
        self.model = _GINEConvParams(dim_in, dim_out)
        self.precision = precision
        self._param_names = [n for n, _ in self.named_parameters()]
        self._plan_cache = {}

    def _eps_host(self):
        """model.eps as a float, read from the buffer once per change of it (load_state_dict bumps its version)."""
        t = self.model.eps
        key = (t.data_ptr(), t._version, t.device)
        hit = self.__dict__.get("_eps_cache")
        if hit is None or hit[0] != key:
            hit = (key, float(t.reshape(-1)[0].item()))
            self.__dict__["_eps_cache"] = hit
        return hit[1]

    def __repr__(self):
        return "{}({}, {}, residual={}, backend=libgps_b200(sm_90a), precision={})".format(
            self.__class__.__name__, self.dim_in, self.dim_out, self.residual, self.precision)
