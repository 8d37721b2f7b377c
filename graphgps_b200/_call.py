"""The call path every layer shares: one library call per direction under one autograd node.

A layer (GPSLayer, GraphormerLayer, SANLayer, GatedGCNLayer, GINEConvLayer) keeps what is its own: its args struct,
its batch reads and its gradient buffers.  It declares these hooks for `LayerFn`:

    _entry                                   library prefix: <entry>_forward, <entry>_backward
    _dropout_live()                          whether a dropout probability is > 0 (read in training only)
    _args(call, inputs, named, grads=None)   the args struct with configuration, graph, parameter and gradient pointers
    _plan(args, call)                        (saved_bytes, workspace_bytes, wplanes_bytes), from a PlanCache
    _bind_forward(args, call, inputs, plan, params) -> (outputs, extra, keep)
    _grads(named) -> (grads, flags, parameter gradients in parameter order)
    _bind_backward(args, call, inputs, g_outs, needs, keep) -> (input gradients, extra)

`call` is the layer's per-call state (its graph structure and batch-dependent sizes), `inputs` the tensors autograd
differentiates other than the parameters, `extra` the positional arguments the library takes between the args struct and
the stream, and `keep` whatever the backward must see again (hand-off and weight-plane buffers).
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib

_workspaces = {}
_drop_counters = {}


def dropout_counter(device):
    """The device-resident Philox counter of `device`, created at zero on first use."""
    ctr = _drop_counters.get(device)
    if ctr is None:
        ctr = torch.zeros(1, dtype=torch.int64, device=device)
        _drop_counters[device] = ctr
    return ctr


def next_dropout_offset(device):
    """Device-resident Philox offset for this call: counter += 4096; snapshot = counter.

    Kept on the device (two tiny stream-ordered ops) so that a captured CUDA graph draws fresh dropout
    masks on every replay; the snapshot tensor is what forward and backward of this call both read."""
    ctr = dropout_counter(device)
    ctr.add_(4096)
    return ctr.clone()


def dropout_seed():
    return int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF


def workspace(device, nbytes):
    """Transient scratch for one C call, one buffer per (device, stream): layers running on different streams never
    share it, and a buffer is never freed while the process lives (a captured CUDA graph may hold its address) -
    growth keeps the old ones.  Under stream capture the buffer is allocated from the graph's own pool instead."""
    if torch.cuda.is_current_stream_capturing():
        return torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=device)
    key = (device, torch.cuda.current_stream(device).cuda_stream)
    held = _workspaces.setdefault(key, [])
    if not held or held[-1].numel() < nbytes:
        held.append(torch.empty(int(nbytes * 1.25) + 256, dtype=torch.uint8, device=device))
    return held[-1]


class PlanCache:
    """(saved_bytes, workspace_bytes, wplanes_bytes) of `<entry>_plan`, which is pure in the sizes and modes of its
    args: the layer keys each plan by exactly what it depends on.  Cleared past 64 entries."""

    def __init__(self, entry, plan_type):
        self._fn, self._type, self._hits = entry + "_plan", plan_type, {}

    def __call__(self, key, args):
        hit = self._hits.get(key)
        if hit is None:
            plan = self._type()
            _lib.check(getattr(_lib.load(), self._fn)(C.byref(args), C.byref(plan)), self._fn)
            hit = (int(plan.saved_bytes), int(max(plan.fwd_workspace_bytes, plan.bwd_workspace_bytes)),
                   int(getattr(plan, "wplanes_bytes", 0)))
            if len(self._hits) > 64:
                self._hits.clear()
            self._hits[key] = hit
        return hit


def weight_planes(layer, args, nbytes, params, device):
    """The padded weight planes this forward and its backward read (the autograd node holds the buffer).

    A packed buffer is never written again: while every parameter is the same tensor at the same version, forwards
    share the layer's current buffer without packing (once per optimiser step); otherwise the forward packs into a
    fresh one, so a backward still outstanding reads the weights its own forward used.  Under CUDA-graph capture
    each call packs into a buffer of its own from the graph's pool, which every replay re-packs."""
    valid = 0
    if torch.cuda.is_current_stream_capturing():
        buf = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=device)
    else:
        key = (tuple((p.data_ptr(), p._version) for p in params), layer.precision, nbytes, device)
        cur = layer.__dict__.get("_wplanes")
        if cur is not None and cur[1] == key:
            buf, valid = cur[0], 1
        else:
            buf = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=device)
            layer.__dict__["_wplanes"] = (buf, key)
    args.wplanes, args.wplanes_bytes, args.wplanes_valid = buf.data_ptr(), buf.numel(), valid
    return buf


def check_params(layer, named):
    """The library reads raw fp32 device pointers of every parameter and floating buffer: refuse anything else (the
    reference would cast or raise)."""
    bufs = [(n, b) for n, b in layer.named_buffers() if b.is_floating_point()]
    for n, t in list(named.items()) + bufs:
        if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
            raise TypeError(f"graphgps_b200.{type(layer).__name__}: parameter/buffer '{n}' must be a contiguous float32 "
                            f"CUDA tensor (got {t.dtype} on {t.device})")


def linear(weight, bias, gw=None, gb=None):
    return _lib.GpsLinear(_lib.ptr(weight), _lib.ptr(bias), _lib.ptr(gw), _lib.ptr(gb))


def batch_norm(mod, gw=None, gb=None):
    return _lib.GpsBatchNorm(_lib.ptr(mod.weight), _lib.ptr(mod.bias), _lib.ptr(mod.running_mean),
                             _lib.ptr(mod.running_var), _lib.ptr(mod.num_batches_tracked),
                             _lib.ptr(gw), _lib.ptr(gb))


def zeroed_grads(named):
    """Gradient buffers zeroed in one multi-tensor fill, so the library skips its memsets (GPS_FLAG_GRADS_ZEROED)."""
    grads = {n: torch.empty_like(p) for n, p in named.items()}
    torch._foreach_zero_(list(grads.values()))
    return grads


def read_x(batch, layer, d=None):
    """batch.x: a float32 CUDA tensor, [num_nodes, d] when d is given."""
    x = batch.x
    if not x.is_cuda:
        raise RuntimeError(f"graphgps_b200.{type(layer).__name__} runs on CUDA tensors only; there is no CPU fallback")
    if x.dtype != torch.float32:
        raise TypeError("batch.x must be float32")
    if d is not None and (x.dim() != 2 or x.shape[1] != d):
        raise ValueError(f"batch.x must have shape [num_nodes, {d}] (got {tuple(x.shape)})")
    return x.contiguous()


def read_edge_attr(batch, x, layer, d):
    """batch.edge_attr [num_edges, d]: float32 on the device of x."""
    e = getattr(batch, "edge_attr", None)
    if e is None:
        raise ValueError(f"graphgps_b200.{type(layer).__name__} needs batch.edge_attr")
    if not torch.is_tensor(e) or e.dtype != torch.float32 or e.device != x.device:
        raise TypeError("batch.edge_attr must be a float32 tensor on the device of batch.x")
    E = int(batch.edge_index.shape[1])
    if e.dim() != 2 or tuple(e.shape) != (E, d):
        raise ValueError(f"batch.edge_attr must have shape [num_edges, {d}] = [{E}, {d}] (got {tuple(e.shape)})")
    return e.contiguous()


def read_attn_bias(batch, x, gs, layer, required):
    """batch.attn_bias [num_graphs * heads, Nmax, Nmax], row g * heads + h for graph g and head h, Nmax = the largest
    graph: float32 on the device of x, or None for no bias (as torch's MultiheadAttention treats attn_mask=None).  A
    missing attribute raises AttributeError when `required`, else it means no bias as well."""
    if required and not hasattr(batch, "attn_bias"):
        raise AttributeError(f"graphgps_b200.{type(layer).__name__} reads batch.attn_bias [num_graphs * heads, Nmax, "
                             "Nmax], which this batch does not have (Graphormer's BiasEncoder writes it)")
    ab = getattr(batch, "attn_bias", None)
    if ab is None:
        return None
    if not torch.is_tensor(ab) or ab.dtype != torch.float32 or ab.device != x.device:
        raise TypeError("batch.attn_bias must be a float32 tensor on the device of batch.x (got "
                        f"{getattr(ab, 'dtype', type(ab))} on {getattr(ab, 'device', None)})")
    want = (gs.B * layer.num_heads, gs.nmax, gs.nmax)
    if tuple(ab.shape) != want:
        raise ValueError(f"batch.attn_bias must have shape [num_graphs * heads, Nmax, Nmax] = {list(want)} "
                         f"(got {list(ab.shape)})")
    if gs.nmax == 0:   # no nodes: nothing attends
        return None
    return ab.contiguous()


class LayerFn(torch.autograd.Function):
    """One autograd node per layer call: forward = <entry>_forward, backward = <entry>_backward.

    apply(layer, call, *inputs, *params), params in layer._param_names order."""

    @staticmethod
    def forward(ctx, layer, call, *tensors):
        n_in = len(tensors) - len(layer._param_names)
        inputs, params = tensors[:n_in], tensors[n_in:]
        dev = inputs[0].device
        named = dict(zip(layer._param_names, params))
        args = layer._args(call, inputs, named)
        args.seed = dropout_seed()
        plan = layer._plan(args, call)
        saved = torch.empty(max(plan[0], 256), dtype=torch.uint8, device=dev)
        ws = workspace(dev, plan[1])
        args.saved, args.saved_bytes = saved.data_ptr(), saved.numel()
        args.workspace, args.workspace_bytes = ws.data_ptr(), ws.numel()
        outs, extra, keep = layer._bind_forward(args, call, inputs, plan, params)
        # Without a live dropout every site has p = 0 and the library reads no offset; with one, the offset is the
        # device-resident snapshot alone (args.offset stays 0)
        snap = None
        if layer.training and layer._dropout_live():
            snap = next_dropout_offset(dev)
            args.offset_dev = snap.data_ptr()
        fn = layer._entry + "_forward"
        _lib.check(getattr(_lib.load(), fn)(C.byref(args), *extra, torch.cuda.current_stream(dev).cuda_stream), fn)
        # the saved buffer lives as long as the autograd node: backward(retain_graph=True) may run again
        ctx.layer, ctx.call, ctx.saved_buf, ctx.keep, ctx.snap = layer, call, saved, keep, snap
        ctx.seed, ctx.training = args.seed, args.training
        ctx.save_for_backward(*tensors)
        return outs if len(outs) > 1 else outs[0]

    @staticmethod
    def backward(ctx, *g_outs):
        layer, call = ctx.layer, ctx.call
        tensors = ctx.saved_tensors
        n_in = len(tensors) - len(layer._param_names)
        inputs, params = tensors[:n_in], tensors[n_in:]
        dev = inputs[0].device
        named = dict(zip(layer._param_names, params))
        grads, flags, g_params = layer._grads(named)
        args = layer._args(call, inputs, named, grads)
        args.flags = flags
        args.seed, args.training = ctx.seed, ctx.training
        if ctx.snap is not None:
            args.offset_dev = ctx.snap.data_ptr()
        g_outs = tuple(None if g is None else g.contiguous() for g in g_outs)
        plan = layer._plan(args, call)
        ws = workspace(dev, plan[1])
        args.saved, args.saved_bytes = ctx.saved_buf.data_ptr(), ctx.saved_buf.numel()
        args.workspace, args.workspace_bytes = ws.data_ptr(), ws.numel()
        g_inputs, extra = layer._bind_backward(args, call, inputs, g_outs, ctx.needs_input_grad[2:], ctx.keep)
        fn = layer._entry + "_backward"
        _lib.check(getattr(_lib.load(), fn)(C.byref(args), *extra, torch.cuda.current_stream(dev).cuda_stream), fn)
        return (None, None) + tuple(g_inputs) + tuple(g_params)
