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

import torch
import torch.nn as nn

from . import _lib
from ._call import LayerFn, PlanCache, batch_norm, check_params, linear, read_edge_attr, read_x, weight_planes
from .graph import graph_of

_ACTS = ("relu", "gelu")


class _CustomGnnBase(nn.Module):
    """What both layers share: argument block, plan key, weight planes and forward."""

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

    # ------------------------------------------------------------------ hooks of _call.LayerFn; call = the graph
    _entry = "gps_custom_gnn"

    def _dropout_live(self):
        return self.dropout > 0

    def _args(self, gs, inputs, named, grads=None):
        g = grads or {}
        check_params(self, named)
        a = _lib.GpsCustomGnnArgs()
        a.d = self.out_dim
        a.kind = _lib.CUSTOM_GATEDGCN if self._gated else _lib.CUSTOM_GINE
        a.act = _lib.ACT[self.act] if self._gated else 0
        a.training = 1 if self.training else 0
        a.precision = _lib.PRECISION[self.precision]
        a.residual = 1 if self.residual else 0
        a.dropout = float(self.dropout)
        a.graph = gs.desc

        def lin(prefix):
            w, b = prefix + ".weight", prefix + ".bias"
            return linear(named[w], named[b], g.get(w), g.get(b))

        if self._gated:
            a.A, a.B, a.C, a.D, a.E = (lin(n) for n in "ABCDE")
            a.bn_node_x = batch_norm(self.bn_node_x, g.get("bn_node_x.weight"), g.get("bn_node_x.bias"))
            a.bn_edge_e = batch_norm(self.bn_edge_e, g.get("bn_edge_e.weight"), g.get("bn_edge_e.bias"))
        else:
            a.nn0, a.nn2 = lin("model.nn.0"), lin("model.nn.2")
            a.gine_eps = self._eps_host()
        return a

    def _plan(self, args, gs):
        """gps_custom_gnn_plan is pure in its arguments' sizes and modes."""
        return self._plans((gs.N, gs.E, self.precision, bool(args.training), self.dropout > 0), args)

    def _bind_forward(self, args, gs, inputs, plan, params):
        x, e = inputs
        x_out = torch.empty_like(x)
        e_out = torch.empty_like(e) if self._gated else None
        wp = weight_planes(self, args, plan[2], params, x.device)
        args.x, args.edge_attr, args.x_out, args.edge_out = x.data_ptr(), e.data_ptr(), x_out.data_ptr(), _lib.ptr(e_out)
        return ((x_out, e_out) if self._gated else (x_out,)), (), wp

    def _grads(self, named):
        grads = {n: torch.empty_like(p) for n, p in named.items()}   # the library writes every gradient whole
        return grads, 0, tuple(grads[n] for n in self._param_names)

    def _bind_backward(self, args, gs, inputs, g_outs, needs, wp):
        x, e = inputs
        g_x = torch.empty_like(x)
        g_e = torch.empty_like(e) if needs[1] else None
        args.x, args.edge_attr = x.data_ptr(), e.data_ptr()
        args.grad_x_out, args.grad_edge_out = g_outs[0].data_ptr(), _lib.ptr(g_outs[1]) if self._gated else 0
        args.grad_x, args.grad_edge_attr = g_x.data_ptr(), _lib.ptr(g_e)
        args.wplanes, args.wplanes_bytes, args.wplanes_valid = wp.data_ptr(), wp.numel(), 1
        return (g_x, g_e), ()

    def forward(self, batch):
        x = read_x(batch, self, self.out_dim)
        e = read_edge_attr(batch, x, self, self.out_dim)
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
        out = LayerFn.apply(self, gs, x, e, *params)
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
        self._plans = PlanCache(self._entry, _lib.GpsCustomGnnPlan)

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
        self._plans = PlanCache(self._entry, _lib.GpsCustomGnnPlan)

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
