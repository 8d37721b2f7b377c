"""H100-native drop-ins for the node-prediction heads of the node-level configs and their losses:
`graphgps.head.inductive_node.GNNInductiveNodeHead` (`gnn.head: inductive_node`), GraphGym's `GNNNodeHead`
(`gnn.head: node`), `graphgps.loss.weighted_cross_entropy` and GraphGym's multiclass `cross_entropy`.

Same `forward(batch)` contract as the reference, with GraphGym's MLP of L = layers_post_mp Linears (PyG 2.2):

    h = x; h = normalize(relu(Linear(h))) for the L - 1 hidden layers (width dim_inner); batch.x = Linear(h)
    InductiveNodeHead   returns (batch.x, batch.y)
    NodeHead            returns (batch.x[mask], batch.y[mask]), mask = batch[f'{batch.split}_mask']

normalize(h) = h / max(||h||_2, 1e-12) per row: GraphGym builds the hidden layers from LayerConfig's defaults (no
BatchNorm, no dropout, ReLU, L2 normalisation), whatever cfg.gnn says.  The state dict keeps GraphGym's names.

NodeHead turns the split's boolean mask into a row list with one host read per (batch, split, mask version) and caches
it, with the selected labels, on the batch: the next call on that batch reads nothing from the device and returns the
same label tensor.  The losses check the labels once per label tensor (one host read, cached on the tensor), keep the
loss on the device, and compute pred_score in the same pass; pred_score is differentiable.

One C call per direction (libgps_b200.so, sm_90a); there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from ._call import LayerFn, PlanCache, check_params, linear, read_x, workspace
from .graph import _cache_get, _cache_put

_ROWS_ATTR = "_gps_b200_node_rows"
_LABEL_ATTR = "_gps_b200_label_check"


class _GymLinear(nn.Module):
    """torch_geometric.graphgym.models.layer.Linear: its parameters live in `model` (torch_geometric.nn.Linear)."""

    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.model = nn.Linear(dim_in, dim_out, bias=True)


class _GymGeneralLayer(nn.Module):
    """GeneralLayer('linear') from LayerConfig defaults: `layer` holds the Linear; ReLU and the L2 normalisation have no
    parameters."""

    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.layer = _GymLinear(dim_in, dim_out)


class _GymMultiLayer(nn.Module):
    """GeneralMultiLayer: Layer_0 .. Layer_{n-1}."""

    def __init__(self, n, dim_in, dim_inner):
        super().__init__()
        for i in range(n):
            self.add_module(f"Layer_{i}", _GymGeneralLayer(dim_in if i == 0 else dim_inner, dim_inner))


class _GymMLP(nn.Module):
    """GraphGym's MLP: `model` = Sequential(GeneralMultiLayer, Linear) for L > 1, Sequential(Linear) for L = 1."""

    def __init__(self, dim_in, dim_out, L, dim_inner):
        super().__init__()
        if L > 1:
            self.model = nn.Sequential(_GymMultiLayer(L - 1, dim_in, dim_inner), _GymLinear(dim_inner, dim_out))
        else:
            self.model = nn.Sequential(_GymLinear(dim_in, dim_out))


class _Call:
    """Per-call state of LayerFn: N, and the selected rows (int64 [M]) or None."""

    def __init__(self, N, rows):
        self.N, self.rows = N, rows
        self.M = 0 if rows is None else int(rows.shape[0])


class _NodeHead(nn.Module):
    _entry = "gps_node_head"

    def __init__(self, dim_in, dim_out, layers_post_mp=1, dim_inner=None, precision="fp32"):
        super().__init__()
        if precision not in _lib.PRECISION:
            raise ValueError(f"precision must be one of {tuple(_lib.PRECISION)} (got {precision!r})")
        L = int(layers_post_mp)
        if not 1 <= L <= _lib.NODE_HEAD_MAX_L:
            raise NotImplementedError(f"graphgps_b200.{type(self).__name__}: 1 <= layers_post_mp <= "
                                      f"{_lib.NODE_HEAD_MAX_L} (got {layers_post_mp})")
        dim_inner = int(dim_in) if dim_inner is None else int(dim_inner)   # MLP: dim_in when cfg.gnn.dim_inner is None
        for w in (dim_in, dim_out, dim_inner):
            if not 1 <= int(w) <= 4096:
                raise NotImplementedError(f"graphgps_b200.{type(self).__name__}: needs 1 <= dim_in, dim_inner, "
                                          f"dim_out <= 4096 (got {dim_in}, {dim_inner}, {dim_out})")
        self.dim_in, self.dim_out, self.dim_inner, self.L = int(dim_in), int(dim_out), dim_inner, L
        self.precision = precision
        # GraphGym's modules in its construction order, so the same seed draws the same parameters
        self.layer_post_mp = _GymMLP(self.dim_in, self.dim_out, L, dim_inner)
        self._param_names = [n for n, _ in self.named_parameters()]
        self._plans = PlanCache(self._entry, _lib.GpsNodeHeadPlan)

    # ------------------------------------------------------------------ hooks of _call.LayerFn
    def _dropout_live(self):
        return False

    def _args(self, call, inputs, named, grads=None):
        g = grads or {}
        check_params(self, named)
        a = _lib.GpsNodeHeadArgs()
        a.L, a.precision = self.L, _lib.PRECISION[self.precision]
        a.training = 1 if self.training else 0
        a.dim_in, a.dim_inner, a.dim_out = self.dim_in, self.dim_inner, self.dim_out
        a.N, a.M = call.N, call.M
        a.x = inputs[0].data_ptr()
        a.rows = _lib.ptr(call.rows)
        names = self._param_names
        for i in range(self.L):
            w, b = names[2 * i], names[2 * i + 1]
            a.fc[i] = linear(named[w], named[b], g.get(w), g.get(b))
        return a

    def _plan(self, args, call):
        return self._plans((call.N, self.precision), args)

    def _bind_forward(self, args, call, inputs, plan, params):
        x = inputs[0]
        y = torch.empty(call.N, self.dim_out, dtype=torch.float32, device=x.device)
        args.y = y.data_ptr()
        if call.rows is None:
            return (y,), (), None
        pred = torch.empty(call.M, self.dim_out, dtype=torch.float32, device=x.device)
        args.pred = pred.data_ptr()
        return (y, pred), (), None

    def _grads(self, named):
        grads = {n: torch.empty_like(p) for n, p in named.items()}   # the library writes every gradient whole
        return grads, 0, tuple(grads[n] for n in self._param_names)

    def _bind_backward(self, args, call, inputs, g_outs, needs, keep):
        g_x = torch.empty_like(inputs[0])
        args.grad_y = _lib.ptr(g_outs[0])
        if call.rows is not None:
            args.grad_pred = _lib.ptr(g_outs[1])
        args.grad_x = g_x.data_ptr()
        return (g_x,), ()

    def _run(self, batch, rows):
        x = read_x(batch, self, self.dim_in)
        params = [p for _, p in self.named_parameters()]
        return LayerFn.apply(self, _Call(x.shape[0], rows), x, *params)

    def extra_repr(self):
        return (f"dim_in={self.dim_in}, dim_out={self.dim_out}, layers_post_mp={self.L}, dim_inner={self.dim_inner}, "
                f"backend=libgps_b200(sm_90a), precision={self.precision}")


class InductiveNodeHead(_NodeHead):
    """Inductive node-prediction head (reference: graphgps/head/inductive_node.py, GNNInductiveNodeHead)."""

    def forward(self, batch):
        batch.x = self._run(batch, None)
        return batch.x, batch.y


class _Rows:
    """The row list and selected labels of one (batch, split): valid while the mask and labels are the same tensors at
    the same versions."""

    def __init__(self):
        self.by_split = {}


def _rows_of(batch, x):
    split = batch.split
    mask, y = getattr(batch, f"{split}_mask"), batch.y
    if not torch.is_tensor(mask) or mask.dtype != torch.bool or tuple(mask.shape) != (x.shape[0],) or \
            mask.device != x.device:
        raise ValueError(f"batch.{split}_mask must be a bool [num_nodes] = [{x.shape[0]}] tensor on {x.device}")
    key = (mask.data_ptr(), mask._version, y.data_ptr(), y._version, tuple(y.shape))
    cache = _cache_get(batch, _ROWS_ATTR, _Rows)
    if cache is None:
        cache = _Rows()
        _cache_put(batch, cache, _ROWS_ATTR)
    hit = cache.by_split.get(split)
    if hit is not None and hit[0] == key:
        return hit[1], hit[2]
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError("graphgps_b200.NodeHead reads the split's mask on the host once per batch and cannot do so "
                           "inside a CUDA-graph capture: run the head on this batch once before capturing")
    rows = mask.nonzero().flatten()   # the one host read per (batch, split, mask version)
    labels = y[rows]
    cache.by_split[split] = (key, rows, labels)
    return rows, labels


class NodeHead(_NodeHead):
    """Transductive node-prediction head (reference: GraphGym's GNNNodeHead, `gnn.head: node`): the MLP over every
    node, then the rows of the batch's current split."""

    def forward(self, batch):
        x = read_x(batch, self, self.dim_in)
        rows, labels = _rows_of(batch, x)
        y, pred = self._run(batch, rows)
        batch.x = y
        return pred, labels


# ---------------------------------------------------------------------------------------------------------- losses
def _check_labels(true, K):
    """int64 labels in [0, K): one host read per label tensor (data, version, shape), cached on the tensor."""
    if true.dtype != torch.int64:
        raise TypeError(f"labels must be int64 (got {true.dtype})")
    key = (true.data_ptr(), true._version, tuple(true.shape), K)
    if getattr(true, _LABEL_ATTR, None) == key:
        return
    if true.numel():
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("graphgps_b200: the labels are checked on the host once per label tensor and cannot be "
                               "inside a CUDA-graph capture: run the loss on them once before capturing")
        has_ignore, lo, hi = torch.stack([(true == -100).any().long(), true.min(), true.max()]).tolist()
        if has_ignore:
            raise NotImplementedError("graphgps_b200: label -100 (ignore_index) is not built")
        if lo < 0 or hi >= K:
            raise IndexError(f"labels must lie in [0, {K}) (got [{lo}, {hi}])")
    setattr(true, _LABEL_ATTR, key)


class _LossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, true, weighted):
        M = pred.shape[0]
        Cn = pred.shape[1] if pred.dim() == 2 else 1
        a = _lib.GpsNodeLossArgs(M=M, C=Cn, weighted=int(weighted))
        plan = _lib.GpsNodeLossPlan()
        lib = _lib.load()
        _lib.check(lib.gps_node_loss_plan(C.byref(a), C.byref(plan)), "gps_node_loss_plan")
        dev = pred.device
        saved = torch.empty(max(int(plan.saved_bytes), 256), dtype=torch.uint8, device=dev)
        ws = workspace(dev, int(plan.fwd_workspace_bytes))
        loss = torch.empty((), dtype=torch.float32, device=dev)
        score = torch.empty_like(pred)
        a.pred, a.label, a.loss, a.pred_score = _lib.ptr(pred), _lib.ptr(true), loss.data_ptr(), _lib.ptr(score)
        a.saved, a.saved_bytes, a.workspace, a.workspace_bytes = saved.data_ptr(), saved.numel(), ws.data_ptr(), ws.numel()
        st = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.gps_node_loss_forward(C.byref(a), st), "gps_node_loss_forward")
        ctx.args, ctx.saved_buf = (M, Cn, int(weighted)), saved
        # an unused output's gradient arrives as None, not zeros: a zero loss gradient over weights that sum to 0 is
        # NaN (as in torch), where no loss gradient at all leaves the pred_score path finite
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(true, score)
        return loss, score

    @staticmethod
    def backward(ctx, g_loss, g_score):
        true, score = ctx.saved_tensors
        M, Cn, weighted = ctx.args
        grad = torch.empty_like(score)
        a = _lib.GpsNodeLossArgs(M=M, C=Cn, weighted=weighted)
        a.label, a.pred_score, a.grad_pred = _lib.ptr(true), _lib.ptr(score), _lib.ptr(grad)
        a.grad_loss = _lib.ptr(None if g_loss is None else g_loss.contiguous())
        a.grad_score = _lib.ptr(None if g_score is None else g_score.contiguous())
        a.saved, a.saved_bytes = ctx.saved_buf.data_ptr(), ctx.saved_buf.numel()
        _lib.check(_lib.load().gps_node_loss_backward(C.byref(a), torch.cuda.current_stream(score.device).cuda_stream),
                   "gps_node_loss_backward")
        return grad, None, None


def _loss(pred, true, weighted, what):
    if not (pred.is_cuda and true.is_cuda):
        raise RuntimeError(f"graphgps_b200.{what} runs on CUDA tensors only; there is no CPU fallback")
    if pred.dtype != torch.float32:
        raise TypeError(f"graphgps_b200.{what}: pred must be float32 (got {pred.dtype})")
    if true.device != pred.device:
        raise ValueError(f"graphgps_b200.{what}: pred and labels must be on one device")
    if pred.dim() not in (1, 2) or (pred.dim() == 1 and not weighted) or true.dim() != 1 or \
            true.shape[0] != pred.shape[0]:
        raise ValueError(f"graphgps_b200.{what}: needs pred [M, C] (or [M], weighted) and labels [M] (got "
                         f"{list(pred.shape)} and {list(true.shape)})")
    Cn = pred.shape[1] if pred.dim() == 2 else 1
    if weighted and Cn == 1 and pred.dim() == 2:
        raise ValueError(f"graphgps_b200.{what}: a binary pred is 1-D, as compute_loss squeezes it")
    if not 1 <= Cn <= _lib.NODE_LOSS_MAX_C:
        raise NotImplementedError(f"graphgps_b200.{what}: 1 <= C <= {_lib.NODE_LOSS_MAX_C} (got {Cn})")
    _check_labels(true, max(Cn, 2))
    return _LossFn.apply(pred.contiguous(), true.contiguous(), weighted)


def weighted_cross_entropy(pred, true):
    """graphgps/loss/weighted_cross_entropy.py: (loss, log_softmax(pred)) for pred [M, C], (loss, sigmoid(pred)) for a
    binary pred [M], with the class weights w_c = (M - count_c) / M of this batch."""
    return _loss(pred, true, True, "weighted_cross_entropy")


def cross_entropy(pred, true):
    """GraphGym's multiclass cross_entropy: (nll_loss(log_softmax(pred), true), log_softmax(pred)) for pred [M, C]."""
    return _loss(pred, true, False, "cross_entropy")
