"""RWSE, the random-walk structural encoding, on the device.

`rw_landing_probs(batch, ksteps)` computes what the reference precomputes per graph on the CPU before training
(graphgps/transform/posenc_stats.py:get_rw_landing_probs, master_loader.py:199-215):

    out[i, j] = (P^ksteps[j])[i, i],   P = D_out^-1 A of i's graph,   out [num_nodes, len(ksteps)] float32

with A[s, d] the number of edges s -> d of batch.edge_index (duplicates add up, self-loops count), a node without
out-edges a zero row of P, and P^0 = I.  P is block-diagonal over the graphs of a batch, so the result equals the
reference applied graph by graph and concatenated in node order.

`KernelPENodeEncoder` is the drop-in for graphgps/encoder/kernel_pos_encoder.py:KernelPENodeEncoder (model "linear"):

    batch.x = cat(h, pe_encoder(raw_norm(pestat)))      h = linear_x(batch.x) with expand_x, else batch.x

Same state_dict names, module order and initial draws as the reference.  One C call per direction (libgps_b200.so,
sm_90a); there is no CPU fallback.  The landing probabilities read the batch's cached graph structure and its Nmax
(one host read per batch object), so a step can be captured in a CUDA graph once that is cached.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from ._call import LayerFn, PlanCache, batch_norm, check_params, linear, workspace
from .graph import graph_of

KERNEL_TYPES = ("RWSE", "HKdiagSE", "ElstaticSE")


def _ksteps(ksteps):
    ks = [int(k) for k in ksteps]
    if not ks:
        raise ValueError("ksteps must not be empty")
    if any(k < 0 for k in ks):
        raise ValueError(f"ksteps must be >= 0 (got {ks})")
    if len(ks) > _lib.RWSE_MAX_COLS or max(ks) > _lib.RWSE_MAX_STEPS:
        raise NotImplementedError(f"graphgps_b200.rw_landing_probs: at most {_lib.RWSE_MAX_COLS} ksteps of at most "
                                  f"{_lib.RWSE_MAX_STEPS} steps are built (got {len(ks)}, max {max(ks)})")
    return ks


def rw_landing_probs(batch, ksteps) -> torch.Tensor:
    """Random-walk landing probabilities [num_nodes, len(ksteps)] float32 of every node of `batch`, on its device."""
    ks = _ksteps(ksteps)
    ei = batch.edge_index
    if not torch.is_tensor(ei) or not ei.is_cuda:
        raise RuntimeError("graphgps_b200.rw_landing_probs runs on CUDA tensors only; there is no CPU fallback")
    gs = graph_of(batch)
    out = torch.empty(gs.N, len(ks), dtype=torch.float32, device=ei.device)
    if gs.N == 0:
        return out
    ws = workspace(ei.device, 8 * gs.N)
    arr = (C.c_int32 * len(ks))(*ks)
    rc = _lib.load().gps_rwse_landing(C.byref(gs.desc), arr, len(ks), gs.nmax, out.data_ptr(), ws.data_ptr(),
                                      ws.numel(), torch.cuda.current_stream(ei.device).cuda_stream)
    _lib.check(rc, "gps_rwse_landing")
    return out


def cached_rw_landing_probs(batch, ksteps) -> torch.Tensor:
    """`rw_landing_probs`, computed once per batch object and ksteps and kept on the batch's graph structure (which
    `graph_of` builds once per batch object), so the layers, a second encoder and a CUDA-graph capture share it."""
    gs = graph_of(batch)
    cache = gs.__dict__.setdefault("_rwse", {})
    key = tuple(int(k) for k in ksteps)
    hit = cache.get(key)
    if hit is None:
        hit = cache[key] = rw_landing_probs(batch, key)
    return hit


class KernelPENodeEncoder(nn.Module):
    """Kernel-based structural encoding node encoder (reference: graphgps/encoder/kernel_pos_encoder.py).

    The reference reads dim_in and its `posenc_<kernel_type>` settings from GraphGym's cfg; here they are arguments
    (graphgps_b200.graphgym.install_rwse binds them from cfg).  With `ksteps` (RWSE only) the statistics are computed on
    the device from the batch's edges instead of read from `batch.pestat_RWSE`, which is then set to them."""

    _entry = "gps_kernel_pe"

    def __init__(self, dim_in, dim_emb, num_kernel_times, dim_pe, kernel_type="RWSE", raw_norm_type="batchnorm",
                 model="linear", expand_x=True, ksteps=None, pass_as_var=False):
        super().__init__()
        if kernel_type not in KERNEL_TYPES:
            raise ValueError(f"kernel_type must be one of {KERNEL_TYPES} (got {kernel_type!r})")
        dim_in, dim_emb, K, dim_pe = int(dim_in), int(dim_emb), int(num_kernel_times), int(dim_pe)
        if dim_emb - dim_pe < 0:   # the reference's check and message
            raise ValueError(f"PE dim size {dim_pe} is too large for desired embedding size of {dim_emb}.")
        model = str(model).lower()
        if model == "mlp":
            raise NotImplementedError("graphgps_b200.KernelPENodeEncoder: model 'mlp' is not built (no shipped config "
                                      "uses it; 'linear' is)")
        if model != "linear":
            raise ValueError(f"{type(self).__name__}: Does not support '{model}' encoder model.")
        if pass_as_var:
            raise NotImplementedError("graphgps_b200.KernelPENodeEncoder: pass_as_var is not built")
        if not (1 <= dim_in <= 4096 and 1 <= dim_pe and dim_emb <= 4096 and 1 <= K <= _lib.RWSE_MAX_COLS):
            raise NotImplementedError(f"graphgps_b200.KernelPENodeEncoder: needs 1 <= dim_in, dim_pe and dim_emb <= "
                                      f"4096 and 1 <= num_kernel_times <= {_lib.RWSE_MAX_COLS} (got {dim_in}, "
                                      f"{dim_pe}, {dim_emb}, {K})")
        if ksteps is not None:
            if kernel_type != "RWSE":
                raise ValueError("ksteps (statistics computed on the device) is built for kernel_type 'RWSE' only")
            ksteps = tuple(_ksteps(ksteps))
            if len(ksteps) != K:
                raise ValueError(f"len(ksteps) = {len(ksteps)} must equal num_kernel_times = {K}")
        self.kernel_type, self.ksteps = kernel_type, ksteps
        self.dim_in, self.dim_emb, self.dim_pe, self.num_kernel_times = dim_in, dim_emb, dim_pe, K
        self.pass_as_var = False
        # the reference's modules in its order, so the same seed draws the same parameters (kernel_pos_encoder.py:53-80)
        if expand_x and dim_emb - dim_pe > 0:
            self.linear_x = nn.Linear(dim_in, dim_emb - dim_pe)
        self.expand_x = expand_x and dim_emb - dim_pe > 0
        if not self.expand_x and dim_in != dim_emb - dim_pe:
            raise ValueError(f"without expand_x, batch.x is concatenated as it is: dim_in must be dim_emb - dim_pe = "
                             f"{dim_emb - dim_pe} (got {dim_in})")
        self.raw_norm = nn.BatchNorm1d(K) if str(raw_norm_type).lower() == "batchnorm" else None
        self.pe_encoder = nn.Linear(K, dim_pe)
        self._param_names = [n for n, _ in self.named_parameters()]
        self._plans = PlanCache(self._entry, _lib.GpsKernelPePlan)

    # ------------------------------------------------------------------ hooks of _call.LayerFn
    def _dropout_live(self):
        return False

    def _args(self, N, inputs, named, grads=None):
        g = grads or {}
        check_params(self, named)
        a = _lib.GpsKernelPeArgs()
        a.N, a.K, a.dim_in, a.dim_emb, a.dim_pe = N, self.num_kernel_times, self.dim_in, self.dim_emb, self.dim_pe
        a.expand_x = 1 if self.expand_x else 0
        a.batch_norm = 1 if self.raw_norm is not None else 0
        a.training = 1 if self.training else 0
        a.x, a.pestat = inputs[0].data_ptr(), inputs[1].data_ptr()
        a.pe_encoder = linear(named["pe_encoder.weight"], named["pe_encoder.bias"], g.get("pe_encoder.weight"),
                              g.get("pe_encoder.bias"))
        if self.expand_x:
            a.linear_x = linear(named["linear_x.weight"], named["linear_x.bias"], g.get("linear_x.weight"),
                                g.get("linear_x.bias"))
        if self.raw_norm is not None:
            a.raw_norm = batch_norm(self.raw_norm, g.get("raw_norm.weight"), g.get("raw_norm.bias"))
        return a

    def _plan(self, args, N):
        return self._plans((N, self.training), args)

    def _bind_forward(self, args, N, inputs, plan, params):
        out = torch.empty(N, self.dim_emb, dtype=torch.float32, device=inputs[0].device)
        args.out = out.data_ptr()
        return (out,), (), None

    def _grads(self, named):
        grads = {n: torch.empty_like(p) for n, p in named.items()}   # the library writes every gradient whole
        return grads, 0, tuple(grads[n] for n in self._param_names)

    def _bind_backward(self, args, N, inputs, g_outs, needs, keep):
        g_x = torch.empty_like(inputs[0])
        args.grad_out, args.grad_x = _lib.ptr(g_outs[0]), g_x.data_ptr()
        return (g_x, None), ()

    # ------------------------------------------------------------------ forward
    def _pestat(self, batch):
        if self.ksteps is not None:
            pestat = cached_rw_landing_probs(batch, self.ksteps)
            batch.pestat_RWSE = pestat
            return pestat
        name = f"pestat_{self.kernel_type}"
        if not hasattr(batch, name):   # the reference's check and message
            raise ValueError(f"Precomputed '{name}' variable is required for {type(self).__name__}; set config "
                             f"'posenc_{self.kernel_type}.enable' to True, and also set 'posenc.kernel.times' values")
        return getattr(batch, name)

    def forward(self, batch):
        x = batch.x
        if not torch.is_tensor(x) or not x.is_cuda:
            raise RuntimeError(f"graphgps_b200.{type(self).__name__} runs on CUDA tensors only; there is no CPU "
                               "fallback")
        if x.dtype != torch.float32 or x.dim() != 2 or x.shape[1] != self.dim_in:
            raise ValueError(f"batch.x must be float32 [num_nodes, {self.dim_in}] (got {x.dtype} {list(x.shape)})")
        N = int(x.shape[0])
        pestat = self._pestat(batch)
        if not torch.is_tensor(pestat) or pestat.dtype != torch.float32 or pestat.device != x.device or \
                tuple(pestat.shape) != (N, self.num_kernel_times):
            raise ValueError(f"pestat_{self.kernel_type} must be float32 [num_nodes, {self.num_kernel_times}] = "
                             f"[{N}, {self.num_kernel_times}] on {x.device} (got {getattr(pestat, 'dtype', None)} "
                             f"{list(getattr(pestat, 'shape', []))} on {getattr(pestat, 'device', None)})")
        if self.training and self.raw_norm is not None and N <= 1:   # as BatchNorm1d refuses it
            raise ValueError(f"Expected more than 1 value per channel when training, got input size "
                             f"{[N, self.num_kernel_times]}")
        params = [p for _, p in self.named_parameters()]
        batch.x = LayerFn.apply(self, N, x.contiguous(), pestat.detach().contiguous(), *params)
        return batch

    def extra_repr(self):
        return (f"kernel_type={self.kernel_type}, dim_in={self.dim_in}, dim_emb={self.dim_emb}, dim_pe={self.dim_pe}, "
                f"num_kernel_times={self.num_kernel_times}, expand_x={self.expand_x}, ksteps={self.ksteps}, "
                "backend=libgps_b200(sm_90a)")
