"""Data-parallel plumbing for the GPSLayer hot path (SURVEY.md section 8e).

Graph mini-batches are independent units: every rank runs its own 256-graph batch through the full
layer with per-replica BatchNorm statistics (the reference has no SyncBN), and the only exchange is
the all-reduce (mean) of the parameter gradients, once per optimiser step over NCCL/NVLink
(the reference's hook would sit between `loss.backward()` and `optimizer.step()`,
graphgps/train/custom_train.py:32-38; the reference itself has no distributed code at all).

`GradBucket` is the product path: ONE static flat fp32 buffer holds the gradients of a set of layers;
every parameter's `.grad` is a view of it and `gps_layer_backward` adds its gradients straight into
those views (GpsLayerArgs.flags, GPS_FLAG_GRADS_ACCUMULATE).  CUDA-graph replays, the optimiser and the collective
therefore all see the same memory: the all-reduce runs in place on the bucket (ReduceOp.AVG on NCCL,
no copy-in / scale / copy-out) and can be captured in the same CUDA graph as the step.  Parameters are
laid out in three contiguous groups per layer in the order the backward pass finishes them - "early" (FFN,
attention output projection, the three GPSLayer norms), "mid" (the local model: A..E / GINE nn / GCN lin and its
BatchNorms, minus the rows of the fused node projection) and "late" (the fused node projection A,B,D,E + in_proj /
to_q,k,v, whose one weight-gradient GEMM is the last kernel of the pass) - and the library records an event per
group, so each group's collective is issued on a communication stream while the rest of the backward pass
(and, in a stack, the backward of the layers below) still runs (`enable_overlap()` / `allreduce_overlapped()`).
"""
from __future__ import annotations

import torch
import torch.distributed as dist

# gradient groups of a GPSLayer in the order the backward pass finishes them (csrc/layer.cu: ev_grads_early / _mid / _done)
_EARLY_PREFIXES = ("ff_linear1.", "ff_linear2.", "norm2.", "norm1_local.", "norm1_attn.",
                   "self_attn.out_proj.", "self_attn.to_out.")
_LATE_PREFIXES = ("self_attn.in_proj", "self_attn.to_q.", "self_attn.to_k.", "self_attn.to_v.",
                  "local_model.A.", "local_model.B.", "local_model.D.", "local_model.E.", "local_model.lin.",
                  "local_model.lin_src.", "local_model.pre_nns.",
                  "self_attn.encoder.layers.0.attention.self.")   # Wcat rows
EARLY, MID, LATE = 0, 1, 2


def _group(name):
    if name.startswith(_EARLY_PREFIXES):
        return EARLY
    return LATE if name.startswith(_LATE_PREFIXES) else MID


def shard_graph_range(num_graphs: int, rank: int, world: int):
    """Graphs [lo, hi) of a global batch that rank `rank` owns (contiguous, balanced)."""
    base, rem = divmod(num_graphs, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class GradBucket:
    """Static flat gradient storage for one or more `graphgps_b200.GPSLayer`s (or any nn.Modules).

    After construction `p.grad` of every parameter is a view of `self.flat`.  Keep them that way:
    zero with `bucket.zero_()` (or `optimizer.zero_grad(set_to_none=False)`), never `set_to_none=True`.
    """

    def __init__(self, layers, device=None):
        self.layers = list(layers)
        entries = []   # (layer index, group, name, param)
        for li, layer in enumerate(self.layers):
            for n, p in layer.named_parameters():
                entries.append((li, _group(n), n, p))
        if not entries:
            raise ValueError("GradBucket: no parameters")
        device = device or entries[0][3].device
        # layer-major; inside a layer early, mid, late.  16-float alignment keeps every view 64-byte aligned.
        order = sorted(range(len(entries)), key=lambda i: (entries[i][0], entries[i][1]))
        offs, off = {}, 0
        self.segments = []   # (layer, group, begin, end) in element offsets
        cur = None
        for i in order:
            li, early, n, p = entries[i]
            if cur is None or cur[0] != li or cur[1] != early:
                if cur is not None:
                    self.segments.append((cur[0], cur[1], cur[2], off))
                cur = [li, early, off]
            offs[i] = off
            off += (p.numel() + 15) // 16 * 16
        self.segments.append((cur[0], cur[1], cur[2], off))
        self.flat = torch.zeros(off, dtype=torch.float32, device=device)
        for i, (li, early, n, p) in enumerate(entries):
            if p.dtype != torch.float32 or p.device != self.flat.device:
                raise TypeError(f"GradBucket: parameter {n} must be float32 on {self.flat.device}")
            p.grad = self.flat[offs[i]:offs[i] + p.numel()].view_as(p)
        self._params = [(li, n, p) for li, _, n, p in entries]
        lo = self.flat.data_ptr()
        hi = lo + self.flat.numel() * 4
        for layer in self.layers:
            layer.__dict__["_grad_bucket"] = (lo, hi)

    def zero_(self):
        self.flat.zero_()
        return self

    def check_attached(self):
        """Raises if some parameter's .grad is no longer a view of this bucket (e.g. after
        `optimizer.zero_grad(set_to_none=True)`): a collective on the bucket would then reduce stale memory."""
        lo = self.flat.data_ptr()
        hi = lo + self.flat.numel() * 4
        for li, n, p in self._params:
            g = p.grad
            if g is None or not (lo <= g.data_ptr() < hi):
                raise RuntimeError(f"GradBucket: .grad of layer {li} parameter '{n}' is not a view of the bucket any "
                                   "more; zero gradients with bucket.zero_() / zero_grad(set_to_none=False)")

    def enable_overlap(self):
        """Give every layer the three events gps_layer_backward records as its gradient groups become final (early:
        FFN / out-proj / GPSLayer norms; mid: local model; done: everything incl. in_proj) and a communication stream on
        which `allreduce_overlapped` runs the collectives."""
        dev = self.flat.device
        self.comm_stream = torch.cuda.Stream(device=dev)
        self.events = []
        for layer in self.layers:
            evs = tuple(torch.cuda.Event() for _ in range(3))
            for ev in evs:
                ev.record(torch.cuda.current_stream(dev))     # materialise the cudaEvent_t handles
            layer.__dict__["grad_events"] = evs
            self.events.append(evs)
        return self

    def allreduce_overlapped(self, group=None):
        """Call right after backward() has been enqueued (layers ran last-to-first).  Every segment is reduced as soon as
        its event fires: under the rest of that layer's backward pass and under the backward of the layers below it.
        Only the last-finished segment (layer 0's fused-projection gradients, 7d^2 floats) is exposed; the caller's stream
        waits for the communication stream at the end.  Works after a CUDA-graph replay of the step as well: the library
        records the events as external event nodes under capture, so the collectives stay outside the graph (NCCL kernels
        captured inside a graph cost ~0.5 ms of host time per launch with torch 2.11 / NCCL 2.28)."""
        self.check_attached()
        cur = torch.cuda.current_stream(self.flat.device)
        cs = self.comm_stream
        with torch.cuda.stream(cs):
            for li in reversed(range(len(self.layers))):
                for grp in (EARLY, MID, LATE):
                    seg = self.segment(li, grp)
                    if seg is None:
                        continue
                    cs.wait_event(self.events[li][grp])
                    self.allreduce(group, segments=[seg])
        cur.wait_stream(cs)

    def segment(self, layer: int, grp):
        grp = {True: EARLY, False: None}.get(grp, grp) if isinstance(grp, bool) else grp
        if grp is None:   # legacy "not early": everything after the early group of this layer
            parts = [(b, en) for li, g, b, en in self.segments if li == layer and g != EARLY]
            return self.flat[min(b for b, _ in parts):max(e for _, e in parts)] if parts else None
        for li, g, b, en in self.segments:
            if li == layer and g == grp:
                return self.flat[b:en]
        return None

    def allreduce(self, group=None, segments=None):
        """In-place mean over ranks of the whole bucket (or of the given list of flat slices)."""
        world = dist.get_world_size(group)
        if world == 1:
            return
        if segments is None:
            self.check_attached()
        parts = segments if segments is not None else [self.flat]
        avg = dist.get_backend(group) == "nccl"
        for t in parts:
            if avg:
                dist.all_reduce(t, op=dist.ReduceOp.AVG, group=group)
            else:   # gloo has no AVG
                dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
                t.mul_(1.0 / world)


def allreduce_gradients(params, bucket=None, group=None):
    """Generic fallback for parameters whose .grad is NOT bucket-backed: all-reduce (mean) through a flat staging
    buffer (copy in, reduce, copy out).  Returns the staging buffer for reuse."""
    grads = [p.grad for p in params if p.grad is not None]
    if not grads:
        return bucket
    n = sum(g.numel() for g in grads)
    if bucket is None or bucket.numel() != n or bucket.device != grads[0].device:
        bucket = torch.empty(n, dtype=grads[0].dtype, device=grads[0].device)
    views, off = [], 0
    for g in grads:
        views.append(bucket[off:off + g.numel()].view_as(g))
        off += g.numel()
    torch._foreach_copy_(views, grads)
    world = dist.get_world_size(group)
    dist.all_reduce(bucket, op=dist.ReduceOp.SUM, group=group)
    bucket.mul_(1.0 / world)
    torch._foreach_copy_(grads, views)
    return bucket
