"""Per-mini-batch graph structure (CSR by destination, CSC by source, graph offsets) on the GPU.

Built once per batch by `gps_graph_build` and cached on the batch object, so the L layers of a
GPSModel and their backward passes share it.  This replaces what the reference redoes in every
layer: PyG propagate's index_select/scatter bookkeeping (graphgps/layer/gatedgcn_layer.py:67-70,
118-123) and to_dense_batch's bincount/cumsum/max().item() host sync (gps_layer.py:199).
"""
from __future__ import annotations

import ctypes as C
import os
import weakref

import torch

from . import _lib

_CACHE_ATTR = "_gps_b200_graph"


class GraphStructure:
    """Owns the int32 storage and the C-side GpsGraph descriptor."""

    def __init__(self, edge_index: torch.Tensor, batch: torch.Tensor, num_graphs: int):
        if not edge_index.is_cuda:
            raise RuntimeError("graphgps_b200 runs on CUDA tensors only (no CPU fallback)")
        if edge_index.dtype != torch.int64 or batch.dtype != torch.int64:
            raise TypeError("edge_index and batch must be int64 (as PyG collation produces)")
        if edge_index.dim() != 2 or edge_index.shape[0] != 2:
            raise ValueError("edge_index must have shape [2, E]")
        lib = _lib.load()
        if os.environ.get("GPS_B200_CHECK", "0") == "1" and edge_index.numel():
            # debug switch: the CSR build scatters through edge_index unchecked (one host sync when enabled)
            lo, hi = int(edge_index.min()), int(edge_index.max())
            if lo < 0 or hi >= int(batch.shape[0]):
                raise IndexError(f"edge_index values [{lo}, {hi}] out of range for {int(batch.shape[0])} nodes")
        self.N = int(batch.shape[0])
        self.E = int(edge_index.shape[1])
        self.B = int(num_graphs)
        self.edge_index = edge_index.contiguous()
        self.batch = batch.contiguous()
        nbytes = lib.gps_graph_bytes(self.N, self.E, self.B)
        self.storage = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=edge_index.device)
        self.desc = _lib.GpsGraph()
        stream = torch.cuda.current_stream(edge_index.device).cuda_stream
        rc = lib.gps_graph_build(self.edge_index.data_ptr(), self.batch.data_ptr(), self.N, self.E, self.B,
                                 self.storage.data_ptr(), self.storage.numel(), C.byref(self.desc), stream)
        _lib.check(rc, "gps_graph_build")
        self.key = (edge_index.data_ptr(), batch.data_ptr(), self.N, self.E, edge_index._version, batch._version)

    @property
    def nmax(self) -> int:
        """Size of the largest graph (to_dense_batch's Nmax, the side of batch.attn_bias).  Read from the device once
        per batch and cached; inside a CUDA-graph capture it must already be cached (GPSStack.capture reads it in its
        warm-up), because the read synchronises."""
        v = self.__dict__.get("_nmax")
        if v is None:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("GraphStructure.nmax is read from the device and cannot be read inside a CUDA-graph "
                                   "capture: read graph_of(batch).nmax before capturing")
            v = int(torch.diff(self.graph_ptr).max()) if self.B > 0 else 0
            self.__dict__["_nmax"] = v
        return v

    def _view(self, addr, n):
        off = addr - self.storage.data_ptr()
        return self.storage[off:off + 4 * n].view(torch.int32)

    # int32 tensor views (for tests / debugging)
    @property
    def dst_ptr(self): return self._view(self.desc.dst_ptr, self.N + 1)
    @property
    def dst_src(self): return self._view(self.desc.dst_src, self.E)
    @property
    def dst_eid(self): return self._view(self.desc.dst_eid, self.E)
    @property
    def src_ptr(self): return self._view(self.desc.src_ptr, self.N + 1)
    @property
    def src_dst(self): return self._view(self.desc.src_dst, self.E)
    @property
    def src_eid(self): return self._view(self.desc.src_eid, self.E)
    @property
    def graph_ptr(self): return self._view(self.desc.graph_ptr, self.B + 1)


def _num_graphs(batch_obj) -> int:
    ng = getattr(batch_obj, "num_graphs", None)
    if ng is not None:
        return int(ng)
    ptr = getattr(batch_obj, "ptr", None)
    if ptr is not None:
        return int(ptr.shape[0]) - 1
    b = batch_obj.batch
    # one device->host sync per *batch* (not per layer); PyG Batch objects never reach this line
    return int(b[-1].item()) + 1 if b.numel() else 0


_side_cache = weakref.WeakKeyDictionary()   # {attribute: value} of batch objects whose attributes do not round-trip


def _cache_get(batch_obj, attr=_CACHE_ATTR, typ=GraphStructure):
    """The value cached on `batch_obj` under `attr` if it is a `typ`, else None (by default its graph structure)."""
    # PyG Data/Batch route setattr/getattr through their storage object (underscore names included), so read the
    # way we write; a plain __dict__ lookup would never hit there and the CSR build would rerun in every layer
    try:
        hit = getattr(batch_obj, attr, None)
    except Exception:
        hit = None
    if hit is None:
        try:
            hit = _side_cache.get(batch_obj, {}).get(attr)
        except TypeError:
            hit = None
    return hit if isinstance(hit, typ) else None


def _cache_put(batch_obj, value, attr=_CACHE_ATTR):
    try:
        setattr(batch_obj, attr, value)
        if getattr(batch_obj, attr, None) is value:
            return
    except Exception:
        pass
    try:
        _side_cache.setdefault(batch_obj, {})[attr] = value
    except TypeError:  # not weak-referenceable: still works, the value is recomputed per call
        pass


def graph_of(batch_obj) -> GraphStructure:
    """Returns the cached structure of `batch_obj`, building it on first use."""
    ei, bv = batch_obj.edge_index, batch_obj.batch
    cached = _cache_get(batch_obj)
    key = (ei.data_ptr(), bv.data_ptr(), int(bv.shape[0]), int(ei.shape[1]), ei._version, bv._version)
    if cached is not None and cached.key == key:
        return cached
    gs = GraphStructure(ei, bv, _num_graphs(batch_obj))
    _cache_put(batch_obj, gs)
    return gs
