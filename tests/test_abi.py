"""CPU: the C-ABI library loads and exports every symbol include/gps_b200.h declares; the Python
module keeps the reference's constructor contract and state_dict layout (no compute calls)."""
import os
import re

import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib
from oracle.gps_oracle import OracleGPSLayer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "gps_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(gps_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    syms = header_symbols()
    assert len(syms) >= 10
    for s in syms:
        assert hasattr(lib, s), f"libgps_b200.so does not export {s}"
        assert s in _lib.SYMBOLS, f"ctypes binding missing for {s}"
    assert lib.gps_abi_version() == 4
    assert lib.gps_build_arch() == b"sm_90a"


def test_graph_bytes_is_pure():
    lib = _lib.load()
    assert lib.gps_graph_bytes(10, 20, 2) > 0
    assert lib.gps_graph_bytes(0, 0, 0) >= 0


@pytest.mark.parametrize("local,glob", [("CustomGatedGCN", "Transformer"), ("GINE", "Transformer"),
                                        ("CustomGatedGCN", "Performer"), ("None", "Transformer"),
                                        ("GINE", "None"), ("CustomGatedGCN", "None"), ("GCN", "Transformer")])
def test_state_dict_layout_matches_reference(local, glob):
    ours = graphgps_b200.GPSLayer(64, local, glob, 4)
    ref = OracleGPSLayer(64, local, glob, 4)   # same keys as the reference (tests/test_oracle.py pins that)
    so, sr = ours.state_dict(), ref.state_dict()
    assert set(so) == set(sr)
    for k in so:
        assert tuple(so[k].shape) == tuple(sr[k].shape), k
    ours.load_state_dict(sr, strict=True)


def test_constructor_errors_follow_reference():
    G = graphgps_b200.GPSLayer
    with pytest.raises(ValueError):
        G(64, "NoSuchGNN", "Transformer", 4)                 # gps_layer.py:98
    with pytest.raises(ValueError):
        G(64, "GINE", "NoSuchFormer", 4)                     # gps_layer.py:121
    with pytest.raises(ValueError):
        G(64, "GINE", "Transformer", 4, layer_norm=True, batch_norm=True)   # gps_layer.py:125-126
    with pytest.raises(NotImplementedError):
        G(64, "GINE", "Performer", 4, log_attn_weights=True)  # gps_layer.py:36-41
    with pytest.raises(NotImplementedError):
        G(64, "PNA", "Transformer", 4)                        # known to the reference, not built here


def test_cpu_tensors_fail_loudly():
    layer = graphgps_b200.GPSLayer(32, "CustomGatedGCN", "Transformer", 4)
    b = graphgps_b200.make_batch("zinc-gatedgcn", dim=32, num_graphs=2)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        layer(b)


def test_graphgym_glue_rebinds_and_registers(monkeypatch):
    """INTEGRATION.md section 1: rebinding gps_model.GPSLayer, and @register_layer-style registration driven by cfg.gt."""
    import sys
    import types
    from graphgps_b200 import graphgym

    gm = types.ModuleType("graphgps.network.gps_model")
    gm.GPSLayer = object
    assert graphgym.install(gm) is object and gm.GPSLayer is graphgps_b200.GPSLayer

    registry = {}

    def register_layer(key, module=None):
        if key in registry:
            raise KeyError(key)
        registry[key] = module
        return module

    ns = types.SimpleNamespace
    cfg = ns(gt=ns(layer_type="GINE+Transformer", n_heads=4, dropout=0.1, attn_dropout=0.2, layer_norm=False,
                   batch_norm=True), gnn=ns(act="gelu"))
    for name, attrs in (("torch_geometric", {}), ("torch_geometric.graphgym", {}),
                        ("torch_geometric.graphgym.register", {"register_layer": register_layer}),
                        ("torch_geometric.graphgym.config", {"cfg": cfg})):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        monkeypatch.setitem(sys.modules, name, m)
    cls = graphgym.register("gpslayer_b200")
    assert registry["gpslayer_b200"] is cls
    layer = cls(ns(dim_out=32))
    assert (layer.dim_h, layer.local_gnn_type, layer.global_model_type, layer.num_heads) == (32, "GINE", "Transformer", 4)
    assert layer.act == "gelu" and layer.dropout == 0.1 and layer.attn_dropout == 0.2
    with pytest.raises(KeyError):
        graphgym.register("gpslayer_b200")


def test_graph_cache_round_trips_on_storage_backed_batches():
    """PyG Data/Batch keep attributes (underscore names included) in a storage object, not in __dict__: the cache
    must be read the way it is written (ADVICE r1).  No GPU needed: the cached object is only compared by identity."""
    from graphgps_b200 import graph as G

    class StoreBacked:                      # mimics torch_geometric.data.Data attribute routing
        def __init__(self):
            object.__setattr__(self, "_store", {})

        def __setattr__(self, k, v):
            self._store[k] = v

        def __getattr__(self, k):
            try:
                return object.__getattribute__(self, "_store")[k]
            except KeyError:
                raise AttributeError(k)

    class Frozen:                           # refuses new attributes -> weak side cache
        __slots__ = ("__weakref__",)

    gs = object.__new__(G.GraphStructure)
    for obj in (StoreBacked(), Frozen()):
        assert G._cache_get(obj) is None
        G._cache_put(obj, gs)
        assert G._cache_get(obj) is gs
    sb = StoreBacked()
    G._cache_put(sb, gs)
    assert G._CACHE_ATTR not in sb.__dict__ and G._cache_get(sb) is gs


def test_collate_matches_pyg_conventions():
    """graphgps_b200.loader.collate: node-offset edge indices, sorted batch vector, ptr offsets (what the layer needs
    from a PyG Batch), including an empty graph and a graph without edges."""
    import torch
    from graphgps_b200.loader import collate
    g = torch.Generator().manual_seed(0)
    graphs = [(torch.randn(3, 4, generator=g), torch.tensor([[0, 1, 2], [1, 2, 0]]), torch.randn(3, 4, generator=g)),
              (torch.zeros(0, 4), torch.zeros(2, 0, dtype=torch.int64), torch.zeros(0, 4)),
              (torch.randn(2, 4, generator=g), torch.zeros(2, 0, dtype=torch.int64), torch.zeros(0, 4)),
              (torch.randn(4, 4, generator=g), torch.tensor([[3, 0], [0, 3]]), torch.randn(2, 4, generator=g))]
    b = collate(graphs)
    assert b.num_graphs == 4 and b.ptr.tolist() == [0, 3, 3, 5, 9]
    assert b.batch.tolist() == [0, 0, 0, 2, 2, 3, 3, 3, 3]
    assert b.edge_index.tolist() == [[0, 1, 2, 8, 5], [1, 2, 0, 5, 8]]
    assert b.x.shape == (9, 4) and b.edge_attr.shape == (5, 4)


def test_stack_and_bucket_structure_on_cpu():
    """GPSStack mirrors GPSModel's `layers` Sequential (same per-layer state_dict keys); GradBucket groups a GPSLayer's
    parameters early / mid / late in the order the backward pass finishes them and aliases every .grad to one buffer."""
    import torch
    import graphgps_b200
    from graphgps_b200.dp import EARLY, LATE, MID, GradBucket, _group
    st = graphgps_b200.GPSStack(2, 16, "CustomGatedGCN", "Transformer", 2)
    keys = list(st.state_dict().keys())
    assert "layers.0.local_model.A.weight" in keys and "layers.1.self_attn.in_proj_weight" in keys
    assert _group("ff_linear1.weight") == EARLY and _group("norm1_attn.bias") == EARLY
    assert _group("local_model.C.weight") == MID and _group("local_model.bn_edge_e.bias") == MID
    assert _group("local_model.A.weight") == LATE and _group("self_attn.in_proj_bias") == LATE
    bucket = GradBucket(list(st.layers))
    lo, n = bucket.flat.data_ptr(), bucket.flat.numel()
    total = 0
    for p in st.parameters():
        assert lo <= p.grad.data_ptr() < lo + 4 * n and p.grad.shape == p.shape
        total += p.numel()
    assert n >= total
    segs = [(li, g) for li, g, _, _ in bucket.segments]
    assert segs == [(0, EARLY), (0, MID), (0, LATE), (1, EARLY), (1, MID), (1, LATE)]
    p = st.layers[1].ff_linear2.weight
    p.grad.fill_(2.0)
    assert float(bucket.segment(1, EARLY).sum()) >= 2.0 * p.numel()
    bucket.check_attached()
    p.grad = None                     # what optimizer.zero_grad(set_to_none=True) does
    import pytest
    with pytest.raises(RuntimeError, match="not a view of the bucket"):
        bucket.check_attached()
