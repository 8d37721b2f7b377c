"""CPU: the BigBird global model (gps_layer.py:115-119,207-208; bigbird_layer.py of the reference).

The fp64 oracle (tests/bigbird_oracle.py) against the reference layer run verbatim (reference_live) and against every
fixture of tests/golden/bigbird/; the random-block table builder against the reference's own tables; the duplicates
in those tables; the parameter container, the config mutation and the constructor errors; the GraphGym build; and
the C entry points' refusal of malformed arguments before any CUDA call."""
import ctypes as C
import glob as _glob
import os
import sys
import types

import numpy as np
import pytest
import torch

import graphgps_b200
from graphgps_b200 import _lib, bigbird as bbmod
from bigbird_oracle import attach_bigbird, bigbird_cfg, bigbird_oracle_layer
from util import GOLDEN_DIR, golden_batch

BB_DIR = os.path.join(GOLDEN_DIR, "bigbird")
FIXTURES = sorted(os.path.basename(p)[:-3] for p in _glob.glob(os.path.join(BB_DIR, "*.pt"))
                  if not p.endswith("tables.pt"))
LIVE = "reference_live_GINE_BigBird"


def _load(name):
    return torch.load(os.path.join(BB_DIR, name + ".pt"), weights_only=False)


def _oracle(fix, dtype=torch.float64, dedup=False):
    c = fix["config"]
    cfg = types.SimpleNamespace(**c["bigbird"])
    layer = bigbird_oracle_layer(c["d"], c["local"], c["heads"], cfg, batch_norm=c["batch_norm"])
    layer.load_state_dict(fix["state"], strict=True)
    layer.self_attn.table = fix["table"].numpy()
    layer.self_attn.dedup = dedup
    layer = layer.to(dtype)
    layer.train(c["training"])
    return layer


def _run(layer, fix, dtype=torch.float64):
    b = golden_batch(fix, dtype=dtype)
    b.x.requires_grad_(True)
    b.edge_attr.requires_grad_(True)
    x_in, e_in = b.x, b.edge_attr
    out = layer(b)
    loss = (out.x * fix["ct_x"].to(dtype)).sum()
    res = {"out_x": out.x.detach()}
    if "ct_e" in fix:
        loss = loss + (out.edge_attr * fix["ct_e"].to(dtype)).sum()
        res["out_e"] = out.edge_attr.detach()
    if "grad_x" in fix:
        loss.backward()
        res["grad_x"] = x_in.grad
        if e_in.grad is not None:
            res["grad_e"] = e_in.grad
        res["grad_params"] = {n: p.grad for n, p in layer.named_parameters() if p.grad is not None}
    return res


def _max_err(res, fix, keys=("out_x", "out_e", "grad_x", "grad_e")):
    errs = {}
    for k in keys:
        if k in fix and k in res:
            errs[k] = float((res[k].double() - fix[k].double()).abs().max())
    for n, g in fix.get("grad_params", {}).items():
        errs["grad:" + n] = float((res["grad_params"][n].double() - g.double()).abs().max())
    return errs


def test_fixtures_exist():
    assert LIVE in FIXTURES and len(FIXTURES) >= 14


def test_oracle_equals_reference_live_bigbird():
    fix = _load(LIVE)
    errs = _max_err(_run(_oracle(fix), fix), fix)
    assert errs["out_x"] <= 1e-10, errs
    assert max(v for k, v in errs.items() if k != "out_x") <= 1e-9, errs
    assert len(fix["grad_params"]) == len([n for n, _ in _oracle(fix).named_parameters()])


@pytest.mark.parametrize("name", [n for n in FIXTURES if n != LIVE])
def test_oracle_matches_fixture_fp64(name):
    fix = _load(name)
    errs = _max_err(_run(_oracle(fix), fix), fix)
    scale = {k: max(1.0, float(fix[k].abs().max())) for k in ("out_x", "grad_x") if k in fix}
    for k, e in errs.items():
        ref = fix[k] if k in fix else fix["grad_params"][k[5:]]
        assert e / max(1.0, float(ref.abs().max())) <= 2e-6, (name, k, e, scale)


def test_fixtures_hold_duplicate_key_blocks_that_matter():
    """Nearly every table repeats a key block within one query block's list; counting each once moves the output."""
    from bigbird_oracle import key_block_lists
    dup_tables = 0
    for name in FIXTURES:
        fix = _load(name)
        R = fix["table"].numpy()
        nb = R.shape[1] + 2
        if any(len(row) != len(set(row)) for rows in key_block_lists(R, nb) for row in rows):
            dup_tables += 1
    assert dup_tables >= len(FIXTURES) - 2
    fix = _load("gine_bigbird_relu")
    a = _run(_oracle(fix), fix)["out_x"]
    b = _run(_oracle(fix, dedup=True), fix)["out_x"]
    assert float((a - b).abs().max()) > 1e-2


# ------------------------------------------------------------------------------------------------- random-block table
def test_table_matches_reference_tables():
    t = _load("tables")
    n = 0
    for (bs, r, H, S), ref in t["tables"].items():
        got = bbmod.random_table(S, bs, H, r)
        assert got.shape == tuple(ref.shape) and (got == ref.numpy()).all(), (bs, r, H, S)
        n += 1
    for (bs, r, H, S, ml), ref in t["legacy"].items():
        got = bbmod.random_table(S, bs, H, r, ml)
        assert (got == ref.numpy()).all()
    assert n > 150


def test_table_raises_where_the_reference_raises():
    t = _load("tables")
    for (bs, r, H), bad in t["raises"].items():
        for nb in range(1, 48):
            S = nb * bs
            if nb < 4 or S in bad:
                with pytest.raises(NotImplementedError):
                    bbmod.random_table(S, bs, H, r)
            else:
                bbmod.random_table(S, bs, H, r)
    assert t["raises"][(3, 5, 2)] == [12, 36]
    # legacy lengths drawn for max_position_embeddings = 128 tokens cannot cover the batch
    with pytest.raises(NotImplementedError):
        bbmod.random_table(1024, 8, 2, 2, 128)


def test_table_fixtures_match_builder():
    for name in FIXTURES:
        fix = _load(name)
        c = fix["config"]["bigbird"]
        R = fix["table"].numpy()
        S = (R.shape[1] + 2) * c["block_size"]
        got = bbmod.random_table(S, c["block_size"], fix["config"]["heads"], c["num_random_blocks"])
        assert (got == R).all(), name


def test_table_leaves_numpy_global_rng_alone():
    np.random.seed(123)
    before = np.random.get_state()
    bbmod.random_table(36, 3, 8, 3)
    after = np.random.get_state()
    assert before[0] == after[0] and (before[1] == after[1]).all() and before[2:] == after[2:]


def test_block_lists_are_transposes_with_multiplicity():
    R = bbmod.random_table(33, 3, 4, 3)
    nb = 11
    kptr, kidx, qptr, qidx = bbmod.block_lists(R, nb)
    assert kptr.shape == qptr.shape == (4 * (nb + 1),)
    for h in range(4):
        cnt_k = np.zeros((nb, nb), int)
        cnt_q = np.zeros((nb, nb), int)
        for i in range(nb):
            for kb in kidx[kptr[h * (nb + 1) + i]:kptr[h * (nb + 1) + i + 1]]:
                cnt_k[i, kb] += 1
            lst = qidx[qptr[h * (nb + 1) + i]:qptr[h * (nb + 1) + i + 1]]
            assert list(lst) == sorted(lst)
            for qb in lst:
                cnt_q[qb, i] += 1
            assert list(kidx[kptr[h * (nb + 1) + i]:kptr[h * (nb + 1) + i + 1]]) == bbmod.key_blocks(R[h], i, nb)
        assert (cnt_k == cnt_q).all()
        assert cnt_k.max() >= 2


# ------------------------------------------------------------------------------------------------- module
def _ref_keys(fix):
    return list(fix["state"].keys())


def test_state_dict_keys_shapes_and_order():
    for name in ("gine_bigbird_relu", "gatedgcn_bigbird_sigmoid_bias", "none_bigbird_relu", "gine_bigbird_nonorm"):
        fix = _load(name)
        c = fix["config"]
        layer = graphgps_b200.GPSLayer(c["d"], c["local"], "BigBird", c["heads"], batch_norm=c["batch_norm"],
                                       bigbird_cfg=types.SimpleNamespace(**c["bigbird"]))
        sd = layer.state_dict()
        assert list(sd.keys()) == _ref_keys(fix), name
        assert all(tuple(sd[k].shape) == tuple(v.shape) for k, v in fix["state"].items())
        layer.load_state_dict(fix["state"], strict=True)
    assert "self_attn.encoder.layers.0.attention.self.query.bias" in _load("gatedgcn_bigbird_sigmoid_bias")["state"]
    assert "self_attn.encoder.layers.0.attention.self.query.bias" not in _load("gine_bigbird_relu")["state"]


def test_config_mutation_matches_reference():
    cfg = bigbird_cfg()
    graphgps_b200.GPSLayer(56, "GINE", "BigBird", 8, dropout=0.3, attn_dropout=0.7, bigbird_cfg=cfg)
    assert (cfg.dim_hidden, cfg.n_heads, cfg.dropout) == (56, 8, 0.3)
    # any object read by attribute
    ns = types.SimpleNamespace(block_size=2, num_random_blocks=1)
    layer = graphgps_b200.GPSLayer(16, "None", "BigBird", 4, bigbird_cfg=ns)
    assert layer.self_attn.cfg.block_size == 2 and ns.dim_hidden == 16


@pytest.mark.parametrize("over,exc", [
    (dict(attention_type="original_full"), NotImplementedError),
    (dict(is_decoder=True), NotImplementedError),
    (dict(add_cross_attention=True, is_decoder=True), NotImplementedError),
    (dict(chunk_size_feed_forward=4), NotImplementedError),
    (dict(hidden_act="gelu"), NotImplementedError),
])
def test_constructor_refuses(over, exc):
    with pytest.raises(exc):
        graphgps_b200.GPSLayer(56, "GINE", "BigBird", 8, bigbird_cfg=bigbird_cfg(**over))


def test_constructor_errors():
    with pytest.raises(NotImplementedError):
        graphgps_b200.GPSLayer(56, "GINE", "BigBird", 8, bigbird_cfg=None)
    with pytest.raises(ValueError):
        graphgps_b200.GPSLayer(56, "GINE", "BigBird", 5, bigbird_cfg=bigbird_cfg())


def test_graphgym_register_builds_gine_bigbird(monkeypatch):
    reg = {}
    cfg = types.SimpleNamespace(
        gt=types.SimpleNamespace(layer_type="GINE+BigBird", n_heads=8, dropout=0.0, attn_dropout=0.0, layer_norm=False,
                                 batch_norm=True, pna_degrees=None, bigbird=bigbird_cfg()),
        gnn=types.SimpleNamespace(act="relu"))
    monkeypatch.setitem(sys.modules, "torch_geometric", types.ModuleType("torch_geometric"))
    monkeypatch.setitem(sys.modules, "torch_geometric.graphgym", types.ModuleType("torch_geometric.graphgym"))
    monkeypatch.setitem(sys.modules, "torch_geometric.graphgym.register",
                        types.SimpleNamespace(register_layer=lambda n, c: reg.__setitem__(n, c)))
    monkeypatch.setitem(sys.modules, "torch_geometric.graphgym.config", types.SimpleNamespace(cfg=cfg))
    from graphgps_b200.graphgym import register
    cls = register("gpslayer_b200_bigbird_test")
    layer = cls(types.SimpleNamespace(dim_out=56))
    assert layer.global_model_type == "BigBird" and layer.local_gnn_type == "GINE"
    assert list(layer.state_dict().keys()) == _ref_keys(_load("gine_bigbird_relu"))
    assert reg["gpslayer_b200_bigbird_test"] is cls


def test_gradient_groups():
    from graphgps_b200 import dp
    assert dp._group("self_attn.encoder.layers.0.attention.self.query.weight") == dp.LATE
    assert dp._group("self_attn.encoder.layers.0.output.LayerNorm.weight") == dp.MID
    assert dp._group("self_attn.encoder.layers.0.intermediate.dense.bias") == dp.MID


# ------------------------------------------------------------------------------------------------- C ABI
def _lib_or_skip():
    try:
        return _lib.load()
    except (RuntimeError, OSError) as e:   # pragma: no cover - the library is built by build()
        pytest.skip(str(e))


def _args(global_type=_lib.GLOBAL["BigBird"], local=_lib.LOCAL["GINE"], d=56, heads=8, bb=None):
    a = _lib.GpsLayerArgs()
    a.d, a.heads, a.local_type, a.global_type = d, heads, local, global_type
    a.graph.N, a.graph.E, a.graph.B = 10, 0, 1
    if bb is not None:
        a.bigbird = bb
    return a


def _bb(nb=4, bs=3, lists=True):
    b = _lib.GpsBigBird()
    b.block_size, b.num_blocks, b.hidden_act, b.ln_eps = bs, nb, 0, 1e-6
    if lists:
        b.key_ptr = b.key_idx = b.query_ptr = b.query_idx = 16   # never dereferenced: refused first
    return b


def test_abi_constants():
    assert _lib.GLOBAL == {"None": 0, "Transformer": 1, "Performer": 2, "BigBird": 3}
    assert _lib.GLOBAL_BIGBIRD == _lib.GLOBAL["BigBird"] == 3
    hdr = open(os.path.join(os.path.dirname(GOLDEN_DIR), "..", "include", "gps_b200.h")).read()
    assert "GPS_GLOBAL_BIGBIRD = 3" in hdr


def test_entry_points_refuse_malformed_arguments():
    lib = _lib_or_skip()
    ARG = _lib.GPS_ERR_ARG
    for fn in (lib.gps_layer_forward, lib.gps_layer_backward):
        assert fn(C.byref(_args()), None) == ARG                                  # GpsBigBird left empty
        assert fn(C.byref(_args(bb=_bb(nb=3))), None) == ARG                      # nb < 4
        assert fn(C.byref(_args(bb=_bb(bs=0))), None) == ARG
        assert fn(C.byref(_args(bb=_bb(lists=False))), None) == ARG
        assert fn(C.byref(_args(heads=5, bb=_bb())), None) == ARG                 # d % heads
        # a well-formed GpsBigBird with missing parameters: refused by the parameter check
        assert fn(C.byref(_args(bb=_bb())), None) == ARG
    # an attention bias needs the Transformer
    a = _args(bb=_bb())
    a.attn_bias = _lib.GpsAttnBias(16, 4, 0)
    assert lib.gps_layer_forward(C.byref(a), None) == ARG
    # stages
    g = _lib.GpsGraph()
    assert lib.gps_bigbird_attention_forward(C.byref(g), 8, 7, None, 16, 16, 16, 56, 16, 56, 16, None) == ARG
    assert lib.gps_bigbird_attention_forward(C.byref(g), 8, 7, C.byref(_bb()), 0, 16, 16, 56, 16, 56, 16, None) == ARG
    assert lib.gps_bigbird_attention_forward(C.byref(g), 8, 7, C.byref(_bb(nb=2)), 16, 16, 16, 56, 16, 56, 16,
                                             None) == ARG
    assert lib.gps_bigbird_attention_backward(C.byref(g), 8, 7, C.byref(_bb()), 16, 16, 16, 56, 16, 16, 56, 16, 0, 16,
                                              16, 16, 56, None) == ARG
    assert lib.gps_layernorm_forward(0, 4, 8, 16, 16, 1e-6, 16, 16, 16, None) == ARG
    assert lib.gps_layernorm_backward(16, 16, 4, 8, 16, 16, 16, 16, 0, 0, 0, 0, None) == ARG
    assert lib.gps_layernorm_forward(16, 4, 6, 16, 16, 1e-6, 16, 16, 16, None) == _lib.GPS_ERR_UNSUPPORTED
