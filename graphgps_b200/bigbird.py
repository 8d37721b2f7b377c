"""BigBird global model of GPSLayer (reference: graphgps/layer/gps_layer.py:115-119,207-208 and
graphgps/layer/bigbird_layer.py:1667-1706, the SingleBigBirdLayer it builds).

This module holds what the layer needs on the host side:
  * the configuration (cfg.gt.bigbird, read by attribute) and the checks of what is built;
  * the parameter container, whose state_dict has the reference's keys, shapes and order;
  * the random-block table R [heads, nb - 2, num_random_blocks] of block-sparse attention, drawn as the reference draws
    it in every forward call (np.random.seed(0), then the same `permutation` calls in the same order), but on a private
    RandomState so that numpy's global generator is left alone;
  * the two CSR lists the kernels read, per head, with duplicate blocks kept: the key blocks of every query block, and
    the query blocks of every key block.  They depend on the batch only through nb, the number of blocks of the padded
    length, and are uploaded once per (device, nb, heads, block_size, num_random_blocks, max_position_embeddings).

Attention pattern (query block i of nb, lists are multisets):
  i = 0 and i = nb - 1      every block;
  i = 1                     [0, 1, 2, nb - 1] + R[h][0];
  i = nb - 2                [0, nb - 3, nb - 2, nb - 1] + R[h][nb - 3];
  2 <= i <= nb - 3          [0, i - 1, i, i + 1, nb - 1] + R[h][i - 1].
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from . import _lib

_ACTS = ("relu", "sigmoid")
# padded lengths at which the reference draws the table with the plan of the BigBird paper
_LEGACY_LENGTHS = (1024, 3072, 4096)


# ------------------------------------------------------------------------------------------------ configuration
class BigBirdConfig:
    """The fields of cfg.gt.bigbird the layer reads (gt_config.py:52-72 defaults)."""

    def __init__(self, cfg):
        def get(name, default):
            return getattr(cfg, name, default)

        self.attention_type = get("attention_type", "block_sparse")
        self.chunk_size_feed_forward = get("chunk_size_feed_forward", 0)
        self.is_decoder = bool(get("is_decoder", False))
        self.add_cross_attention = bool(get("add_cross_attention", False))
        self.hidden_act = get("hidden_act", "relu")
        self.max_position_embeddings = int(get("max_position_embeddings", 128))
        self.use_bias = bool(get("use_bias", False))
        self.num_random_blocks = int(get("num_random_blocks", 3))
        self.block_size = int(get("block_size", 3))
        self.layer_norm_eps = float(get("layer_norm_eps", 1e-6))

    def check(self):
        """NotImplementedError for what the reference does differently from block-sparse self-attention."""
        if self.attention_type != "block_sparse":
            raise NotImplementedError(
                f"BigBird attention_type '{self.attention_type}' is not built in graphgps_b200: the reference's "
                "SingleBigBirdLayer asserts attention_type == 'block_sparse' (bigbird_layer.py:1674)")
        if self.add_cross_attention:
            raise NotImplementedError(
                "BigBird add_cross_attention=True is not built in graphgps_b200: the reference then switches the "
                "layer to attention_type 'original_full' (bigbird_layer.py:1489-1493) and builds a cross-attention "
                "block that GPSLayer never feeds")
        if self.is_decoder:
            raise NotImplementedError(
                "BigBird is_decoder=True is not built in graphgps_b200: the reference's decoder path returns the "
                "self-attention cache as the layer's output (bigbird_layer.py:1308-1310,1347-1348)")
        if self.chunk_size_feed_forward != 0:
            raise NotImplementedError(
                "BigBird chunk_size_feed_forward != 0 is not built in graphgps_b200: the reference then splits the "
                "feed-forward along the padded sequence (apply_chunking_to_forward, bigbird_layer.py:49-112)")
        if self.hidden_act not in _ACTS:
            raise NotImplementedError(
                f"BigBird hidden_act '{self.hidden_act}' is not built in graphgps_b200: the reference's ACT2FN holds "
                f"{_ACTS} only (bigbird_layer.py:32-46) and raises KeyError for any other name")
        if self.block_size < 1 or self.num_random_blocks < 1:
            raise NotImplementedError(
                f"BigBird needs block_size >= 1 and num_random_blocks >= 1 (got {self.block_size}, "
                f"{self.num_random_blocks})")


# ------------------------------------------------------------------------------------------------ parameters
class _Self(nn.Module):
    def __init__(self, d, bias):
        super().__init__()
        self.query = nn.Linear(d, d, bias=bias)
        self.key = nn.Linear(d, d, bias=bias)
        self.value = nn.Linear(d, d, bias=bias)


class _DenseNorm(nn.Module):
    def __init__(self, d, eps):
        super().__init__()
        self.dense = nn.Linear(d, d)
        self.LayerNorm = nn.LayerNorm(d, eps=eps)


class _Attention(nn.Module):
    def __init__(self, d, bias, eps):
        super().__init__()
        self.self = _Self(d, bias)
        self.output = _DenseNorm(d, eps)


class _Intermediate(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.dense = nn.Linear(d, d)


class _Layer(nn.Module):
    def __init__(self, d, bias, eps):
        super().__init__()
        self.attention = _Attention(d, bias, eps)
        self.intermediate = _Intermediate(d)
        self.output = _DenseNorm(d, eps)


class _Encoder(nn.Module):
    def __init__(self, d, bias, eps):
        super().__init__()
        self.layers = nn.ModuleList([_Layer(d, bias, eps)])


class BigBirdParams(nn.Module):
    """Names of the reference's SingleBigBirdLayer (one BigBirdLayer): encoder.layers.0.attention.self.{query,key,value}
    (bias only with use_bias), .attention.output.{dense,LayerNorm}, .intermediate.dense, .output.{dense,LayerNorm},
    registered in the reference's order with torch's default initialisation (post_init is not called there)."""

    def __init__(self, d, heads, cfg: BigBirdConfig):
        super().__init__()
        self.cfg = cfg
        self.heads = heads
        self.encoder = _Encoder(d, cfg.use_bias, cfg.layer_norm_eps)

    @property
    def layer(self):
        return self.encoder.layers[0]


# ------------------------------------------------------------------------------------------------ random blocks
def _put(table, row, c0, c1, picked, where):
    """table[row, c0:c1] = picked with numpy's assignment rules: a pick of the slot's width, or one block repeated."""
    if len(picked) != c1 - c0 and len(picked) != 1:
        raise NotImplementedError(
            f"BigBird cannot fill its random-block table at {where}: {c1 - c0} random blocks are drawn from "
            f"{len(picked)} candidates (the reference fails to assign the row with a ValueError)")
    table[row, c0:c1] = picked


def _plan(S, bs, r):
    """Bands of key blocks the random blocks come from, as (band end in tokens, random blocks per band)."""
    nb = S // bs
    if 2 * r + 5 < nb:
        return [(2 * r + 5) * bs, S], [r, 0]
    if r + 5 < nb:
        return [(r + 5) * bs, S], [r // 2, r - r // 2]
    return [S], [r]


def _table_banded(S, bs, heads, r, rng):
    ends, counts = _plan(S, bs, r)
    nb = S // bs
    bands = [e // bs for e in ends]             # band p covers key blocks [bands[p - 1], bands[p])
    cols = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    tabs = [np.zeros((nb, int(cols[-1])), dtype=np.int32) for _ in range(heads)]

    def draw(rows, band, lo):
        c0, c1 = int(cols[band]), int(cols[band + 1])
        for row in rows:
            for h in range(heads):
                picked = rng.permutation(np.arange(lo, bands[band], dtype=np.int32))[:c1 - c0]
                _put(tabs[h], row, c0, c1, picked, f"padded length {S}, query block {row}, head {h}")

    for p in range(len(bands)):
        if p > 0:
            # rows of the earlier bands draw their share of band p; rows of band p draw from every earlier band
            if counts[p] > 0:
                draw(range(1, bands[p - 1]), p, bands[p - 1])
            for q in range(p):
                if counts[q] > 0:
                    draw(range(bands[p - 1], bands[p]), q, bands[q - 1] if q > 0 else 0)
        if counts[p] > 0:
            lo = bands[p - 1] if p > 0 else 0
            draw(range(lo if p > 0 else 1, bands[p]), p, lo)
    return np.stack([t[1:nb - 1] for t in tabs])


def _table_legacy(S, bs, heads, r, max_len, rng):
    """The plan of the BigBird paper for padded lengths 1024 / 3072 / 4096: rows for max_len tokens, drawn up to 1024."""
    nb = S // bs
    nbm = max_len // bs
    if nbm < nb or nbm < 2:
        raise NotImplementedError(
            f"BigBird at padded length {S} draws its random blocks for max_position_embeddings = {max_len} tokens, "
            f"{nbm} blocks of {bs}, which cannot cover the {nb} blocks of the batch (the reference fails there)")
    mid = np.arange(1, nbm - 1, dtype=np.int32)
    last = 1024 // bs - 1 if 1024 > 2 * bs else nbm - 1
    out = []
    for h in range(heads):
        tab = np.zeros((nbm - 2, r), dtype=np.int32)
        for i in range(1, nbm - 1):
            if i == 1:
                cand = mid[2:last]
            elif i == 2:
                cand = mid[3:last]
            elif i in (nbm - 3, nbm - 2):
                cand = mid[:last]
            elif i - 2 > last:
                cand = mid[:last]
            elif i + 1 == last:
                cand = mid[:i - 2]
            else:
                cand = np.concatenate((mid[:i - 2], mid[i + 1:last]))
            _put(tab, i - 1, 0, r, rng.permutation(cand)[:r], f"padded length {S}, query block {i}, head {h}")
        out.append(tab[:nb - 2])
    return np.stack(out)


def padded_length(nmax, bs):
    """to_dense_batch's Nmax padded up to a multiple of the block size (_pad_to_block_size)."""
    return nmax + (bs - nmax % bs) % bs


def random_table(S, bs, heads, r, max_len=128):
    """R [heads, S / bs - 2, r] (int32) for padded length S, as the reference draws it with seed 0.
    NotImplementedError where the reference cannot run: fewer than 4 blocks, or a row the plan cannot fill."""
    nb = S // bs
    if S % bs != 0 or nb < 4:
        raise NotImplementedError(
            f"BigBird block-sparse attention needs at least 4 blocks of block_size = {bs} (padded length {S}: "
            f"{nb} blocks); the reference cannot run such a batch")
    rng = np.random.RandomState(0)
    if S in _LEGACY_LENGTHS:
        return _table_legacy(S, bs, heads, r, max_len, rng)
    return _table_banded(S, bs, heads, r, rng)


def key_blocks(R, i, nb):
    """Key blocks (a multiset, in the kernels' order) of query block i for one head's table R [nb - 2, r]."""
    if i == 0 or i == nb - 1:
        return list(range(nb))
    if i == 1:
        base = [0, 1, 2, nb - 1]
    elif i == nb - 2:
        base = [0, nb - 3, nb - 2, nb - 1]
    else:
        base = [0, i - 1, i, i + 1, nb - 1]
    return base + [int(b) for b in R[i - 1]]


def block_lists(R, nb):
    """The two CSR lists of the kernels, all heads concatenated: (key_ptr [H*(nb+1)], key_idx, query_ptr [H*(nb+1)],
    query_idx); ptr entries are absolute offsets into idx.  Duplicates are kept; query blocks per key block ascend."""
    kptr, kidx, qptr, qidx = [], [], [], []
    for h in range(R.shape[0]):
        rows = [key_blocks(R[h], i, nb) for i in range(nb)]
        cols = [[] for _ in range(nb)]
        for i, row in enumerate(rows):
            for kb in row:
                cols[kb].append(i)
        for lst, ptr, idx in ((rows, kptr, kidx), (cols, qptr, qidx)):
            for row in lst:
                ptr.append(len(idx))
                idx.extend(row)
            ptr.append(len(idx))
    return (np.asarray(kptr, np.int32), np.asarray(kidx, np.int32), np.asarray(qptr, np.int32),
            np.asarray(qidx, np.int32))


_device_lists = {}


def device_lists(device, nb, heads, bs, r, max_len):
    """(key_ptr, key_idx, query_ptr, query_idx) int32 tensors on `device`, built and uploaded once per key."""
    key = (str(device), nb, heads, bs, r, max_len)
    hit = _device_lists.get(key)
    if hit is None:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError(
                f"BigBird's block lists for {nb} blocks are built on the host and cannot be uploaded inside a CUDA-graph "
                "capture: run the layer once on a batch of the same padded length before capturing")
        R = random_table(nb * bs, bs, heads, r, max_len)
        hit = tuple(torch.from_numpy(a).to(device) for a in block_lists(R, nb))
        _device_lists[key] = hit
    return hit


def gps_bigbird(params: BigBirdParams, named, grads, prefix):
    """GpsBigBird of the C ABI from the container's parameters (named / grads: name -> tensor).  num_blocks and the
    block lists belong to the batch and are left 0 / NULL."""
    cfg = params.cfg
    g = grads or {}
    p = prefix + "encoder.layers.0."

    def lin(name, bias=True):
        return _lib.GpsLinear(_lib.ptr(named[p + name + ".weight"]), _lib.ptr(named.get(p + name + ".bias")),
                              _lib.ptr(g.get(p + name + ".weight")), _lib.ptr(g.get(p + name + ".bias")))

    return _lib.GpsBigBird(cfg.block_size, 0, _lib.BIGBIRD_ACT[cfg.hidden_act], cfg.layer_norm_eps, 0, 0, 0, 0,
                           lin("attention.self.query"), lin("attention.self.key"), lin("attention.self.value"),
                           lin("attention.output.dense"), lin("attention.output.LayerNorm"),
                           lin("intermediate.dense"), lin("output.dense"), lin("output.LayerNorm"))


