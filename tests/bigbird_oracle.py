"""TEST INFRASTRUCTURE - CPU restatement (pure torch) of the reference GPSLayer with global_model_type='BigBird'.

Restates graphgps/layer/bigbird_layer.py (paths relative to the reference checkout) in a dense form:
  * :1667-1706  SingleBigBirdLayer: to_dense_batch's Nmax padded to a multiple of block_size, one BigBirdLayer;
  * :316-765    block-sparse attention, as a block-multiplicity matrix W [heads, S, S]: W[h, q, k] = how often key k's
                block appears in the key-block list of q's block (duplicates of the random-block table count twice).
                Padded keys are excluded (the reference adds -10000), p = W exp(s - m) / sum(W exp(s - m)), padded query
                rows are not computed (the reference multiplies them by 0 and drops them);
  * :1116-1127  a = LayerNorm(dropout(dense(ctx)) + x);  :1215-1242  out = LayerNorm(dropout(dense(act(dense(a)))) + a).
The random-block table is an INPUT (`table`, [heads, nb - 2, r]): the fixtures store the reference's own table; without
one the oracle asks graphgps_b200.bigbird.random_table, which tests/test_bigbird.py pins to the stored tables.

Pinned to the reference itself: tests/test_bigbird.py::test_oracle_equals_reference_live_bigbird holds this file to the
reference layer's fp64 outputs and gradients stored by tests/golden/make_bigbird_golden.py.
"""
from __future__ import annotations

import types

import torch
import torch.nn as nn
import torch.nn.functional as F

from graphgps_b200.bigbird import BigBirdConfig, BigBirdParams
from oracle.gps_oracle import OracleGPSLayer

DEFAULT_CFG = dict(attention_type="block_sparse", chunk_size_feed_forward=0, is_decoder=False,
                   add_cross_attention=False, hidden_act="relu", max_position_embeddings=128, use_bias=False,
                   num_random_blocks=3, block_size=3, layer_norm_eps=1e-6)


def bigbird_cfg(**kw):
    """cfg.gt.bigbird as a SimpleNamespace with the gt_config.py:52-72 defaults."""
    return types.SimpleNamespace(**dict(DEFAULT_CFG, **kw))


def key_block_lists(R, nb):
    """Per head and query block, the key blocks it attends (a list with duplicates): blocks 0 and nb-1 attend every
    block; block 1 [0, 1, 2, nb-1] + R[0]; block nb-2 [0, nb-3, nb-2, nb-1] + R[nb-3]; others [0, i-1, i, i+1, nb-1] +
    R[i-1]."""
    out = []
    for h in range(R.shape[0]):
        rows = []
        for i in range(nb):
            if i in (0, nb - 1):
                rows.append(list(range(nb)))
                continue
            if i == 1:
                base = [0, 1, 2, nb - 1]
            elif i == nb - 2:
                base = [0, nb - 3, nb - 2, nb - 1]
            else:
                base = [0, i - 1, i, i + 1, nb - 1]
            rows.append(base + [int(v) for v in R[h][i - 1]])
        out.append(rows)
    return out


def multiplicity(R, nb, bs, dedup=False):
    """W [heads, S, S] (float64) of the block lists; dedup=True counts every block once (for the duplicate test)."""
    H, S = R.shape[0], nb * bs
    W = torch.zeros(H, S, S, dtype=torch.float64)
    for h, rows in enumerate(key_block_lists(R, nb)):
        for i, row in enumerate(rows):
            for kb in (sorted(set(row)) if dedup else row):
                W[h, i * bs:(i + 1) * bs, kb * bs:(kb + 1) * bs] += 1
    return W


class OracleBigBird(nn.Module):
    """SingleBigBirdLayer restated; same parameter names as the reference (state_dicts load both ways)."""

    def __init__(self, dim_h, num_heads, cfg):
        super().__init__()
        self.cfg = BigBirdConfig(cfg)
        self.heads = num_heads
        self.dropout = float(getattr(cfg, "dropout", 0.0))
        p = BigBirdParams(dim_h, num_heads, self.cfg)
        self.encoder = p.encoder
        self.table = None       # [heads, nb - 2, r]; None: graphgps_b200.bigbird.random_table
        self.dedup = False      # count every key block once (the duplicate test)
        self.masks = None       # {"self_out": keep [N, d], "output": keep [N, d]} 0/1 in packed row order, or None
        self.last_table = None

    def _drop(self, t, key, rows):
        if not self.training or self.dropout == 0.0:
            return t
        if self.masks is None:
            return F.dropout(t, self.dropout, True)
        return t * self.masks[key][rows].to(t.dtype) / (1.0 - self.dropout)

    def forward(self, h_dense, mask):
        from graphgps_b200.bigbird import random_table
        L = self.encoder.layers[0]
        B, nmax, d = h_dense.shape
        bs, H = self.cfg.block_size, self.heads
        S = nmax + (bs - nmax % bs) % bs
        nb = S // bs
        R = self.table if self.table is not None else random_table(S, bs, H, self.cfg.num_random_blocks,
                                                                   self.cfg.max_position_embeddings)
        self.last_table = R
        W = multiplicity(R, nb, bs, self.dedup).to(h_dense.dtype)
        hd = d // H
        act = torch.relu if self.cfg.hidden_act == "relu" else torch.sigmoid
        out = h_dense.new_zeros(B, nmax, d)
        row0 = 0
        for g in range(B):
            n = int(mask[g].sum())
            x = h_dense[g, :n]
            rows = torch.arange(row0, row0 + n)
            row0 += n
            q = L.attention.self.query(x).view(n, H, hd).transpose(0, 1)
            k = L.attention.self.key(x).view(n, H, hd).transpose(0, 1)
            v = L.attention.self.value(x).view(n, H, hd).transpose(0, 1)
            s = q @ k.transpose(1, 2) / hd ** 0.5
            w = W[:, :n, :n]
            s = s.masked_fill(w == 0, float("-inf"))
            e = w * torch.exp(s - s.amax(-1, keepdim=True))
            ctx = ((e / e.sum(-1, keepdim=True)) @ v).transpose(0, 1).reshape(n, d)
            a = L.attention.output.LayerNorm(self._drop(L.attention.output.dense(ctx), "self_out", rows) + x)
            o = L.output.LayerNorm(self._drop(L.output.dense(act(L.intermediate.dense(a))), "output", rows) + a)
            out[g, :n] = o
        return out


def attach_bigbird(layer, dim_h, num_heads, cfg, dropout=0.0):
    """Turn an oracle GPSLayer built with global_model_type='None' into its BigBird version."""
    cfg.dim_hidden, cfg.n_heads, cfg.dropout = dim_h, num_heads, dropout
    layer.self_attn = OracleBigBird(dim_h, num_heads, cfg)
    layer.global_model_type = "BigBird"
    return layer


def bb_batch(sizes, d, seed=0, dtype=torch.float32):
    """A batch of ring graphs with one chord each (local ids), of the given sizes."""
    from graphgps_b200.batch import batch_from_lists
    edges = []
    for n in sizes:
        el = [(i, (i + 1) % n) for i in range(n)] + [((i + 1) % n, i) for i in range(n)] if n > 1 else []
        if n > 3:
            el += [(0, n // 2), (n // 2, 0)]
        edges.append(el)
    b = batch_from_lists(sizes, edges, d, seed=seed)
    b.x, b.edge_attr = b.x.to(dtype), b.edge_attr.to(dtype)
    return b


def bigbird_oracle_layer(dim_h, local_gnn_type, num_heads, cfg, **kw):
    """OracleGPSLayer(dim_h, local, 'BigBird', ...) for local in {None, GINE, GCN, CustomGatedGCN}."""
    layer = OracleGPSLayer(dim_h, local_gnn_type, "None", num_heads, **kw)
    return attach_bigbird(layer, dim_h, num_heads, cfg, kw.get("dropout", 0.0))
