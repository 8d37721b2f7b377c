"""TEST INFRASTRUCTURE - CPU restatement (pure torch) of the reference GPSLayer with global_model_type='BiasedTransformer'.

Extends oracle/gps_oracle.py (unchanged) with Graphormer's additive attention bias, graphgps/layer/gps_layer.py (paths
relative to the reference checkout):
  * :104-106  self_attn = nn.MultiheadAttention(dim_h, num_heads, dropout=attn_dropout, batch_first=True), the module of
              the Transformer case, so parameters, initial draws and state_dict are the Transformer's
  * :202-204  h_attn = _sa_block(h_dense, batch.attn_bias, ~mask)[mask]
  * :234-241  self_attn(x, x, x, attn_mask=attn_mask, key_padding_mask=key_padding_mask, need_weights=False)[0]
batch.attn_bias is a float tensor [num_graphs * heads, Nmax, Nmax] (row g * heads + h), added to the scaled scores.

Pinned to the reference itself: tests/test_biased.py::test_oracle_equals_reference_live_biased holds this file to the
reference layer's fp64 outputs and gradients (the attn_bias gradient included) stored by tests/golden/make_biased_golden.py.
"""
from __future__ import annotations

import torch.nn as nn

from oracle.gps_oracle import OracleGPSLayer


class _BiasedMHA(nn.MultiheadAttention):
    """torch's MultiheadAttention that adds the bias handed over in `self.attn_bias` as its float attn_mask (the base
    layer calls self_attn(..., attn_mask=None, key_padding_mask=~mask, need_weights=False))."""

    attn_bias = None

    def forward(self, query, key, value, attn_mask=None, **kw):
        return super().forward(query, key, value, attn_mask=self.attn_bias, **kw)


class OracleGPSLayerBiased(OracleGPSLayer):
    """OracleGPSLayer(..., 'BiasedTransformer', ...): reads batch.attn_bias in every forward call."""

    def __init__(self, dim_h, local_gnn_type, global_model_type, num_heads, **kw):
        assert global_model_type == "BiasedTransformer"
        super().__init__(dim_h, local_gnn_type, "Transformer", num_heads, **kw)
        # same module, same draws, same state_dict keys: only the forward reads the bias (global_model_type stays
        # "Transformer", the branch of the base forward that calls torch's module)
        self.self_attn.__class__ = _BiasedMHA

    def forward(self, batch):
        self.self_attn.attn_bias = batch.attn_bias      # AttributeError when the batch has none, as in the reference
        try:
            return super().forward(batch)
        finally:
            self.self_attn.attn_bias = None
