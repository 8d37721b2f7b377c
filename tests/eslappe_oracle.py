"""TEST INFRASTRUCTURE - CPU restatement (pure torch) of the reference GPSLayer with equivstable_pe=True.

Extends oracle/gps_oracle.py (unchanged) with the EquivStableLapPE edge gate of GatedGCN,
graphgps/layer/gatedgcn_layer.py (paths relative to the reference checkout):
  * :29-35    mlp_r_ij = Sequential(Linear(1, d), act(), Linear(d, 1), Sigmoid())
  * :65-70    PE = batch.pe_EquivStableLapPE, passed to propagate
  * :101-104  r_ij = sum_c (PE_i - PE_j)^2 ;  sigma_ij = sigmoid(e_ij) * mlp_r_ij(r_ij)
and the flag's handling in graphgps/layer/gps_layer.py: GatedGCN receives the PE (:92-96, :164-171); GCN and None
never read it (:176-187); GINE + equivstable_pe builds GINEConvESLapPE, whose __init__ calls reset_parameters()
(gine_conv_layer.py:35) before :44 defines mlp_r_ij, so the reference raises AttributeError and the pair is refused here.

Pinned to the reference itself: tests/test_eslappe.py::test_oracle_equals_reference_live_eslappe holds this file to the
reference layer's fp64 outputs and gradients (grad_pe included) stored by tests/golden/make_eslappe_golden.py.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.gps_oracle import _ACTS, OracleGatedGCN, OracleGPSLayer, OraclePerformerSelfAttention


class OracleGatedGCNESLapPE(OracleGatedGCN):
    """OracleGatedGCN with the EquivStableLapPE gate.  The PE of the current call is handed over in `self.pe` by
    OracleGPSLayerESLapPE.forward (the base layer calls local_model(x, e, edge_index))."""

    def __init__(self, dim, dropout, act="relu"):
        super().__init__(dim, dropout, act)
        self.mlp_r_ij = nn.Sequential(nn.Linear(1, dim), _ACTS[act](), nn.Linear(dim, 1), nn.Sigmoid())   # :29-35
        self.pe = None

    def forward(self, x, e, edge_index):
        pe = self.pe
        src, dst = edge_index[0], edge_index[1]          # j = source, i = target
        x_in, e_in = x, e                                  # :52-54
        Ax, Bx, Ce, Dx, Ex = self.A(x), self.B(x), self.C(e), self.D(x), self.E(x)   # :57-61
        e_ij = Dx[dst] + Ex[src] + Ce                      # :96
        sigma = torch.sigmoid(e_ij)                        # :97
        r_ij = ((pe[dst] - pe[src]) ** 2).sum(dim=-1, keepdim=True)   # :102 (PE_i - PE_j)
        sigma = sigma * self.mlp_r_ij(r_ij)                # :103-104
        num = torch.zeros_like(Bx).index_add_(0, dst, sigma * Bx[src])   # :117-119
        den = torch.zeros_like(Bx).index_add_(0, dst, sigma)             # :121-123
        x = Ax + num / (den + 1e-6)                        # :125, :133
        e = e_ij                                           # :106, :134
        x = self.act_fn_x(self.bn_node_x(x))               # :72, :75
        e = self.act_fn_e(self.bn_edge_e(e))               # :73, :76
        x = F.dropout(x, self.dropout, training=self.training)   # :78
        e = F.dropout(e, self.dropout, training=self.training)   # :79
        return x_in + x, e_in + e                          # :81-83


class OracleGPSLayerESLapPE(OracleGPSLayer):
    """OracleGPSLayer(..., equivstable_pe=True): GatedGCN gets the gate; GCN / None ignore the flag; GINE raises.

    Parameters are drawn in the reference's order (local model incl. mlp_r_ij, then the global model, then the FFN:
    gps_layer.py:44-153), so under the same torch seed the initial state equals the reference layer's."""

    def __init__(self, dim_h, local_gnn_type, global_model_type, num_heads, act="relu", dropout=0.0,
                 attn_dropout=0.0, **kw):
        if local_gnn_type == "GINE":
            raise NotImplementedError("GINE with equivstable_pe=True does not construct in the reference "
                                      "(gine_conv_layer.py:35,44)")
        rng = torch.get_rng_state()
        super().__init__(dim_h, local_gnn_type, global_model_type, num_heads, act=act, dropout=dropout,
                         attn_dropout=attn_dropout, **kw)
        self.equivstable_pe = local_gnn_type == "CustomGatedGCN"
        if self.equivstable_pe:
            # re-draw from the constructor's starting RNG state in the reference's order: the gated local model with
            # mlp_r_ij (gatedgcn_layer.py:21-38), then everything the base constructor built after the local model
            # (BatchNorms and dropouts draw nothing)
            torch.set_rng_state(rng)
            self.local_model = OracleGatedGCNESLapPE(dim_h, dropout, act)
            if global_model_type == "Transformer":
                self.self_attn = nn.MultiheadAttention(dim_h, num_heads, dropout=attn_dropout, batch_first=True)
            elif global_model_type == "Performer":
                self.self_attn = OraclePerformerSelfAttention(dim_h, num_heads, dropout=attn_dropout)
            self.ff_linear1 = nn.Linear(dim_h, dim_h * 2)
            self.ff_linear2 = nn.Linear(dim_h * 2, dim_h)

    def forward(self, batch):
        if not self.equivstable_pe:
            return super().forward(batch)
        self.local_model.pe = batch.pe_EquivStableLapPE    # gps_layer.py:164-171
        try:
            return super().forward(batch)
        finally:
            self.local_model.pe = None
