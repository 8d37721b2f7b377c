"""Float64 restatement of Graphormer's attention-bias encoder (graphgps/encoder/graphormer_encoder.py:140-183), straight
from its formula; its backward is autograd's.  For pair p = (b, i, j) of graph b with sd_p = max(1, spatial_types[p]):

    bias[b, h, o + i, o + j] = spatial[s_p, h] + (1 / sd_p) sum_k sum_h' edge[spt[p, k], h'] W[k, h', h]

W[k, h', h] = edge_dis_encoder.weight[k * H * H + h' * H + h]; the edge term only with shortest_path_types.  Entries no
pair covers are 0.  With the graph token (o = 1) the block is padded by one leading row and column, both filled with
graph_token[h].  Output [B * H, N', N'] with B = batch.max() + 1 and N' = Nmax + o, row b * H + h.
"""
from __future__ import annotations

import torch


def bias_forward(state, spatial_types, graph_index, batch, heads, shortest_path_types=None, use_graph_token=True):
    sp = state["spatial_encoder.weight"]
    dtype = sp.dtype
    H = heads
    B = int(batch.max()) + 1
    counts = torch.bincount(batch, minlength=B)
    ptr = torch.zeros(B + 1, dtype=torch.int64, device=batch.device)
    ptr[1:] = torch.cumsum(counts, 0)
    nmax = int(counts.max())
    i, j = graph_index[0], graph_index[1]
    b = batch[i]
    il, jl = i - ptr[b], j - ptr[b]
    val = sp[spatial_types]                                                        # [P, H]
    if shortest_path_types is not None:
        S = shortest_path_types.shape[1]
        W = state["edge_dis_encoder.weight"].reshape(S, H, H)
        E = state["edge_encoder.weight"]
        sd = spatial_types.clamp(min=1).to(dtype)
        val = val + torch.einsum("pkq,kqh->ph", E[shortest_path_types], W) / sd[:, None]
    o = 1 if use_graph_token else 0
    n = nmax + o
    dense = torch.zeros(B, n, n, H, dtype=dtype, device=val.device).index_put((b, il + o, jl + o), val)
    if use_graph_token:
        edge = torch.zeros(n, n, dtype=torch.bool, device=val.device)
        edge[0, :] = True
        edge[:, 0] = True
        dense = torch.where(edge[None, :, :, None], state["graph_token"].reshape(1, 1, 1, H), dense)
    return dense.permute(0, 3, 1, 2).reshape(B * H, n, n)


def bias_inputs(fix, device="cpu"):
    """(spatial_types, graph_index, batch, shortest_path_types or None) of a fixture on `device`."""
    spt = fix.get("shortest_path_types")
    return (fix["spatial_types"].to(device), fix["graph_index"].to(device), fix["batch"].to(device),
            None if spt is None else spt.to(device))
