"""Dense float64 restatement of the Graphormer layer (graphgps/layer/graphormer_layer.py:39-49), graph by graph, and
the batches of the Graphormer tests.

    h   = LayerNorm(x)                                   input_norm, eps 1e-5
    a   = MHA(h, h, h) restricted to each graph           scale 1/sqrt(hd), + attn_bias[g*H + h] after scaling
    x1  = a + x
    out = W2 GELU(W1 LayerNorm(x1) + b1) + b2 + x1        mlp.0 .. mlp.5 (exact erf GELU)

Dropout is not restated: the fixtures and the dense comparisons run with it off (the GPU tests replay the masks).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def graphormer_forward(state, x, batch, num_graphs, heads, attn_bias=None, return_attn=False):
    """out [N, d] of the layer with parameters `state` (the reference's state_dict names)."""
    d = x.shape[1]
    hd = d // heads
    s = {k: v.to(x.dtype) for k, v in state.items()}
    h = F.layer_norm(x, (d,), s["input_norm.weight"], s["input_norm.bias"], 1e-5)
    qkv = h @ s["attention.in_proj_weight"].t() + s["attention.in_proj_bias"]
    q, k, v = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
    O = attention(q, k, v, batch, num_graphs, heads, attn_bias)
    a = O @ s["attention.out_proj.weight"].t() + s["attention.out_proj.bias"]
    x1 = a + x
    h2 = F.layer_norm(x1, (d,), s["mlp.0.weight"], s["mlp.0.bias"], 1e-5)
    hid = F.gelu(h2 @ s["mlp.1.weight"].t() + s["mlp.1.bias"])
    return hid @ s["mlp.4.weight"].t() + s["mlp.4.bias"] + x1


def attention(q, k, v, batch, num_graphs, heads, attn_bias=None):
    """Softmax attention of every node over its own graph's nodes; q, k, v [N, heads * hd] -> O [N, heads * hd]."""
    N, D = q.shape
    hd = D // heads
    counts = torch.bincount(batch, minlength=num_graphs).tolist()
    out = torch.zeros_like(q)
    start = 0
    for g, n in enumerate(counts):
        if n:
            sl = slice(start, start + n)
            Q = q[sl].view(n, heads, hd).transpose(0, 1) / math.sqrt(hd)
            K = k[sl].view(n, heads, hd).transpose(0, 1)
            V = v[sl].view(n, heads, hd).transpose(0, 1)
            S = Q @ K.transpose(1, 2)
            if attn_bias is not None:
                S = S + attn_bias[g * heads:(g + 1) * heads, :n, :n].to(S.dtype)
            out[sl] = (torch.softmax(S, -1) @ V).transpose(0, 1).reshape(n, D)
        start += n
    return out


def graphormer_batch(sizes, d, seed=0, token=False, dtype=torch.float32):
    """A batch of ring graphs with one chord each; token=True makes the first node of every graph a graph token (one
    shared feature row and no edges, as add_graph_token prepends it)."""
    from graphgps_b200.batch import batch_from_lists
    edges = []
    for n in sizes:
        base = 1 if token else 0
        m = n - base
        el = [(base + i, base + (i + 1) % m) for i in range(m)] + [(base + (i + 1) % m, base + i) for i in range(m)] \
            if m > 1 else []
        if m > 3:
            el += [(base, base + m // 2), (base + m // 2, base)]
        edges.append(el)
    b = batch_from_lists(sizes, edges, d, seed=seed)
    x = b.x.to(dtype)
    if token:
        g = torch.Generator().manual_seed(seed + 7)
        tok = torch.randn(d, generator=g).to(dtype)
        starts = [0]
        for n in sizes[:-1]:
            starts.append(starts[-1] + n)
        x[starts] = tok
    b.x = x
    b.edge_attr = b.edge_attr.to(dtype)
    return b


def random_bias(sizes, heads, seed=0, dtype=torch.float32):
    """attn_bias [B * heads, Nmax, Nmax]; the padded entries hold large values that a kernel must never read."""
    nmax = max(sizes)
    g = torch.Generator().manual_seed(seed)
    ab = torch.full((len(sizes) * heads, nmax, nmax), 1e4, dtype=torch.float64)
    for gi, n in enumerate(sizes):
        ab[gi * heads:(gi + 1) * heads, :n, :n] = torch.randn(heads, n, n, generator=g, dtype=torch.float64) * 0.7
    return ab.to(dtype)
