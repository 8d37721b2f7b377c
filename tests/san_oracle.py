"""Float64 restatement of the SAN layer (graphgps/layer/san_layer.py:10-210 with full_graph=True, batch_norm=True,
layer_norm=False, residual=True, use_bias=False) and a SAN batch generator with dataset-like shapes.

The restatement follows the reference line by line:
  * MultiHeadAttentionLayer.forward (san_layer.py:89-120): Q_h, K_h, V_h, Q_2h, K_2h from x, E from edge_attr,
    E_2 = E_2(fake_edge_emb.weight[0]), all without bias, viewed as [*, H, hd];
  * propagate_attention (san_layer.py:38-87): per real edge j -> i the score exp(clamp(sum(K_j Q_i / sqrt(hd) E), -5,
    5)) / (gamma + 1), per fake pair gamma exp(clamp(sum(K2_j Q2_i / sqrt(hd) E_2), -5, 5)) / (gamma + 1); wV and Z are
    scatter-sums over the destination; h = wV / (Z + 1e-6);
  * the fake pairs are negate_edge_index's complement (graphgps/utils.py:12-65): every ordered pair of a graph without
    a real edge, self pairs removed, built here with a dense boolean matrix per graph (fake_pairs);
  * SANLayer.forward (san_layer.py:169-210): h1 = BN1(x + O_h(dropout(h))), out = BN2(h1 + FFN2(dropout(relu(FFN1(h1)))))
    with nn.BatchNorm1d's batch statistics (biased variance) in training and the running ones in eval.
Dropout masks (the library's, 0 or 1/(1-p)) can be injected at both sites.
"""
import math

import torch


def fake_pairs(edge_index, batch, num_graphs):
    """(src, dst) of every pair j -> i, j != i, of the same graph without a real edge j -> i."""
    batch = batch.cpu()
    ei = edge_index.cpu()
    counts = torch.bincount(batch, minlength=num_graphs)
    ptr = torch.zeros(num_graphs + 1, dtype=torch.int64)
    ptr[1:] = torch.cumsum(counts, 0)
    srcs, dsts = [], []
    for g in range(num_graphs):
        n, p0 = int(counts[g]), int(ptr[g])
        adj = torch.ones(n, n, dtype=torch.bool)
        m = (batch[ei[0]] == g) & (batch[ei[1]] == g)
        adj[ei[0, m] - p0, ei[1, m] - p0] = False
        adj.fill_diagonal_(False)
        s, d = adj.nonzero(as_tuple=True)
        srcs.append(s + p0)
        dsts.append(d + p0)
    if not srcs:
        return torch.zeros(2, 0, dtype=torch.int64, device=edge_index.device)
    return torch.stack([torch.cat(srcs), torch.cat(dsts)]).to(edge_index.device)


def san_attention(Q, K, V, Q2, K2, E, E2, edge_index, fake_index, H, gamma):
    """h_out [N, d] of propagate_attention + forward (san_layer.py:38-120); Q..K2 [N, d], E [E, d], E2 [d]."""
    N, d = Q.shape
    hd = d // H
    v = lambda t: t.reshape(-1, H, hd)  # noqa: E731
    src, dst = edge_index[0], edge_index[1]
    score = (v(K)[src] * v(Q)[dst] / math.sqrt(hd) * v(E)).sum(-1, keepdim=True)
    score = torch.exp(score.clamp(-5, 5)) / (gamma + 1)
    fs, fd = fake_index[0], fake_index[1]
    score2 = (v(K2)[fs] * v(Q2)[fd] / math.sqrt(hd) * E2.reshape(1, H, hd)).sum(-1, keepdim=True)
    score2 = gamma * torch.exp(score2.clamp(-5, 5)) / (gamma + 1)
    wV = torch.zeros(N, H, hd, dtype=Q.dtype, device=Q.device)
    wV = wV.index_add(0, dst, v(V)[src] * score).index_add(0, fd, v(V)[fs] * score2)
    Z = torch.zeros(N, H, 1, dtype=Q.dtype, device=Q.device)
    Z = Z.index_add(0, dst, score).index_add(0, fd, score2)
    return (wV / (Z + 1e-6)).reshape(N, d)


def _bn(z, w, b, rm, rv, training):
    if training:
        mu = z.mean(0)
        var = z.var(0, unbiased=False)
    else:
        mu, var = rm, rv
    return (z - mu) / torch.sqrt(var + 1e-5) * w + b


def san_forward(state, x, edge_attr, edge_index, fake_index, H, gamma, training=True, masks=None, prefix=""):
    """One SANLayer in float64.  state: the layer's parameters (and, for eval, running statistics) by state_dict name;
    masks: optional (m_attn [N, d], m_ffn [N, 2d]) dropout scales."""
    s = lambda n: state[prefix + n]  # noqa: E731
    lin = lambda t, n, bias=True: t @ s(n + ".weight").t() + (s(n + ".bias") if bias else 0)  # noqa: E731
    emb = s("attention.fake_edge_emb.weight")[0]
    E2 = s("attention.E_2.weight") @ emb
    h = san_attention(lin(x, "attention.Q", False), lin(x, "attention.K", False), lin(x, "attention.V", False),
                      lin(x, "attention.Q_2", False), lin(x, "attention.K_2", False),
                      lin(edge_attr, "attention.E", False), E2, edge_index, fake_index, H, gamma)
    if masks is not None:
        h = h * masks[0]
    z1 = x + lin(h, "O_h")
    h1 = _bn(z1, s("batch_norm1_h.weight"), s("batch_norm1_h.bias"), state.get(prefix + "batch_norm1_h.running_mean"),
             state.get(prefix + "batch_norm1_h.running_var"), training)
    t = torch.relu(lin(h1, "FFN_h_layer1"))
    if masks is not None:
        t = t * masks[1]
    z2 = h1 + lin(t, "FFN_h_layer2")
    return _bn(z2, s("batch_norm2_h.weight"), s("batch_norm2_h.bias"), state.get(prefix + "batch_norm2_h.running_mean"),
               state.get(prefix + "batch_norm2_h.running_var"), training)


# ------------------------------------------------------------------------------------------ batches
class SanBatch:
    """x [N, d], edge_attr [E, d], edge_index [2, E], batch [N], num_graphs; size(0) = N as PyG's Batch.size."""

    def __init__(self, x, edge_attr, edge_index, batch, num_graphs):
        self.x, self.edge_attr, self.edge_index, self.batch, self.num_graphs = x, edge_attr, edge_index, batch, num_graphs

    def size(self, dim=None):
        return self.x.shape[0] if dim in (0, None) else self.x.shape[dim]

    def to(self, dev):
        return SanBatch(self.x.to(dev), self.edge_attr.to(dev), self.edge_index.to(dev), self.batch.to(dev),
                        self.num_graphs)


def _graph_edges(kind, n, g):
    """Directed edge list (src, dst) of one graph of n nodes, local indices.  Approximate published statistics:
    molecules (ZINC / ogbg-mol*: ~23-26 atoms, bonds both ways), peptide chains (~150 residues, chain plus a few
    contacts), SBM graphs (PATTERN / CLUSTER: ~118 nodes, ~40 % density), superpixel kNN graphs (COCO / VOC: ~480
    nodes, ~8 in-edges per node)."""
    if n == 1:
        return torch.zeros(2, 0, dtype=torch.int64)
    if kind in ("mol", "chain"):
        src = torch.arange(n - 1)
        dst = src + 1
        extra = max(1, n // (6 if kind == "mol" else 20))
        a = torch.randint(0, n, (extra,), generator=g)
        b = torch.randint(0, n, (extra,), generator=g)
        keep = a != b
        src, dst = torch.cat([src, a[keep]]), torch.cat([dst, b[keep]])
        return torch.cat([torch.stack([src, dst]), torch.stack([dst, src])], 1)
    if kind == "sbm":
        p = torch.rand(n, n, generator=g)
        adj = torch.triu(p < 0.4, 1)
        adj = adj | adj.t()
        s, d = adj.nonzero(as_tuple=True)
        return torch.stack([s, d])
    if kind == "knn":
        pos = torch.rand(n, 2, generator=g)
        dist = torch.cdist(pos, pos)
        dist.fill_diagonal_(float("inf"))
        k = min(8, n - 1)
        nb = dist.topk(k, largest=False).indices          # the k nearest sources of every node
        dst = torch.arange(n).repeat_interleave(k)
        return torch.stack([nb.reshape(-1), dst])
    raise ValueError(kind)


def san_batch(kind, sizes, d, seed, dtype=torch.float32, scale=1.0):
    """Graphs of the given sizes and kind, node and edge features ~ N(0, scale^2)."""
    g = torch.Generator().manual_seed(seed)
    eis, batch, off = [], [], 0
    for gi, n in enumerate(sizes):
        eis.append(_graph_edges(kind, n, g) + off)
        batch.append(torch.full((n,), gi, dtype=torch.int64))
        off += n
    ei = torch.cat(eis, 1) if eis else torch.zeros(2, 0, dtype=torch.int64)
    x = torch.randn(off, d, generator=g, dtype=torch.float64) * scale
    e = torch.randn(ei.shape[1], d, generator=g, dtype=torch.float64) * scale
    return SanBatch(x.to(dtype), e.to(dtype), ei, torch.cat(batch), len(sizes))


def dataset_sizes(kind, count, seed):
    """Graph sizes drawn around the datasets' published mean sizes."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = {"mol": (10, 38), "chain": (120, 180), "sbm": (100, 137), "knn": (420, 520)}[kind]
    return torch.randint(lo, hi + 1, (count,), generator=g).tolist()
