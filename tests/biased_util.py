"""Helpers of the BiasedTransformer tests: fixtures under tests/golden/biased/ and the attention biases they use."""
import glob
import os

import numpy as np
import torch

from util import GOLDEN_DIR, compare, golden_batch, run_layer

BIASED_DIR = os.path.join(GOLDEN_DIR, "biased")
LIVE_NAME = "reference_live_GINE_BiasedTransformer"
PAD_VALUE = 30.0   # padded entries of every generated bias: a kernel that reads one shifts its softmax visibly


def biased_names():
    names = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(BIASED_DIR, "*.pt")))
    return [n for n in names if n != LIVE_NAME]


def load_biased(name):
    return torch.load(os.path.join(BIASED_DIR, name + ".pt"), weights_only=False)


def biased_batch(fix, device="cpu", dtype=torch.float32):
    b = golden_batch(fix, device, dtype)
    b.attn_bias = fix["attn_bias"].to(device=device, dtype=dtype)
    return b


def graph_sizes(batch_vec, num_graphs):
    return torch.bincount(batch_vec.cpu(), minlength=num_graphs)


def make_bias(batch_vec, num_graphs, heads, seed, kind="random", edge_index=None, std=2.0):
    """[num_graphs * heads, Nmax, Nmax] float32 bias, row g * heads + h.

    random:      independent N(0, std^2) entries: asymmetric, different per head and per graph;
    graph_token: random, with row 0 and column 0 of every graph holding one value per head (Graphormer's graph token,
                 graphormer_encoder.py BiasEncoder with use_graph_token);
    spd:         a per-head table looked up by the shortest-path distance from query to key (scipy csgraph, unreachable
                 pairs get a table entry of their own), so values repeat as in real Graphormer batches.
    Padded entries (query or key beyond the graph) hold PAD_VALUE."""
    g = torch.Generator().manual_seed(seed)
    n = graph_sizes(batch_vec, num_graphs)
    nmax = int(n.max()) if num_graphs else 0
    B, H = num_graphs, heads
    bias = torch.full((B * H, nmax, nmax), PAD_VALUE)
    if kind == "spd":
        from scipy.sparse import coo_matrix
        from scipy.sparse.csgraph import shortest_path
        maxd = 6
        table = std * torch.randn(H, maxd + 2, generator=g)
        ptr = torch.zeros(B + 1, dtype=torch.int64)
        ptr[1:] = torch.cumsum(n, 0)
        ei = edge_index.cpu()
    for gi in range(B):
        ng = int(n[gi])
        if kind == "spd":
            sel = (ei[1] >= ptr[gi]) & (ei[1] < ptr[gi + 1])
            src, dst = (ei[0, sel] - ptr[gi]).numpy(), (ei[1, sel] - ptr[gi]).numpy()
            adj = coo_matrix((np.ones(len(src)), (src, dst)), shape=(ng, ng)).tocsr()
            d = shortest_path(adj, directed=True, unweighted=True)
            idx = torch.from_numpy(np.where(np.isinf(d), maxd + 1, np.minimum(d, maxd))).long()
            for h in range(H):
                bias[gi * H + h, :ng, :ng] = table[h][idx]
        else:
            bias[gi * H:(gi + 1) * H, :ng, :ng] = std * torch.randn(H, ng, ng, generator=g)
            if kind == "graph_token" and ng > 0:
                tok = std * torch.randn(H, generator=g)
                bias[gi * H:(gi + 1) * H, 0, :ng] = tok[:, None]
                bias[gi * H:(gi + 1) * H, :ng, 0] = tok[:, None]
    return bias


def run_biased(layer, batch, fix, backward=True):
    """util.run_layer plus the gradient w.r.t. batch.attn_bias (res["grad_attn_bias"])."""
    ab = batch.attn_bias.requires_grad_(backward)
    res = run_layer(layer, batch, fix, backward)
    if backward:
        res["grad_attn_bias"] = ab.grad.detach().cpu()
    return res


# util.compare checks grad_attn_bias itself whenever the fixture has it
compare_biased = compare
