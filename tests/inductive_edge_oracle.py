"""Float64 restatement of the inductive link-prediction head (dot decoding, one post-MP Linear) and of its ranking
statistics, with the library's tie rule: rank = 1 + #{k != j in the graph : <y_i, y_k> > <y_i, y_j>}."""
import torch

STATS = ("hits@1", "hits@3", "hits@10", "mrr")

_MASK31 = 0x7FFFFFFF


def hashed_x(n, d, seed):
    """Node features [n, d] float64 as a pure function of (n, d, seed): an integer hash of each element's index (31-bit
    products, so no int64 overflow), mapped to k / 64 with k in [-128, 128).  Every value is exact in bf16 and fp32, and
    the same on every machine and torch version, so a fixture stores the seed and a checksum instead of the tensor."""
    h = torch.arange(n * d, dtype=torch.int64)
    h = (h * 1103515245 + (seed & _MASK31) * 69069 + 12345) & _MASK31
    h = h ^ (h >> 13)
    h = (h * 1664525 + 1013904223) & _MASK31
    h = h ^ (h >> 16)
    h = (h * 22695477 + 1) & _MASK31
    k = ((h >> 12) & 255) - 128
    return (k.double() / 64.0).reshape(n, d)


def fixture_x(fix):
    """The fixture's node features, rebuilt from its seed and checked against its exact checksum."""
    n, d = fix["x_shape"]
    x = hashed_x(n, d, fix["x_seed"])
    assert float(x.sum()) == fix["x_sum"] and float((x * x).sum()) == fix["x_sumsq"], "hashed_x drifted"
    return x


def head_forward(x, weight, bias, eli):
    """y = x W^T + b and pred[k] = <y[s_k], y[t_k]>."""
    y = x @ weight.t() + bias
    return y, (y[eli[0]] * y[eli[1]]).sum(-1)


def rank_stats(y, eli, label, ptr):
    """{'hits@1', 'hits@3', 'hits@10', 'mrr'}: per graph (node offsets ptr [B+1]) the means over its positives, 0 for a
    graph without positives, then the mean over the graphs.  A positive's graph is its source node's."""
    y = y.detach().double()
    ptr = [int(v) for v in ptr]
    B = len(ptr) - 1
    pos = (label == 1).nonzero().flatten().tolist()
    src, dst = eli[0].tolist(), eli[1].tolist()
    per_graph = {g: [] for g in range(B)}
    graph_of = torch.bucketize(torch.tensor([src[k] for k in pos], dtype=torch.int64),
                               torch.tensor(ptr[1:], dtype=torch.int64), right=True).tolist()
    for k, g in zip(pos, graph_of):
        i, j = src[k], dst[k]
        n0, n1 = ptr[g], ptr[g + 1]
        scores = y[n0:n1] @ y[i]
        above = scores > scores[j - n0]
        above[j - n0] = False
        per_graph[g].append(1 + int(above.sum()))
    totals = [0.0] * 4
    for g in range(B):
        ranks = torch.tensor(per_graph[g], dtype=torch.float64)
        if ranks.numel():
            vals = [float((ranks <= 1).double().mean()), float((ranks <= 3).double().mean()),
                    float((ranks <= 10).double().mean()), float((1.0 / ranks).mean())]
            totals = [a + v for a, v in zip(totals, vals)]
    return {name: (t / B if B else 0.0) for name, t in zip(STATS, totals)}
