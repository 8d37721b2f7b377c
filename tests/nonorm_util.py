"""Helpers of the GPSLayer(..., batch_norm=False) tests: fixtures under tests/golden/nonorm/ and seeded single-graph
node-level batches (full-batch transductive tasks: the whole graph is the batch).

The sizes of NODE_SHAPES follow the public statistics of the datasets the six GCN+Transformer configs train on
(actor-GPS, wn-{squirrel,chameleon}-GPS, webkb-{cor,tex,wis}-GPS); the edges are synthetic, not the datasets'."""
import collections
import glob
import os

import torch

from graphgps_b200.batch import GraphBatch
from util import GOLDEN_DIR

NONORM_DIR = os.path.join(GOLDEN_DIR, "nonorm")
LIVE_NAME = "reference_live_GCN_Transformer"

# name -> nodes, directed edges, dim_h, heads, attn_dropout of the config
NodeShape = collections.namedtuple("NodeShape", "N E d heads attn_dropout")
NODE_SHAPES = {
    "webkb": NodeShape(183, 325, 64, 4, 0.0),          # WebKB Texas
    "chameleon": NodeShape(2277, 36101, 96, 4, 0.5),   # WikipediaNetwork chameleon (head dim 24)
    "squirrel": NodeShape(5201, 217073, 64, 4, 0.0),   # WikipediaNetwork squirrel: heavy-tailed in-degree
    "actor": NodeShape(7600, 30019, 64, 4, 0.0),       # Actor
}


def nonorm_names():
    names = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(NONORM_DIR, "*.pt")))
    return [n for n in names if n != LIVE_NAME]


def load_nonorm(name):
    return torch.load(os.path.join(NONORM_DIR, name + ".pt"), weights_only=False)


def node_graph(N, E, d, seed=0, tail=1.5, dtype=torch.float32):
    """One directed graph as a batch of one: E edges j -> i with uniform sources and destinations drawn from Pareto
    (shape `tail`) node weights, so a few nodes have in-degrees in the thousands at the squirrel shape.  Self loops and
    duplicate edges occur as they come.  Vectorised: 217 k edges take milliseconds."""
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(N, generator=g, dtype=torch.float64).clamp_min(1e-12) ** (-1.0 / tail)
    dst = torch.multinomial(w, E, replacement=True, generator=g)
    src = torch.randint(0, N, (E,), generator=g)
    x = torch.randn(N, d, generator=g).to(dtype)
    edge_attr = torch.randn(E, d, generator=g).to(dtype)
    return GraphBatch(x=x, edge_index=torch.stack([src, dst]), edge_attr=edge_attr,
                      batch=torch.zeros(N, dtype=torch.int64), num_graphs=1, ptr=torch.tensor([0, N]))


def node_shape_batch(name, seed=0):
    s = NODE_SHAPES[name]
    return node_graph(s.N, s.E, s.d, seed=seed)


def with_edge_cases(b, seed=0):
    """b with every edge at its last node removed (an isolated node), a self loop at node 0 and a duplicate of edge 0."""
    ei, ea = b.edge_index, b.edge_attr
    last = b.x.shape[0] - 1
    keep = (ei[0] != last) & (ei[1] != last)
    ei, ea = ei[:, keep], ea[keep]
    g = torch.Generator().manual_seed(seed)
    ei = torch.cat([ei, torch.tensor([[0], [0]]), ei[:, :1]], dim=1)
    ea = torch.cat([ea, torch.randn(1, ea.shape[1], generator=g).to(ea.dtype), ea[:1]], dim=0)
    return GraphBatch(x=b.x, edge_index=ei, edge_attr=ea, batch=b.batch, num_graphs=b.num_graphs, ptr=b.ptr)
