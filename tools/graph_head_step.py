"""Cost of the graph-prediction heads: graphgps_b200.SANGraphHead / GraphormerHead against the reference heads
(graphgps/head/san_graph.py, graphormer_graph.py with PyG's pooling) restated in eager torch.

    python tools/graph_head_step.py [--steps 50] [--rounds 5]

  1. head forward + backward from a fixed cotangent of pred at four shapes: the library recorded into a CUDA graph and
     replayed, against eager torch (PyG's pooling with size=None reads batch.max() to the host; to_dense_batch reads its
     batch size and Nmax);
  2. one training step of 5 GatedGCNLayers (d 304, PCQM4Mv2-shaped batch) -> SANGraphHead (mean) -> L1 loss ->
     backward, captured whole in one CUDA graph, against the same step without the head (layers -> L1 loss on x).
Each round times every arm `steps` times between two CUDA events; rounds alternate the arms and the median ms over the
rounds is printed with the launches per call, the GPU name and its power limit."""
import argparse
import os
import statistics
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import graphgps_b200  # noqa: E402
from graphgps_b200 import _lib  # noqa: E402
from graphgps_b200.graph import graph_of  # noqa: E402
from graphormer_step import gpu_info, timed  # noqa: E402
from inductive_edge_step import kernels_of  # noqa: E402

DEV = "cuda"


def torch_pool(x, batch, pooling):
    """PyG's global_mean_pool / global_add_pool (size=None) and graph_token's to_dense_batch(x, batch)[:, 0]."""
    B = int(batch.max()) + 1   # host read
    if pooling != "graph_token":
        s = x.new_zeros(B, x.shape[1]).index_add_(0, batch, x)
        if pooling == "add":
            return s
        return s / torch.bincount(batch, minlength=B).clamp(min=1).to(x.dtype).unsqueeze(1)
    n = torch.bincount(batch, minlength=B)
    ptr = torch.cat([n.new_zeros(1), torch.cumsum(n, 0)])
    nmax = int(n.max())        # host read
    dense = x.new_zeros(B, nmax, x.shape[1])
    dense[batch, torch.arange(x.shape[0], device=x.device) - ptr[batch]] = x
    return dense[:, 0]


def torch_head(head, x, batch):
    if isinstance(head, graphgps_b200.GraphormerHead):
        h = torch_pool(head.ln(x), batch, head.graph_pooling)
        return head.layers(h)
    h = torch_pool(x, batch, head.graph_pooling)
    act = torch.relu if head.act == "relu" else F.gelu
    for l, fc in enumerate(head.FC_layers):
        h = fc(h)
        if l < head.L:
            h = act(h)
    return h


def shape_batch(B, lo, hi, d, seed, token=False):
    g = torch.Generator().manual_seed(seed)
    sizes = (torch.randint(lo, hi + 1, (B,), generator=g) + (1 if token else 0)).tolist()
    batch = torch.repeat_interleave(torch.arange(B), torch.tensor(sizes))
    return types.SimpleNamespace(x=torch.randn(len(batch), d, generator=g).to(DEV), batch=batch.to(DEV),
                                 edge_index=torch.zeros(2, 0, dtype=torch.int64, device=DEV), num_graphs=B,
                                 y=torch.zeros(B, device=DEV))


# name, head, graphs, sizes lo..hi, d, dim_out, pooling
SHAPES = [("pcqm4m", "san", 256, 1, 51, 304, 1, "mean"),
          ("zinc", "san", 32, 9, 37, 64, 1, "add"),
          ("molpcba-SAN", "san", 512, 5, 40, 304, 128, "add"),
          ("zinc-Graphormer", "graphormer", 256, 10, 38, 80, 1, "graph_token")]


def capture(step):
    step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    return graph


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/graph_head_step.py needs a CUDA device")
    name, plim = gpu_info()
    print(f"GPU: {name}, power limit {plim}")
    lib = _lib.load()
    torch.manual_seed(0)

    # 1. the head alone
    for i, (label, kind, B, lo, hi, d, dout, pooling) in enumerate(SHAPES):
        data = shape_batch(B, lo, hi, d, i, token=kind == "graphormer")
        head = (graphgps_b200.SANGraphHead(d, dout, graph_pooling=pooling) if kind == "san" else
                graphgps_b200.GraphormerHead(d, dout)).to(DEV).train()
        x = data.x.clone().requires_grad_(True)
        ct = torch.randn(B, dout, device=DEV)
        params = [x] + list(head.parameters())

        def lib_step():
            data.x = x
            pred, _ = head(data)
            data.graph_feature = None   # a graph kept alive from the previous step would tie the capture to its stream
            return torch.autograd.grad((pred * ct).sum(), params)

        def torch_step():
            pred = torch_head(head, x, data.batch)
            return torch.autograd.grad((pred * ct).sum(), params)

        a, b = lib_step(), torch_step()
        err = max(float((u - v).abs().max()) / max(float(v.abs().max()), 1e-30) for u, v in zip(a, b))
        graph = capture(lib_step)
        c0 = lib.gps_launch_count()
        lib_step()
        launches = lib.gps_launch_count() - c0
        tk = kernels_of(torch_step)
        t = {"library": [], "torch": []}
        for _ in range(args.rounds):
            t["library"].append(timed(graph.replay, args.steps))
            t["torch"].append(timed(torch_step, args.steps))
        lt, tt = statistics.median(t["library"]), statistics.median(t["torch"])
        print(f"1. {label}: {type(head).__name__}, {B} graphs, {data.x.shape[0]} nodes, d {d} -> {dout}, {pooling}: "
              f"library captured {1e3 * lt:.1f} us ({launches} launches, 0 host reads) | eager torch {1e3 * tt:.1f} us "
              f"({tk} kernels and copies, {1 if pooling != 'graph_token' else 2} host reads) | x{tt / lt:.1f} | "
              f"max rel diff {err:.1e}")

    # 2. a captured training step: 5 GatedGCNLayers -> head -> L1
    d = 304
    gb = graphgps_b200.make_batch("pcqm4m-small", seed=1, dim=d).to(DEV)
    B = int(gb.num_graphs)
    y = torch.randn(B, 1, device=DEV)
    layers = [graphgps_b200.GatedGCNLayer(d, d, 0.0, True).to(DEV).train() for _ in range(5)]
    head = graphgps_b200.SANGraphHead(d, 1, graph_pooling="mean").to(DEV).train()
    x0, e0 = gb.x.clone().requires_grad_(True), gb.edge_attr.clone()
    lparams = [p for layer in layers for p in layer.parameters()]
    graph_of(gb)

    def stack():
        gb.x, gb.edge_attr = x0, e0
        for layer in layers:
            layer(gb)
        return gb

    def release():   # nothing of this step's autograd graph outlives it (see lib_step)
        gb.x, gb.edge_attr, gb.graph_feature = x0, e0, None

    def with_head():
        pred, _ = head(stack())
        release()
        return torch.autograd.grad(F.l1_loss(pred, y), lparams + list(head.parameters()))

    def without_head():
        h = stack().x
        release()
        return torch.autograd.grad(F.l1_loss(h, torch.zeros_like(h)), lparams)

    gb.y = y
    g_with, g_without = capture(with_head), capture(without_head)
    counts = []
    for fn in (with_head, without_head):
        c0 = lib.gps_launch_count()
        fn()
        counts.append(lib.gps_launch_count() - c0)
    t = {"with": [], "without": []}
    for _ in range(args.rounds):
        t["with"].append(timed(g_with.replay, args.steps))
        t["without"].append(timed(g_without.replay, args.steps))
    mw, mo = statistics.median(t["with"]), statistics.median(t["without"])
    print(f"2. captured training step, 5 GatedGCNLayers, {B} graphs, {gb.x.shape[0]} nodes, d {d}: with SANGraphHead "
          f"{mw:.3f} ms ({counts[0]} launches) | layers alone {mo:.3f} ms ({counts[1]} launches) | head "
          f"{1e3 * (mw - mo):.1f} us ({100 * (mw - mo) / mw:.1f} % of the step)")


if __name__ == "__main__":
    main()
