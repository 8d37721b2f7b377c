"""Cost of RWSE on the device (run on an H100): prints the card, its power limit and one JSON line of timings.

  * rw_landing_probs per batch at the PCQM4Mv2, ZINC, molpcba, cifar10 and MalNet-Tiny shapes (device time, CUDA
    events, the batch's graph structure already built);
  * the landing probabilities of a whole synthetic PCQM4Mv2 (3.75 M graphs, 256 per batch; device time of the landing
    calls only, over 64 distinct batches cycled);
  * the CPU baseline: the float32 dense restatement of the reference (D^-1 A and its matrix powers per graph, numpy)
    on this host for a fixed number of PCQM4Mv2-sized graphs, scaled to 3.75 M graphs;
  * the encoder's forward + backward at PCQM4Mv2 shape, captured in a CUDA graph, against an eager-torch float32
    restatement of the reference encoder;
  * its share of a captured PCQM4Mv2 training step: encoder + 5 GatedGCN+Transformer GPSLayers + SANGraphHead.

    python tools/rwse_step.py
"""
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import graphgps_b200  # noqa: E402
from graphgps_b200.graph import graph_of  # noqa: E402

DEV = "cuda:0"
PCQM_GRAPHS = 3_746_620


def molecules(rng, sizes, directed_knn=0):
    """Edges of undirected random trees with a ring closure (or directed k-NN graphs), batched by node offset."""
    src, dst, off = [], [], 0
    for n in sizes:
        n = int(n)
        if directed_knn:
            p = rng.random((n, 2))
            d = ((p[:, None] - p[None]) ** 2).sum(-1)
            np.fill_diagonal(d, np.inf)
            nb = np.argsort(d, 1)[:, :directed_knn]
            s, t = np.repeat(np.arange(n), directed_knn), nb.ravel()
        else:
            par = np.array([rng.integers(0, i) for i in range(1, n)], dtype=np.int64)
            s, t = np.arange(1, n), par
            if n > 5:
                s, t = np.append(s, 0), np.append(t, n - 1)
            s, t = np.concatenate([s, t]), np.concatenate([t, s])
        src.append(s + off)
        dst.append(t + off)
        off += n
    ei = torch.from_numpy(np.stack([np.concatenate(src), np.concatenate(dst)]).astype(np.int64))
    bvec = torch.repeat_interleave(torch.arange(len(sizes)), torch.as_tensor(np.asarray(sizes, dtype=np.int64)))
    return types.SimpleNamespace(edge_index=ei.to(DEV), batch=bvec.to(DEV), num_graphs=len(sizes))


def hubs(rng, n, m=2):
    src, dst, deg = [], [], np.ones(n)
    for i in range(1, n):
        t = rng.choice(i, min(m, i), replace=False, p=deg[:i] / deg[:i].sum())
        src += [i] * len(t)
        dst += list(t)
        deg[t] += 1
    return np.array([src, dst]), n


def malnet(rng, graphs=16, mean_nodes=1410):
    parts, off, sizes = [], 0, []
    for n in rng.integers(mean_nodes // 2, mean_nodes * 3 // 2, graphs):
        e, n = hubs(rng, int(n))
        parts.append(e + off)
        off += n
        sizes.append(n)
    ei = torch.from_numpy(np.concatenate(parts, 1).astype(np.int64))
    bvec = torch.repeat_interleave(torch.arange(graphs), torch.as_tensor(sizes))
    return types.SimpleNamespace(edge_index=ei.to(DEV), batch=bvec.to(DEV), num_graphs=graphs)


def device_ms(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def dense_cpu(ei, n, ks):
    """float32 dense restatement of get_rw_landing_probs for one graph (consecutive ksteps from 1)."""
    A = np.zeros((n, n), np.float32)
    np.add.at(A, (ei[0], ei[1]), 1.0)
    deg = A.sum(1)
    dinv = np.where(deg > 0, 1.0 / np.where(deg > 0, deg, 1), 0).astype(np.float32)
    P = dinv[:, None] * A
    Pk, out = P.copy(), []
    for _ in ks:
        out.append(np.diagonal(Pk).copy())
        Pk = Pk @ P
    return np.stack(out, 1)


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("device:", torch.cuda.get_device_name(0), "|", q)
    rng = np.random.default_rng(0)
    ks16 = list(range(1, 17))
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}
    shapes = {
        "pcqm4m_256x14": (molecules(rng, rng.integers(3, 26, 256)), ks16),
        "zinc_128x23": (molecules(rng, rng.integers(9, 38, 128)), list(range(1, 21))),
        "molpcba_512x26": (molecules(rng, rng.integers(5, 48, 512)), ks16),
        "cifar10_128x117_knn8": (molecules(rng, rng.integers(85, 150, 128), directed_knn=8), ks16),
        "malnet_16x1410": (malnet(rng), ks16),
    }
    for name, (b, ks) in shapes.items():
        graph_of(b).nmax
        res[f"landing_ms_{name}"] = device_ms(lambda: graphgps_b200.rw_landing_probs(b, ks), 20)

    batches = [molecules(rng, rng.integers(3, 26, 256)) for _ in range(64)]
    for b in batches:
        graph_of(b).nmax
    steps = PCQM_GRAPHS // 256 + 1
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for i in range(steps):
        graphgps_b200.rw_landing_probs(batches[i % 64], ks16)
    e.record()
    torch.cuda.synchronize()
    res["landing_s_all_pcqm4m_device"] = s.elapsed_time(e) / 1e3

    ei = batches[0].edge_index.cpu().numpy()
    ptr = np.concatenate([[0], np.cumsum(np.bincount(batches[0].batch.cpu().numpy()))])
    graphs = [(ei[:, (ei[0] >= ptr[g]) & (ei[0] < ptr[g + 1])] - ptr[g], int(ptr[g + 1] - ptr[g]))
              for g in range(len(ptr) - 1)]
    n_cpu = 2048
    t0 = time.perf_counter()
    for i in range(n_cpu):
        e_, n = graphs[i % len(graphs)]
        dense_cpu(e_, n, ks16)
    res["cpu_dense_fp32_s_per_graph"] = (time.perf_counter() - t0) / n_cpu
    res["cpu_dense_fp32_s_all_pcqm4m_scaled"] = res["cpu_dense_fp32_s_per_graph"] * PCQM_GRAPHS

    # encoder forward + backward at PCQM4Mv2 shape (d 304, dim_pe 20, K 16, expand_x False), captured vs eager torch
    b = batches[0]
    N, d, K, dpe = int(b.batch.numel()), 304, 16, 20
    pestat = graphgps_b200.rw_landing_probs(b, ks16)
    x = torch.randn(N, d - dpe, device=DEV, requires_grad=True)
    g = torch.randn(N, d, device=DEV)
    enc = graphgps_b200.KernelPENodeEncoder(d - dpe, d, K, dpe, expand_x=False).to(DEV).train()
    params = list(enc.parameters())

    def ours():
        bb = types.SimpleNamespace(x=x, pestat_RWSE=pestat)
        out = enc(bb).x
        return torch.autograd.grad(out, [x] + params, g)

    ref_bn, ref_lin = torch.nn.BatchNorm1d(K).to(DEV), torch.nn.Linear(K, dpe).to(DEV)
    ref_params = [x] + list(ref_bn.parameters()) + list(ref_lin.parameters())

    def eager():
        out = torch.cat([x, ref_lin(ref_bn(pestat))], 1)
        return torch.autograd.grad(out, ref_params, g)

    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        for _ in range(3):
            ours()
    torch.cuda.current_stream().wait_stream(st)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ours()
    res["encoder_fwd_bwd_ms_captured"] = device_ms(graph.replay, 200)
    res["encoder_fwd_bwd_ms_eager_torch_reference"] = device_ms(eager, 200)

    try:
        bvec = b.batch
        ea = torch.randn(b.edge_index.shape[1], d, device=DEV)
        y = torch.randn(b.num_graphs, 1, device=DEV)
        layers = [graphgps_b200.GPSLayer(d, "CustomGatedGCN", "Transformer", 4).to(DEV).train() for _ in range(5)]
        head = graphgps_b200.SANGraphHead(d, 1).to(DEV)
        all_params = params + [p for m in layers + [head] for p in m.parameters()]

        def train_step():
            bb = types.SimpleNamespace(x=x, pestat_RWSE=pestat, edge_index=b.edge_index, batch=bvec,
                                       num_graphs=b.num_graphs)
            h = enc(bb).x
            gb = graphgps_b200.GraphBatch(x=h, edge_index=b.edge_index, edge_attr=ea, batch=bvec,
                                          num_graphs=b.num_graphs)
            gb._gps_b200_graph = graph_of(b)
            for lay in layers:
                gb = lay(gb)
            pred, _ = head(types.SimpleNamespace(x=gb.x, batch=bvec, edge_index=b.edge_index, num_graphs=b.num_graphs,
                                                 y=y))
            return torch.autograd.grad((pred - y).abs().mean(), all_params, allow_unused=True)

        with torch.cuda.stream(st):
            for _ in range(3):
                train_step()
        torch.cuda.current_stream().wait_stream(st)
        g2 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g2):
            train_step()
        res["train_step_ms_captured"] = device_ms(g2.replay, 50)
        res["encoder_share_of_step"] = res["encoder_fwd_bwd_ms_captured"] / res["train_step_ms_captured"]
    except Exception as ex:   # reported, not hidden
        res["train_step_error"] = f"{type(ex).__name__}: {ex}"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
