"""Cost of the PCQM-Contact link-prediction head: graphgps_b200.InductiveEdgeHead against the reference's composition
(graphgps/head/inductive_edge.py) restated in eager torch, on a contact-shaped batch.

    python tools/inductive_edge_step.py [--contacts 8] [--d 138] [--steps 20] [--rounds 5]

Batch: 256 graphs of 15..50 nodes; `--contacts` positive pairs per graph on average (uniform in [0, 2 * contacts]),
each with two negatives, as the reference's PCQM-Contact loader labels them.  The number of contacts per graph is not
part of this repository, so it is an argument and every result line states it.
  1. eval head: forward with the ranking statistics, read to the host; the library against the restated per-graph loop
     (to_data_list slices, x x^T, the two boolean masks, cat, argsort, nonzero and four .item() reads per graph);
  2. training head: forward + backward from a fixed cotangent of pred; the library recorded into a CUDA graph and
     replayed, against eager torch (Linear, gather, sum, autograd);
  3. an eval step of 5 GatedGCNLayers (library) followed by the head: the head's share with the library head and with
     the eager torch head in its place.
Each round times every arm `steps` times between two CUDA events; rounds alternate the arms and the median ms over the
rounds is printed, with the launches and host reads per batch, the GPU name and its power limit."""
import argparse
import os
import statistics
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch  # noqa: E402

import graphgps_b200  # noqa: E402
from graphgps_b200 import _lib  # noqa: E402
from graphgps_b200.batch import GraphBatch  # noqa: E402
from graphormer_step import gpu_info, timed  # noqa: E402

DEV = "cuda"


def contact_batch(d, contacts, seed=0):
    g = torch.Generator().manual_seed(seed)
    sizes = torch.randint(15, 51, (256,), generator=g).tolist()
    eli, lab, ei, off = [], [], [], 0
    for n in sizes:
        m = int(torch.randint(0, 2 * contacts + 1, (1,), generator=g))
        s, t = torch.randint(0, n, (m,), generator=g), torch.randint(0, n, (m,), generator=g)
        k1, k2 = torch.randint(0, n, (m,), generator=g), torch.randint(0, n, (m,), generator=g)
        eli.append(torch.stack([torch.cat([s, s, t]), torch.cat([t, k1, k2])]) + off)
        lab.append(torch.cat([torch.ones(m, dtype=torch.int64), torch.zeros(2 * m, dtype=torch.int64)]))
        a = torch.arange(n - 1)   # a chain for the message-passing layers, both directions
        ei.append(torch.cat([torch.stack([a, a + 1]), torch.stack([a + 1, a])], 1) + off)
        off += n
    batch = torch.repeat_interleave(torch.arange(256), torch.tensor(sizes))
    ei = torch.cat(ei, 1)
    return dict(sizes=sizes, x=torch.randn(off, d, generator=g), edge_index=ei, edge_attr=torch.randn(ei.shape[1], d,
                generator=g), eli=torch.cat(eli, 1), label=torch.cat(lab), batch=batch)


class TorchHead:
    """The reference's forward and compute_mrr restated in eager torch on the library head's parameters."""

    def __init__(self, head):
        self.lin = head.layer_post_mp.model[0].model
        self.host_reads = 0

    def __call__(self, x, eli, label, sizes, npairs, training):
        y = self.lin(x)
        v = y[eli]
        pred = torch.sum(v[0] * v[1], dim=-1)
        if training:
            return pred
        stats, n0, p0 = {}, 0, 0
        for n, p in zip(sizes, npairs):
            xg, eg, lg = y[n0:n0 + n], eli[:, p0:p0 + p] - n0, label[p0:p0 + p]
            n0, p0 = n0 + n, p0 + p
            s = xg @ xg.transpose(0, 1)
            pos = eg[:, lg == 1]
            self.host_reads += 1                         # boolean-mask indexing synchronises
            npos = pos.shape[1]
            pp = s[pos[0], pos[1]]
            if npos > 0:
                mask = torch.ones([npos, n], dtype=torch.bool, device=x.device)
                mask[torch.arange(npos, device=x.device), pos[1]] = False
                neg = s[pos[0]][mask].view(npos, -1)
                self.host_reads += 1
            else:
                neg = pp
            yp = torch.cat([pp.view(-1, 1), neg], 1) if npos > 0 else pp.view(-1, 1)
            order = torch.argsort(yp, dim=1, descending=True)
            rk = torch.nonzero(order == 0, as_tuple=False)[:, 1] + 1
            self.host_reads += 1
            for name, val in (("hits@1", (rk <= 1).float()), ("hits@3", (rk <= 3).float()),
                              ("hits@10", (rk <= 10).float()), ("mrr", 1.0 / rk.float())):
                f = float(val.mean().item())
                self.host_reads += 1
                stats.setdefault(name, []).append(0.0 if f != f else f)
        return pred, {k: sum(v) / len(v) for k, v in stats.items()}


def kernels_of(fn):
    """CUDA kernels and copies one call of fn enqueues (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--contacts", type=int, default=8)
    ap.add_argument("--d", type=int, default=138)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/inductive_edge_step.py needs a CUDA device")
    name, plim = gpu_info()
    print(f"GPU: {name}, power limit {plim}")
    d = args.d
    cb = contact_batch(d, args.contacts)
    K, P = cb["label"].numel(), int((cb["label"] == 1).sum())
    print(f"batch: 256 graphs, {cb['x'].shape[0]} nodes, d {d}, {K} labeled pairs, {P} positives "
          f"(--contacts {args.contacts})")
    torch.manual_seed(0)
    head = graphgps_b200.InductiveEdgeHead(d, 1).to(DEV)
    th = TorchHead(head)
    x = cb["x"].to(DEV)
    eli, label, bvec = cb["eli"].to(DEV), cb["label"].to(DEV), cb["batch"].to(DEV)
    sizes = cb["sizes"]
    npairs = torch.bincount(cb["batch"][cb["eli"][0]], minlength=256).tolist()
    # pairs of graph b are contiguous: the restated loop slices them in order
    data = types.SimpleNamespace(x=x, edge_index_labeled=eli, edge_label=label, batch=bvec, num_graphs=256)
    lib = _lib.load()

    def lib_eval():
        data.x = x
        return head(data)[2]

    def torch_eval():
        return th(x, eli, label, sizes, npairs, False)[1]

    head.eval()
    with torch.no_grad():
        a, b = lib_eval(), torch_eval()
        print("  eval stats: library", {k: round(v, 6) for k, v in a.items()}, "torch", {k: round(v, 6) for k, v in b.items()})
        c0 = lib.gps_launch_count()
        lib_eval()
        lib_launches = lib.gps_launch_count() - c0
        th.host_reads = 0
        torch_eval()
        torch_reads = th.host_reads
        torch_kernels = kernels_of(torch_eval)
        ev = {"library": [], "torch": []}
        for _ in range(args.rounds):
            ev["library"].append(timed(lib_eval, args.steps))
            ev["torch"].append(timed(torch_eval, max(1, args.steps // 4)))
    le, te = statistics.median(ev["library"]), statistics.median(ev["torch"])
    print(f"1. eval head (--contacts {args.contacts}): library {le:.3f} ms ({lib_launches} launches, 1 host read) | "
          f"eager torch {te:.3f} ms ({torch_kernels} kernels and copies, {torch_reads} host reads) | x{te / le:.1f}")

    # 2. training head, forward + backward
    head.train()
    ct = torch.randn(K, device=DEV)
    xg = x.clone().requires_grad_(True)
    params = [xg] + list(head.parameters())

    def lib_step():
        data.x = xg
        pred, _ = head(data)
        return torch.autograd.grad((pred * ct).sum(), params)

    def torch_step():
        pred = th(xg, eli, label, sizes, npairs, True)
        return torch.autograd.grad((pred * ct).sum(), params)

    lib_step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        lib_step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        lib_step()
    c0 = lib.gps_launch_count()
    lib_step()
    lib_tr = lib.gps_launch_count() - c0
    torch_tr = kernels_of(torch_step)
    tr = {"library": [], "torch": []}
    for _ in range(args.rounds):
        tr["library"].append(timed(graph.replay, args.steps))
        tr["torch"].append(timed(torch_step, args.steps))
    lt, tt = statistics.median(tr["library"]), statistics.median(tr["torch"])
    print(f"2. training head fwd+bwd: library captured {lt:.3f} ms ({lib_tr} launches, 0 host reads) | eager torch "
          f"{tt:.3f} ms ({torch_tr} kernels and copies, 0 host reads) | x{tt / lt:.1f}")

    # 3. eval step: 5 GatedGCNLayers + head
    layers = [graphgps_b200.GatedGCNLayer(d, d, 0.0, True).to(DEV).eval() for _ in range(5)]
    gb = GraphBatch(x=x, edge_index=cb["edge_index"].to(DEV), edge_attr=cb["edge_attr"].to(DEV), batch=bvec,
                    num_graphs=256, edge_index_labeled=eli, edge_label=label)
    e0 = gb.edge_attr

    def stack():
        gb.x, gb.edge_attr = x, e0
        for layer in layers:
            layer(gb)
        return gb

    def step_lib():
        return head.eval()(stack())[2]

    def step_torch():
        h = stack()
        return th(h.x, eli, label, sizes, npairs, False)[1]

    head.eval()
    with torch.no_grad():
        step_lib()
        step_torch()
        st = {"stack": [], "library": [], "torch": []}
        for _ in range(args.rounds):
            st["stack"].append(timed(stack, args.steps))
            st["library"].append(timed(step_lib, args.steps))
            st["torch"].append(timed(step_torch, max(1, args.steps // 4)))
    ms, ml, mt = (statistics.median(st[k]) for k in ("stack", "library", "torch"))
    print(f"3. eval step, 5 GatedGCNLayers + head (--contacts {args.contacts}): layers alone {ms:.3f} ms | with the "
          f"library head {ml:.3f} ms (head {100 * (ml - ms) / ml:.0f} %) | with the eager torch head {mt:.3f} ms "
          f"(head {100 * (mt - ms) / mt:.0f} %)")


if __name__ == "__main__":
    main()
