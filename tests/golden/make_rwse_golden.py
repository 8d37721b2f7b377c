"""Generates tests/golden/rwse/*.pt: RWSE fixtures from the REFERENCE's own graphgps/transform/posenc_stats.py
(get_rw_landing_probs) and graphgps/encoder/kernel_pos_encoder.py (KernelPENodeEncoder), run verbatim (loaded by path).
Their PyG imports are stubbed here, after PyG 2.x's source:

  * torch_geometric.utils.to_dense_adj(edge_index, max_num_nodes): [1, n, n] edge counts in the default dtype (PyG
    fills missing edge attributes with torch.ones); scatter(src, index, dim, dim_size, reduce='sum'): index_add;
    maybe_num_nodes: the given count or max + 1.  The other names the file imports are never called here;
  * torch_geometric.graphgym.config.cfg: share.dim_in and posenc_<type> (dim_pe, kernel.times, model, layers,
    raw_norm_type, pass_as_var), read at construction; torch_geometric.graphgym.register: register_node_encoder.

    python tests/golden/make_rwse_golden.py [REFERENCE_GRAPHGPS_DIR]

The reference's landing probabilities run per graph, in float64 (edge_weight float64 ones) and in float32 as it runs
by default; each fixture keeps the float64 result of its first rows (at most 40 000 entries, so every file stays under
1 MB) and the largest relative deviation of the float32 result from it over all rows.  The encoder runs in float64 on
the float32 fixture parameters, with pestat = float32(landing probabilities), x and the cotangent of out from seeds
(tests/rwse_oracle.py:hashed); a fixture keeps its parameter gradients and running statistics, and out / grad_x are
taken from tests/rwse_oracle.py, which reference_live pins to the reference at 1e-10 (reference_live keeps everything in
float64, and `init_state`, the reference encoder's state_dict right after construction from torch.manual_seed(1357)).
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from rwse_oracle import encoder as oracle_encoder, hashed, landing as oracle_landing  # noqa: E402

OUT = os.path.join(HERE, "rwse")
REF = "/root/reference/graphgps"
INIT_SEED = 1357
STORE = 40_000


def to_dense_adj(edge_index, batch=None, edge_attr=None, max_num_nodes=None):
    n = int(max_num_nodes)
    adj = torch.zeros(1, n, n)
    w = torch.ones(edge_index.shape[1]) if edge_attr is None else edge_attr
    adj[0].index_put_((edge_index[0], edge_index[1]), w.to(adj.dtype), accumulate=True)
    return adj


def scatter(src, index, dim=0, dim_size=None, reduce="sum"):
    assert reduce == "sum" and dim == 0
    return src.new_zeros(dim_size).index_add_(0, index, src)


def maybe_num_nodes(edge_index, num_nodes=None):
    return int(num_nodes) if num_nodes is not None else (int(edge_index.max()) + 1 if edge_index.numel() else 0)


CFG = types.SimpleNamespace(share=types.SimpleNamespace(dim_in=1))


def load_reference(ref=REF):
    """(get_rw_landing_probs, RWSENodeEncoder) of the reference, with the stubbed PyG they import."""
    utils = types.ModuleType("torch_geometric.utils")
    utils.to_dense_adj, utils.scatter = to_dense_adj, scatter
    for name in ("get_laplacian", "to_scipy_sparse_matrix", "to_undirected"):
        setattr(utils, name, None)
    num_nodes = types.ModuleType("torch_geometric.utils.num_nodes")
    num_nodes.maybe_num_nodes = maybe_num_nodes
    gr = types.ModuleType("graphgps.encoder.graphormer_encoder")
    gr.graphormer_pre_processing = None
    config = types.ModuleType("torch_geometric.graphgym.config")
    config.cfg = CFG
    register = types.ModuleType("torch_geometric.graphgym.register")
    register.register_node_encoder = lambda name: (lambda cls: cls)
    pyg = types.ModuleType("torch_geometric")
    gym = types.ModuleType("torch_geometric.graphgym")
    gym.register, gym.config = register, config
    mods = {"torch_geometric": pyg, "torch_geometric.utils": utils, "torch_geometric.utils.num_nodes": num_nodes,
            "torch_geometric.graphgym": gym, "torch_geometric.graphgym.config": config,
            "torch_geometric.graphgym.register": register, "graphgps.encoder.graphormer_encoder": gr}
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update(mods)
    try:
        loaded = []
        for mod, rel in (("posenc_stats", "transform/posenc_stats.py"), ("kernel_pos_encoder",
                                                                        "encoder/kernel_pos_encoder.py")):
            spec = importlib.util.spec_from_file_location(f"ref_{mod}", os.path.join(ref, rel))
            m = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(m)
            loaded.append(m)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return loaded[0].get_rw_landing_probs, loaded[1].RWSENodeEncoder


# ------------------------------------------------------------------------------------------------ graphs
def molecule(rng, n):
    """An undirected molecule-like graph: a random tree plus a few ring closures, both directions of every bond."""
    e = [(int(rng.integers(0, i)), i) for i in range(1, n)]
    for _ in range(int(rng.integers(0, 3)) if n > 4 else 0):
        a, b = rng.choice(n, 2, replace=False)
        e.append((int(a), int(b)))
    e = np.array(e, dtype=np.int64).reshape(-1, 2)
    return np.concatenate([e.T, e.T[::-1]], 1)


def knn_graph(rng, n, k=8):
    """A directed k-nearest-neighbour graph of random points in the plane (cifar10 superpixels)."""
    p = rng.random((n, 2))
    d = ((p[:, None] - p[None]) ** 2).sum(-1)
    np.fill_diagonal(d, np.inf)
    nb = np.argsort(d, 1)[:, :k]
    return np.stack([np.repeat(np.arange(n), k), nb.ravel()])


def hub_graph(rng, n, m=3):
    """A directed graph with high-in-degree hubs (MalNet call graphs): preferential attachment of each new node's m
    out-edges, and a few edges back from the hubs."""
    src, dst, deg = [], [], np.ones(n)
    for i in range(1, n):
        t = rng.choice(i, min(m, i), replace=False, p=deg[:i] / deg[:i].sum())
        src += [i] * len(t)
        dst += list(t)
        deg[t] += 1
    hubs = np.argsort(-deg)[:20]
    for h in hubs:
        back = rng.choice(n, 5, replace=False)
        src += [int(h)] * 5
        dst += list(back)
    return np.array([src, dst], dtype=np.int64)


def edge_case_graphs():
    g = [
        (1, np.zeros((2, 0), np.int64)),                                         # single isolated node
        (3, np.array([[0, 0, 1], [0, 1, 0]])),                                   # self-loop, node 2 isolated
        (4, np.array([[0, 0, 1, 2, 3, 3], [1, 1, 2, 3, 0, 0]])),                 # duplicates on a directed 4-cycle
        (5, np.array([[0, 1, 2, 3, 4], [1, 2, 3, 4, 0]])),                       # directed 5-cycle
        (6, np.array([[0, 0, 1, 2, 3, 3, 4, 5], [3, 4, 5, 3, 0, 1, 2, 0]])),     # bipartite {0,1,2} -> {3,4,5} -> ...
        (3, np.array([[0, 1], [1, 2]])),                                          # a directed path: sink node 2
        (2, np.array([[0, 1, 1], [1, 0, 1]])),                                   # self-loop with a back edge
    ]
    return g


def batch_of(graphs):
    sizes = [n for n, _ in graphs]
    ptr = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    ei = [e + ptr[i] for i, (_, e) in enumerate(graphs)]
    return ptr, np.concatenate(ei, 1) if ei else np.zeros((2, 0), np.int64)


def reference_landing(get_rw, graphs, ksteps, dtype):
    out = []
    for n, e in graphs:
        ei = torch.as_tensor(e, dtype=torch.int64).reshape(2, -1)
        old = torch.get_default_dtype()
        torch.set_default_dtype(dtype)
        try:
            out.append(get_rw(list(ksteps), ei, edge_weight=torch.ones(ei.shape[1], dtype=dtype), num_nodes=n))
        finally:
            torch.set_default_dtype(old)
    return torch.cat(out, 0).to(dtype)


def reference_encoder(RWSE, cfg, state, x, pestat, g_out, training):
    CFG.share.dim_in = cfg["dim_in"] if cfg["expand_x"] else cfg["dim_emb"] - cfg["dim_pe"]
    CFG.posenc_RWSE = types.SimpleNamespace(dim_pe=cfg["dim_pe"], kernel=types.SimpleNamespace(times=cfg["ksteps"]),
                                            model="Linear", layers=1, pass_as_var=False,
                                            raw_norm_type="BatchNorm" if cfg["batch_norm"] else "none")
    enc = RWSE(cfg["dim_emb"], expand_x=cfg["expand_x"]).double()
    if state is not None:
        enc.load_state_dict(state)
    enc.train(training)
    xx = x.double().clone().requires_grad_(True)
    b = types.SimpleNamespace(x=xx, pestat_RWSE=pestat.double())
    out = enc(b).x
    out.backward(g_out.double())
    grads = {k: p.grad for k, p in enc.named_parameters()}
    run = (enc.raw_norm.running_mean.clone(), enc.raw_norm.running_var.clone()) if cfg["batch_norm"] else None
    return enc, out.detach(), xx.grad, grads, run


def make(name, get_rw, RWSE, graphs, ksteps, dim_in, dim_emb, dim_pe, expand_x, training=True, batch_norm=True,
         seed=0, running=None):
    ptr, ei = batch_of(graphs)
    N = int(ptr[-1])
    r64 = reference_landing(get_rw, graphs, ksteps, torch.float64)
    r32 = reference_landing(get_rw, graphs, ksteps, torch.float32)
    ora = torch.from_numpy(oracle_landing(ei, ptr, ksteps))
    assert float((ora - r64).abs().max()) < 1e-12, name
    dev32 = float(((r32.double() - r64).abs() / (r64.abs() + 1e-7)).max()) if N else 0.0
    cfg = dict(ksteps=list(ksteps), dim_in=dim_in, dim_emb=dim_emb, dim_pe=dim_pe, expand_x=expand_x,
               batch_norm=batch_norm, training=training)
    torch.manual_seed(seed)
    init = {k: v for k, v in reference_encoder(RWSE, cfg, None, torch.zeros(2, dim_in if expand_x else dim_emb - dim_pe),
                                               torch.rand(2, len(ksteps)), torch.zeros(2, dim_emb), False)[0]
            .state_dict().items()}
    state = {k: (v.float() if v.is_floating_point() else v) for k, v in init.items()}
    for k in state:   # non-trivial affine parameters and running statistics
        if k == "raw_norm.weight":
            state[k] = 1.0 + 0.2 * hashed(seed + 7, state[k].shape)
        elif k == "raw_norm.bias":
            state[k] = 0.1 * hashed(seed + 8, state[k].shape)
    if running is not None:
        state["raw_norm.running_mean"], state["raw_norm.running_var"] = running
    x_seed = 1000 + seed
    x = hashed(x_seed, (N, dim_in))
    g = hashed(x_seed + 1, (N, dim_emb))
    pestat = r64.float()
    _, out, gx, grads, run = reference_encoder(RWSE, cfg, {k: v.double() if v.is_floating_point() else v
                                                          for k, v in state.items()}, x, pestat, g, training)
    o_out, o_gx, o_grads, o_run = oracle_encoder(state, cfg, x, pestat, g, training)
    assert float((o_out - out).abs().max()) < 1e-10 and float((o_gx - gx).abs().max()) < 1e-10, name
    for k, v in grads.items():
        assert float((o_grads[k] - v).abs().max()) < 1e-10, (name, k)
    rows = min(N, STORE // len(ksteps))
    fix = dict(config=cfg, ptr=torch.from_numpy(ptr), edge_index=torch.from_numpy(ei).to(torch.int32),
               rw64=r64[:rows].clone(), ref32_rel_dev=dev32, state=state, x_seed=x_seed,
               grads={k: v.clone() for k, v in grads.items()}, running=run)
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".pt")
    torch.save(fix, path)
    print(f"{name}: N={N} E={ei.shape[1]} K={len(ksteps)} ref fp32 rel dev {dev32:.2e} "
          f"{os.path.getsize(path) / 1024:.0f} KB")
    return fix


def main(ref=REF):
    get_rw, RWSE = load_reference(ref)
    rng = np.random.default_rng(2024)
    zinc = [(n, molecule(rng, n)) for n in rng.integers(9, 38, 32)]
    make("zinc_k20_pe28", get_rw, RWSE, zinc, range(1, 21), 36, 64, 28, False, seed=1)
    make("zinc_eval", get_rw, RWSE, zinc, range(1, 21), 36, 64, 28, False, training=False, seed=2,
         running=(0.3 * hashed(5, (20,)).abs(), 0.05 + hashed(6, (20,)).abs()))
    pcqm = [(int(n), molecule(rng, int(n)) if n > 1 else np.zeros((2, 0), np.int64))
            for n in np.concatenate([[1, 1, 1, 2], rng.integers(3, 30, 252)])]
    rng.shuffle(pcqm)
    make("pcqm4m_k16_pe20_d304", get_rw, RWSE, pcqm, range(1, 17), 284, 304, 20, False, seed=3)
    pcba = [(int(n), molecule(rng, int(n))) for n in rng.integers(5, 50, 512)]
    make("molpcba_k16_pe20_d384", get_rw, RWSE, pcba, range(1, 17), 364, 384, 20, False, seed=4)
    cifar = [(int(n), knn_graph(rng, int(n))) for n in rng.integers(100, 135, 8)]
    make("cifar10_knn8_expand_d52", get_rw, RWSE, cifar, range(1, 17), 5, 52, 24, True, seed=5)
    make("malnet_hubs_5000", get_rw, RWSE, [(5000, hub_graph(rng, 5000))], range(1, 17), 5, 64, 16, True, seed=6)
    ec = edge_case_graphs()
    make("edge_cases_k3183", get_rw, RWSE, ec, [3, 1, 8, 3], 3, 16, 8, True, seed=7)
    make("edge_cases_range5", get_rw, RWSE, ec, range(0, 5), 3, 16, 8, True, seed=8)
    make("edge_cases_no_norm", get_rw, RWSE, ec, range(1, 9), 8, 16, 8, False, batch_norm=False, seed=9)
    # reference_live: small, every output kept in float64, and the reference's initial state
    live = edge_case_graphs() + [(n, molecule(rng, n)) for n in (7, 12)]
    fix = make("reference_live", get_rw, RWSE, live, [2, 1, 5, 0, 7], 4, 24, 12, True, seed=10)
    ptr, ei = batch_of(live)
    cfg = fix["config"]
    N = int(ptr[-1])
    x, g = hashed(fix["x_seed"], (N, 4)), hashed(fix["x_seed"] + 1, (N, 24))
    r64 = reference_landing(get_rw, live, cfg["ksteps"], torch.float64)
    st = {k: v.double() if v.is_floating_point() else v for k, v in fix["state"].items()}
    _, out, gx, grads, run = reference_encoder(RWSE, cfg, st, x, r64.float(), g, True)
    torch.manual_seed(INIT_SEED)
    CFG.share.dim_in = 5
    CFG.posenc_RWSE.dim_pe, CFG.posenc_RWSE.kernel.times = 20, list(range(1, 17))
    init_state = RWSE(64, expand_x=True).state_dict()
    fix.update(rw64=r64, out=out, grad_x=gx, grads=grads, running=run, init_state=init_state,
               init_config=dict(dim_in=5, dim_emb=64, dim_pe=20, K=16))
    torch.save(fix, os.path.join(OUT, "reference_live.pt"))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else REF)
