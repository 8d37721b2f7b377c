"""Float64 restatement of RWSE: the random-walk landing probabilities and KernelPENodeEncoder (model "linear"), forward
and backward.  Pinned to the reference run verbatim (tests/golden/rwse/reference_live.pt) at 1e-10, and to the
reference's float64 results stored in every fixture.

The landing probabilities walk every source of a graph at once, V <- V P with V = I, P = D_out^-1 A as a sparse
matrix, so a graph of 5 000 nodes costs n x E per step rather than the reference's dense n^3."""
import os

import numpy as np
import scipy.sparse as sp
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rwse")
BN_EPS, BN_MOMENTUM = 1e-5, 0.1


def graph_landing(edge_index, n, ksteps):
    """diag(P^k) [n, len(ksteps)] float64 of one graph; edge_index [2, E] local node ids (numpy or torch)."""
    ei = np.asarray(edge_index, dtype=np.int64).reshape(2, -1)
    src, dst = ei[0], ei[1]
    out = np.zeros((n, len(ksteps)), dtype=np.float64)
    if n == 0:
        return out
    A = sp.csr_matrix((np.ones(src.size), (src, dst)), shape=(n, n))   # duplicates add up
    deg = np.asarray(A.sum(axis=1)).ravel()
    dinv = np.where(deg > 0, 1.0 / np.where(deg > 0, deg, 1.0), 0.0)
    P = sp.diags(dinv) @ A
    PT = P.T.tocsr()
    V = np.eye(n)
    for t in range(max(ksteps) + 1):
        if t > 0:
            V = (PT @ V.T).T
        d = np.diagonal(V)
        for j, k in enumerate(ksteps):
            if k == t:
                out[:, j] = d
    return out


def landing(edge_index, ptr, ksteps):
    """The batch: every graph of node offsets ptr [B+1] separately, concatenated in node order (P is block-diagonal)."""
    ei = np.asarray(edge_index, dtype=np.int64).reshape(2, -1)
    ptr = np.asarray(ptr, dtype=np.int64)
    gid = np.searchsorted(ptr, ei[0], side="right") - 1
    parts = []
    for g in range(ptr.size - 1):
        m = gid == g
        parts.append(graph_landing(ei[:, m] - ptr[g], int(ptr[g + 1] - ptr[g]), ksteps))
    return np.concatenate(parts, 0) if parts else np.zeros((0, len(ksteps)))


def landing_batched(edge_index, N, ksteps):
    """The same computation on the whole batch as one block-diagonal graph."""
    return graph_landing(edge_index, N, ksteps)


def encoder(state, cfg, x, pestat, g_out, training, running=None):
    """KernelPENodeEncoder in float64: returns out, grad_x, {param: grad}, and the running statistics after the call
    (running: (running_mean, running_var) before it, default the state's)."""
    p = {k: v.detach().double().clone().requires_grad_(v.is_floating_point() and not k.startswith("raw_norm.run"))
         for k, v in state.items() if not k.endswith("num_batches_tracked")}
    x = x.detach().double().clone().requires_grad_(True)
    pe = pestat.detach().double()
    rm, rv = running if running is not None else (state.get("raw_norm.running_mean"), state.get("raw_norm.running_var"))
    if cfg["batch_norm"]:
        rm, rv = rm.double(), rv.double()
        if training:
            mean, var = pe.mean(0), pe.var(0, unbiased=False)
            n = pe.shape[0]
            rm = (1 - BN_MOMENTUM) * rm + BN_MOMENTUM * mean
            rv = (1 - BN_MOMENTUM) * rv + BN_MOMENTUM * var * n / (n - 1)
        else:
            mean, var = rm, rv
        z = (pe - mean) / torch.sqrt(var + BN_EPS) * p["raw_norm.weight"] + p["raw_norm.bias"]
    else:
        z = pe
    enc = z @ p["pe_encoder.weight"].T + p["pe_encoder.bias"]
    h = x @ p["linear_x.weight"].T + p["linear_x.bias"] if "linear_x.weight" in p else x
    out = torch.cat([h, enc], 1)
    out.backward(g_out.double())
    grads = {k: v.grad for k, v in p.items() if v.requires_grad}
    return out.detach(), x.grad, grads, (rm, rv)


def hashed(seed, shape, scale=1.0):
    """Seeded float32 values, reproducible on any machine (torch's CPU generator)."""
    g = torch.Generator().manual_seed(int(seed))
    return (torch.randn(*shape, generator=g) * scale).float()


def load(name):
    return torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)


def fixture_names():
    return sorted(p[:-3] for p in os.listdir(GOLDEN) if p.endswith(".pt") and p != "reference_live.pt")


def fixture_inputs(fix):
    """x, the cotangent of out and the encoder's pestat input, float32(the landing probabilities), of a fixture."""
    c = fix["config"]
    N = int(fix["ptr"][-1])
    x = hashed(fix["x_seed"], (N, c["dim_in"]))
    g = hashed(fix["x_seed"] + 1, (N, c["dim_emb"]))
    pestat = torch.from_numpy(landing(fix["edge_index"].long().numpy(), fix["ptr"].numpy(), c["ksteps"])).float()
    return x, g, pestat
