"""Float64 restatement of the SAN2 layer (graphgps/layer/san2_layer.py with full_graph=True, batch_norm=True,
layer_norm=False, residual=True, use_bias=False).

The restatement follows the reference line by line:
  * MultiHeadAttention2Layer.forward (san2_layer.py:111-142): Q_h, K_h, V_h, Q_2h, K_2h from x, E from edge_attr,
    E_2 = E_2(fake_edge_emb.weight[0]), all without bias, viewed as [*, H, hd];
  * propagate_attention (san2_layer.py:65-108): per real edge j -> i the score t = sum(K_j Q_i / sqrt(hd) E), per fake
    pair u = sum(K2_j Q2_i / sqrt(hd) E_2); pyg_softmax (san2_layer.py:11-33) over each destination's real edges and,
    separately, over its fake pairs: exp(s - max) / (sum exp(s - max) + 1e-16), the max of an empty segment 0 as
    torch_scatter's scatter_max gives it; then h = (sum alpha V + gamma sum beta V) / (gamma + 1);
  * the fake pairs are negate_edge_index's complement (tests/san_oracle.py fake_pairs);
  * SAN2Layer.forward (san2_layer.py:191-232): the trunk of tests/san_oracle.py's san_forward.
gamma is read from the state (`attention.gamma`), so a float64 leaf there receives its gradient.  Dropout masks (the
library's, 0 or 1/(1-p)) can be injected at both sites.
"""
import math

import torch

from san_oracle import _bn, fake_pairs, san_batch  # noqa: F401  (fake_pairs, san_batch: the SAN batch helpers)


def pyg_softmax(src, index, num_nodes):
    """src [M, H] grouped by index [M] over num_nodes destinations: exp(src - max) / (sum + 1e-16), per group."""
    H = src.shape[1]
    idx = index.view(-1, 1).expand(-1, H)
    mx = torch.zeros(num_nodes, H, dtype=src.dtype, device=src.device)
    mx = mx.scatter_reduce(0, idx, src, reduce="amax", include_self=False)
    out = (src - mx[index]).exp()
    den = torch.zeros(num_nodes, H, dtype=src.dtype, device=src.device).index_add(0, index, out)
    return out / (den[index] + 1e-16)


def san2_parts(Q, K, V, Q2, K2, E, E2, edge_index, fake_index, H):
    """(R, F) [N, H, hd]: the real-edge and fake-pair softmax outputs sum alpha V and sum beta V."""
    N, d = Q.shape
    hd = d // H
    v = lambda t: t.reshape(-1, H, hd)  # noqa: E731
    src, dst = edge_index[0], edge_index[1]
    t = (v(K)[src] * v(Q)[dst] / math.sqrt(hd) * v(E)).sum(-1)
    fs, fd = fake_index[0], fake_index[1]
    u = (v(K2)[fs] * v(Q2)[fd] / math.sqrt(hd) * E2.reshape(1, H, hd)).sum(-1)
    alpha = pyg_softmax(t, dst, N)
    beta = pyg_softmax(u, fd, N)
    R = torch.zeros(N, H, hd, dtype=Q.dtype, device=Q.device).index_add(0, dst, v(V)[src] * alpha[..., None])
    F = torch.zeros(N, H, hd, dtype=Q.dtype, device=Q.device).index_add(0, fd, v(V)[fs] * beta[..., None])
    return R, F


def san2_attention(Q, K, V, Q2, K2, E, E2, edge_index, fake_index, H, gamma):
    """h_out [N, d] of propagate_attention + forward (san2_layer.py:65-142); Q..K2 [N, d], E [E, d], E2 [d]; gamma a
    float or a 0-d tensor."""
    R, F = san2_parts(Q, K, V, Q2, K2, E, E2, edge_index, fake_index, H)
    return ((R + gamma * F) / (gamma + 1)).reshape(Q.shape)


def scores(Q, K, Q2, K2, E, E2, edge_index, fake_index, H):
    """The real and fake pre-softmax scores t [E, H], u [F, H]."""
    hd = Q.shape[1] // H
    v = lambda t: t.reshape(-1, H, hd)  # noqa: E731
    t = (v(K)[edge_index[0]] * v(Q)[edge_index[1]] * v(E)).sum(-1) / math.sqrt(hd)
    u = (v(K2)[fake_index[0]] * v(Q2)[fake_index[1]] * E2.reshape(1, H, hd)).sum(-1) / math.sqrt(hd)
    return t, u


def san2_forward(state, x, edge_attr, edge_index, fake_index, H, training=True, masks=None, prefix="", taps=None):
    """One SAN2Layer in float64.  state: the layer's parameters (and, for eval, running statistics) by state_dict name,
    `attention.gamma` included; masks: optional (m_attn [N, d], m_ffn [N, 2d]) dropout scales; taps: optional dict that
    receives R and F [N, d] and the attention output "attn" [N, d] (its .grad retained after a backward)."""
    s = lambda n: state[prefix + n]  # noqa: E731
    lin = lambda t, n, bias=True: t @ s(n + ".weight").t() + (s(n + ".bias") if bias else 0)  # noqa: E731
    emb = s("attention.fake_edge_emb.weight")[0]
    E2 = s("attention.E_2.weight") @ emb
    R, F = san2_parts(lin(x, "attention.Q", False), lin(x, "attention.K", False), lin(x, "attention.V", False),
                      lin(x, "attention.Q_2", False), lin(x, "attention.K_2", False),
                      lin(edge_attr, "attention.E", False), E2, edge_index, fake_index, H)
    gamma = s("attention.gamma")
    h = ((R + gamma * F) / (gamma + 1)).reshape(x.shape)
    if taps is not None:
        h.retain_grad()
        taps.update(R=R.reshape(x.shape), F=F.reshape(x.shape), attn=h)
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
