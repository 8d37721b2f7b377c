"""Float64 restatement of the node-prediction heads and their losses: GraphGym's MLP (hidden layers Linear -> ReLU ->
row L2 normalisation, then a Linear), the row selection of GNNNodeHead, weighted_cross_entropy with the float32 class
weights w_c = (V - count_c) / V * [count_c > 0], and the multiclass cross_entropy."""
import torch
import torch.nn.functional as F

from graph_head_oracle import _Bf16Linear
from inductive_edge_oracle import hashed_x


def mlp(x, weights, biases, bf16=False):
    """y = W_{L-1} n(relu(... n(relu(W_0 x + b_0)) ...)) + b_{L-1}, n(h) = h / max(||h||, 1e-12) per row.  bf16: every
    product takes bf16-rounded operands, as the library's bf16 mode does."""
    h = x
    for l, (w, b) in enumerate(zip(weights, biases)):
        h = _Bf16Linear.apply(h, w, b) if bf16 else h @ w.t() + b
        if l < len(weights) - 1:
            h = torch.relu(h)
            h = h / h.norm(dim=1, keepdim=True).clamp_min(1e-12)
    return h


def class_weights(true, K):
    """The reference's float32 weights over K classes, as float64."""
    V = true.shape[0]
    counts = torch.bincount(true, minlength=K)[:K]
    w = (V - counts).float() / V
    return (w * (counts > 0).float()).double()


def weighted_cross_entropy(pred, true):
    """(loss, pred_score): multiclass nll of log_softmax with weights w, or binary BCE-with-logits weighted by w[true]."""
    if pred.dim() > 1:
        w = class_weights(true, pred.shape[1])
        lp = F.log_softmax(pred, dim=-1)
        return F.nll_loss(lp, true, weight=w), lp
    w = class_weights(true, 2)
    return F.binary_cross_entropy_with_logits(pred, true.double(), weight=w[true]), torch.sigmoid(pred)


def cross_entropy(pred, true):
    lp = F.log_softmax(pred, dim=-1)
    return F.nll_loss(lp, true), lp


LOSSES = {"weighted_cross_entropy": weighted_cross_entropy, "cross_entropy": cross_entropy}


# ------------------------------------------------------------------------------------------------ fixtures
def fixture_x(fix):
    """The fixture's node features, rebuilt from its seed, checked against its exact checksum, with its zero rows."""
    n, d = fix["x_shape"]
    x = hashed_x(n, d, fix["x_seed"])
    x[fix["config"].get("zero_rows", [])] = 0.0
    assert float(x.sum()) == fix["x_sum"] and float((x * x).sum()) == fix["x_sumsq"], "hashed_x drifted"
    return x


def fixture_labels(fix):
    return fix["labels"].long()


def fixture_rows(fix):
    """The selected rows (node head) or None."""
    if fix["config"]["head"] != "node":
        return None
    return fix["masks"][fix["config"]["split"]].nonzero().flatten()


def fixture_ct(fix):
    """The cotangent of pred_score [M, C] ([M] for a binary head)."""
    M = int(fix["num_pred"])
    C = fix["config"]["dout"]
    ct = hashed_x(M, C, fix["ct_seed"])
    assert float(ct.sum()) == fix["ct_sum"], "hashed_x drifted"
    return ct.flatten() if C == 1 else ct


def param_names(L):
    if L == 1:
        return ["layer_post_mp.model.0.model"]
    return [f"layer_post_mp.model.0.Layer_{i}.layer.model" for i in range(L - 1)] + ["layer_post_mp.model.1.model"]


def fixture_params(fix):
    return {k: v.double().clone().requires_grad_(True) for k, v in fix["state"].items()}


def head_loss(fix, x, params, bf16=False):
    """(pred, label, loss, pred_score) of the fixture's head and loss on x."""
    c = fix["config"]
    names = param_names(c["L"])
    y = mlp(x, [params[n + ".weight"] for n in names], [params[n + ".bias"] for n in names], bf16)
    true = fixture_labels(fix)
    rows = fixture_rows(fix)
    if rows is not None:
        y, true = y[rows], true[rows]
    pred = y.squeeze(-1) if y.shape[1] == 1 else y
    loss, score = LOSSES[c["loss"]](pred, true)
    return pred, true, loss, score


def ambiguous_rows(fix, rel=2.0 ** -16):
    """bool [N]: rows with a hidden pre-activation within rel of its term scale sum |x_k w_k| + |b| of zero.  The
    library's fp32 mode runs each product as three bf16 MMAs on hi / lo planes (about 2^-16 relative), so such a
    ReLU can fall the other way than in float64 and move that row's gradients."""
    c = fix["config"]
    names = param_names(c["L"])
    x = fixture_x(fix)
    out = torch.zeros(x.shape[0], dtype=torch.bool)
    h = x
    for n in names[:-1]:
        w, b = fix["state"][n + ".weight"].double(), fix["state"][n + ".bias"].double()
        pre = h @ w.t() + b
        out |= (pre.abs() <= rel * (h.abs() @ w.abs().t() + b.abs())).any(1)
        h = torch.relu(pre)
        h = h / h.norm(dim=1, keepdim=True).clamp_min(1e-12)
    return out


def oracle(fix, mode="loss", bf16=False):
    """loss, pred_score, grad_x and the parameter gradients in float64, under loss.backward() (mode 'loss') or under the
    fixture's cotangent on pred_score (mode 'ct')."""
    x = fixture_x(fix).requires_grad_(True)
    params = fixture_params(fix)
    _, _, loss, score = head_loss(fix, x, params, bf16)
    out = loss if mode == "loss" else (score * fixture_ct(fix)).sum()
    grads = torch.autograd.grad(out, [x] + list(params.values()), allow_unused=True)
    gx = grads[0] if grads[0] is not None else torch.zeros_like(x)
    gp = {k: (g if g is not None else torch.zeros_like(p)) for (k, p), g in zip(params.items(), grads[1:])}
    return loss.detach(), score.detach(), gx, gp
