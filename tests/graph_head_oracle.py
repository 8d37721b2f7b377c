"""Float64 restatement of the graph-prediction heads: SANGraphHead (pooling, L hidden Linears with the activation, the
output Linear) and GraphormerHead (LayerNorm, pooling, one Linear), over graphs given by their node offsets ptr [B+1]."""
import torch
import torch.nn.functional as F

from inductive_edge_oracle import fixture_x, hashed_x  # noqa: F401  (the fixtures' node features)


def pool(x, ptr, pooling):
    """[B, d]: mean = sum / max(count, 1), add = sum, graph_token = the first row; an empty graph gives a zero row."""
    ptr = [int(v) for v in ptr]
    rows = []
    for g in range(len(ptr) - 1):
        xs = x[ptr[g]:ptr[g + 1]]
        if xs.shape[0] == 0:
            rows.append(x.new_zeros(x.shape[1]))
        elif pooling == "graph_token":
            rows.append(xs[0])
        elif pooling == "add":
            rows.append(xs.sum(0))
        else:
            rows.append(xs.sum(0) / xs.shape[0])
    return torch.stack(rows) if rows else x.new_zeros(0, x.shape[1])


def _bf(t):
    return t.float().to(torch.bfloat16).double()


class _Bf16Linear(torch.autograd.Function):
    """y = bf(h) bf(W)^T + b with the library's bf16 backward: g_h = bf(g) bf(W), g_W = bf(g)^T bf(h), g_b = sum g."""

    @staticmethod
    def forward(ctx, h, w, b):
        ctx.save_for_backward(h, w)
        return _bf(h) @ _bf(w).t() + b

    @staticmethod
    def backward(ctx, g):
        h, w = ctx.saved_tensors
        return _bf(g) @ _bf(w), _bf(g).t() @ _bf(h), g.sum(0)


def _linear(h, w, b, bf16):
    return _Bf16Linear.apply(h, w, b) if bf16 else h @ w.t() + b


def san_head(x, ptr, pooling, act, weights, biases, bf16=False):
    """pred = W_L act(... act(W_0 pool(x) + b_0) ...) + b_L; act 'relu' or 'gelu' (exact erf).  bf16: every product
    takes bf16-rounded operands, as the library's bf16 mode does."""
    h = pool(x, ptr, pooling)
    fn = torch.relu if act == "relu" else F.gelu
    for l, (w, b) in enumerate(zip(weights, biases)):
        h = _linear(h, w, b, bf16)
        if l < len(weights) - 1:
            h = fn(h)
    return h


def graphormer_head(x, ptr, pooling, gamma, beta, w, b, bf16=False):
    """pred = pool(LayerNorm(x)) W^T + b, eps 1e-5."""
    h = F.layer_norm(x, (x.shape[1],), gamma, beta, 1e-5)
    return _linear(pool(h, ptr, pooling), w, b, bf16)


def fixture_ct(fix):
    """The fixture's cotangent of pred [B, dim_out], rebuilt from its seed and checked against its checksum."""
    ct = hashed_x(fix["num_graphs"], fix["config"]["dout"], fix["ct_seed"])
    assert float(ct.sum()) == fix["ct_sum"], "hashed_x drifted"
    return ct


def fixture_batch(fix):
    """batch.batch [N] from the fixture's graph offsets."""
    return torch.repeat_interleave(torch.arange(fix["num_graphs"]), torch.diff(fix["ptr"]))


def fixture_params(fix):
    """The fixture's parameters as float64 leaves in the head's state-dict order."""
    return {k: v.double().clone().requires_grad_(True) for k, v in fix["state"].items()}


def head_forward(fix, x, params, bf16=False):
    """The fixture's head on x with params (fixture_params)."""
    cfg = fix["config"]
    if cfg["kind"] == "san_graph":
        L = cfg["L"]
        ws = [params[f"FC_layers.{l}.weight"] for l in range(L + 1)]
        bs = [params[f"FC_layers.{l}.bias"] for l in range(L + 1)]
        return san_head(x, fix["ptr"], cfg["pooling"], cfg["act"], ws, bs, bf16)
    return graphormer_head(x, fix["ptr"], cfg["pooling"], params["ln.weight"], params["ln.bias"],
                           params["layers.0.weight"], params["layers.0.bias"], bf16)


def oracle(fix, bf16=False):
    """pred, grad_x and the parameter gradients of the fixture's head under its cotangent, in float64 (bf16: with the
    bf16-rounded product operands of the library's bf16 mode)."""
    x = fixture_x(fix).requires_grad_(True)
    params = fixture_params(fix)
    pred = head_forward(fix, x, params, bf16)
    (pred * fixture_ct(fix)).sum().backward()
    return pred.detach(), x.grad, {k: p.grad for k, p in params.items()}
