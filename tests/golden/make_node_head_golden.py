"""Generates tests/golden/node_head/*.pt: node-prediction head and loss fixtures from the REFERENCE's own
graphgps/head/inductive_node.py and graphgps/loss/weighted_cross_entropy.py, run verbatim (loaded by path).  The
reference pins PyG 2.2; its imports are stubbed here after PyG 2.2's torch_geometric/graphgym/models/{layer,head}.py
and graphgym/loss.py:

  * cfg: cfg.gnn.layers_post_mp, cfg.gnn.dim_inner and cfg.model.loss_fun, read where the reference reads them;
  * register: register_head / register_loss decorators that record into head_dict / loss_dict;
  * new_layer_config(dim_in, dim_out, L, has_act, has_bias, cfg) and MLP: for L > 1, GeneralMultiLayer('linear') of
    L - 1 GeneralLayers built from LayerConfig's defaults (Linear with bias, ReLU, then F.normalize(p=2, dim=1); no
    BatchNorm, no dropout, whatever cfg.gnn says), then Linear(dim_inner -> dim_out); for L = 1 one Linear.  Each
    Linear keeps its torch Linear in `.model`; the MLP writes batch.x;
  * GNNNodeHead (`node`): the MLP, then (batch.x[batch[f'{split}_mask']], batch.y[...]);
  * compute_loss: squeezes a trailing size-1 dim off pred and true, tries every loss_dict entry, then the built-in
    multiclass cross_entropy nll_loss(log_softmax(pred), true).

The reference's weighted loss computes its class weights in float32 (as it does on the device); torch refuses a float32
weight next to a float64 input, so the two loss calls it makes (F.nll_loss, F.binary_cross_entropy_with_logits) get
their weight and target cast to the input's dtype, and the head and loss run in float64 on the float32 parameters.

    python tests/golden/make_node_head_golden.py [REFERENCE_GRAPHGPS_DIR]

Each fixture holds the config, x as tests/inductive_edge_oracle.py's hashed_x seed with an exact checksum (and the rows
it zeroes), the labels, the split masks (node head), the state_dict (float32), the loss and pred_score, and the
gradients of every parameter (and of x where they stay small) under loss.backward() and under a hashed_x cotangent on
pred_score.  pred_score and grad_x are stored where they stay small and otherwise taken from tests/node_head_oracle.py,
which is pinned to the reference: every fixture stays under 1 MB.  reference_live keeps float64 for two small cases,
pins the oracle at 1e-10, and holds the reference heads' initial state_dicts from torch.manual_seed(INIT_SEED).
"""
import importlib.util
import os
import sys
import types
import zlib

import torch
import torch.nn as nn
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from inductive_edge_oracle import hashed_x  # noqa: E402
OUT = os.path.join(HERE, "node_head")
REF = "/root/reference/graphgps"
INIT_SEED = 2468
KEEP_MAX = 60_000   # elements of pred_score / grad_x a fixture stores

CFG = types.SimpleNamespace(gnn=types.SimpleNamespace(layers_post_mp=1, dim_inner=None),
                            model=types.SimpleNamespace(loss_fun="weighted_cross_entropy"))


# ------------------------------------------------------------------------------------------------ PyG 2.2 stubs
class LayerConfig(types.SimpleNamespace):
    def __init__(self, **kw):
        base = dict(has_batchnorm=False, bn_eps=1e-5, bn_mom=0.1, mem_inplace=False, dim_in=-1, dim_out=-1,
                    edge_dim=-1, dim_inner=None, num_layers=2, has_bias=True, has_l2norm=True, dropout=0.0,
                    has_act=True, final_act=True, act="relu", keep_edge=0.5)
        base.update(kw)
        super().__init__(**base)


def new_layer_config(dim_in, dim_out, num_layers, has_act, has_bias, cfg):
    return LayerConfig(dim_in=dim_in, dim_out=dim_out, num_layers=num_layers, has_act=has_act, has_bias=has_bias,
                       dim_inner=cfg.gnn.dim_inner)


class Linear(nn.Module):
    def __init__(self, lc):
        super().__init__()
        self.model = nn.Linear(lc.dim_in, lc.dim_out, bias=lc.has_bias)

    def forward(self, batch):
        if isinstance(batch, torch.Tensor):
            return self.model(batch)
        batch.x = self.model(batch.x)
        return batch


class GeneralLayer(nn.Module):
    def __init__(self, lc):
        super().__init__()
        self.has_l2norm = lc.has_l2norm
        lc.has_bias = not lc.has_batchnorm
        self.layer = Linear(lc)
        self.post_layer = nn.Sequential(*([nn.ReLU()] if lc.has_act else []))

    def forward(self, batch):
        batch = self.layer(batch)
        batch.x = self.post_layer(batch.x)
        if self.has_l2norm:
            batch.x = F.normalize(batch.x, p=2, dim=1)
        return batch


class GeneralMultiLayer(nn.Module):
    def __init__(self, lc):
        super().__init__()
        dim_inner = lc.dim_out if lc.dim_inner is None else lc.dim_inner
        for i in range(lc.num_layers):
            d_in = lc.dim_in if i == 0 else dim_inner
            d_out = lc.dim_out if i == lc.num_layers - 1 else dim_inner
            has_act = lc.final_act if i == lc.num_layers - 1 else True
            sub = LayerConfig(**{**vars(lc), "dim_in": d_in, "dim_out": d_out, "has_act": has_act})
            self.add_module(f"Layer_{i}", GeneralLayer(sub))

    def forward(self, batch):
        for layer in self.children():
            batch = layer(batch)
        return batch


class MLP(nn.Module):
    def __init__(self, lc):
        super().__init__()
        dim_inner = lc.dim_in if lc.dim_inner is None else lc.dim_inner
        lc.has_bias = True
        layers = []
        if lc.num_layers > 1:
            layers.append(GeneralMultiLayer(LayerConfig(num_layers=lc.num_layers - 1, dim_in=lc.dim_in,
                                                        dim_out=dim_inner, dim_inner=dim_inner, final_act=True)))
            layers.append(Linear(LayerConfig(**{**vars(lc), "dim_in": dim_inner})))
        else:
            layers.append(Linear(lc))
        self.model = nn.Sequential(*layers)

    def forward(self, batch):
        for layer in self.model:
            batch = layer(batch)
        return batch


class GNNNodeHead(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.layer_post_mp = MLP(new_layer_config(dim_in, dim_out, CFG.gnn.layers_post_mp, has_act=False,
                                                  has_bias=True, cfg=CFG))

    def forward(self, batch):
        batch = self.layer_post_mp(batch)
        mask = f"{batch.split}_mask"
        return batch.x[batch[mask]], batch.y[batch[mask]]


class Batch(types.SimpleNamespace):
    def __getitem__(self, k):
        return getattr(self, k)


def _cast_to(t, like):
    return None if t is None else t.to(like.dtype)


F_SHIM = types.SimpleNamespace(
    log_softmax=F.log_softmax,
    nll_loss=lambda input, target, weight=None: F.nll_loss(input, target, weight=_cast_to(weight, input)),
    binary_cross_entropy_with_logits=lambda input, target, weight=None: F.binary_cross_entropy_with_logits(
        input, target.to(input.dtype), weight=_cast_to(weight, input)))


def load_reference(ref=REF):
    """The reference's GNNInductiveNodeHead, its weighted_cross_entropy and the stubbed compute_loss."""
    register = types.ModuleType("torch_geometric.graphgym.register")
    register.head_dict, register.loss_dict = {}, {}

    def deco(d):
        return lambda name: (lambda obj: d.__setitem__(name, obj) or obj)

    register.register_head, register.register_loss = deco(register.head_dict), deco(register.loss_dict)
    mods = {"torch_geometric": {}, "torch_geometric.graphgym": {},
            "torch_geometric.graphgym.config": {"cfg": CFG},
            "torch_geometric.graphgym.models": {},
            "torch_geometric.graphgym.models.layer": {"new_layer_config": new_layer_config, "MLP": MLP}}
    for name, attrs in mods.items():
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        m.__path__ = []
        sys.modules[name] = m
    sys.modules["torch_geometric.graphgym.register"] = register
    out = {}
    for rel in ("head/inductive_node.py", "loss/weighted_cross_entropy.py"):
        spec = importlib.util.spec_from_file_location("graphgps." + rel[:-3].replace("/", "."), os.path.join(ref, rel))
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        out[rel] = m
    out["loss/weighted_cross_entropy.py"].F = F_SHIM

    def compute_loss(pred, true):
        pred = pred.squeeze(-1) if pred.ndim > 1 else pred
        true = true.squeeze(-1) if true.ndim > 1 else true
        for func in register.loss_dict.values():
            value = func(pred, true)
            if value is not None:
                return value
        assert CFG.model.loss_fun == "cross_entropy" and pred.ndim > 1 and true.ndim == 1
        pred = F.log_softmax(pred, dim=-1)
        return F.nll_loss(pred, true), pred

    return register.head_dict["inductive_node"], GNNNodeHead, compute_loss


def build_head(classes, head, d, dout, L, dim_inner):
    CFG.gnn.layers_post_mp, CFG.gnn.dim_inner = L, dim_inner
    inductive, node, _ = classes
    return inductive(d, dout) if head == "inductive_node" else node(d, dout)


def graph_sizes(B, lo, hi, seed):
    return torch.randint(lo, hi + 1, (B,), generator=torch.Generator().manual_seed(seed)).tolist()


def run_case(classes, name, head, d, dout, L, dim_inner, loss_fun, N, labels_fn, split=None, masks_fn=None,
             zero_rows=(), neg_bias=False, dtype=torch.float32):
    seed = zlib.crc32(name.encode()) % (2 ** 31)
    torch.manual_seed(seed)
    model = build_head(classes, head, d, dout, L, dim_inner)
    if neg_bias:   # every unit of the first hidden layer is negative on a zero row: ReLU zeroes it entirely
        with torch.no_grad():
            model.layer_post_mp.model[0].Layer_0.layer.model.bias.abs_().neg_().sub_(0.05)
    if dtype != torch.float64:
        model.float()
    model.double()
    x = hashed_x(N, d, seed)
    x[list(zero_rows)] = 0.0
    g = torch.Generator().manual_seed(seed + 2)
    labels = labels_fn(N, g)
    masks = masks_fn(N, g) if masks_fn else None
    fix = {"config": dict(name=name, head=head, d=d, dout=dout, L=L, dim_inner=dim_inner, loss=loss_fun, split=split,
                          zero_rows=list(zero_rows)),
           "x_seed": seed, "x_shape": (N, d), "x_sum": float(x.sum()), "x_sumsq": float((x * x).sum()),
           "labels": labels.to(torch.int16), "state": {k: v.detach().to(dtype).clone() for k, v in
                                                        model.state_dict().items()}}
    if masks is not None:
        fix["masks"] = masks
    CFG.model.loss_fun = loss_fun
    keep = (lambda t: t.detach().clone()) if dtype == torch.float64 else (lambda t: t.detach().float())
    for mode in ("loss", "ct"):
        xr = x.clone().requires_grad_(True)
        batch = Batch(x=xr, y=labels.clone(), split=split, **({f"{k}_mask": v for k, v in (masks or {}).items()}))
        pred, true = model(batch)
        loss, score = classes[2](pred, true)
        M = pred.shape[0]
        fix["num_pred"] = M
        if mode == "loss":
            fix["loss"] = float(loss.detach())
            if score.numel() <= KEEP_MAX or dtype == torch.float64:
                fix["pred_score"] = keep(score)
            fix["pred_score_sum"] = float(score.sum())
            out = loss
        else:
            ct = hashed_x(M, dout, seed + 1)
            fix.update(ct_seed=seed + 1, ct_sum=float(ct.sum()))
            out = (score * (ct.flatten() if dout == 1 else ct)).sum()
        model.zero_grad(set_to_none=True)
        out.backward()
        sfx = "" if mode == "loss" else "_ct"
        fix["grads" + sfx] = {k: keep(p.grad) if p.grad is not None else torch.zeros_like(p, dtype=dtype)
                              for k, p in model.named_parameters()}
        if N * d <= KEEP_MAX or dtype == torch.float64:
            fix["grad_x" + sfx] = keep(xr.grad) if xr.grad is not None else torch.zeros(N, d, dtype=dtype)
    return fix


def uniform_labels(C, present=None):
    def fn(N, g):
        lab = torch.randint(0, C, (N,), generator=g)
        if present is not None:
            pool = torch.tensor(present)
            lab = pool[torch.randint(0, len(present), (N,), generator=g)]
        return lab
    return fn


def split_masks(fracs=(0.6, 0.2, 0.2), empty=None):
    def fn(N, g):
        perm = torch.randperm(N, generator=g)
        n0, n1 = int(fracs[0] * N), int((fracs[0] + fracs[1]) * N)
        out = {}
        for name, idx in (("train", perm[:n0]), ("val", perm[n0:n1]), ("test", perm[n1:])):
            m = torch.zeros(N, dtype=torch.bool)
            if name != empty:
                m[idx] = True
            out[name] = m
        return out
    return fn


W = "weighted_cross_entropy"
CE = "cross_entropy"
CASES = [
    # name, head, d, C, L, dim_inner, loss, N, labels, kwargs
    ("pattern_d64_L3", "inductive_node", 64, 2, 3, None, W, sum(graph_sizes(32, 100, 136, 1)), uniform_labels(2), {}),
    ("cluster_d48_L3", "inductive_node", 48, 6, 3, None, W, sum(graph_sizes(16, 100, 136, 2)), uniform_labels(6), {}),
    ("voc_d96_L3", "inductive_node", 96, 21, 3, None, W, sum(graph_sizes(32, 440, 520, 3)), uniform_labels(21), {}),
    ("voc_gatedgcn_d108_L3", "inductive_node", 108, 21, 3, None, W, sum(graph_sizes(32, 440, 520, 4)),
     uniform_labels(21), {}),
    ("coco_d96_L3", "inductive_node", 96, 81, 3, None, W, sum(graph_sizes(16, 440, 520, 5)), uniform_labels(81), {}),
    ("odd_d37_inner40_L2", "inductive_node", 37, 3, 2, 40, W, 301, uniform_labels(3), {}),
    ("absent_class_C5", "inductive_node", 32, 5, 3, None, W, 200, uniform_labels(5, [0, 1, 3]), {}),
    ("one_class_C4", "inductive_node", 32, 4, 3, None, W, 150, uniform_labels(4, [2]), {}),
    ("relu_zero_rows", "inductive_node", 24, 3, 3, None, W, 120, uniform_labels(3),
     dict(zero_rows=[0, 7, 8, 50, 119], neg_bias=True)),
    ("binary_d64_L3", "inductive_node", 64, 1, 3, None, W, 900, uniform_labels(2), {}),
    ("actor_d64_C5_train", "node", 64, 5, 1, None, CE, 7600, uniform_labels(5),
     dict(split="train", masks_fn=split_masks())),
    ("webkb_d64_C5_val", "node", 64, 5, 1, None, CE, 183, uniform_labels(5),
     dict(split="val", masks_fn=split_masks((0.48, 0.32, 0.2)))),
    ("empty_mask_test", "node", 64, 5, 1, None, CE, 183, uniform_labels(5),
     dict(split="test", masks_fn=split_masks(empty="test"))),
]
LIVE = [
    ("live_inductive", "inductive_node", 20, 4, 3, 24, W, 90, uniform_labels(4),
     dict(zero_rows=[3, 40], neg_bias=True)),
    ("live_node", "node", 12, 3, 2, 16, CE, 70, uniform_labels(3), dict(split="train", masks_fn=split_masks())),
    ("live_binary", "inductive_node", 16, 1, 2, None, W, 50, uniform_labels(2), {}),
]


def main():
    classes = load_reference(sys.argv[1] if len(sys.argv) > 1 else REF)
    os.makedirs(OUT, exist_ok=True)
    for name, head, d, C, L, di, loss, N, lab, kw in CASES:
        fix = run_case(classes, name, head, d, C, L, di, loss, N, lab, **kw)
        p = os.path.join(OUT, name + ".pt")
        torch.save(fix, p)
        print(name, "N", N, "M", fix["num_pred"], "loss", fix["loss"], "grad_x" in fix, "pred_score" in fix,
              f"{os.path.getsize(p) / 1e3:.0f} kB")
    live = {"cases": {}, "init_seed": INIT_SEED}
    for name, head, d, C, L, di, loss, N, lab, kw in LIVE:
        live["cases"][name] = run_case(classes, name, head, d, C, L, di, loss, N, lab, dtype=torch.float64, **kw)
    for key, args in (("init_state_L3", ("inductive_node", 64, 2, 3, None)), ("init_state_L1", ("node", 64, 5, 1, None)),
                      ("init_state_L2_inner", ("inductive_node", 37, 3, 2, 40))):
        torch.manual_seed(INIT_SEED)
        live[key] = {k: v.clone() for k, v in build_head(classes, *args).state_dict().items()}
    p = os.path.join(OUT, "reference_live.pt")
    torch.save(live, p)
    print("reference_live", f"{os.path.getsize(p) / 1e3:.0f} kB")


if __name__ == "__main__":
    main()
