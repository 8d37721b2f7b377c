"""Shared helpers for the parity tests."""
import glob
import os

import torch

from graphgps_b200.batch import GraphBatch

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = "cuda:0"


def golden_names():
    return sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(GOLDEN_DIR, "*.pt")))


def load_golden(name):
    return torch.load(os.path.join(GOLDEN_DIR, name + ".pt"), weights_only=False)


def golden_batch(fix, device="cpu", dtype=torch.float32):
    return GraphBatch(x=fix["x"].to(device=device, dtype=dtype), edge_index=fix["edge_index"].to(device),
                      edge_attr=fix["edge_attr"].to(device=device, dtype=dtype), batch=fix["batch"].to(device),
                      num_graphs=fix["num_graphs"])


def run_layer(layer, batch, fix, backward=True):
    """forward (+backward with the fixture's cotangents). Returns dict of outputs/grads on CPU."""
    cfg = fix["config"]
    batch.x.requires_grad_(backward)
    batch.edge_attr.requires_grad_(backward)
    x_in, e_in = batch.x, batch.edge_attr
    out = layer(batch)
    res = {"out_x": out.x.detach().cpu()}
    dev, dt = out.x.device, out.x.dtype
    loss = (out.x * fix["ct_x"].to(device=dev, dtype=dt)).sum()
    if cfg["local"] == "CustomGatedGCN":
        res["out_e"] = out.edge_attr.detach().cpu()
        loss = loss + (out.edge_attr * fix["ct_e"].to(device=dev, dtype=dt)).sum()
    if backward:
        loss.backward()
        res["grad_x"] = x_in.grad.detach().cpu()
        if e_in.grad is not None:
            res["grad_e"] = e_in.grad.detach().cpu()
        res["grad_params"] = {n: p.grad.detach().cpu() for n, p in layer.named_parameters() if p.grad is not None}
    res["state_after"] = {k: v.detach().cpu() for k, v in layer.state_dict().items()
                          if "running" in k or "num_batches" in k}
    return res


def pin_dropout_counter(device, value):
    """Sets the library's device-resident dropout counter, so the next layer call draws the masks of offset
    value + 4096."""
    from graphgps_b200 import _call
    _call.dropout_counter(torch.device(device)).fill_(value)


def rel_err(a, b):
    """max |a-b| / max(1, max|b|): absolute on O(1) (BatchNorm-normalised) data, relative on large."""
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / max(1.0, float(b.abs().max())))


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / max(float(b.norm()), 1e-30))


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _nan(*shape, dtype=torch.float32):
    """A device tensor that starts as NaN, so an element a kernel leaves unwritten fails the check that reads it."""
    return torch.full(shape, float("nan"), device=DEV, dtype=dtype)


def _elem_check(worst, name, got, ref, bound):
    """|got - ref| <= bound elementwise (bounds from the float64 restatements: actual reduction lengths, per element).
    Records the worst error as a fraction of its bound in worst[name]."""
    got, ref, bound = got.double().cpu(), ref.double().cpu(), bound.double().cpu()
    assert got.shape == ref.shape == bound.shape, (name, got.shape, ref.shape, bound.shape)
    assert not torch.isnan(got).any(), f"{name}: NaN left in the output"
    err = (got - ref).abs()
    frac = float((err / (bound + 1e-300)).max()) if got.numel() else 0.0
    worst[name] = max(worst.get(name, 0.0), frac)
    assert bool((err <= bound).all()), f"{name}: error {frac:.3g} x its bound"
    return frac


def compare(res, fix, tol, what="", grad_l2_tol=None, zero=None, zero_tol=None):
    """Forward outputs (out_x, out_e) and BatchNorm running statistics: max|a-b| / max(1, max|b|) <= tol; integer
    state (num_batches_tracked) exactly.

    Gradients (grad_x, grad_e, grad_attn_bias, every grad_params entry): the same max-abs criterion, OR (when
    grad_l2_tol is given) relative L2 error <= grad_l2_tol, one bound for all keys or a dict {key: bound} whose missing
    keys fall back to its "default" entry.  The second criterion exists because the derivative of a ReLU network is
    discontinuous: a pre-activation within rounding distance of 0 flips its mask between two correct arithmetics (the
    reference's own fp32 vs fp64 runs differ by 1.8e-2 max-abs on ff_linear1.weight at the code2 shape for exactly this
    reason), which moves a handful of gradient entries by O(|g|) while leaving the L2 error at the rounding level.  A
    real defect (wrong operand, missing term) shows up as an L2 error of order 1.

    zero(key, expected) marks gradients that are zero in exact arithmetic, which no relative measure can bound: such a
    gradient that fails the criteria above passes when max|a| <= zero_tol.

    Every gradient and state entry of the fixture must be present in res.
    """
    errs, bad = {}, {}

    def check_fwd(key, a, b):
        e = rel_err(a, b)
        errs[key] = e
        errs["raw:" + key] = float((a.double() - b.double()).abs().max())   # unscaled max-abs beside the scaled one
        if not e <= tol:
            bad[key] = e

    def check_grad(key, a, b):
        e = rel_err(a, b)
        errs[key] = e
        errs["raw:" + key] = float((a.double() - b.double()).abs().max())
        if e <= tol:
            return
        if zero is not None and zero(key, b) and float(a.abs().max()) <= zero_tol:
            return
        if grad_l2_tol is not None:
            bound = grad_l2_tol.get(key, grad_l2_tol["default"]) if isinstance(grad_l2_tol, dict) else grad_l2_tol
            l2 = rel_l2(a, b)
            errs[key + "(l2)"] = l2
            if l2 <= bound:
                return
            bad[key] = (e, l2, bound)
        else:
            bad[key] = e

    for k in ("out_x", "out_e"):
        if k in fix and k in res:
            check_fwd(k, res[k], fix[k])
    for k in ("grad_x", "grad_e", "grad_attn_bias"):
        if k in fix:
            if k in res:
                check_grad(k, res[k], fix[k])
            else:
                bad[k] = "missing"
    for n, g in fix.get("grad_params", {}).items():
        if n in res.get("grad_params", {}):
            check_grad("grad:" + n, res["grad_params"][n], g)
        else:
            bad["grad:" + n] = "missing"
    for n, v in fix.get("state_after", {}).items():
        if n not in res["state_after"]:
            bad["state:" + n] = "missing"
        elif v.is_floating_point():
            check_fwd("state:" + n, res["state_after"][n], v)
        elif not torch.equal(res["state_after"][n], v):
            bad["state:" + n] = "differs"
    assert not bad, f"{what} tolerance {tol} (grad L2 {grad_l2_tol}) exceeded: {bad}"
    return errs
