"""Helpers of the EquivStableLapPE (GPSLayer(..., equivstable_pe=True)) tests: fixtures under tests/golden/eslappe/."""
import glob
import os

import torch

from util import GOLDEN_DIR, compare, golden_batch, rel_err, rel_l2, run_layer

ESLAP_DIR = os.path.join(GOLDEN_DIR, "eslappe")
LIVE_NAME = "reference_live_CustomGatedGCN_Transformer"


def eslap_names():
    names = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(ESLAP_DIR, "*.pt")))
    return [n for n in names if n != LIVE_NAME]


def load_eslap(name):
    return torch.load(os.path.join(ESLAP_DIR, name + ".pt"), weights_only=False)


def eslap_batch(fix, device="cpu", dtype=torch.float32):
    b = golden_batch(fix, device, dtype)
    b.pe_EquivStableLapPE = fix["pe"].to(device=device, dtype=dtype)
    return b


def run_eslap(layer, batch, fix, backward=True):
    """util.run_layer plus the gradient w.r.t. batch.pe_EquivStableLapPE (res["grad_pe"])."""
    pe = batch.pe_EquivStableLapPE.requires_grad_(backward)
    res = run_layer(layer, batch, fix, backward)
    if backward:
        res["grad_pe"] = pe.grad.detach().cpu()
    return res


def compare_eslap(res, fix, tol, what="", grad_l2_tol=None):
    """util.compare, and grad_pe under the same gradient criterion (max-abs, or relative L2 when given)."""
    errs = compare(res, fix, tol, what, grad_l2_tol)
    if "grad_pe" in fix:
        e = rel_err(res["grad_pe"], fix["grad_pe"])
        errs["grad_pe"] = e
        if e > tol:
            l2 = rel_l2(res["grad_pe"], fix["grad_pe"])
            errs["grad_pe(l2)"] = l2
            assert grad_l2_tol is not None and l2 <= grad_l2_tol, f"{what} grad_pe: max-abs {e}, L2 {l2}"
    return errs


def make_pe(N, k, seed):
    """PE rows with norms spread over (0.3, 2.1), as tests/golden/make_eslappe_golden.py draws them."""
    g = torch.Generator().manual_seed(seed)
    rows = torch.randn(N, k, generator=g)
    rows = rows / rows.norm(dim=1, keepdim=True).clamp_min(1e-6)
    return rows * (0.3 + 1.8 * torch.rand(N, 1, generator=g))


def calibrate_gate(layer, pe, edge_index):
    """Rescale / shift mlp_r_ij.2 of layer (in place) so that rho spans (0.05, 0.95) over the edges."""
    mlp = layer.local_model.mlp_r_ij
    with torch.no_grad():
        r = ((pe[edge_index[1]] - pe[edge_index[0]]) ** 2).sum(-1, keepdim=True).double()
        h = mlp[1](r @ mlp[0].weight.double().t() + mlp[0].bias.double())
        z = h @ mlp[2].weight.double().t()
        lo, hi = float(z.min()), float(z.max())
        f = 6.0 / max(hi - lo, 1e-12)
        mlp[2].weight.mul_(f)
        mlp[2].bias.fill_(-f * (hi + lo) / 2)
