"""Generates tests/golden/eslappe/*.pt: GPSLayer(..., equivstable_pe=True) fixtures from the REFERENCE ITSELF (its own
layer files run verbatim under oracle/ref_shim.py, fp64), next to the fixtures of tests/golden/make_golden.py.

    python tests/golden/make_eslappe_golden.py [REFERENCE_LAYER_DIR]

The fixtures live in a subdirectory because tests/util.py::golden_names() feeds every tests/golden/*.pt to tests that
build layers without the flag.  Each holds what a make_golden.py fixture holds (config, inputs, reference state_dict,
cotangents, fp64 outputs / gradients / running statistics stored as fp32) plus the positional encoding `pe` [N, k]
(config["pe_dim"] = k) and its gradient `grad_pe`.  reference_live_CustomGatedGCN_Transformer.pt is the
reference_live-style case (fp64 inputs, weights, outputs and gradients) that pins the oracle at 1e-9.

A unit-normal PE at k = 64 gives r_ij = |PE_i - PE_j|^2 ~ 128 and saturates the gate rho = mlp_r_ij(r_ij), which hides
gradient bugs.  So the PE rows get norms spread over (0.3, 2.1) (r_ij spans about two decades), and mlp_r_ij.2 is
rescaled and shifted so that its pre-activation spans (-3, 3) over the case's edges: rho spans (0.05, 0.95).  The
range of rho of each case is printed.  Every fixture stays below 1 MB.
"""
import os
import sys
import zlib

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from graphgps_b200.batch import make_batch  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "eslappe")

# name, local, global, shape, d, heads, act, num_graphs, training, k (PE width)
CASES = [
    ("gatedgcn_transformer_relu_pe", "CustomGatedGCN", "Transformer", "zinc-gatedgcn", 64, 4, "relu", 5, True, 64),
    ("gatedgcn_transformer_gelu_pe", "CustomGatedGCN", "Transformer", "pcqm4m-small", 48, 4, "gelu", 12, True, 48),
    ("gatedgcn_performer_relu_pe", "CustomGatedGCN", "Performer", "zinc-gatedgcn", 48, 2, "relu", 6, True, 48),
    ("gatedgcn_transformer_eval_pe", "CustomGatedGCN", "Transformer", "zinc-gatedgcn", 64, 4, "relu", 6, False, 64),
    ("gatedgcn_transformer_k7_pe", "CustomGatedGCN", "Transformer", "zinc-gatedgcn", 32, 4, "gelu", 6, True, 7),
]
LIVE_NAME = "reference_live_CustomGatedGCN_Transformer"


def make_pe(N, k, seed):
    g = torch.Generator().manual_seed(seed)
    rows = torch.randn(N, k, generator=g)
    rows = rows / rows.norm(dim=1, keepdim=True).clamp_min(1e-6)
    return rows * (0.3 + 1.8 * torch.rand(N, 1, generator=g))


def calibrate_gate(layer, pe, edge_index):
    """Rescale / shift mlp_r_ij.2 (in place) so that its pre-activation spans (-3, 3) over the edges."""
    mlp = layer.local_model.mlp_r_ij
    with torch.no_grad():
        r = ((pe[edge_index[1]] - pe[edge_index[0]]) ** 2).sum(-1, keepdim=True).double()
        h = mlp[1](r @ mlp[0].weight.double().t() + mlp[0].bias.double())
        z = h @ mlp[2].weight.double().t()
        lo, hi = float(z.min()), float(z.max())
        f = 6.0 / max(hi - lo, 1e-12)
        mlp[2].weight.mul_(f)
        mlp[2].bias.fill_(-f * (hi + lo) / 2)


def gate_range(layer, pe, edge_index):
    """min / max of rho = mlp_r_ij(|PE_i - PE_j|^2) over the edges."""
    with torch.no_grad():
        r = ((pe[edge_index[1]] - pe[edge_index[0]]) ** 2).sum(-1, keepdim=True)
        rho = layer.local_model.mlp_r_ij(r.to(layer.local_model.mlp_r_ij[0].weight.dtype))
    return float(rho.min()), float(rho.max())


def run_case(ref, name, local, glob, shape, d, heads, act, B, training, pe_dim):
    torch.manual_seed(zlib.crc32(name.encode()) % (2 ** 31))
    layer = ref.GPSLayer(d, local, glob, heads, act=act, equivstable_pe=True)
    # non-trivial BatchNorm affine + running stats so they are actually exercised
    with torch.no_grad():
        for m in layer.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.3, 0.3)
                m.running_mean.uniform_(-0.2, 0.2)
                m.running_var.uniform_(0.6, 1.4)
    batch = make_batch(shape, seed=11, dim=d, num_graphs=B)
    pe = make_pe(batch.x.shape[0], pe_dim, zlib.crc32(name.encode()) % 1000)
    calibrate_gate(layer, pe, batch.edge_index)
    state = {k: v.clone() for k, v in layer.state_dict().items()}
    fix = {"config": dict(name=name, local=local, glob=glob, d=d, heads=heads, act=act, training=training,
                          pe_dim=pe_dim),
           "x": batch.x.clone(), "edge_index": batch.edge_index.clone(), "edge_attr": batch.edge_attr.clone(),
           "batch": batch.batch.clone(), "num_graphs": B, "state": state, "pe": pe}
    layer = layer.double()
    layer.train(training)
    b = batch.clone()
    b.x = b.x.double().requires_grad_(True)
    b.edge_attr = b.edge_attr.double().requires_grad_(True)
    b.pe_EquivStableLapPE = pe.double().requires_grad_(True)
    x_in, e_in, pe_in = b.x, b.edge_attr, b.pe_EquivStableLapPE
    fix["rho_range"] = gate_range(layer, pe.double(), b.edge_index)
    out = layer(b)
    g = torch.Generator().manual_seed(5)
    ct_x = torch.randn(out.x.shape, generator=g)
    ct_e = torch.randn(out.edge_attr.shape, generator=g)
    fix["ct_x"], fix["ct_e"] = ct_x, ct_e
    fix["out_x"] = out.x.detach().float()
    fix["out_e"] = out.edge_attr.detach().float()
    loss = (out.x * ct_x.double()).sum() + (out.edge_attr * ct_e.double()).sum()
    if training:
        loss.backward()
        fix["grad_x"] = x_in.grad.float()
        fix["grad_e"] = e_in.grad.float()
        fix["grad_pe"] = pe_in.grad.float()
        fix["grad_params"] = {n: p.grad.float() for n, p in layer.named_parameters() if p.grad is not None}
    fix["state_after"] = {k: v.detach().float() if v.is_floating_point() else v.clone()
                          for k, v in layer.state_dict().items() if "running" in k or "num_batches" in k}
    return fix


def run_live_case(ref):
    """The reference layer in fp64 on seeded inputs (d = k = 32, 4 heads, 7 zinc-shaped graphs), grad_pe included."""
    torch.manual_seed(3)
    R = ref.GPSLayer(32, "CustomGatedGCN", "Transformer", 4, equivstable_pe=True)
    b = make_batch("zinc-gatedgcn", seed=5, dim=32, num_graphs=7, dtype=torch.float64)
    pe = make_pe(b.x.shape[0], 32, 6).double()
    calibrate_gate(R, pe, b.edge_index)
    state = {k: v.clone() for k, v in R.state_dict().items()}
    R = R.double()
    fix = {"local": "CustomGatedGCN", "glob": "Transformer", "state": state, "x": b.x.clone(),
           "edge_index": b.edge_index.clone(), "edge_attr": b.edge_attr.clone(), "batch": b.batch.clone(),
           "num_graphs": 7, "pe": pe.clone()}
    b.x.requires_grad_(True)
    b.edge_attr.requires_grad_(True)
    b.pe_EquivStableLapPE = pe.requires_grad_(True)
    x_in = b.x
    o = R(b)
    (o.x ** 2).sum().backward()
    fix["out_x"] = o.x.detach().clone()
    fix["grad_x"] = x_in.grad.clone()
    fix["grad_pe"] = pe.grad.clone()
    fix["grad_params"] = {n: p.grad.clone() for n, p in R.named_parameters() if p.grad is not None}
    fix["rho_range"] = gate_range(R, pe.detach(), b.edge_index)
    return fix


def main():
    args = sys.argv[1:]
    ref = load_reference(args[0] if args else None)
    os.makedirs(OUT, exist_ok=True)
    for case in CASES:
        fix = run_case(ref, *case)
        path = os.path.join(OUT, case[0] + ".pt")
        torch.save(fix, path)
        print(case[0], "N", fix["x"].shape[0], "E", fix["edge_index"].shape[1], "rho in (%.3f, %.3f)" %
              fix["rho_range"], f"{os.path.getsize(path)/1e3:.0f} kB")
    fix = run_live_case(ref)
    path = os.path.join(OUT, LIVE_NAME + ".pt")
    torch.save(fix, path)
    print(LIVE_NAME, "rho in (%.3f, %.3f)" % fix["rho_range"], f"{os.path.getsize(path)/1e3:.0f} kB")


if __name__ == "__main__":
    main()
