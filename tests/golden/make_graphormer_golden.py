"""Generates tests/golden/graphormer/*.pt: GraphormerLayer fixtures from the REFERENCE's own graphormer_layer.py run
verbatim in fp64 (loaded by path; its only third-party import, torch_geometric.utils.to_dense_batch, comes from
oracle/ref_shim.py).

    python tests/golden/make_graphormer_golden.py [REFERENCE_LAYER_DIR] [CASE ...]

Each fixture holds the config, the batch (x, edge_index, batch, num_graphs), the attention bias (or how the batch
lacks one), the reference state_dict, the cotangent, the output and every gradient including grad_attn_bias, stored
as fp32; reference_live keeps fp64 and pins tests/graphormer_oracle.py at 1e-10 / 1e-9.  reference_live also holds
`init_state`, the reference layer's state_dict right after construction from torch.manual_seed(INIT_SEED).  Dropout is
0 in every fixture.
"""
import importlib.util
import os
import sys
import types
import zlib

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from graphormer_oracle import graphormer_batch, random_bias  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402

OUT = os.path.join(HERE, "graphormer")
INIT_SEED = 1234

# name, d, heads, sizes, graph token, bias ("tensor" / "none" = attribute set to None / "absent"), training
ZINC = [24, 19, 30, 12, 27, 21]
CASES = [
    ("hd10_bias_token_train", 80, 8, ZINC, True, "tensor", True),
    ("hd10_bias_token_eval", 80, 8, ZINC, True, "tensor", False),
    ("hd10_no_attr", 80, 8, ZINC, True, "absent", True),
    ("hd10_bias_none", 80, 8, ZINC, True, "none", True),
    ("hd16_bias", 64, 4, [17, 33, 9, 25], False, "tensor", True),
    ("hd7_bias", 56, 8, [23, 17, 30, 21, 12], True, "tensor", True),
    ("hd16_bias_wgmma", 64, 4, [72, 64], False, "tensor", True),   # N >= 64 B: the wgmma forward
]
LIVE = ("reference_live", 24, 4, [9, 14, 6], True, "tensor", True)       # hd 6


def load_graphormer(layer_dir=None):
    """The reference's graphormer_layer.py loaded verbatim (after ref_shim installed its stubs)."""
    ref = load_reference(layer_dir)
    path = os.path.join(ref.layer_dir, "graphormer_layer.py")
    if not os.path.isfile(path):
        path = "/root/reference/graphgps/layer/graphormer_layer.py"
    spec = importlib.util.spec_from_file_location("graphgps.layer.graphormer_layer", path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _prepare(layer):
    with torch.no_grad():
        for m in layer.modules():
            if isinstance(m, torch.nn.LayerNorm):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.3, 0.3)
        layer.attention.in_proj_bias.uniform_(-0.2, 0.2)
        layer.attention.out_proj.bias.uniform_(-0.2, 0.2)


def run_case(grm, name, d, heads, sizes, token, bias_kind, training, dtype=torch.float32):
    seed = zlib.crc32(name.encode()) % (2 ** 31)
    torch.manual_seed(seed)
    layer = grm.GraphormerLayer(d, heads, 0.0, 0.0, 0.0)
    _prepare(layer)
    b = graphormer_batch(sizes, d, seed % 1000, token, dtype)
    bias = random_bias(sizes, heads, seed % 997, dtype) if bias_kind == "tensor" else None
    fix = {"config": dict(name=name, d=d, heads=heads, sizes=list(sizes), token=token, bias=bias_kind,
                          training=training),
           "x": b.x.clone(), "edge_index": b.edge_index.clone(), "batch": b.batch.clone(), "num_graphs": len(sizes),
           "attn_bias": None if bias is None else bias.clone(), "state": {k: v.clone() for k, v in layer.state_dict().items()}}
    layer = layer.double()
    layer.train(training)
    data = types.SimpleNamespace(x=b.x.double().clone().requires_grad_(True), batch=b.batch)
    x_in = data.x
    ab = None
    if bias_kind == "tensor":
        ab = bias.double().clone().requires_grad_(True)
        data.attn_bias = ab
    elif bias_kind == "none":
        data.attn_bias = None
    out = layer(data).x
    g = torch.Generator().manual_seed(5)
    ct = torch.randn(out.shape, generator=g, dtype=torch.float64)
    (out * ct).sum().backward()
    keep = (lambda t: t.detach().clone()) if dtype == torch.float64 else (lambda t: t.detach().float())
    fix["ct"] = ct.to(dtype)
    fix["out"] = keep(out)
    fix["grad_x"] = keep(x_in.grad)
    fix["grad_attn_bias"] = keep(ab.grad) if ab is not None else None
    fix["grad_params"] = {n: keep(p.grad) for n, p in layer.named_parameters()}
    return fix


def main():
    """python make_graphormer_golden.py [REFERENCE_LAYER_DIR] [CASE ...]: every fixture, or the named ones."""
    args = sys.argv[1:]
    names = {c[0] for c in CASES} | {LIVE[0]}
    layer_dir = args[0] if args and args[0] not in names else None
    only = [a for a in args if a in names]
    grm = load_graphormer(layer_dir)
    os.makedirs(OUT, exist_ok=True)
    for case in CASES:
        if only and case[0] not in only:
            continue
        fix = run_case(grm, *case)
        path = os.path.join(OUT, case[0] + ".pt")
        torch.save(fix, path)
        print(case[0], "N", fix["x"].shape[0], f"{os.path.getsize(path)/1e3:.0f} kB")
    if only and LIVE[0] not in only:
        return
    fix = run_case(grm, *LIVE, dtype=torch.float64)
    torch.manual_seed(INIT_SEED)
    fix["init_seed"] = INIT_SEED
    fix["init_state"] = {k: v.clone() for k, v in grm.GraphormerLayer(80, 8, 0.1, 0.1, 0.1).state_dict().items()}
    path = os.path.join(OUT, LIVE[0] + ".pt")
    torch.save(fix, path)
    print(LIVE[0], f"{os.path.getsize(path)/1e3:.0f} kB")


if __name__ == "__main__":
    main()
