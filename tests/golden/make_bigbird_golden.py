"""Generates tests/golden/bigbird/*.pt: GPSLayer(dim_h, <local>, 'BigBird', ...) fixtures from the REFERENCE's own
gps_layer.py and bigbird_layer.py run verbatim in fp64 (gps_layer.py under oracle/ref_shim.py, whose stub for
graphgps.layer.bigbird_layer is replaced here by the real file, loaded by path).

    python tests/golden/make_bigbird_golden.py [REFERENCE_LAYER_DIR]

Each layer fixture holds the config (with the bigbird config), inputs, the reference state_dict, the cotangent, the
reference's own random-block table `table` [heads, nb - 2, r] (drawn by its _get_rand_attn_plan /
_bigbird_block_rand_mask_with_head with np.random.seed(0), as its forward does), fp64 outputs, every gradient and the
running statistics (stored as fp32; reference_live_GINE_BigBird keeps fp64 and pins the oracle at 1e-10 / 1e-9).
tables.pt holds the reference's table for a sweep of (block_size, r, heads, padded length), legacy 1024 included,
and the padded lengths at which the reference raises.
"""
import importlib.util
import os
import sys
import types
import zlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from bigbird_oracle import bb_batch, bigbird_cfg  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402

OUT = os.path.join(HERE, "bigbird")

# name, local, d, heads, sizes, training, batch_norm, cfg overrides
CASES = [
    ("gine_bigbird_relu", "GINE", 56, 8, [23, 17, 30, 21, 12, 26], True, True, {}),
    ("gine_bigbird_eval", "GINE", 56, 8, [23, 17, 30, 21, 12, 26], False, True, {}),
    ("gatedgcn_bigbird_sigmoid_bias", "CustomGatedGCN", 56, 8, [19, 24, 11, 28], True, True,
     dict(use_bias=True, hidden_act="sigmoid")),
    ("none_bigbird_relu", "None", 56, 8, [20, 33, 14], True, True, {}),
    ("gine_bigbird_nonorm", "GINE", 56, 8, [23, 17, 30, 21], True, False, {}),
    ("gine_bigbird_bs2", "GINE", 56, 8, [15, 22, 9, 18], True, True, dict(block_size=2, num_random_blocks=1)),
    ("gine_bigbird_bs4", "GINE", 56, 8, [31, 22, 40, 18], True, True, dict(block_size=4, num_random_blocks=2)),
    ("gine_bigbird_plan3", "GINE", 56, 8, [20, 13, 16], True, True, {}),            # Nmax 20: one band
    ("gine_bigbird_plan2", "GINE", 56, 8, [30, 13, 26], True, True, {}),            # Nmax 30: two bands (r//2)
    ("gine_bigbird_plan1", "GINE", 56, 8, [37, 13, 26], True, True, {}),            # Nmax 37: two bands (r, 0)
    ("gine_bigbird_nb4", "GINE", 56, 8, [12, 7, 10, 4], True, True, {}),            # Nmax 12: nb = 4
    ("gine_bigbird_lastpad", "GINE", 56, 8, [34, 12, 20, 9, 27], True, True, {}),   # last block real in one graph
    ("gine_bigbird_d64", "GINE", 64, 4, [23, 17, 30, 21], True, True, dict(num_random_blocks=2)),
]
LIVE = ("reference_live_GINE_BigBird", "GINE", 16, 4, [14, 9, 13], True, True, dict(num_random_blocks=2))


def load_bigbird(ref):
    """The reference's bigbird_layer.py loaded verbatim, installed as gps_layer.py's SingleBigBirdLayer."""
    path = os.path.join(ref.layer_dir, "bigbird_layer.py")
    if not os.path.isfile(path):
        path = "/root/reference/graphgps/layer/bigbird_layer.py"
    spec = importlib.util.spec_from_file_location("graphgps.layer.bigbird_layer", path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    sys.modules["graphgps.layer.gps_layer"].SingleBigBirdLayer = m.SingleBigBirdLayer
    return m


def ref_table(bbm, S, bs, r, H, max_len=128):
    """The reference's random-block table for padded length S, drawn as its forward draws it."""
    cfg = types.SimpleNamespace(max_position_embeddings=max_len, dim_hidden=H, n_heads=H, num_random_blocks=r,
                                block_size=bs, use_bias=False)
    a = bbm.BigBirdBlockSparseAttention(cfg, seed=0)
    state = np.random.get_state()
    try:
        np.random.seed(0)
        if S in (1024, 3072, 4096):
            t = [a._bigbird_block_rand_mask(max_len, max_len, bs, bs, r, last_idx=1024)[:S // bs - 2] for _ in range(H)]
        else:
            pl, pr = a._get_rand_attn_plan(S, bs, r)
            t = a._bigbird_block_rand_mask_with_head(from_seq_length=S, to_seq_length=S, from_block_size=bs,
                                                     to_block_size=bs, num_heads=H, plan_from_length=pl,
                                                     plan_num_rand_blocks=pr)
        return np.stack(t, 0)
    finally:
        np.random.set_state(state)


def _prepare(layer):
    with torch.no_grad():
        for m in layer.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.3, 0.3)
                m.running_mean.uniform_(-0.2, 0.2)
                m.running_var.uniform_(0.6, 1.4)
            if isinstance(m, torch.nn.LayerNorm):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.3, 0.3)


def run_case(ref, bbm, name, local, d, heads, sizes, training, batch_norm, over, dtype=torch.float32):
    seed = zlib.crc32(name.encode()) % (2 ** 31)
    torch.manual_seed(seed)
    cfg = bigbird_cfg(**over)
    layer = ref.GPSLayer(d, local, "BigBird", heads, act="relu", batch_norm=batch_norm, bigbird_cfg=cfg)
    _prepare(layer)
    batch = bb_batch(sizes, d, seed % 1000, dtype)
    nmax = max(sizes)
    bs = cfg.block_size
    S = nmax + (bs - nmax % bs) % bs
    fix = {"config": dict(name=name, local=local, glob="BigBird", d=d, heads=heads, act="relu", training=training,
                          batch_norm=batch_norm, bigbird={k: v for k, v in vars(cfg).items()}),
           "x": batch.x.clone(), "edge_index": batch.edge_index.clone(), "edge_attr": batch.edge_attr.clone(),
           "batch": batch.batch.clone(), "num_graphs": batch.num_graphs,
           "table": torch.from_numpy(ref_table(bbm, S, bs, cfg.num_random_blocks, heads)),
           "state": {k: v.clone() for k, v in layer.state_dict().items()}}
    layer = layer.double()
    layer.train(training)
    b = batch.clone()
    b.x = b.x.double().requires_grad_(True)
    b.edge_attr = b.edge_attr.double().requires_grad_(True)
    x_in, e_in = b.x, b.edge_attr
    out = layer(b)
    g = torch.Generator().manual_seed(5)
    ct_x = torch.randn(out.x.shape, generator=g, dtype=torch.float64).to(dtype)
    fix["ct_x"] = ct_x
    keep = (lambda t: t.detach().clone()) if dtype == torch.float64 else (lambda t: t.detach().float())
    fix["out_x"] = keep(out.x)
    loss = (out.x * ct_x.double()).sum()
    if local == "CustomGatedGCN":
        ct_e = torch.randn(out.edge_attr.shape, generator=g, dtype=torch.float64).to(dtype)
        fix["ct_e"] = ct_e
        fix["out_e"] = keep(out.edge_attr)
        loss = loss + (out.edge_attr * ct_e.double()).sum()
    if training or dtype == torch.float64:
        loss.backward()
        fix["grad_x"] = keep(x_in.grad)
        if e_in.grad is not None:
            fix["grad_e"] = keep(e_in.grad)
        fix["grad_params"] = {n: keep(p.grad) for n, p in layer.named_parameters() if p.grad is not None}
    fix["state_after"] = {k: (keep(v) if v.is_floating_point() else v.clone())
                          for k, v in layer.state_dict().items() if "running" in k or "num_batches" in k}
    return fix


def tables(bbm):
    """The reference's table over (block_size, r, heads) and padded lengths, and the lengths where it raises."""
    out = {"tables": {}, "raises": {}}
    for bs, r, H in ((3, 3, 8), (2, 1, 2), (4, 2, 3), (3, 5, 2), (1, 3, 2)):
        bad = []
        for nb in range(4, 48):
            S = nb * bs
            try:
                out["tables"][(bs, r, H, S)] = torch.from_numpy(ref_table(bbm, S, bs, r, H))
            except Exception:
                bad.append(S)
        out["raises"][(bs, r, H)] = bad
    # the plan of the BigBird paper at padded length 1024 (max_position_embeddings 1024, so the table covers it)
    out["legacy"] = {(8, 2, 2, 1024, 1024): torch.from_numpy(ref_table(bbm, 1024, 8, 2, 2, 1024))}
    return out


def main():
    args = sys.argv[1:]
    ref = load_reference(args[0] if args else None)
    bbm = load_bigbird(ref)
    os.makedirs(OUT, exist_ok=True)
    torch.save(tables(bbm), os.path.join(OUT, "tables.pt"))
    for case in CASES:
        fix = run_case(ref, bbm, *case)
        path = os.path.join(OUT, case[0] + ".pt")
        torch.save(fix, path)
        print(case[0], "N", fix["x"].shape[0], "table", tuple(fix["table"].shape), f"{os.path.getsize(path)/1e3:.0f} kB")
    fix = run_case(ref, bbm, *LIVE, dtype=torch.float64)
    path = os.path.join(OUT, LIVE[0] + ".pt")
    torch.save(fix, path)
    print(LIVE[0], f"{os.path.getsize(path)/1e3:.0f} kB")


if __name__ == "__main__":
    main()
