"""SAN layer on the GPU: the fixtures from the reference in fp32-grade and bf16, the attention stage at every shipped
head dim against float64, dropout at both sites with the library's masks injected into the oracle, the shared
embedding over two layers, reproducibility, retained graphs, CUDA-graph capture, the launch count, and the full
zinc-, molpcba- and coco-SAN shapes against the float64 oracle run on the GPU.  The checks SAN2Layer runs as well are
in tests/san_harness.py."""
import pytest
import torch

from graphgps_b200.graph import graph_of
from san_harness import (_full, _gb, _load, _module, _seq_step, _stage, check_bitwise_reproducible_and_retain_graph,
                         check_dropout_both_sites_with_injected_masks, check_eval_mode_leaves_running_statistics,
                         check_fixture, check_launch_count, check_shared_embedding_gradient_over_two_layers,
                         check_training_updates_running_statistics, fixtures)
from san_oracle import dataset_sizes, san_batch
from util import DEV, pin_dropout_counter

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", fixtures("SAN"))
def test_fixture(name, precision):
    if name == "saturate_hd8" and precision == "bf16":
        # scores of |t| ~ 20 carry bf16 rounding of ~2^-9 |t| ~ 0.04: the clamp mask of every pair that close to +-5
        # flips, which moves the fake-pair weight gradients by O(10 %) in L2; fp32-grade holds this fixture instead
        pytest.skip("saturated scores are checked in fp32-grade only")
    if name == "two_layer_shared_hd6" and precision == "bf16":
        # 61 rows per BatchNorm column through two layers: bf16 rounding moves the near-cancelling BatchNorm-bias and
        # FFN1-bias gradients by ~0.2 relative L2; the shared-embedding gradient is held in fp32-grade
        pytest.skip("two stacked layers on 61 rows are checked in fp32-grade only")
    check_fixture("SAN", _load("SAN", name), precision)


def test_eval_mode_leaves_running_statistics():
    check_eval_mode_leaves_running_statistics("SAN")


def test_training_updates_running_statistics():
    check_training_updates_running_statistics("SAN")


# ------------------------------------------------------------------------------------------ attention stage
# every shipped head dim: zinc 7, cluster 6, pattern 8, molhiv 16, molpcba 76, coco / voc 11, peptides 21
@pytest.mark.parametrize("hd,H,kind,gamma", [(7, 8, "mol", 1e-5), (6, 8, "sbm", 0.1), (8, 10, "sbm", 1e-5),
                                             (16, 4, "mol", 1e-5), (76, 4, "mol", 1e-5), (11, 8, "knn", 1e-6),
                                             (21, 4, "chain", 0.1)])
def test_attention_stage_head_dims(hd, H, kind, gamma):
    sizes = dataset_sizes(kind, 3 if kind in ("mol", "sbm") else 1, hd) + [1]
    errs, info = _stage("SAN", kind, sizes, H, hd, gamma, seed=hd, scale=1.6)
    print(hd, kind, {k: f"{v:.1e}" for k, v in errs.items()}, f"saturated {info['saturated']:.2f}",
          "excluded nodes", info["excluded"])
    assert info["saturated"] > 0.01          # a share of the scores lies beyond the clamp
    assert max(errs.values()) < 2e-5, errs


def test_dropout_both_sites_with_injected_masks():
    check_dropout_both_sites_with_injected_masks("SAN", 1e-5)


def test_shared_embedding_gradient_over_two_layers():
    check_shared_embedding_gradient_over_two_layers("SAN")


def test_bitwise_reproducible_and_retain_graph():
    check_bitwise_reproducible_and_retain_graph("SAN")


# ------------------------------------------------------------------------------------------ capture
@pytest.mark.parametrize("p", [0.0, 0.2])
def test_captured_two_layer_stack(p):
    torch.manual_seed(4)
    seq = _module("SAN", dict(d=56, heads=8, gamma=1e-5, layers=2), "fp32", p).to(DEV)
    sb = san_batch("mol", dataset_sizes("mol", 6, 6), 56, 6).to(DEV)
    b = _gb(sb.x, sb.edge_attr, sb.edge_index, sb.batch, 6)
    graph_of(b).nmax   # read before capture (the read synchronises); the eager step below also caches it
    ct = torch.randn(sb.x.shape, device=DEV)
    x = sb.x.clone().requires_grad_(True)
    e = sb.edge_attr.clone().requires_grad_(True)
    pin_dropout_counter(DEV, 4096 * 1000)
    eager_g, eager_out = _seq_step(seq, x, e, b, ct)
    eager_out = eager_out.detach()
    x = x.detach().clone().requires_grad_(True)
    e = e.detach().clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            _seq_step(seq, x, e, b, ct)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, capture_error_mode="thread_local"):
        cap_g, cap_out = _seq_step(seq, x, e, b, ct)
    pin_dropout_counter(DEV, 4096 * 1000)
    graph.replay()
    torch.cuda.synchronize()
    first = cap_out.clone()
    assert torch.equal(first, eager_out)
    for a, r in zip(cap_g, eager_g):
        assert torch.equal(a, r)
    graph.replay()
    torch.cuda.synchronize()
    if p > 0.0:
        assert not torch.equal(first, cap_out)   # fresh masks on every replay
    else:
        assert torch.equal(first, cap_out)


def test_launch_count():
    check_launch_count("SAN")


# ------------------------------------------------------------------------------------------ full size
def test_full_size_zinc_san():
    _full("SAN", "mol", 32, 56, 8, 1e-5, 0.0, 21)


def test_full_size_molpcba_san():
    _full("SAN", "mol", 512, 304, 4, 1e-5, 0.2, 22)


def test_full_size_coco_san():
    _full("SAN", "knn", 8, 88, 8, 1e-6, 0.0, 23)
