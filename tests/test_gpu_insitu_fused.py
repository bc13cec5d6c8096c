"""The fused attention forward inside the UNMODIFIED reference engine (tools/insitu.py run_fused): the
reference's `AttentionLayer.forward` re-bound by `patch_minisgl_attention` (`--patch fused`) against the same
engine with our norm / RoPE kernels as separate launches (`--patch model`), at page sizes 64 and 1, Qwen3-0.6B
shape, dummy weights, teacher-forced on the tokens of the free-running fi run.  Skipped when build() found no
reference checkout.

Gates:
  * bit identity: the fused launch computes exactly what q-norm, k-norm, RoPE and attention compute as four
    launches (tests/test_gpu_elementwise.py, tests/test_gpu_attention.py), so the logits of every forward
    and the K / V rows of every appended token equal the unfused run's bit for bit;
  * launches: per layer, a decode forward (eager, or being captured into a graph) makes 3 launches fewer
    (q-norm, k-norm, RoPE) and a prefill forward 2 fewer (the three become one);
  * the fused run passes the same logits gate against the reference's fi backend as the unfused one
    (tests/test_gpu_insitu.py);
  * `install_into_minisgl()` with the b200 backend computes what `--patch fused` computes, and with the
    reference's own fi backend it leaves the launches and outputs of the unpatched attention layer alone.
"""
import argparse
import json
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import insitu  # noqa: E402

pytestmark = pytest.mark.gpu

LOGITS_TOL = 1e-3
LAYERS = 28


@pytest.fixture(scope="module")
def runs():
    if not insitu.reference_available():
        pytest.skip("reference package not installed (build() copies it when a reference checkout is readable)")
    return insitu.run_fused(argparse.Namespace(layers=LAYERS))


def _load(path):
    import torch

    return torch.load(path)


def _assert_same_bits(runs, a, b):
    assert insitu.logits_bit_identical(runs[a], runs[b]), f"{a} vs {b}: logits differ"
    s = insitu.compare(runs[a], runs[b])
    for key in ("k_first_bit_exact", "v_first_bit_exact", "k_last_bit_exact", "v_last_bit_exact"):
        assert s[key], (a, b, s)
    return s


@pytest.mark.parametrize("page", [64, 1])
def test_fused_equals_unfused_bit_for_bit(runs, page):
    s = _assert_same_bits(runs, f"b200_p{page}_fused", f"b200_p{page}_patched")
    assert s["graph_replays"] >= 10 and s["chunked_reqs"] >= 2 and s["extend_reqs_with_cache_hit"] >= 2, s


@pytest.mark.parametrize("page", [64, 1])
def test_fused_saves_three_launches_per_decode_layer(runs, page):
    fused, unfused = _load(runs[f"b200_p{page}_fused"]), _load(runs[f"b200_p{page}_patched"])
    fwd = fused["forwards"]
    assert fwd == unfused["forwards"], (fwd, unfused["forwards"])
    assert fwd["prefill"] > 0 and fwd["decode"] > 0, fwd
    saved = unfused["b200_launches"] - fused["b200_launches"]
    want = LAYERS * (3 * fwd["decode"] + 2 * fwd["prefill"])
    print(json.dumps({"page": page, "forwards": fwd, "unfused": unfused["b200_launches"],
                      "fused": fused["b200_launches"], "saved": saved}))
    assert saved == want, (saved, want, fwd)


def test_fused_passes_the_reference_fi_gate(runs):
    spread = insitu.compare(runs["fi_tc_p64"], runs["fi_p64"])["logits_rel_worst"]
    got = insitu.compare(runs["b200_p64_fused"], runs["fi_p64"])["logits_rel_worst"]
    bound = max(LOGITS_TOL, 2.0 * spread)
    print(json.dumps({"rel": got, "reference_fi_tc_vs_fi": spread, "bound": bound}))
    assert got <= bound, (got, bound)


def test_install_into_minisgl_runs_the_fused_forward(runs):
    _assert_same_bits(runs, "b200_p64_installed", "b200_p64_fused")


def test_install_into_minisgl_leaves_the_fi_backend_alone(runs):
    _assert_same_bits(runs, "fi_p64_installed", "fi_p64_installed_unfused")
    a, b = _load(runs["fi_p64_installed"]), _load(runs["fi_p64_installed_unfused"])
    assert a["b200_launches"] == b["b200_launches"] > 0, (a["b200_launches"], b["b200_launches"])
