"""Kernel census of the UNMODIFIED reference engine with `install_into_minisgl()` and the b200 backend
(tools/insitu.py run_census, torch.profiler with CUDA activities): one eager prefill forward and one decode graph
replay of a Qwen3-0.6B-shaped engine launch no FlashInfer kernel, the MLP activation is ours in every layer, and
the installed prefill forward makes exactly one b200 launch per layer more than the engine patched layer by layer,
which keeps FlashInfer's activation.  Skipped when build() found no reference checkout."""
import argparse
import json
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import insitu  # noqa: E402

pytestmark = pytest.mark.gpu

LAYERS = 28


@pytest.fixture(scope="module")
def census():
    if not insitu.reference_available():
        pytest.skip("reference package not installed (build() copies it when a reference checkout is readable)")
    return insitu.run_census(argparse.Namespace(layers=LAYERS, out=None))


def _activation_launches(groups, group):
    return sum(n for name, n in groups[group].items() if "silu_and_mul" in name or "act_and_mul" in name)


def test_installed_forward_launches_no_flashinfer_kernel(census):
    inst = census["installed"]
    for part in ("prefill_forward", "decode_replay"):
        assert inst[part]["flashinfer"] == {}, (part, inst[part]["flashinfer"])
        assert _activation_launches(inst[part], "ours") == LAYERS, (part, inst[part]["ours"])
    print(json.dumps({"sampler": inst["sampler"]}))


def test_layer_patched_engine_still_runs_flashinfer_activation(census):
    ref = census["patched_layers"]
    for part in ("prefill_forward", "decode_replay"):
        assert _activation_launches(ref[part], "flashinfer") == LAYERS, (part, ref[part]["flashinfer"])


def test_one_more_b200_launch_per_layer(census):
    c = census["checks"]
    assert c["installed_prefill_b200_launches_minus_patched_layers"] == LAYERS, c
    assert c["ok"], c
