"""Prefill at the page geometries and GQA groups decode already covers.

Page sizes: 8 and 32 (8- and 32-row TMA boxes: a box that straddles cached_len is loaded row by row, the fused
append stores the partial boxes that hold a unit's first and last new rows row by row), 128 and 256 (pages of
several 64-row boxes), and 24, 48 and 96 (not powers of two: boxes of 8, 16 and 32 rows), with cached lengths
that fall inside boxes (test_gpu_attention_probes.PREFILL_LENS); decode needles and the exact-tail on / off
equality at 24, 48 and 96.  GQA groups of 9 to 16 query heads per kv head (96/8, 128/8, 64/4 and the odd 9/1,
15/1) through the wgmma prefill kernel: needles and ramps, the fp32 oracle, and a radix-shared prefix."""
import pytest
import torch

from test_gpu_attention import _run_case
from test_gpu_attention_probes import PREFILL_LENS, _decode_needles, _prefill_probe
from test_gpu_decode_tail import _check, _tail_lens

pytestmark = pytest.mark.gpu

PAGE_SIZES = [8, 24, 32, 48, 96, 128, 256]
# cached lengths inside a box at every box size: 100, 37, 129 and 1
ORACLE_LENS = [(100, 300), (37, 200), (129, 130), (1, 140), (0, 333)]
GQA_SHAPES = [(96, 8), (128, 8), (64, 4), (9, 1), (15, 1)]
GQA_IDS = [f"hq{hq}-hkv{hkv}" for hq, hkv in GQA_SHAPES]


@pytest.mark.parametrize("order", [0, 1], ids=["size-sorted", "request-major"])
@pytest.mark.parametrize("page_size", PAGE_SIZES)
def test_prefill_probes_page_sizes(b200, native_lib, page_size, order):
    _prefill_probe(b200, page_size=page_size, hq=16, hkv=8, dtype=torch.bfloat16, lens=PREFILL_LENS,
                   opts={"prefill_impl": 1, "prefill_order": order})


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("page_size", PAGE_SIZES)
def test_prefill_oracle_page_sizes(b200, native_lib, page_size, dtype):
    """fp32 oracle, appended rows bit-exact, every other row of the NaN-poisoned pool untouched."""
    _run_case(b200, page_size=page_size, hq=16, hkv=8, lens=ORACLE_LENS, phase="prefill", dtype=dtype)


@pytest.mark.parametrize("plan", ["unsplit", "split"])
@pytest.mark.parametrize("page_size", [24, 48, 96])
def test_decode_needles_non_power_of_two_pages(b200, native_lib, page_size, plan):
    _decode_needles(b200, page_size=page_size, hq=16, hkv=8, dtype=torch.bfloat16, plan=plan)


@pytest.mark.parametrize("page_size", [24, 48, 96])
def test_decode_exact_tail_non_power_of_two_pages(b200, native_lib, page_size):
    _check(b200, page_size=page_size, lens=_tail_lens(page_size))


@pytest.mark.parametrize("hq,hkv", GQA_SHAPES, ids=GQA_IDS)
def test_prefill_probes_large_groups(b200, native_lib, hq, hkv):
    _prefill_probe(b200, page_size=16, hq=hq, hkv=hkv, dtype=torch.bfloat16, lens=PREFILL_LENS[:5], opts={})


@pytest.mark.parametrize("page_size", [1, 64])
@pytest.mark.parametrize("hq,hkv", GQA_SHAPES, ids=GQA_IDS)
def test_prefill_oracle_large_groups(b200, native_lib, hq, hkv, page_size):
    _run_case(b200, page_size=page_size, hq=hq, hkv=hkv, lens=[(0, 130), (64, 300), (0, 7), (37, 200)],
              phase="prefill")


@pytest.mark.parametrize("hq,hkv", [(16, 1), (128, 8)], ids=["hq16-hkv1", "hq128-hkv8"])
def test_prefill_radix_shared_prefix_large_group_fp16(b200, native_lib, hq, hkv):
    """Requests whose leading page-table entries are identical (radix-shared pages), at a group of 16, fp16."""
    _run_case(b200, page_size=16, hq=hq, hkv=hkv, lens=[(128, 300), (128, 260), (128, 400)], phase="prefill",
              share_prefix=0, dtype=torch.float16)
