"""Page-size independence of the attention kernels.  Below page size 8 the decode and prefill producers gather the
pool's K/V token rows with cp.async (row mode); from page size 8 on they load whole page pieces with TMA boxes (box
mode).  The way rows reach shared memory must not change a single bit: the same logical batch -- the same token rows,
lengths and inputs -- laid out at page sizes 1, 2, 4 and 12 (row mode) and 64 (box mode), pages in random order and
every pool row no request owns NaN, gives the same outputs and the same pool rows at every page size."""
import random

import numpy as np
import pytest
import torch

from helpers import (SPLIT_PLAN, GpuWorld, add_requests, assert_bits_equal, attn_tolerance_ok, make_inputs,
                     make_world, options, oracle_forward, padded_reqs, poison_unowned, run_attention, tail_range_ends)
from oracle import metadata as o_meta

pytestmark = pytest.mark.gpu

D = 128
PAGE_SIZES = [1, 2, 4, 12, 64]


def _world(page_size, lens, *, hq, hkv, dtype, seed, share_prefix=None, pad_to=None):
    """A NaN-poisoned world whose requests hold the same token rows at every page size.  With share_prefix, the
    requests after the first reuse its cached pages (radix matches are page aligned, so how many rows are shared
    depends on the page size); their first cached_len rows equal the first request's, so the contents do not."""
    n_pages = sum(-(-d // page_size) for _, d in lens) + (pad_to or 0) + 8
    w = make_world(seed=seed, page_size=page_size, hq=hq, hkv=hkv, dtype=dtype,
                   max_reqs=max(len(lens), pad_to or 0) + 1, max_seq=max(d for _, d in lens) + 8, num_pages=n_pages)
    add_requests(w, lens, share_prefix_from=share_prefix)
    poison_unowned(w)
    g = torch.Generator().manual_seed(seed + 7)
    rows = [torch.randn((2, d, hkv, D), generator=g).to(dtype) for _, d in lens]
    if share_prefix is not None:
        for i, (c, _) in enumerate(lens):
            if i > 0 and c > 0:
                rows[i][:, :c] = rows[share_prefix][:, :c]
    for (t, _, d), r in zip(w.reqs, rows):
        w.pool_cpu[:, 0, torch.from_numpy(w.page_table[t, :d].astype(np.int64))] = r
    return w


def _fused_args(dtype, norms):
    from oracle.rope import ref_cos_sin_cache

    g = torch.Generator().manual_seed(5)
    qw = (torch.rand(D, generator=g) + 0.5).to(dtype).cuda() if norms else None
    kw = (torch.rand(D, generator=g) + 0.5).to(dtype).cuda() if norms else None
    return ref_cos_sin_cache(D, 8192, 1e6).cuda(), qw, kw, 1e-6


def _run(b200, page_size, lens, *, phase, hq, hkv, dtype=torch.bfloat16, fused=None, graph=False, pad_to=None,
         share_prefix=None, seed=0):
    """One launch; returns (outputs of the real requests, K rows and V rows of every request in logical order after
    the launch, and the world, metadata and q / k / v for an oracle check)."""
    w = _world(page_size, lens, hq=hq, hkv=hkv, dtype=dtype, seed=seed, share_prefix=share_prefix, pad_to=pad_to)
    reqs = padded_reqs(w, pad_to)
    md = o_meta.ref_prepare_metadata(w.page_table, reqs, page_size)
    qkv, q, k, v = make_inputs(w, seed + 1, reqs=reqs)
    gw = GpuWorld(b200, w)
    out, _, kc, vc = run_attention(gw, gw.batch(phase, pad_to=pad_to, md=md), qkv.cuda(), fused=fused, graph=graph)
    n_out = len(lens) if phase == "decode" else sum(d - c for c, d in lens)
    idx = torch.from_numpy(np.concatenate([w.page_table[t, :d] for t, _, d in w.reqs]).astype(np.int64)).cuda()
    return out[:n_out], kc[idx], vc[idx], (w, md, q, k, v)


def _same_bits(b200, lens, page_sizes=PAGE_SIZES, oracle=True, **kw):
    """Runs lens at every page size, requires bit-identical outputs and pool rows; checks the first page size's
    output against the fp32 oracle (oracle/tolerance.py) when `oracle` (unfused launches only)."""
    first = None
    for ps in page_sizes:
        out, kr, vr, ctx = _run(b200, ps, lens, **kw)
        if first is None:
            first = (ps, out, kr, vr)
            if oracle and kw.get("fused") is None:
                w, md, q, k, v = ctx
                n_real = len(lens)
                reqs = padded_reqs(w, kw.get("pad_to"))
                ref, _, _ = oracle_forward(w, 0, q, k, v, md, reqs=reqs)
                attn_tolerance_ok(out, ref[: out.shape[0]], f"{kw['phase']} page size {ps}")
            continue
        what = f"page size {ps} vs {first[0]}"
        assert_bits_equal(out, first[1], f"{what}: outputs")
        assert_bits_equal(kr, first[2], f"{what}: K rows")
        assert_bits_equal(vr, first[3], f"{what}: V rows")


def _tile_end_lens(seed=0):
    """Decode requests whose streamed range (kv_len - 1 keys) ends at every row of a 128-row tile, in the first and
    in a later tile, plus the box-mode tail offsets of page size 64, shuffled."""
    ns = set(range(1, 129)) | {n + 256 for n in range(0, 128, 3)} | set(tail_range_ends(64))
    lens = [(n, n + 1) for n in sorted(ns)]
    random.Random(seed).shuffle(lens)
    return lens


# ------------------------------------------------------------------------------------------------- decode
@pytest.mark.parametrize("hq,hkv", [(16, 8), (8, 1), (12, 1), (128, 8)])
def test_decode_same_bits_at_every_page_size(b200, native_lib, hq, hkv):
    _same_bits(b200, _tile_end_lens(), phase="decode", hq=hq, hkv=hkv, oracle=hq <= 16)


@pytest.mark.parametrize("norms", [True, False], ids=["qk-norm", "no-norm"])
@pytest.mark.parametrize("hq,hkv", [(16, 8), (12, 1)])
def test_fused_decode_same_bits_at_every_page_size(b200, native_lib, hq, hkv, norms):
    _same_bits(b200, _tile_end_lens(1), phase="decode", hq=hq, hkv=hkv, fused=_fused_args(torch.bfloat16, norms))


@pytest.mark.parametrize("merge", [1, 0], ids=["in-kernel-merge", "combine-launch"])
@pytest.mark.parametrize("fused", [False, True], ids=["plain", "fused"])
def test_split_decode_same_bits_at_every_page_size(b200, native_lib, merge, fused):
    lens = _tile_end_lens(2)[:40] + [(1999, 2000), (1500, 1501), (700, 701), (1025, 1026)]
    with options(b200, **SPLIT_PLAN, decode_fused_combine=merge):
        _same_bits(b200, lens, phase="decode", hq=16, hkv=2, fused=_fused_args(torch.bfloat16, True) if fused else None)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_padded_graph_decode_same_bits_at_every_page_size(b200, native_lib, dtype):
    """The fused launch captured into a CUDA graph on dummy requests and replayed on a padded batch (the producers
    then stream K/V before the predecessor has finished), in both 16-bit types."""
    _same_bits(b200, _tile_end_lens(3)[:30], phase="decode", hq=16, hkv=8, dtype=dtype,
               fused=_fused_args(dtype, True), graph=True, pad_to=36)


def test_decode_more_units_than_the_unit_cache_same_bits(b200, native_lib):
    """1600 requests x 8 kv heads = 12 800 work units, more than the 96 a CTA decodes into shared memory on 132 SMs:
    the units past the cache are decoded from global memory.  Box mode at page size 16 keeps the pool small."""
    lens = [(n, n + 1) for n in np.random.default_rng(4).integers(1, 16, 1600).tolist()]
    _same_bits(b200, lens, page_sizes=[1, 2, 4, 16], phase="decode", hq=16, hkv=8, oracle=False)


# ------------------------------------------------------------------------------------------------ prefill
PREFILL_CASES = {
    "fresh": dict(lens=[(0, 70), (0, 300), (0, 129), (0, 1)]),
    "cached-unaligned": dict(lens=[(300, 700), (1000, 1100), (77, 200), (129, 130), (63, 64)]),
    "radix-shared": dict(lens=[(300, 700), (256, 400), (128, 129), (299, 301)], share_prefix=0),
    "long-prompt": dict(lens=[(0, 4096), (5, 64)]),
}


@pytest.mark.parametrize("hq,hkv", [(16, 2), (32, 2)], ids=["gqa8", "gqa16"])
@pytest.mark.parametrize("case", sorted(PREFILL_CASES))
def test_prefill_same_bits_at_every_page_size(b200, native_lib, case, hq, hkv):
    _same_bits(b200, phase="prefill", hq=hq, hkv=hkv, **PREFILL_CASES[case])


def test_fp16_prefill_same_bits_at_every_page_size(b200, native_lib):
    _same_bits(b200, phase="prefill", hq=16, hkv=2, dtype=torch.float16, **PREFILL_CASES["cached-unaligned"])


# ------------------------------------------------------------------------------------------------ tracing
@pytest.mark.parametrize("phase", ["decode", "prefill"])
def test_row_mode_traced_equals_untraced_with_producer_events(b200, native_lib, phase):
    """Page size 4: a traced launch computes the same bits as an untraced one, and every producer warp records a
    slot wait, the slot becoming free and the loads issued for each tile it fills."""
    import importlib

    from test_gpu_attn_trace import DECODE_LENS, Case, _traced_equals_untraced

    tr = importlib.import_module("mini-sglang_b200.trace")
    if phase == "decode":
        case = Case(b200, phase="decode", page_size=4, hq=16, hkv=2, lens=DECODE_LENS)
        producers = (0, 1, 2, 3)
    else:
        case = Case(b200, phase="prefill", page_size=4, hq=16, hkv=2, lens=[(300, 700), (0, 257), (77, 200)])
        producers = (0, 1)
    (launch,), _ = _traced_equals_untraced(b200, case, epw=4096)
    assert launch.header["box_rows"] == 0 and launch.header["page_size"] == 4
    for c in range(launch.header["grid"]):
        for w in producers:
            codes = launch.warp_events(c, w)["code"]
            n = int((codes == tr.ISSUED).sum())
            assert int((codes == tr.EMPTY_WAIT).sum()) == n and int((codes == tr.EMPTY_DONE).sum()) == n, (c, w)
    assert int((launch.events["code"] == tr.ISSUED).sum()) > 0
