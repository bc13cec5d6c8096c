"""Exact-tail K/V loads of the decode kernel (option decode_exact_tail): at page sizes >= 8 the page piece that holds
the end of a KV range is loaded only up to its last valid row (8-row boxes), pieces past the end are not loaded, and
the stage rows left unwritten keep whatever an earlier tile put there.  Every case runs the launch with the option at
1 and at 0 on a pool whose unowned rows are NaN, requires the two to agree bit for bit (output, appended rows, the
rest of the pool) and checks the output against the oracle."""
import random

import numpy as np
import pytest
import torch

from helpers import (SPLIT_PLAN, GpuWorld, add_requests, assert_bits_equal, attn_tolerance_ok, make_inputs,
                     make_world, options, oracle_forward, padded_reqs, poison_unowned, run_attention, tail_range_ends)
from oracle import metadata as o_meta

pytestmark = pytest.mark.gpu

HQ, HKV, D = 16, 8, 128
EPS = 1e-6


def _check(b200, *, page_size, lens, mode="eager", pad_to=None, force_split=False, seed=0):
    """Runs `lens` ((kv_len - 1, kv_len) decode requests) with decode_exact_tail 1 and 0; returns the plan.
    mode: "eager" (forward), "fused" (forward_decode_fused) or "graph" (the fused launch captured like the engine's
    decode graphs: the K/V producers start before the predecessor finishes)."""
    from oracle.layer import ref_pre_attention
    from oracle.rope import ref_cos_sin_cache

    w = make_world(seed=seed, page_size=page_size, hq=HQ, hkv=HKV, max_reqs=max(len(lens), pad_to or 0) + 1,
                   max_seq=max(d for _, d in lens) + 8)
    add_requests(w, lens)
    poison_unowned(w)  # page tails past a range end are what a whole-box load streams in
    n_real = len(w.reqs)
    reqs = padded_reqs(w, pad_to)
    ref_md = o_meta.ref_prepare_metadata(w.page_table, reqs, page_size)
    qkv, q, k, v = make_inputs(w, seed + 1, reqs=reqs)
    fused = None
    if mode != "eager":
        cache = ref_cos_sin_cache(D, 4096, 1e6)
        g = torch.Generator().manual_seed(seed)
        qw = (torch.rand(D, generator=g) + 0.5).to(torch.bfloat16)
        kw = (torch.rand(D, generator=g) + 0.5).to(torch.bfloat16)
        q, k, v = ref_pre_attention(qkv, torch.from_numpy(ref_md.positions), HQ, HKV, D, cache, qw, kw, EPS)
        fused = (cache.cuda(), qw.cuda(), kw.cuda(), EPS)
    ref_out, ref_kc, ref_vc = oracle_forward(w, 0, q, k, v, ref_md, reqs=reqs)

    arms = []
    with options(b200, **(SPLIT_PLAN if force_split else {})):
        for exact in (1, 0):
            with options(b200, decode_exact_tail=exact):
                gw = GpuWorld(b200, w)
                arms.append(run_attention(gw, gw.batch("decode", pad_to=pad_to, md=ref_md), qkv.cuda(), fused=fused,
                                          graph=mode == "graph"))
    (o1, plan, k1, v1), (o0, _, k0, v0) = arms
    assert_bits_equal(o1[:n_real], o0[:n_real], "outputs")
    # the whole pool, except the slot the padding requests all append to (many writers)
    keep = torch.ones(k1.shape[0], dtype=torch.bool)
    keep[torch.from_numpy(ref_md.out_loc[n_real:].astype(np.int64))] = False
    assert_bits_equal(k1[keep], k0[keep], "k pool")
    assert_bits_equal(v1[keep], v0[keep], "v pool")
    attn_tolerance_ok(o1[:n_real], ref_out[:n_real], f"exact tail {mode} ps={page_size}")
    slots = torch.from_numpy(ref_md.out_loc[:n_real].astype(np.int64))
    assert_bits_equal(v1[slots], ref_vc[slots], "appended v rows")
    if mode == "eager":  # the fused modes append the roped k row, which the fp32 oracle may round differently
        assert_bits_equal(k1[slots], ref_kc[slots], "appended k rows")
    return plan.cpu()


def _tail_lens(page_size, seed=0):
    """Decode requests whose streamed range n = kv_len - 1 ends at every offset of interest in its last page and
    tile: tail_range_ends(page_size), a last valid row that is the first row of a tile (n mod 128 == 1) and a range
    that ends on a tile boundary (n mod 128 == 0).  Repeated and shuffled so that each CTA runs several units and
    reuses its ring stages (their unloaded rows then hold an earlier tile)."""
    ns = set(tail_range_ends(page_size)) | {128, 129, 256, 257, 385, 512}
    lens = [(n, n + 1) for n in sorted(ns)] * 3
    random.Random(seed).shuffle(lens)
    return lens


@pytest.mark.parametrize("page_size", [8, 16, 32, 64])
def test_exact_tail_every_box_size(b200, native_lib, page_size):
    _check(b200, page_size=page_size, lens=_tail_lens(page_size))


@pytest.mark.parametrize("page_size", [8, 16, 32, 64])
def test_exact_tail_range_is_one_partial_piece(b200, native_lib, page_size):
    """kv_len 2..9: the whole streamed range (1..8 keys) lies in the first piece of the first page."""
    lens = [(n - 1, n) for n in range(2, 10)] * 40
    random.Random(1).shuffle(lens)
    _check(b200, page_size=page_size, lens=lens)


@pytest.mark.parametrize("page_size", [16, 64, 256])
def test_exact_tail_split_kv(b200, native_lib, page_size):
    """Split-KV plans of 128-key chunks: at page size 256 chunk ends fall inside pages; only the last chunk of a
    request stops short of the appended token."""
    lens = _tail_lens(64, seed=2)[:24] + [(1999, 2000), (1500, 1501), (700, 701)]
    plan = _check(b200, page_size=page_size, lens=lens, force_split=True)
    assert int(plan[0]) == 128 and int(plan[1]) > len(lens)  # really split


@pytest.mark.parametrize("page_size", [16, 64])
def test_exact_tail_fused_pre_attention(b200, native_lib, page_size):
    _check(b200, page_size=page_size, lens=_tail_lens(page_size, seed=3), mode="fused")


@pytest.mark.parametrize("page_size", [8, 64])
def test_exact_tail_cuda_graph_replay(b200, native_lib, page_size):
    """Fused launch captured into a CUDA graph and replayed on a padded batch, as bench.py's decode step runs."""
    lens = _tail_lens(page_size, seed=4)[:20]
    _check(b200, page_size=page_size, lens=lens, mode="graph", pad_to=24)
