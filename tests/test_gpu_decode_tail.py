"""Exact-tail K/V loads of the decode kernel (option decode_exact_tail): at page sizes >= 8 the page piece that holds
the end of a KV range is loaded only up to its last valid row (8-row boxes), pieces past the end are not loaded, and
the stage rows left unwritten keep whatever an earlier tile put there.  Every case runs the launch with the option at
1 and at 0 on a pool whose unowned rows are NaN, requires the two to agree bit for bit (output, appended rows, the
rest of the pool) and checks the output against the oracle."""
import random

import numpy as np
import pytest
import torch

from helpers import GpuWorld, add_requests, attn_tolerance_ok, make_inputs, make_world, options, oracle_forward
from oracle import metadata as o_meta

pytestmark = pytest.mark.gpu

HQ, HKV, D = 16, 8, 128
EPS = 1e-6


def _box_rows(page_size):
    rb = 64
    while page_size % rb:
        rb >>= 1
    return rb


def _run_arm(b200, w, ref_md, qkv, exact, mode, pad_to, pre):
    with options(b200, decode_exact_tail=exact):
        try:
            gw = GpuWorld(b200, w)
            backend = gw.backend
            x = qkv.cuda()
            bs = x.shape[0]
            positions = torch.from_numpy(ref_md.positions).cuda()
            out_loc = torch.from_numpy(ref_md.out_loc).cuda()
            if mode == "graph":
                # captured like the engine's decode graphs: the K/V producers start before the predecessor finishes
                backend.init_capture_graph(w.page_table.shape[1], [bs])
                dummy = b200.Req(table_idx=w.page_table.shape[0] - 1, cached_len=0, device_len=1)
                qkv_buf = torch.zeros_like(x)
                pos_buf = torch.zeros(bs, dtype=torch.int32, device="cuda")
                loc_buf = torch.full((bs,), int(w.page_table[-1, 0]), dtype=torch.int32, device="cuda")
                out_buf = torch.zeros(bs, HQ, D, dtype=x.dtype, device="cuda")
                cap = b200.Batch([dummy] * bs, "decode")
                cap.padded_reqs = cap.reqs
                backend.prepare_for_capture(cap)
                cap.out_loc, cap.positions = loc_buf, pos_buf

                def run():
                    q, k, v = qkv_buf.split([HQ * D, HKV * D, HKV * D], dim=-1)
                    out_buf.copy_(backend.forward_decode_fused(q.view(-1, HQ, D), k, v, 0, cap, pos_buf, *pre))

                stream = torch.cuda.Stream()
                with torch.cuda.stream(stream):
                    run()
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph, stream=stream):
                        run()
                torch.cuda.synchronize()
                batch = gw.batch("decode", pad_to=pad_to)
                batch.out_loc, batch.positions = out_loc, positions
                backend.prepare_metadata(batch)
                with torch.cuda.stream(stream):
                    qkv_buf.copy_(x)
                    pos_buf.copy_(positions)
                    loc_buf.copy_(out_loc)
                    backend.prepare_for_replay(batch)
                    graph.replay()
                out = out_buf
            else:
                batch = gw.batch("decode", pad_to=pad_to)
                batch.out_loc, batch.positions = out_loc, positions
                backend.prepare_metadata(batch)
                q, k, v = x.split([HQ * D, HKV * D, HKV * D], dim=-1)
                if mode == "fused":
                    out = backend.forward_decode_fused(q.view(-1, HQ, D), k, v, 0, batch, positions, *pre)
                else:
                    out = backend.forward(q.view(-1, HQ, D), k, v, 0, batch)
            torch.cuda.synchronize()
            plan = batch.attn_metadata.decode_plan.cpu()
            kc, vc = gw.pool_rows(0)
            return out.cpu(), kc, vc, plan
        finally:
            b200.core.set_global_ctx(None)


def _check(b200, *, page_size, lens, mode="eager", pad_to=None, force_split=False, seed=0):
    """Runs `lens` ((kv_len - 1, kv_len) decode requests) with decode_exact_tail 1 and 0; returns the plan."""
    from oracle.layer import ref_pre_attention
    from oracle.rope import ref_cos_sin_cache

    w = make_world(seed=seed, page_size=page_size, hq=HQ, hkv=HKV, max_reqs=max(len(lens), pad_to or 0) + 1,
                   max_seq=max(d for _, d in lens) + 8)
    add_requests(w, lens)
    # every pool row no request owns is NaN: page tails past a range end are what a whole-box load streams in
    used = np.zeros(w.pool_cpu.shape[2], dtype=bool)
    for (t, _, d) in w.reqs:
        used[w.page_table[t, :d]] = True
    w.pool_cpu[:, :, torch.from_numpy(~used)] = float("nan")
    n_real = len(w.reqs)
    triples = list(w.reqs) + [(w.page_table.shape[0] - 1, 0, 1)] * ((pad_to or 0) - n_real)
    ref_md = o_meta.ref_prepare_metadata(w.page_table, triples, page_size)
    saved, w.reqs = w.reqs, triples
    qkv, q, k, v = make_inputs(w, seed + 1)
    pre = ()
    if mode != "eager":
        cache = ref_cos_sin_cache(D, 4096, 1e6)
        g = torch.Generator().manual_seed(seed)
        qw = (torch.rand(D, generator=g) + 0.5).to(torch.bfloat16)
        kw = (torch.rand(D, generator=g) + 0.5).to(torch.bfloat16)
        q, k, v = ref_pre_attention(qkv, torch.from_numpy(ref_md.positions), HQ, HKV, D, cache, qw, kw, EPS)
        pre = (cache.cuda(), qw.cuda(), kw.cuda(), EPS)
    ref_out, ref_kc, ref_vc = oracle_forward(w, 0, q, k, v, ref_md)
    w.reqs = saved

    # force_split: split every request into 128-key chunks (as many items as the policy allows)
    with options(b200, **({"decode_plan_nosplit": 0, "decode_plan_target": 16} if force_split else {})):
        (o1, k1, v1, plan), (o0, k0, v0, _) = [_run_arm(b200, w, ref_md, qkv, arm, mode, pad_to, pre) for arm in (1, 0)]
    assert torch.equal(o1[:n_real].view(torch.int16), o0[:n_real].view(torch.int16)), \
        f"outputs differ: max |d| {(o1[:n_real].float() - o0[:n_real].float()).abs().max().item():.3e}"
    # the whole pool, except the slot the padding requests all append to (many writers)
    keep = torch.ones(k1.shape[0], dtype=torch.bool)
    keep[torch.from_numpy(ref_md.out_loc[n_real:].astype(np.int64))] = False
    assert torch.equal(k1[keep].view(torch.int16), k0[keep].view(torch.int16))
    assert torch.equal(v1[keep].view(torch.int16), v0[keep].view(torch.int16))
    attn_tolerance_ok(o1[:n_real], ref_out[:n_real], f"exact tail {mode} ps={page_size}")
    slots = torch.from_numpy(ref_md.out_loc[:n_real].astype(np.int64))
    assert torch.equal(v1[slots].view(torch.int16), ref_vc[slots].view(torch.int16))
    if mode == "eager":  # the fused modes append the roped k row, which the fp32 oracle may round differently
        assert torch.equal(k1[slots].view(torch.int16), ref_kc[slots].view(torch.int16))
    return plan


def _tail_lens(page_size, seed=0):
    """Decode requests whose streamed range n = kv_len - 1 ends at every offset of interest in its last page and
    tile: n mod page_size in {0, 1, 7, 8, 9, box_rows - 1, page_size - 1}, a last valid row that is the first row of
    a tile (n mod 128 == 1) and a range that ends on a tile boundary (n mod 128 == 0).  Repeated and shuffled so that
    each CTA runs several units and reuses its ring stages (their unloaded rows then hold an earlier tile)."""
    rb = _box_rows(page_size)
    ns = {k * page_size + r for k in (2, 5) for r in (0, 1, 7, 8, 9, rb - 1, page_size - 1)}
    ns |= {128, 129, 256, 257, 385, 512}
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
