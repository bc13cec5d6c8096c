"""Exact-answer probes and adversarial softmax regimes for the decode and prefill kernels (oracle/probes.py).

Needles: every (request, query head) attends to one key chosen on a boundary (tile, chunk, page, the cached /
appended split), all other keys score exactly 0, so the output must be that key's V row bit for bit; a failure
names the position and kv head the kernel attended to instead.  Ramps (prefill): every query row must pick its
own position (rising) or key 0 (falling).  Regimes: peaked, flat, drifting and chunk-offset softmaxes against
the fp64 reference's element-wise bound.  Every pool row no request owns, and every slot this forward appends
to, is NaN before the launch."""
import math
import random

import numpy as np
import pytest
import torch

from helpers import (SPLIT_PLAN, GpuWorld, World, add_requests, assert_bits_equal, options, replan, run_attention,
                     table_align, tail_range_ends)
from oracle import metadata as o_meta
from oracle import probes as P

pytestmark = pytest.mark.gpu

D = 128
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
GQA_SHAPES = [(16, 8), (8, 1), (40, 8), (64, 8), (7, 1), (6, 2)]
# kv_len of the decode probe requests: short ranges, a last chunk holding only the appended token (n % 128 == 1
# and n % 256 == 1), the exact-tail range ends of test_gpu_decode_tail.py, long ranges
DECODE_LENS = [1, 2, 3, 9, 129, 130, 257, 258, 385, 513, 1025, 2048]


def _decode_opts(plan, merge=1, impl=1):
    opts = {"decode_impl": impl, "decode_fused_combine": merge}
    if plan == "unsplit":
        opts["decode_plan_nosplit"] = 1
    else:
        opts.update(SPLIT_PLAN)
    return opts


def _world(*, page_size, hq, hkv, dtype, lens, num_pages=None, top=False, seed=0):
    """Page table for `lens` ((cached_len, device_len) per request).  The pool is NaN (a one-element tensor that
    GpuWorld broadcasts on the device, no CPU copy of the pool).  top: the requests' pages are the highest of
    the pool, starting with the last page before the dummy page."""
    need = sum(-(-d // page_size) for _, d in lens)
    num_pages = num_pages or need + 8
    al = table_align(page_size)
    max_seq = -(-(max(d for _, d in lens) + 8) // al) * al
    table = np.zeros((len(lens) + 1, max_seq), dtype=np.int32)
    table[-1, :] = num_pages * page_size
    if top:
        free = [(num_pages - 1 - i) * page_size for i in range(need)]
    else:
        free = [p * page_size for p in range(num_pages)]
        random.Random(seed).shuffle(free)
    w = World(page_size, num_pages, hq, hkv, D, 1, dtype, table, free, torch.full((1,) * 5, math.nan, dtype=dtype), [])
    add_requests(w, lens)
    return w


def _run(b200, w, phase, build, opts):
    """prepare_metadata, then build(chunk) -> (kv, q) with kv = [(k [n, hkv, d], v [n, hkv, d])] per request
    (positions 0..n-1) and q [nnz, hq, d]; rows below cached_len go into the pool, the rest are this
    forward's k / v inputs.  Checks the appended pool rows bit for bit.  Returns (out, kv, q, gw, batch, qkv)."""
    gw = GpuWorld(b200, w)
    md = o_meta.ref_prepare_metadata(w.page_table, w.reqs, w.page_size)
    batch = gw.batch(phase, md=md)
    with options(b200, **opts):
        gw.backend.prepare_metadata(batch)
        chunk = int(batch.attn_metadata.decode_plan[0])
        assert chunk % 128 == 0
        kv, q = build(chunk)
        pool = gw.pool_rows(0)
        idx = torch.cat([torch.from_numpy(w.page_table[t, :c].astype(np.int64)) for (t, c, _) in w.reqs]).cuda()
        for j in range(2):
            pool[j][idx] = torch.cat([x[j][:c] for x, (_, c, _) in zip(kv, w.reqs)]).cuda()
        new = [torch.cat([x[j][c:dl] for x, (_, c, dl) in zip(kv, w.reqs)]) for j in range(2)]
        nnz = q.shape[0]
        qkv = torch.cat([q.reshape(nnz, -1), new[0].reshape(nnz, -1), new[1].reshape(nnz, -1)], 1).cuda()
        out, _, kc, vc = run_attention(gw, batch, qkv, prepare=False)
    slots = batch.out_loc.long()
    assert_bits_equal(kc[slots], new[0], "appended k rows")
    assert_bits_equal(vc[slots], new[1], "appended v rows")
    return out.cpu(), kv, q, gw, batch, qkv


# ------------------------------------------------------------------------------------------- decode needles
def _decode_build(reqs, hq, hkv, dtype, seed, ties=1):
    """build() for needle decode requests [(kv_len, [pos per query head])]; also fills `want` [bs, hq, d]."""
    G = hq // hkv
    want = torch.empty(len(reqs), hq, D, dtype=dtype)

    def build(chunk):
        gen = torch.Generator().manual_seed(seed)
        kv, q = [], torch.zeros(len(reqs), hq, D)
        for r, (n, pos) in enumerate(reqs):
            k = P.probe_keys(gen, n, hkv, dtype, ramp=False)
            v = P.integer_values(gen, n, hkv, dtype)
            for head in range(hq):
                h, g = divmod(head, G)
                tied = list(dict.fromkeys(pos[(head + 5 * j) % hq] for j in range(ties)))
                tied = tied[:4] if len(tied) >= 4 else tied[:2] if len(tied) >= 2 else tied[:1]
                for p in tied:
                    P.plant_needle(k, p, h, g)
                q[r, head] = P.needle_query(g)
                mean = v[tied, h].double().mean(0)
                assert torch.equal(mean.to(dtype).double(), mean)  # the expected output is exact
                want[r, head] = mean.to(dtype)
            kv.append((k, v))
        return kv, q.to(dtype)

    return build, want


def _check_exact(out, want, kv, reqs, hq, hkv, what):
    G = hq // hkv
    bad = ~(out.view(torch.int16) == want.view(torch.int16)).all(-1)
    if bad.any():
        msgs = []
        for r, head in bad.nonzero().tolist()[:8]:
            n, pos = reqs[r]
            msgs.append(f"  request {r} (kv_len {n}) query head {head} (kv head {head // G}, slot {head % G}), needle at "
                        f"{pos[head]}: {P.diagnose(out[r, head], kv[r][1])}")
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} outputs are not their needle's V row\n" + "\n".join(msgs))


def _decode_needles(b200, *, page_size, hq, hkv, dtype, plan, merge=1, impl=1, lens=None, ties=1, seed=0):
    lens = lens or sorted(set(DECODE_LENS) | ({n + 1 for n in tail_range_ends(page_size)} if page_size >= 8 else set()))
    reqs = P.assign_needles(lens, page_size, hq, seed)
    w = _world(page_size=page_size, hq=hq, hkv=hkv, dtype=dtype, lens=[(n - 1, n) for n, _ in reqs], seed=seed)
    build, want = _decode_build(reqs, hq, hkv, dtype, seed, ties)
    out, kv, _, _, batch, _ = _run(b200, w, "decode", build, _decode_opts(plan, merge, impl))
    plan_t = batch.attn_metadata.decode_plan.cpu()
    chunk, total = int(plan_t[0]), int(plan_t[1])
    if plan == "unsplit":
        assert total == len(reqs)
    else:
        assert total > len(reqs)
        # needles on both sides of every chunk boundary, and a last chunk holding only the appended token
        covered = {(n, p) for n, pos in reqs for p in pos}
        for n in lens:
            for c in range(chunk, n, chunk):
                assert (n, c - 1) in covered and (n, c) in covered, (n, c)
        assert any(n > chunk and n % chunk == 1 for n in lens)
    _check_exact(out, want, kv, reqs, hq, hkv, f"decode ps={page_size} {hq}/{hkv} {plan} merge={merge} ties={ties}")


PLAN_MODES = [("unsplit", 1), ("split", 1), ("split", 0), ("split", 2)]
PLAN_IDS = ["unsplit", "split-inkernel-merge", "split-combine-launch", "split-combine-auto"]


@pytest.mark.parametrize("plan,merge", PLAN_MODES, ids=PLAN_IDS)
@pytest.mark.parametrize("page_size", [1, 8, 16, 64, 256])
def test_decode_needles_page_sizes(b200, native_lib, page_size, plan, merge):
    _decode_needles(b200, page_size=page_size, hq=16, hkv=8, dtype=torch.bfloat16, plan=plan, merge=merge)


@pytest.mark.parametrize("plan,merge", PLAN_MODES, ids=PLAN_IDS)
@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("hq,hkv", GQA_SHAPES)
def test_decode_needles_gqa(b200, native_lib, hq, hkv, dtype, plan, merge):
    _decode_needles(b200, page_size=16, hq=hq, hkv=hkv, dtype=DTYPES[dtype], plan=plan, merge=merge,
                    lens=[2, 129, 257, 700, 1025])


@pytest.mark.parametrize("ties", [2, 4])
@pytest.mark.parametrize("plan,merge", PLAN_MODES[:3], ids=PLAN_IDS[:3])
def test_decode_tied_needles(b200, native_lib, plan, merge, ties):
    """Tied needles in different tiles and chunks: the output is their exact mean (a key dropped or counted
    twice, or a chunk weighted wrong, moves it)."""
    _decode_needles(b200, page_size=64, hq=16, hkv=8, dtype=torch.float16, plan=plan, merge=merge, ties=ties,
                    lens=[129, 257, 513, 1025, 2048])


@pytest.mark.parametrize("plan", ["unsplit", "split"])
@pytest.mark.parametrize("page_size", [1, 16])
def test_decode_needles_bringup_kernel(b200, native_lib, page_size, plan):
    _decode_needles(b200, page_size=page_size, hq=16, hkv=8, dtype=torch.bfloat16, plan=plan, impl=0,
                    lens=[2, 129, 257, 1025])


def test_decode_needles_full_size(b200, native_lib):
    """The cfg1 decode shape (256 requests, kv_len U[100, 2048], page size 64, GQA 16/8): every one of the 4096
    outputs is checked exactly, under the default plan and under a plan built for 8192 CTAs (every request split)."""
    rnd = random.Random(0)
    hq, hkv, ps = 16, 8, 64
    reqs = []
    for _ in range(256):
        n = rnd.randint(100, 2048)
        cand = P.boundary_positions(n, ps)
        rnd.shuffle(cand)
        reqs.append((n, [cand[j] if j < len(cand) else rnd.randrange(n) for j in range(hq)]))
    w = _world(page_size=ps, hq=hq, hkv=hkv, dtype=torch.bfloat16, lens=[(n - 1, n) for n, _ in reqs])
    build, want = _decode_build(reqs, hq, hkv, torch.bfloat16, seed=5)
    out, kv, _, gw, batch, qkv = _run(b200, w, "decode", build, {})
    _check_exact(out, want, kv, reqs, hq, hkv, "full size, default plan")
    # re-plan for a much larger grid: every request split into several chunks (partials + merge)
    replan(gw, batch, 8192)
    # the first forward appended the new rows: the pool now holds every key, the inputs stay the same
    out2, plan, _, _ = run_attention(gw, batch, qkv, prepare=False)
    assert int(plan[1]) > len(reqs)
    _check_exact(out2.cpu(), want, kv, reqs, hq, hkv, "full size, 8192-CTA plan")


# ------------------------------------------------------------------------------------------- prefill needles and ramps
PREFILL_LENS = [(0, 200), (100, 300), (37, 200), (129, 400), (256, 700), (1, 140), (0, 1)]


def _prefill_probe(b200, *, page_size, hq, hkv, dtype, lens, opts, seed=0, w=None):
    """Even query heads run needles (positions cached - 1, cached, cached + 127, cached + 128, the last key and
    a few more, one per head), odd heads ramps (rows with (i >> 3) & 1 == 0 rising, the others falling).  A row
    that sees its head's needle must return its V row exactly; a row before the needle must return the
    uniform mean of its visible keys (fp64 reference and bound)."""
    G = hq // hkv
    w = w or _world(page_size=page_size, hq=hq, hkv=hkv, dtype=dtype, lens=lens, seed=seed)
    plan = {}

    def build(chunk):
        gen = torch.Generator().manual_seed(seed)
        rnd = random.Random(seed)
        kv, qs = [], []
        for (_, c, dl) in w.reqs:
            n, ql = dl, dl - c
            k = P.probe_keys(gen, n, hkv, dtype)
            v = P.integer_values(gen, n, hkv, dtype)
            cand = [x for x in dict.fromkeys([c - 1, c, c + 127, c + 128, n - 1, 0, 127, 128, c + ql // 2]) if 0 <= x < n]
            q = torch.zeros(ql, hq, D)
            heads = {}
            for head in range(hq):
                h, g = divmod(head, G)
                if head % 2 == 0:
                    p = cand[(head // 2) % len(cand)] if head // 2 < len(cand) else rnd.randrange(n)
                    P.plant_needle(k, p, h, g)
                    q[:, head] = P.needle_query(g)
                    heads[head] = ("needle", p)
                else:
                    rising = [(i >> 3) & 1 == 0 for i in range(ql)]
                    q[:, head] = torch.stack([P.ramp_query(dtype, r) for r in rising])
                    heads[head] = ("ramp", rising)
            plan[len(kv)] = heads
            kv.append((k, v))
            qs.append(q)
        return kv, torch.cat(qs).to(dtype)

    out, kv, q, _, _, _ = _run(b200, w, "prefill", build, opts)
    off, errors, worst = 0, [], 0.0
    for r, (_, c, dl) in enumerate(w.reqs):
        ql = dl - c
        k, v = kv[r]
        pos = torch.arange(c, dl)
        for head, (kind, arg) in plan[r].items():
            h = head // G
            got = out[off : off + ql, head]
            if kind == "needle":
                sees = pos >= arg
                want = v[arg, h].expand(ql, D)
            else:
                sees = torch.ones(ql, dtype=torch.bool)
                want = torch.stack([v[c + i, h] if up else v[0, h] for i, up in enumerate(arg)])
            bad = sees & ~(got.view(torch.int16) == want.view(torch.int16)).all(-1)
            for i in bad.nonzero().flatten().tolist()[:3]:
                errors.append(f"  request {r} row {i} (position {c + i}) head {head} {kind} "
                              f"{'at ' + str(arg) if kind == 'needle' else ('rising' if arg[i] else 'falling')}: "
                              f"{P.diagnose(got[i], v)}")
            if (~sees).any():  # rows before the needle: the uniform mean of their visible keys
                rows = (~sees).nonzero().flatten()
                ref, _, bound = P.ref_with_bound(q[off + rows, head], k[:, h], v[:, h], dtype, pos[rows] + 1)
                worst = max(worst, P.bound_excess(got[rows], ref, bound))
        off += ql
    assert not errors, f"prefill {opts}: wrong rows\n" + "\n".join(errors[:12])
    assert worst <= P.P16_EXCESS_TOL, f"rows before their needle: excess {worst:.3e}"


@pytest.mark.parametrize("impl,order", [(1, 0), (1, 1), (0, 0)], ids=["tc-sorted", "tc-request-major", "bringup"])
@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("page_size", [1, 16, 64])
def test_prefill_needles_and_ramps(b200, native_lib, page_size, dtype, impl, order):
    _prefill_probe(b200, page_size=page_size, hq=16, hkv=8, dtype=DTYPES[dtype], lens=PREFILL_LENS,
                   opts={"prefill_impl": impl, "prefill_order": order})


@pytest.mark.parametrize("hq,hkv", [(8, 1), (40, 8), (6, 2), (7, 1)])
def test_prefill_needles_and_ramps_gqa(b200, native_lib, hq, hkv):
    _prefill_probe(b200, page_size=16, hq=hq, hkv=hkv, dtype=torch.bfloat16, lens=PREFILL_LENS[:5], opts={})


# ------------------------------------------------------------------------------------------- far pool slots
FAR_SLOTS = (1 << 20) + (1 << 14)


@pytest.mark.parametrize("phase,page_size", [("decode", 1), ("decode", 64), ("prefill", 64)],
                         ids=["decode-row-mode", "decode-box-mode", "prefill"])
def test_needles_in_far_pool_slots(b200, native_lib, phase, page_size):
    """A pool of 2^20 + 2^14 slots at 8 kv heads (each K and V slice past 2^31 bytes), built on the device;
    the requests' pages are the highest of the pool, up to the last page before the dummy page."""
    hq, hkv, dtype = 16, 8, torch.bfloat16
    need = 2 * (FAR_SLOTS + page_size) * hkv * D * 2
    if torch.cuda.mem_get_info()[0] < 2 * need:
        pytest.skip(f"needs {2 * need / 2**30:.1f} GiB of free device memory (the card is shared)")
    num_pages = FAR_SLOTS // page_size
    if phase == "decode":
        reqs = P.assign_needles([2, 129, 257, 1025], page_size, hq)
        w = _world(page_size=page_size, hq=hq, hkv=hkv, dtype=dtype, lens=[(n - 1, n) for n, _ in reqs],
                   num_pages=num_pages, top=True)
        assert w.page_table[0, 0] == (num_pages - 1) * page_size
        build, want = _decode_build(reqs, hq, hkv, dtype, seed=3)
        for plan in ("unsplit", "split"):
            out, kv, _, gw, _, _ = _run(b200, w, "decode", build, _decode_opts(plan))
            _check_exact(out, want, kv, reqs, hq, hkv, f"far slots ps={page_size} {plan}")
            del gw
            b200.core.set_global_ctx(None)
            torch.cuda.empty_cache()
    else:
        w = _world(page_size=page_size, hq=hq, hkv=hkv, dtype=dtype, lens=PREFILL_LENS[:5], num_pages=num_pages,
                   top=True)
        _prefill_probe(b200, page_size=page_size, hq=hq, hkv=hkv, dtype=dtype, lens=None, opts={}, w=w)
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------- adversarial regimes
@pytest.mark.parametrize("mode", ["unsplit", "split", "prefill"])
@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("name", P.REGIMES)
def test_softmax_regimes_within_bound(b200, native_lib, name, dtype, mode):
    """Every output within the fp64 reference's element-wise bound (oracle/probes.py) up to P16_EXCESS_TOL of
    the (request, head)'s max |out|."""
    hq, hkv, dt = 16, 8, DTYPES[dtype]
    G = hq // hkv
    if mode == "prefill":
        lens, opts, phase = [(256, 556), (0, 300), (100, 101 + 130)], {}, "prefill"
    else:
        lens, opts, phase = [(n - 1, n) for n in (700, 1100, 2048)], _decode_opts(mode), "decode"
    w = _world(page_size=16, hq=hq, hkv=hkv, dtype=dt, lens=lens)

    def build(chunk):
        gen = torch.Generator().manual_seed(11)
        kv, qs = [], []
        for (_, c, dl) in w.reqs:
            q, k, v = P.regime_request(name, gen, dl, dl - c, hq, hkv, dt, block=chunk if mode == "split" else 128)
            kv.append((k, v))
            qs.append(q)
        return kv, torch.cat(qs)

    out, kv, q, _, _, _ = _run(b200, w, phase, build, opts)
    worst, where, off = 0.0, None, 0
    for r, (_, c, dl) in enumerate(w.reqs):
        ql = dl - c
        k, v = kv[r]
        for head in range(hq):
            h = head // G
            ref, _, bound = P.ref_with_bound(q[off : off + ql, head], k[:, h], v[:, h], dt, torch.arange(c + 1, dl + 1))
            e = P.bound_excess(out[off : off + ql, head], ref, bound)
            if e > worst:
                worst, where = e, (r, head)
        off += ql
    assert worst <= P.P16_EXCESS_TOL, f"{name} {dtype} {mode}: excess {worst:.3e} at (request, head) {where}"
