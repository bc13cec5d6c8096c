"""The event trace of the decode and prefill attention kernels on the GPU: a traced launch computes the same bits as
an untraced one (outputs, appended K/V rows, untouched NaN pool rows) with the same number of launches; its events
agree with the plan it ran (every unit once per role, the unit's tiles, the split-KV merges, per-warp time order);
and the buffer limits hold (overflow counted, nothing written past a region, launches past the buffer untraced,
nothing written after tracing is turned off)."""
import ctypes as C
import importlib

import numpy as np
import pytest
import torch

from helpers import (SPLIT_PLAN, GpuWorld, add_requests, assert_bits_equal, make_inputs, make_world, options,
                     padded_reqs, poison_unowned, run_attention)
from oracle import metadata as o_meta

pytestmark = pytest.mark.gpu
tr = importlib.import_module("mini-sglang_b200.trace")

EPW = 2048  # events per warp: enough for every launch below
DECODE_LENS = [(99, 100), (511, 512), (1023, 1024), (256, 257), (700, 701), (64, 65), (1, 2), (1500, 1501),
               (0, 1), (127, 128), (128, 129), (2999, 3000)]
PLANS = {"default": {}, "split": SPLIT_PLAN, "unsplit": {"decode_plan_nosplit": 1}}


class Case:
    """One attention call on a fresh, NaN-poisoned world; run() returns (out, plan, pool K, pool V, launches)."""

    def __init__(self, b200, *, phase, page_size, hq, hkv, lens, dtype=torch.bfloat16, fused=False, graph=False,
                 share_prefix=None, pad_to=None, seed=0):
        self.b200, self.phase, self.ps, self.hq, self.hkv = b200, phase, page_size, hq, hkv
        self.lens, self.dtype, self.fused, self.graph = lens, dtype, fused, graph
        self.share_prefix, self.pad_to, self.seed = share_prefix, pad_to, seed

    def world(self):
        w = make_world(seed=self.seed, page_size=self.ps, hq=self.hq, hkv=self.hkv, dtype=self.dtype,
                       max_reqs=max(len(self.lens), self.pad_to or 0) + 1, max_seq=max(d for _, d in self.lens) + 8)
        add_requests(w, self.lens, share_prefix_from=self.share_prefix)
        poison_unowned(w)
        return w

    def run(self):
        w = self.world()
        reqs = padded_reqs(w, self.pad_to)
        md = o_meta.ref_prepare_metadata(w.page_table, reqs, self.ps)
        qkv = make_inputs(w, self.seed + 1, reqs=reqs)[0].cuda()
        gw = GpuWorld(self.b200, w)
        fused = None
        if self.fused:
            from oracle.rope import ref_cos_sin_cache

            g = torch.Generator().manual_seed(5)
            qw = (torch.rand(128, generator=g) + 0.5).to(self.dtype).cuda()
            kw = (torch.rand(128, generator=g) + 0.5).to(self.dtype).cuda()
            fused = (ref_cos_sin_cache(128, 8192, 1e6).cuda(), qw, kw, 1e-6)
        batch = gw.batch(self.phase, pad_to=self.pad_to, md=md)
        gw.backend.prepare_metadata(batch)
        torch.cuda.synchronize()
        before = self.b200._cabi.launch_count()
        out, plan, kc, vc = run_attention(gw, batch, qkv, fused=fused, graph=self.graph, prepare=False)
        launches = self.b200._cabi.launch_count() - before
        md_dev = batch.attn_metadata
        extra = {"plan": plan.cpu().numpy().copy(), "seq_lens": md_dev.cache_seqlens.cpu().numpy().copy(),
                 "prefill_plan": getattr(md_dev, "prefill_plan", None), "cu_q": md_dev.cu_seqlens_q.cpu().numpy().copy(),
                 "owned": _owned(w)}
        if extra["prefill_plan"] is not None:
            extra["prefill_plan"] = extra["prefill_plan"].cpu().numpy().copy()
        return out, kc, vc, launches, extra


def _owned(w):
    used = np.zeros(w.pool_cpu.shape[2], dtype=bool)
    for (t, _, d) in w.reqs:
        used[w.page_table[t, :d]] = True
    return used


def _traced_equals_untraced(b200, case, epw=EPW):
    out0, kc0, vc0, n0, extra = case.run()
    with tr.AttentionTrace(4, epw) as t:
        out1, kc1, vc1, n1, _ = case.run()
        launches = t.launches()
        counts = t.counts()
    assert_bits_equal(out1, out0, "output")
    assert_bits_equal(kc1, kc0, "pool K")
    assert_bits_equal(vc1, vc0, "pool V")
    free = torch.from_numpy(~extra["owned"]).cuda()
    free[-case.ps:] = False  # the dummy page: the padding requests append there
    assert torch.isnan(kc1[free].float()).all() and torch.isnan(vc1[free].float()).all(), "unowned pool rows"
    assert n1 == n0, f"launches per call: {n1} traced vs {n0} untraced"
    assert counts[0] >= 1 and counts[1] == 0 and len(launches) == counts[0]
    return launches, extra


def _check_warp_order(launch):
    for c in range(launch.header["grid"]):
        for w in range(launch.header["warps"]):
            ev = launch.warp_events(c, w)
            assert len(ev) >= 2 and ev["code"][0] == tr.BEGIN and ev["code"][-1] == tr.END, (c, w)
            assert (np.diff(ev["ns"].astype(np.int64)) >= 0).all(), f"time runs backwards in CTA {c} warp {w}"
    assert not launch.overflow


def _cta_units(total, grid, cta):
    k, out = 0, []
    while True:
        pos = k * grid + ((grid - 1 - cta) if k & 1 else cta)
        if pos >= total:
            return out
        out.append(pos)
        k += 1


def _unit_tiles(ev, count_codes):
    """{k: number of events with a code in count_codes between unit k's begin and end}; every unit is begun once and
    ended before the next one begins."""
    res, cur = {}, None
    for code, arg in zip(ev["code"].tolist(), ev["arg"].tolist()):
        if code == tr.UNIT_BEGIN:
            assert cur is None and arg not in res, f"unit {arg} begun again (open unit: {cur})"
            cur = arg
            res[cur] = 0
        elif code == tr.UNIT_END:
            assert cur == arg, f"unit {arg} ended while unit {cur} was open"
            cur = None
        elif cur is not None and code in count_codes:
            res[cur] += 1
    return res


def _check_decode_plan(launch, extra, hkv):
    plan, seq_lens = extra["plan"], extra["seq_lens"]
    chunk, total_chunks, bs = int(plan[0]), int(plan[1]), int(plan[2])
    order = plan[4 + bs + 1: 4 + bs + 1 + total_chunks]
    grid, box = launch.header["grid"], launch.header["box_rows"] > 0
    assert launch.header["plan_kind"] == int(total_chunks != bs)
    n_split_units, split_pairs = 0, set()
    for c in range(grid):
        tiles = []
        for pos in _cta_units(total_chunks * hkv, grid, c):
            e = int(order[pos // hkv])
            r, ch, n = e & 0xFFFF, (e >> 16) & 0xF, (e >> 20) & 0x1F
            kv_len = int(seq_lens[r])
            begin, end = ch * chunk, min(kv_len, ch * chunk + chunk)
            end_tc = end - 1 if ch == n - 1 else end
            tiles.append(max(0, -(-(end_tc - begin) // 128)))
            if n > 1:
                n_split_units += 1
                split_pairs.add((r, pos % hkv))
        want = {k: t for k, t in enumerate(tiles)}
        for w in range(4, 8):
            assert _unit_tiles(launch.warp_events(c, w), {tr.PV}) == want, f"consumer warp {w} of CTA {c}"
            assert _unit_tiles(launch.warp_events(c, w), {tr.Q_READY}) == {k: int(t > 0) for k, t in want.items()}
        producers = (0, 1) if box else (0, 1, 2, 3)
        for w in producers:
            assert _unit_tiles(launch.warp_events(c, w), {tr.ISSUED}) == want, f"producer warp {w} of CTA {c}"
        assert set(_unit_tiles(launch.warp_events(c, 8), set())) == set(want), f"Q loader of CTA {c}"
        if launch.header["flags"] & tr.FLAG_IN_KERNEL_COMBINE:
            assert set(_unit_tiles(launch.warp_events(c, 9), set())) == set(want), f"combiner of CTA {c}"
    if launch.header["flags"] & tr.FLAG_IN_KERNEL_COMBINE:
        codes = launch.events["code"]
        assert int((codes == tr.ARRIVE_LAST).sum()) == len(split_pairs)
        assert int((codes == tr.MERGE_BEGIN).sum()) == len(split_pairs)
        assert int(((codes == tr.ARRIVE) | (codes == tr.ARRIVE_LAST)).sum()) == n_split_units


def _check_prefill_plan(launch, extra, hq):
    plan, seq_lens, cu_q = extra["prefill_plan"], extra["seq_lens"], extra["cu_q"]
    n_items, grid = int(plan[0]), launch.header["grid"]
    for c in range(grid):
        want = {}
        for k, pos in enumerate(_cta_units(n_items * hq, grid, c)):
            e = int(plan[4 + pos // hq])
            r, q_start = e & 0xFFFF, ((e >> 16) & 0xFFFF) * 128
            q_len, kv_len = int(cu_q[r + 1] - cu_q[r]), int(seq_lens[r])
            kv_hi = min(kv_len, kv_len - q_len + min(q_len, q_start + 128))
            want[k] = -(-kv_hi // 128)
        for w in range(4, 12):
            assert _unit_tiles(launch.warp_events(c, w), {tr.PV, tr.SKIP}) == want, f"consumer warp {w} of CTA {c}"
        for w in (0, 1):
            assert _unit_tiles(launch.warp_events(c, w), {tr.ISSUED}) == want, f"producer warp {w} of CTA {c}"


@pytest.mark.parametrize("page_size", [1, 16, 64])
@pytest.mark.parametrize("group", [2, 8, 12, 16])
@pytest.mark.parametrize("plan", sorted(PLANS))
def test_decode_traced_is_bit_identical_and_matches_the_plan(b200, page_size, group, plan):
    hkv = 2
    with options(b200, **PLANS[plan]):
        case = Case(b200, phase="decode", page_size=page_size, hq=group * hkv, hkv=hkv, lens=DECODE_LENS)
        launches, extra = _traced_equals_untraced(b200, case)
    (launch,) = launches
    assert launch.phase == "decode" and launch.header["group"] == group and launch.header["page_size"] == page_size
    _check_warp_order(launch)
    _check_decode_plan(launch, extra, hkv)
    if plan == "split":
        assert launch.header["plan_kind"] == 1


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("page_size", [1, 64])
def test_fused_decode_traced_is_bit_identical(b200, dtype, page_size):
    case = Case(b200, phase="decode", page_size=page_size, hq=16, hkv=2, lens=DECODE_LENS, dtype=dtype, fused=True)
    (launch,), extra = _traced_equals_untraced(b200, case)
    assert launch.header["flags"] & tr.FLAG_FUSED
    _check_warp_order(launch)
    _check_decode_plan(launch, extra, 2)


def test_fp16_decode_traced_is_bit_identical(b200):
    case = Case(b200, phase="decode", page_size=16, hq=8, hkv=1, lens=DECODE_LENS, dtype=torch.float16)
    (launch,), _ = _traced_equals_untraced(b200, case)
    _check_warp_order(launch)


@pytest.mark.parametrize("page_size", [1, 64])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_prefill_traced_is_bit_identical_and_matches_the_plan(b200, page_size, dtype):
    # a radix-shared prefix (requests 1 and 2 reuse request 0's cached pages) and a 4096-row prompt
    lens = [(300, 700), (256, 400), (128, 129), (0, 4096), (0, 77)]
    case = Case(b200, phase="prefill", page_size=page_size, hq=16, hkv=2, lens=lens, dtype=dtype, share_prefix=0)
    (launch,), extra = _traced_equals_untraced(b200, case, epw=4096)
    assert launch.phase == "prefill"
    _check_warp_order(launch)
    _check_prefill_plan(launch, extra, 16)
    codes = launch.events["code"]
    assert (codes == tr.APPEND).any() and (codes == tr.SKIP).any() and (codes == tr.Q_ISSUED).any()


def test_graph_capture_and_replay_rewrite_the_captured_region(b200):
    case = Case(b200, phase="decode", page_size=16, hq=16, hkv=8, lens=[(99, 100), (511, 512), (300, 301)],
                graph=True, pad_to=4)
    launches, _ = _traced_equals_untraced(b200, case)
    # the warm-up launch and the captured one (written by the replay); the captured launch streams K/V early
    assert [l.header["seq"] for l in launches] == [0, 1]
    assert launches[1].header["flags"] & tr.FLAG_EARLY_KV
    for l in launches:
        _check_warp_order(l)


def _lib(b200):
    return b200._cabi.load()


def _trace_counts(lib):
    t, u = C.c_uint64(), C.c_uint64()
    assert lib.b200_attn_trace_launches(C.byref(t), C.byref(u)) == 0
    return t.value, u.value


def test_small_events_per_warp_overflows_inside_its_region(b200):
    lib = _lib(b200)
    case = Case(b200, phase="decode", page_size=64, hq=16, hkv=2, lens=DECODE_LENS)
    out0, kc0, _, _, _ = case.run()
    epw, guard = 8, 1 << 16
    one = lib.b200_attn_trace_launch_bytes(0, epw)
    buf = torch.zeros(one + guard, dtype=torch.uint8, device="cuda")
    buf[one:] = 0x5A
    torch.cuda.synchronize()
    try:
        assert lib.b200_attn_trace_set(buf.data_ptr(), one, epw) == 0
        out1, kc1, _, _, _ = case.run()
        assert _trace_counts(lib) == (1, 0)
    finally:
        assert lib.b200_attn_trace_set(None, 0, 0) == 0
    assert_bits_equal(out1, out0, "output")
    assert_bits_equal(kc1, kc0, "pool K")
    assert (buf[one:] == 0x5A).all(), "the trace wrote past its region"
    (launch,) = tr.decode_buffer(buf[:one].cpu().numpy().tobytes())
    assert launch.overflow and int(launch.counts.max()) > epw
    assert len(launch.warp_events(0, 4)) == epw


def test_launches_past_the_buffer_run_untraced(b200):
    lib = _lib(b200)
    case = Case(b200, phase="decode", page_size=16, hq=16, hkv=2, lens=DECODE_LENS)
    ref = case.run()[0]
    one = lib.b200_attn_trace_launch_bytes(0, EPW)
    buf = torch.zeros(2 * one, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    try:
        assert lib.b200_attn_trace_set(buf.data_ptr(), buf.numel(), EPW) == 0
        outs = [case.run() for _ in range(3)]
        assert _trace_counts(lib) == (2, 1)
    finally:
        assert lib.b200_attn_trace_set(None, 0, 0) == 0
    for o in outs:
        assert_bits_equal(o[0], ref, "output")
        assert o[3] == outs[0][3]
    assert [l.header["seq"] for l in tr.decode_buffer(buf.cpu().numpy().tobytes())] == [0, 1]


def test_nothing_is_written_after_tracing_is_turned_off(b200):
    lib = _lib(b200)
    case = Case(b200, phase="prefill", page_size=64, hq=16, hkv=2, lens=[(0, 300), (64, 200)])
    buf = torch.zeros(lib.b200_attn_trace_launch_bytes(1, EPW), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert lib.b200_attn_trace_set(buf.data_ptr(), buf.numel(), EPW) == 0
    assert lib.b200_attn_trace_set(None, 0, 0) == 0
    case.run()
    case.run()
    assert int(buf.count_nonzero()) == 0
    assert _trace_counts(lib) == (0, 0)
