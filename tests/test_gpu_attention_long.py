"""Attention at serving-length contexts: decode over 8 193 to 40 960 keys (the Qwen3 models' max_position) and
chunked prefill of 8 192 rows on a 32 768-key cached prefix, where a work unit streams hundreds of K/V tiles
(hundreds of online-softmax rescales and ring-phase flips), fp32 sums run over tens of thousands of keys, the
decode plan's size sort clamps at 127 tiles and CUDA-graph capture data is as wide as the longest context.

Every case is built on the device: a NaN pool (GpuWorld broadcasts one element), of which only the rows the
requests own are written; after every launch the owned rows must hold exactly what was written plus the
appended rows, and every other row must still be NaN.  The checks: needles placed from the plan the metadata
kernel actually built (both sides of every chunk boundary, the first and last tile, the last cached and the
appended key, random keys; four tied needles per query head), adversarial softmax regimes against the fp64
reference's bound (oracle/probes.py: the full reference for decode, sampled rows for prefill), prefill needles
and bf16 ramps.  Each case keeps its pool at about 1 GiB or less, and skips when the shared card has less free
memory than twice that."""
import math
import random

import numpy as np
import pytest
import torch

from helpers import (SPLIT_PLAN, GpuWorld, assert_bits_equal, check_decode_plan, check_prefill_plan, options,
                     run_attention)
from oracle import metadata as o_meta
from oracle import probes as P
from test_gpu_attention_probes import _world

pytestmark = pytest.mark.gpu

D = 128
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
# kv_len of the decode requests: one tile past 8192, the last length below the plan's 127-tile sort clamp and
# the first at it (unsplit: 127 tiles each), past the clamp, a full 2^15 range, the models' max_position
LONG_LENS = [8193, 16256, 16257, 16384 + 129, 32768, 40960]
DECODE_REGIMES = ["temp0", "temp16", "drift_up", "drift_down", "chunk_maxima"]
TIES = 4          # tied needles per query head: their exact mean is the expected output
N_RANDOM = 8      # random needle positions per request length
MAX_SPLITS = 16   # chunks per request the plan never exceeds


def _need_memory(nbytes: int):
    free = torch.cuda.mem_get_info()[0]
    if free < 2 * nbytes:  # leave as much again to the card's other users
        pytest.skip(f"needs {2 * nbytes / 2**30:.1f} GiB of free device memory (the card is shared)")


def _decode_opts(plan, merge=1):
    if plan == "default":
        return {"decode_fused_combine": merge}
    opts = {"decode_impl": 1, "decode_fused_combine": merge}
    opts.update({"decode_plan_nosplit": 1} if plan == "unsplit" else SPLIT_PLAN)
    return opts


class LongCase:
    """One batch of `lens` ((cached_len, kv_len) per request) over a NaN pool on the device; `launch` writes the
    requests' K/V rows (device tensors), runs one attention launch and checks the pool."""

    def __init__(self, b200, *, page_size, hq, hkv, dtype, lens, phase, seed=0):
        pool_bytes = 2 * sum(d for _, d in lens) * hkv * D * 2
        _need_memory(3 * pool_bytes // 2 + (256 << 20))  # the pool and the requests' K/V rows
        self.b200, self.hq, self.hkv, self.dtype, self.phase = b200, hq, hkv, dtype, phase
        self.w = _world(page_size=page_size, hq=hq, hkv=hkv, dtype=dtype, lens=lens, seed=seed)
        self.md = o_meta.ref_prepare_metadata(self.w.page_table, self.w.reqs, page_size)
        self.gw = GpuWorld(b200, self.w)
        self.batch = self.gw.batch(phase, md=self.md)
        self.slots = [torch.from_numpy(self.w.page_table[t, :d].astype(np.int64)).cuda() for (t, _, d) in self.w.reqs]
        owned = torch.zeros(self.gw.pool_rows(0)[0].shape[0], dtype=torch.bool, device="cuda")
        for s in self.slots:
            owned[s] = True
        owned[self.w.num_pages * page_size :] = True  # the dummy page: graph capture's dummy requests append there
        self.unowned = ~owned
        self.nan_bits = torch.full((1,), math.nan, dtype=dtype).view(torch.int16).item()

    def prepare(self, request_major=False):
        """prepare_metadata under the caller's options (request_major: prefill_order = 1 is among them); checks
        the metadata, the decode plan and the prefill plan; returns the decode plan's chunk size."""
        self.gw.backend.prepare_metadata(self.batch)
        md = self.batch.attn_metadata
        torch.cuda.synchronize()
        assert np.array_equal(md.cache_seqlens.cpu().numpy(), self.md.cache_seqlens)
        assert np.array_equal(md.page_table[:, : self.md.max_seqlen_k].cpu().numpy(), self.md.slot_table)
        check_decode_plan(md.decode_plan.cpu().numpy(), self.md.cache_seqlens)
        if md.prefill_plan is not None:
            check_prefill_plan(md.prefill_plan.cpu().numpy(), self.w.reqs, request_major)
        return int(md.decode_plan[0])

    def qkv(self, kv, q):
        """qkv rows [nnz, (hq + 2 hkv) d] of this forward's tokens; writes the cached rows into the pool."""
        kc, vc = self.gw.pool_rows(0)
        new_k, new_v = [], []
        for (k, v), s, (_, c, _) in zip(kv, self.slots, self.w.reqs):
            kc[s[:c]] = k[:c]
            vc[s[:c]] = v[:c]
            new_k.append(k[c:])
            new_v.append(v[c:])
        nnz = q.shape[0]
        return torch.cat([q.reshape(nnz, -1), torch.cat(new_k).reshape(nnz, -1), torch.cat(new_v).reshape(nnz, -1)], 1)

    def check_unowned(self, what=""):
        """Every pool row no request owns is still the NaN it was."""
        for name, x in zip("kv", self.gw.pool_rows(0)):
            bad = (x[self.unowned].view(torch.int16) != self.nan_bits).any(-1).any(-1)
            assert not bad.any(), f"{what}: {int(bad.sum())} {name} pool rows nobody owns were written"

    def check_pool(self, kv, what=""):
        """Owned rows: what was written and appended, bit for bit; every other row: untouched NaN."""
        self.check_unowned(what)
        kc, vc = self.gw.pool_rows(0)
        for r, ((k, v), s) in enumerate(zip(kv, self.slots)):
            c = self.w.reqs[r][1]
            assert_bits_equal(kc[s[c:]], k[c:], f"{what} request {r}: appended k rows")
            assert_bits_equal(vc[s[c:]], v[c:], f"{what} request {r}: appended v rows")
            assert torch.equal(kc[s[:c]].view(torch.int16), k[:c].view(torch.int16)), f"{what} request {r}: cached k rows moved"
            assert torch.equal(vc[s[:c]].view(torch.int16), v[:c].view(torch.int16)), f"{what} request {r}: cached v rows moved"

    def launch(self, kv, q, what="", **kw):
        out, _, _, _ = run_attention(self.gw, self.batch, self.qkv(kv, q), prepare=False, **kw)
        self.check_pool(kv, what)
        return out


# ------------------------------------------------------------------------------------------- decode
def _copies(hq):
    """Requests per length so that every plan position fits: 8 + 2 (MAX_SPLITS - 1) positions plus the random ones."""
    return -(-(8 + 2 * (MAX_SPLITS - 1) + N_RANDOM) // (hq * TIES))


def _decode_needles(case: LongCase, chunk, seed, **kw):
    hq, hkv, dt = case.hq, case.hkv, case.dtype
    G = hq // hkv
    lens = [d for _, _, d in case.w.reqs]
    reqs = P.assign_plan_needles(lens, chunk, hq, seed, TIES, N_RANDOM)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    kv, q = [], torch.zeros(len(reqs), hq, D, device="cuda")
    want = torch.empty(len(reqs), hq, D, dtype=dt, device="cuda")
    for r, (n, pos) in enumerate(reqs):
        k = torch.randn((n, hkv, D), generator=gen, device="cuda")
        k[..., : P.PROBE_DIMS] = 0
        v = torch.randint(-P.V_MAX, P.V_MAX + 1, (n, hkv, D), generator=gen, device="cuda").to(dt)
        for head in range(hq):
            h, g = divmod(head, G)
            k[pos[head], h, P.needle_dim(g)] = P.NEEDLE_K
            q[r, head] = P.needle_query(g).cuda()
            mean = v[pos[head], h].double().mean(0)
            assert torch.equal(mean.to(dt).double(), mean)  # the expected output is exact
            want[r, head] = mean.to(dt)
        kv.append((k.to(dt), v))
    out = case.launch(kv, q.to(dt), "needles", **kw)
    bad = ~(out.view(torch.int16) == want.view(torch.int16)).all(-1)
    if bad.any():
        msgs = []
        for r, head in bad.nonzero().tolist()[:8]:
            n, pos = reqs[r]
            msgs.append(f"  request {r} (kv_len {n}) query head {head}: tied needles at {sorted(pos[head])}, "
                        f"max |out - want| {(out[r, head].float() - want[r, head].float()).abs().max().item():.3g}")
        raise AssertionError(f"needles: {int(bad.sum())} of {bad.numel()} outputs are not their needles' mean\n" + "\n".join(msgs))
    return reqs


def _decode_regime(case: LongCase, name, chunk, seed, split):
    hq, hkv, dt = case.hq, case.hkv, case.dtype
    G = hq // hkv
    gen = torch.Generator(device="cuda").manual_seed(seed)
    kv, qs = [], []
    for (_, c, n) in case.w.reqs:
        q, k, v = P.regime_request(name, gen, n, 1, hq, hkv, dt, block=chunk if split else 128)
        kv.append((k, v))
        qs.append(q)
    q = torch.cat(qs)
    out = case.launch(kv, q, name).cpu()
    q = q.cpu()
    worst, where = 0.0, None
    for r, (k, v) in enumerate(kv):
        k, v = k.cpu(), v.cpu()
        for h in range(hkv):
            heads = slice(h * G, (h + 1) * G)
            ref, _, bound = P.ref_with_bound(q[r, heads], k[:, h], v[:, h], dt)
            e = P.bound_excess(out[r, heads], ref, bound)
            if e > worst:
                worst, where = e, (r, h)
    assert worst <= P.P16_EXCESS_TOL, f"{name}: excess {worst:.3e} at (request, kv head) {where}"


def _long_decode(b200, *, page_size, hq, hkv, dtype, plan, merge=1, lens=None, seed=0):
    lens = lens or [n for n in LONG_LENS for _ in range(_copies(hq))]
    case = LongCase(b200, page_size=page_size, hq=hq, hkv=hkv, dtype=dtype, lens=[(n - 1, n) for n in lens],
                    phase="decode", seed=seed)
    with options(b200, **_decode_opts(plan, merge)):
        chunk = case.prepare()
        total = int(case.batch.attn_metadata.decode_plan[1])
        if plan == "unsplit":
            assert total == len(lens) and chunk >= max(lens)
        elif plan == "split":
            assert total > len(lens)
        _decode_needles(case, chunk, seed)
        for i, name in enumerate(DECODE_REGIMES):
            _decode_regime(case, name, chunk, seed + 1 + i, split=total > len(lens))
    return case


PLAN_MODES = [("unsplit", 1), ("split", 1), ("split", 0), ("split", 2), ("default", 1)]
PLAN_IDS = ["unsplit", "split-inkernel-merge", "split-combine-launch", "split-combine-auto", "default"]


@pytest.mark.parametrize("plan,merge", PLAN_MODES, ids=PLAN_IDS)
@pytest.mark.parametrize("page_size", [1, 64, 256])
def test_long_decode_page_sizes_and_plans(b200, native_lib, page_size, plan, merge):
    """kv_len 8 193 to 40 960 at GQA 16/8, bf16: unsplit units of up to 320 tiles, split units of 20."""
    _long_decode(b200, page_size=page_size, hq=16, hkv=8, dtype=torch.bfloat16, plan=plan, merge=merge)


@pytest.mark.parametrize("plan", ["unsplit", "split"])
@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("hq,hkv", [(16, 8), (8, 1), (128, 8)], ids=["hq16-hkv8", "hq8-hkv1", "hq128-hkv8"])
def test_long_decode_gqa_and_dtypes(b200, native_lib, hq, hkv, dtype, plan):
    _long_decode(b200, page_size=64, hq=hq, hkv=hkv, dtype=DTYPES[dtype], plan=plan)


def test_long_decode_mixed_batch(b200, native_lib):
    """One 40 960-key request among 60 short ones under the default plan, which then splits nothing: the long
    request is one unit of 320 tiles while every other CTA runs short ones."""
    rnd = random.Random(5)
    lens = [rnd.randint(2, 2048) for _ in range(60)]
    lens.insert(23, 40960)
    case = LongCase(b200, page_size=64, hq=16, hkv=8, dtype=torch.bfloat16, lens=[(n - 1, n) for n in lens],
                    phase="decode", seed=5)
    chunk = case.prepare()
    assert int(case.batch.attn_metadata.decode_plan[1]) == len(lens)  # unsplit
    _decode_needles(case, chunk, seed=5)
    for i, name in enumerate(["drift_up", "chunk_maxima"]):
        _decode_regime(case, name, chunk, seed=6 + i, split=False)


def test_long_decode_cuda_graph_replay(b200, native_lib):
    """A decode launch captured with init_capture_graph(max_seq_len 40 960 and up) on dummy requests, replayed on
    the long batch: capture data as wide as the model's context, live slot tables as wide as the batch's."""
    case = LongCase(b200, page_size=64, hq=16, hkv=8, dtype=torch.bfloat16, lens=[(n - 1, n) for n in LONG_LENS],
                    phase="decode", seed=7)
    assert case.w.page_table.shape[1] >= 40960
    chunk = case.prepare()
    _decode_needles(case, chunk, seed=7, graph=True)


@pytest.mark.parametrize("page_size", [1, 64])
def test_long_decode_fused_pre_attention_bit_identical(b200, native_lib, page_size):
    """The fused launch (q/k-norm, RoPE, append, attention) at positions up to 40 959 with the cos/sin cache of
    RotaryEmbedding(128, 128, 40960, 1e6) equals ops.qknorm_rope_inplace followed by forward, bit for bit:
    output, appended rows, the rest of the pool, and the raw q / k rows stay untouched."""
    hq, hkv, dt = 16, 8, torch.bfloat16
    lens = [(n - 1, n) for n in LONG_LENS]
    rope = b200.layers.RotaryEmbedding(D, D, 40960, 1e6, device=torch.device("cuda"))
    cache = rope._cos_sin_cache
    assert cache.shape[0] == 40960
    gen = torch.Generator(device="cuda").manual_seed(8)
    qw = (torch.rand(D, generator=gen, device="cuda") + 0.5).to(dt)
    kw = (torch.rand(D, generator=gen, device="cuda") + 0.5).to(dt)
    kv = [(torch.randn((n, hkv, D), generator=gen, device="cuda").to(dt),
           torch.randn((n, hkv, D), generator=gen, device="cuda").to(dt)) for _, n in lens]
    q = torch.randn((len(lens), hq, D), generator=gen, device="cuda").to(dt)
    arms = []
    for fused in (False, True):
        case = LongCase(b200, page_size=page_size, hq=hq, hkv=hkv, dtype=dt, lens=lens, phase="decode", seed=8)
        case.prepare()
        assert int(case.batch.positions.max()) == 40959
        x = case.qkv(kv, q)
        raw = x.clone()
        if fused:
            out, _, kc, vc = run_attention(case.gw, case.batch, x, prepare=False, fused=(cache, qw, kw, 1e-6))
            assert_bits_equal(x, raw, "raw qkv rows after the fused decode")
        else:
            qq, kk, _ = x.split([hq * D, hkv * D, hkv * D], dim=-1)
            b200.ops.qknorm_rope_inplace(case.batch.positions, qq, kk, D, cache, qw, kw, 1e-6)
            out, _, kc, vc = run_attention(case.gw, case.batch, x, prepare=False)
        case.check_unowned("fused" if fused else "unfused")
        owned = torch.cat(case.slots)
        arms.append((out.cpu(), kc[owned].cpu(), vc[owned].cpu()))
        del case, kc, vc
        b200.core.set_global_ctx(None)
        torch.cuda.empty_cache()
    (o0, k0, v0), (o1, k1, v1) = arms
    assert_bits_equal(o1, o0, "fused output")
    assert_bits_equal(k1, k0, "k rows of the requests")
    assert_bits_equal(v1, v0, "v rows of the requests")


# ------------------------------------------------------------------------------------------- chunked prefill
# (cached_len, kv_len): an 8 192-row chunk on a 32 768-key prefix, 700 rows on an unaligned 16 421-key prefix, and
# a 16 384-row prompt
PREFILL_LONG = [(32768, 40960), (16384 + 37, 16384 + 37 + 700), (0, 16384)]


def _prefill_probe_long(case: LongCase, seed):
    """Even query heads: needles (at cached - 1, cached, cached + 127, cached + 128, the last key, key 0, 127, 128
    and random keys); odd heads: bf16 ramps (rows with (i >> 3) & 1 == 0 rising, the others falling).  Every row
    that sees its head's needle must return that V row and every ramp row its own or key 0's, exactly; sampled
    rows before their needle hold the uniform mean of their visible keys (fp64 reference and bound)."""
    hq, hkv, dt = case.hq, case.hkv, case.dtype
    G = hq // hkv
    rnd = random.Random(seed)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    kv, qs, needles = [], [], []
    for (_, c, n) in case.w.reqs:
        ql = n - c
        k = torch.randn((n, hkv, D), generator=gen, device="cuda")
        k[..., : P.PROBE_DIMS] = 0
        k[..., 8:10] = P.ramp_key_dims(torch.arange(n), dt).cuda()[:, None, :]
        v = torch.randint(-P.V_MAX, P.V_MAX + 1, (n, hkv, D), generator=gen, device="cuda").to(dt)
        cand = [x for x in dict.fromkeys([c - 1, c, c + 127, c + 128, n - 1, 0, 127, 128, c + ql // 2]) if 0 <= x < n]
        q = torch.zeros(ql, hq, D, device="cuda")
        rising = (torch.arange(ql, device="cuda") >> 3) & 1 == 0
        up, down = P.ramp_query(dt, True).cuda(), P.ramp_query(dt, False).cuda()
        pos = {}
        for head in range(0, hq, 2):
            h, g = divmod(head, G)
            p = cand[head // 2] if head // 2 < len(cand) else rnd.randrange(n)
            k[p, h, P.needle_dim(g)] = P.NEEDLE_K
            q[:, head] = P.needle_query(g).cuda()
            pos[head] = p
        for head in range(1, hq, 2):
            q[:, head] = torch.where(rising[:, None], up, down)
        kv.append((k.to(dt), v))
        qs.append(q.to(dt))
        needles.append(pos)
    q = torch.cat(qs)
    out = case.launch(kv, q, "prefill probes")
    errors, worst, off = [], 0.0, 0
    for r, (_, c, n) in enumerate(case.w.reqs):
        ql = n - c
        k, v = kv[r]
        posn = torch.arange(c, n, device="cuda")
        rows = torch.tensor(P.sampled_rows(ql, rnd), device="cuda")
        for head in range(hq):
            h = head // G
            got = out[off : off + ql, head]
            if head % 2 == 0:
                sees = posn >= needles[r][head]
                want = v[needles[r][head], h].expand(ql, D)
            else:
                sees = torch.ones(ql, dtype=torch.bool, device="cuda")
                rising = (torch.arange(ql, device="cuda") >> 3) & 1 == 0
                want = torch.where(rising[:, None], v[c:n, h], v[0, h].expand(ql, D))
            bad = sees & ~(got.view(torch.int16) == want.view(torch.int16)).all(-1)
            for i in bad.nonzero().flatten().tolist()[:3]:
                errors.append(f"  request {r} row {i} (position {c + i}) head {head} "
                              f"{'needle at ' + str(needles[r][head]) if head % 2 == 0 else 'ramp'}: "
                              f"{P.diagnose(got[i].cpu(), v.cpu())}")
            before = rows[~sees[rows]]
            if before.numel():  # sampled rows before the needle: the uniform mean of their visible keys
                ref, _, bound = P.ref_with_bound(q[off + before, head].cpu(), k[:, h].cpu(), v[:, h].cpu(), dt,
                                                 (posn[before] + 1).cpu())
                worst = max(worst, P.bound_excess(got[before], ref, bound))
        off += ql
    assert not errors, "prefill probes: wrong rows\n" + "\n".join(errors[:12])
    assert worst <= P.P16_EXCESS_TOL, f"rows before their needle: excess {worst:.3e}"


def _prefill_regime_long(case: LongCase, name, seed):
    """A regime on every request; sampled rows (P.sampled_rows) of every query head against the fp64 bound."""
    hq, hkv, dt = case.hq, case.hkv, case.dtype
    G = hq // hkv
    rnd = random.Random(seed)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    kv, qs = [], []
    for (_, c, n) in case.w.reqs:
        q, k, v = P.regime_request(name, gen, n, n - c, hq, hkv, dt)
        kv.append((k, v))
        qs.append(q)
    out = case.launch(kv, torch.cat(qs), name)
    worst, where, off = 0.0, None, 0
    for r, (_, c, n) in enumerate(case.w.reqs):
        rows = torch.tensor(P.sampled_rows(n - c, rnd))
        q, k, v = qs[r][rows.cuda()].cpu(), kv[r][0].cpu(), kv[r][1].cpu()
        got = out[off + rows.cuda()].cpu()
        for h in range(hkv):
            for head in range(h * G, (h + 1) * G):
                ref, _, bound = P.ref_with_bound(q[:, head], k[:, h], v[:, h], dt, c + rows + 1)
                e = P.bound_excess(got[:, head], ref, bound)
                if e > worst:
                    worst, where = e, (r, head)
        off += n - c
    assert worst <= P.P16_EXCESS_TOL, f"{name}: excess {worst:.3e} at (request, head) {where}"


@pytest.mark.parametrize("page_size,order", [(1, 0), (64, 0), (64, 1)],
                         ids=["row-mode-size-sorted", "ps64-size-sorted", "ps64-request-major"])
def test_long_chunked_prefill(b200, native_lib, page_size, order):
    case = LongCase(b200, page_size=page_size, hq=16, hkv=8, dtype=torch.bfloat16, lens=PREFILL_LONG,
                    phase="prefill", seed=page_size)
    with options(b200, prefill_order=order):
        case.prepare(request_major=order == 1)
        _prefill_probe_long(case, seed=11)
        _prefill_regime_long(case, "drift_up", seed=12)


def test_long_prefill_plan_clamp(b200, native_lib):
    """The prefill plan of a batch whose heaviest query tiles see more than 1023 K/V tiles (a 131 072-key prefix;
    metadata only, nothing is launched): both orders hold every (request, q_tile) once, heaviest first by
    min(kv tiles, 1023) or request-major."""
    lens = [(131072, 131072 + 300), (200, 1000), (0, 129), (5000, 5001 + 256)]
    _need_memory(2 * sum(d for _, d in lens) * 8 * D * 2)
    w = _world(page_size=64, hq=16, hkv=8, dtype=torch.bfloat16, lens=lens)
    gw = GpuWorld(b200, w)
    md = o_meta.ref_prepare_metadata(w.page_table, w.reqs, 64)
    for order in (0, 1):
        with options(b200, prefill_order=order):
            batch = gw.batch("prefill", md=md)
            gw.backend.prepare_metadata(batch)
            check_prefill_plan(batch.attn_metadata.prefill_plan.cpu().numpy(), w.reqs, request_major=order == 1)
