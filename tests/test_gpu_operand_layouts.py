"""GPU: every kernel reads and writes its operands through the strides it is given.  The engine hands the kernels
slices of one qkv row, so q, k and v share a row stride there; the API (B200AttnBackend.forward, ops.*, the C ABI)
takes row-strided views with independent strides.  Each case runs the same values twice, once in the dense layout
and once in a layout whose strides differ (helpers.LAYOUTS), and requires:

* the output, the appended pool rows and the whole pool bit-identical between the two runs (a layout must not
  change a single bit);
* every padding element of the strided buffers still NaN, bit for bit, and the operands the kernel only reads
  unchanged;
* the strided run within the existing bounds of the oracle.

The padding is NaN and the strides of one call are pairwise distinct in the padded cases, so a kernel that used
one stride where another belongs reads NaN or another operand's rows and fails."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from helpers import (LAYOUTS, SPLIT_PLAN, GpuWorld, add_requests, assert_all_nan_bits, assert_bits_equal,
                     assert_pre_attention_close, attn_tolerance_ok, layout_padding, make_inputs, make_world, options,
                     oracle_forward, padded_reqs, padded_rows, poison_unowned, run_attention, ulp_close)
from oracle import metadata as o_meta
from oracle.index import ref_indexing
from oracle.layer import ref_pre_attention
from oracle.norm import ref_rmsnorm
from oracle.rope import ref_cos_sin_cache
from test_gpu_attention import DECODE_LENS, PREFILL_LENS

pytestmark = pytest.mark.gpu

D = 128
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}


def _distinct(**strides):
    assert len(set(strides.values())) == len(strides), f"strides of one call are not pairwise distinct: {strides}"


# ------------------------------------------------------------------ attention
class _Recorded:
    """A layout of helpers.LAYOUTS that keeps the (q, k, v) views it made, for the checks after the launch."""

    def __init__(self, name: str):
        self.fn, self.views = LAYOUTS[name], []

    def __call__(self, qkv, widths):
        self.views.append(self.fn(qkv, widths))
        return self.views[-1]


def _world(*, page_size, hq, hkv, lens, dtype, pad_to=None, seed=0):
    w = make_world(seed=seed, page_size=page_size, hq=hq, hkv=hkv, max_reqs=max(len(lens), pad_to or 0) + 1,
                   max_seq=max(d for _, d in lens) + 8, dtype=dtype)
    add_requests(w, lens)
    poison_unowned(w)
    reqs = padded_reqs(w, pad_to)
    md = o_meta.ref_prepare_metadata(w.page_table, reqs, page_size)
    qkv, _, _, _ = make_inputs(w, seed + 1, reqs=reqs)
    return w, reqs, md, qkv


def _launch(b200, w, md, qkv, phase, layout, *, fused=None, graph=False, pad_to=None):
    """One attention launch on a fresh device mirror of the world, its operands laid out by LAYOUTS[layout]."""
    gw = GpuWorld(b200, w)
    rec = _Recorded(layout)
    batch = gw.batch(phase, pad_to=pad_to, md=md)
    out, _, kc, vc = run_attention(gw, batch, qkv.cuda(), fused=fused, graph=graph, layout=rec)
    q, k, v = rec.views[-1]
    # the strides the launch was given, under the names of the C ABI; a captured launch reads the backend's
    # static slot table, which prepare_for_replay refreshes from the live metadata
    slot_table = gw.backend.capture.page_table if graph else batch.attn_metadata.page_table
    strides = dict(q_row_stride=q.stride(0), k_row_stride=k.stride(0), v_row_stride=v.stride(0),
                   slot_table_stride=slot_table.stride(0))
    return SimpleNamespace(out=out.cpu(), kc=kc.cpu(), vc=vc.cpu(), views=(q, k, v), strides=strides)


def _check_layout_run(dense, got, qkv, md, n_real, what):
    """got (the layout under test) against dense (one qkv row): output, appended rows and the whole pool
    bit-identical (rows of graph-padding dummies excluded: they all append to one slot), padding still NaN,
    the q / k / v operands unchanged."""
    assert_bits_equal(got.out[:n_real], dense.out[:n_real], f"{what}: output")
    slots = torch.from_numpy(md.out_loc[:n_real].astype(np.int64))
    assert_bits_equal(got.kc[slots], dense.kc[slots], f"{what}: appended k rows")
    assert_bits_equal(got.vc[slots], dense.vc[slots], f"{what}: appended v rows")
    keep = torch.ones(got.kc.shape[0], dtype=torch.bool)
    keep[torch.from_numpy(md.out_loc[n_real:].astype(np.int64))] = False
    assert_bits_equal(got.kc[keep], dense.kc[keep], f"{what}: k pool")
    assert_bits_equal(got.vc[keep], dense.vc[keep], f"{what}: v pool")
    assert_all_nan_bits(layout_padding(got.views), f"{what}: q / k / v buffers")
    for x, want, name in zip(got.views, qkv.split([x.shape[1] for x in got.views], dim=-1), "qkv"):
        assert_bits_equal(x, want, f"{what}: {name} operand after the launch")


def _check_oracle(got, ref, md, n_real, what, pre=None):
    """got against the oracle's (out, k pool, v pool); pre = (qkv, positions, hq, hkv, cache, qw, kw): the k
    rows were normed and roped in the launch, and are held to one ulp of the oracle's chain instead of its bits."""
    ref_out, ref_kc, ref_vc = ref
    attn_tolerance_ok(got.out[:n_real], ref_out[:n_real], what)
    slots = torch.from_numpy(md.out_loc[:n_real].astype(np.int64))
    assert_bits_equal(got.vc[slots], ref_vc[slots], f"{what}: appended v rows vs the oracle")
    if pre is None:
        assert_bits_equal(got.kc[slots], ref_kc[slots], f"{what}: appended k rows vs the oracle")
    else:
        qkv, positions, hq, hkv, cache, qw, kw = pre
        assert_pre_attention_close(None, got.kc[slots].reshape(n_real, -1), qkv[:n_real], positions[:n_real], hq,
                                   hkv, D, cache, qw, kw)


def _decode_operands(qkv, md, hq, hkv, fused, seed):
    """The oracle's (q, k, v) of a decode batch, the `pre` argument of _check_oracle and the `fused` argument of
    _launch.  Fused: both norm weights (drawn from seed), the oracle runs q-norm, k-norm and RoPE first."""
    if not fused:
        q, k, v = qkv.split([hq * D, hkv * D, hkv * D], dim=-1)
        return q, k, v, None, None
    cache = ref_cos_sin_cache(D, 2048, 1e6)
    gen = torch.Generator().manual_seed(seed)
    qw, kw = [(torch.rand(D, generator=gen) + 0.5).to(qkv.dtype) for _ in range(2)]
    positions = torch.from_numpy(md.positions)
    q, k, v = ref_pre_attention(qkv, positions, hq, hkv, D, cache, qw, kw, 1e-6)
    return q, k, v, (qkv, positions, hq, hkv, cache, qw, kw), (cache.cuda(), qw.cuda(), kw.cuda(), 1e-6)


# G = 1, 8 (the N = 8 instantiation of the decode kernel) and 16 (N = 16)
DECODE_GROUPS = [(8, 8), (16, 2), (32, 2)]


@pytest.mark.parametrize("page_size", [1, 64], ids=["ps1", "ps64"])
@pytest.mark.parametrize("hq,hkv", DECODE_GROUPS, ids=[f"hq{a}-hkv{b}" for a, b in DECODE_GROUPS])
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("fused", [False, True], ids=["unfused", "fused"])
@pytest.mark.parametrize("layout", ["separate", "kv_pair", "padded"])
def test_decode_layouts(b200, native_lib, layout, fused, dtype, hq, hkv, page_size):
    """The wgmma decode kernel (page size 1: row loads; 64: box loads), under the default plan and with every
    request split into 128-key chunks, unfused and with the fused q/k-norm + RoPE (both norm weights)."""
    lens = DECODE_LENS["mixed"][:5]
    w, reqs, md, qkv = _world(page_size=page_size, hq=hq, hkv=hkv, lens=lens, dtype=DTYPES[dtype])
    n = len(lens)
    q, k, v, pre, fz = _decode_operands(qkv, md, hq, hkv, fused, seed=5)
    ref = oracle_forward(w, 0, q, k, v, md, reqs=reqs)
    for plan, opts in (("default", {}), ("split", SPLIT_PLAN)):
        what = f"decode {layout} {'fused' if fused else 'unfused'} {dtype} {hq}/{hkv} ps{page_size} {plan} plan"
        with options(b200, **opts):
            dense = _launch(b200, w, md, qkv, "decode", "split", fused=fz)
            got = _launch(b200, w, md, qkv, "decode", layout, fused=fz)
        if layout == "padded":
            _distinct(**got.strides)
        _check_layout_run(dense, got, qkv, md, n, what)
        _check_oracle(got, ref, md, n, what, pre)


@pytest.mark.parametrize("fused", [False, True], ids=["unfused", "fused"])
def test_decode_layout_graph_replay(b200, native_lib, fused):
    """A decode launch captured into a CUDA graph with padded static q / k / v buffers, replayed on a live batch
    padded to the captured size."""
    hq, hkv, pad_to = 16, 8, 8
    lens = DECODE_LENS["mixed"][:3]
    w, reqs, md, qkv = _world(page_size=16, hq=hq, hkv=hkv, lens=lens, dtype=torch.bfloat16, pad_to=pad_to)
    q, k, v, pre, fz = _decode_operands(qkv, md, hq, hkv, fused, seed=6)
    ref = oracle_forward(w, 0, q, k, v, md, reqs=reqs)
    dense = _launch(b200, w, md, qkv, "decode", "split", fused=fz, graph=True, pad_to=pad_to)
    got = _launch(b200, w, md, qkv, "decode", "padded", fused=fz, graph=True, pad_to=pad_to)
    _distinct(**got.strides)
    what = f"graph replay padded {'fused' if fused else 'unfused'}"
    _check_layout_run(dense, got, qkv, md, len(lens), what)
    _check_oracle(got, ref, md, len(lens), what, pre)


def _prefill_lens(page_size):
    """PREFILL_LENS["extend"] with its cached prefixes page aligned (as test_prefill_qwen3_0p6b_shape runs it),
    plus a cached boundary inside a page and inside a K/V tile."""
    lens = [((c // page_size) * page_size, d) for c, d in PREFILL_LENS["extend"]]
    return [(c, max(d, c + 1)) for c, d in lens] + [(37, 200)]


PREFILL_GROUPS = [(16, 8), (16, 1), (32, 2)]


@pytest.mark.parametrize("page_size", [1, 16, 64], ids=["ps1", "ps16", "ps64"])
@pytest.mark.parametrize("hq,hkv", PREFILL_GROUPS, ids=[f"hq{a}-hkv{b}" for a, b in PREFILL_GROUPS])
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("layout", ["kv_pair", "padded_shared_kv"])
def test_prefill_layouts(b200, native_lib, layout, dtype, hq, hkv, page_size):
    """The wgmma prefill kernel (its q and k / v inputs are read through TMA tensor maps built from the row
    strides).  It takes one row stride for k and v, so the padded layout here pads k and v alike."""
    lens = _prefill_lens(page_size)
    w, reqs, md, qkv = _world(page_size=page_size, hq=hq, hkv=hkv, lens=lens, dtype=DTYPES[dtype])
    n = qkv.shape[0]
    what = f"prefill {layout} {dtype} {hq}/{hkv} ps{page_size}"
    dense = _launch(b200, w, md, qkv, "prefill", "split")
    got = _launch(b200, w, md, qkv, "prefill", layout)
    if layout == "padded_shared_kv":
        s = dict(got.strides)
        assert s.pop("k_row_stride") == s["v_row_stride"]
        _distinct(**s)
    _check_layout_run(dense, got, qkv, md, n, what)
    q, k, v = qkv.split([hq * D, hkv * D, hkv * D], dim=-1)
    _check_oracle(got, oracle_forward(w, 0, q, k, v, md, reqs=reqs), md, n, what)


def test_prefill_refuses_k_v_row_strides_that_differ(b200, native_lib):
    """Prefill reads k and v through one row stride and refuses a call whose k and v strides differ, before
    any launch and without touching the pool; the next valid call is correct.  (Decode accepts such operands:
    test_decode_layouts[padded-...].)"""
    hq, hkv = 16, 8
    lens = [(37, 200), (0, 65), (128, 129)]
    w, reqs, md, qkv = _world(page_size=16, hq=hq, hkv=hkv, lens=lens, dtype=torch.bfloat16)
    gw = GpuWorld(b200, w)
    batch = gw.batch("prefill", md=md)
    gw.backend.prepare_metadata(batch)
    q, k, v = LAYOUTS["padded"](qkv.cuda(), (hq * D, hkv * D, hkv * D))
    assert k.stride(0) != v.stride(0)
    kc0, vc0 = [x.cpu() for x in gw.pool_rows(0)]
    launches = b200._cabi.launch_count()
    with pytest.raises(RuntimeError, match="k and v must share a row stride"):
        gw.backend.forward(q.view(-1, hq, D), k, v, 0, batch)
    assert b200._cabi.launch_count() == launches
    kc, vc = gw.pool_rows(0)
    assert_bits_equal(kc, kc0, "k pool after the refused call")
    assert_bits_equal(vc, vc0, "v pool after the refused call")
    out, _, kc, vc = run_attention(gw, batch, qkv.cuda(), prepare=False)
    got = SimpleNamespace(out=out.cpu(), kc=kc.cpu(), vc=vc.cpu())
    q, k, v = qkv.split([hq * D, hkv * D, hkv * D], dim=-1)
    _check_oracle(got, oracle_forward(w, 0, q, k, v, md, reqs=reqs), md, qkv.shape[0], "prefill after a refusal")


# ------------------------------------------------------------------ RoPE and fused qk-norm + RoPE
ROPE_OPS = {"rope": None, "qknorm-both": (True, True), "qknorm-q": (True, False), "qknorm-k": (False, True),
            "qknorm-none": (False, False)}


@pytest.mark.parametrize("pos_dtype", [torch.int32, torch.int64], ids=["pos32", "pos64"])
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("d", [64, 128, 256])
@pytest.mark.parametrize("op", list(ROPE_OPS))
def test_rope_layouts(b200, native_lib, op, d, dtype, pos_dtype):
    """ops.apply_rope_with_cos_sin_cache_inplace and ops.qknorm_rope_inplace with q and k in two padded buffers of
    distinct row strides (q passed 3-D [nnz, hq, d], k 2-D): bit-identical to the run on slices of one qkv row,
    and within one ulp of oracle.layer.ref_pre_attention.  Positions include 0 and max_pos - 1; 7 q and 3 k heads
    put q and k rows of several tokens in one warp at D = 64 and 128."""
    nnz, hq, hkv, max_pos = 67, 7, 3, 1024
    dt = DTYPES[dtype]
    gen = torch.Generator().manual_seed(d)
    qkv = torch.randn(nnz, (hq + 2 * hkv) * d, generator=gen).to(dt)
    pos = torch.randint(0, max_pos, (nnz,), generator=gen).to(pos_dtype)
    pos[0], pos[nnz // 2] = 0, max_pos - 1
    cache = ref_cos_sin_cache(d, max_pos, 1e6)
    weights = [(torch.rand(d, generator=gen) + 0.5).to(dt) for _ in range(2)]
    qw, kw = [x if on else None for x, on in zip(weights, ROPE_OPS[op] or (False, False))]
    pos_g, cache_g = pos.cuda(), cache.cuda()
    qw_g, kw_g = [x.cuda() if x is not None else None for x in (qw, kw)]

    def run(q, k):
        if op == "rope":
            b200.ops.apply_rope_with_cos_sin_cache_inplace(pos_g, q, k, d, cache_g)
        else:
            b200.ops.qknorm_rope_inplace(pos_g, q, k, d, cache_g, qw_g, kw_g, 1e-6)

    widths = (hq * d, hkv * d, hkv * d)
    dense = qkv.cuda()
    run(dense[:, : hq * d], dense[:, hq * d : (hq + hkv) * d])
    q, k, _ = LAYOUTS["padded"](qkv.cuda(), widths)
    _distinct(q_row_stride=q.stride(0), k_row_stride=k.stride(0))
    run(q.view(nnz, hq, d), k)
    assert_bits_equal(q, dense[:, : hq * d], f"{op} q rows")
    assert_bits_equal(k, dense[:, hq * d : (hq + hkv) * d], f"{op} k rows")
    assert_all_nan_bits(layout_padding([q, k]), f"{op} q / k buffers")
    assert_pre_attention_close(q, k, qkv, pos, hq, hkv, d, cache, qw, kw)


# ------------------------------------------------------------------ RMSNorm out of place
# 64 / 128 / 256: the lane-group kernel; 1024: the row kernel at one 16-byte chunk per thread; 4104 and 16384: two
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("rows,dim", [(33, 64), (130, 128), (7, 256), (37, 1024), (9, 4104), (3, 16384)])
def test_rmsnorm_out_of_place_strided_rows(b200, native_lib, rows, dim, dtype):
    """x and out are rows of two differently padded buffers (row strides dim + 8 and dim + 24)."""
    dt = DTYPES[dtype]
    gen = torch.Generator().manual_seed(rows * dim)
    x = (torch.randn(rows, dim, generator=gen) * 3).to(dt)
    w = (torch.randn(dim, generator=gen) * 0.5 + 1).to(dt).cuda()
    dense = x.cuda()
    b200.ops.rmsnorm(dense, w, 1e-6, out=dense)
    xs = padded_rows(x.cuda(), 8)
    out = padded_rows(torch.full_like(x, float("nan")).cuda(), 24)
    _distinct(x_row_stride=xs.stride(0), out_row_stride=out.stride(0))
    assert b200.ops.rmsnorm(xs, w, 1e-6, out=out).data_ptr() == out.data_ptr()
    assert_bits_equal(out, dense, "out of place vs in place")
    assert_bits_equal(xs, x, "x after the norm")
    assert_all_nan_bits(layout_padding([xs, out]), "x / out buffers")
    ulp_close(out, ref_rmsnorm(x, w.cpu(), 1e-6))


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("heads,d", [(5, 64), (3, 128), (2, 256)])
def test_rmsnorm_per_head_out_of_place_strided(b200, native_lib, heads, d, dtype):
    """3-D per-head norm with x = every other head of a wider buffer (head stride 2d, row stride 2 heads d + 8)
    into an out of row stride heads d + 24: all four strides of the call differ."""
    nnz, dt = 41, DTYPES[dtype]
    gen = torch.Generator().manual_seed(heads * d)
    vals = (torch.randn(nnz, heads, d, generator=gen) * 3).to(dt)
    w = (torch.rand(d, generator=gen) + 0.5).to(dt).cuda()
    dense = vals.cuda()
    b200.ops.rmsnorm(dense, w, 1e-6, out=dense)
    x = padded_rows(torch.full((nnz, 2 * heads * d), float("nan"), dtype=dt).cuda(), 8).view(nnz, 2 * heads, d)[:, ::2]
    x.copy_(vals)
    out = padded_rows(torch.full((nnz, heads * d), float("nan"), dtype=dt).cuda(), 24).view(nnz, heads, d)
    _distinct(x_row_stride=x.stride(0), x_head_stride=x.stride(1), out_row_stride=out.stride(0),
              out_head_stride=out.stride(1))
    b200.ops.rmsnorm(x, w, 1e-6, out=out)
    assert_bits_equal(out, dense, "per-head out of place vs in place")
    assert_bits_equal(x, vals, "x after the norm")
    assert_all_nan_bits(layout_padding([x, out]), "x / out buffers (odd heads and row padding)")
    ulp_close(out, ref_rmsnorm(vals, w.cpu(), 1e-6))


# ------------------------------------------------------------------ row gather
@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64], ids=["idx32", "idx64"])
@pytest.mark.parametrize("vocab_range", [None, (700, 1500)], ids=["plain", "vocab-range"])
@pytest.mark.parametrize("dim,dtype", [(1024, "bf16"), (128, "fp16")])
def test_index_rows_into_padded_output(b200, native_lib, dim, dtype, vocab_range, idx_dtype):
    """ops.indexing(output=) into rows of a padded buffer, from a padded table: weight row stride dim + 64,
    output row stride dim + 128 (and row bytes dim): bits equal the oracle's, the padding is untouched."""
    dt, vocab, n = DTYPES[dtype], 3001, 333
    gen = torch.Generator().manual_seed(dim)
    table = torch.randn(vocab, dim, generator=gen).to(dt)
    idx = torch.randint(0, vocab, (n,), generator=gen).to(idx_dtype)
    wide = padded_rows(table.cuda(), 64)
    shard = wide if vocab_range is None else wide[vocab_range[0] : vocab_range[0] + vocab_range[1]]
    out = padded_rows(torch.full((n, dim), float("nan"), dtype=dt).cuda(), 128)
    _distinct(weight_row_stride=shard.stride(0), out_row_stride=out.stride(0), row=dim)
    ret = b200.ops.indexing(shard, idx.cuda(), output=out, vocab_range=vocab_range)
    assert ret.data_ptr() == out.data_ptr()
    ref_table = table if vocab_range is None else table[vocab_range[0] : vocab_range[0] + vocab_range[1]]
    assert_bits_equal(out, ref_indexing(ref_table, idx, vocab_range), "gathered rows")
    assert_bits_equal(wide, table, "table after the gather")
    assert_all_nan_bits(layout_padding([wide, out]), "table / output buffers")
