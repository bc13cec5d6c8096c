"""GPU parity: metadata, decode / prefill attention with fused append, CUDA-graph hooks --
product path (B200AttnBackend -> C ABI -> sm_90a kernels) vs the CPU oracle."""
import random

import numpy as np
import pytest
import torch

from helpers import GpuWorld, add_requests, attn_tolerance_ok, make_inputs, make_world, oracle_forward
from oracle import metadata as o_meta

pytestmark = pytest.mark.gpu


@pytest.fixture(params=[1, 0, 2, 3], ids=["tcgen05", "cpasync", "tcgen05-inorder-combine-launch", "tcgen05-combine-auto"])
def decode_impl(request, b200, native_lib):
    """Both decode kernels are held to the same oracle: the tensor-core + TMA product kernel (wgmma on
    sm_90a; the ids keep the variant names the suite has always used) with the split-KV merge done by
    the last-arriving chunk inside the decode launch -- the default --, as its own launch, and under
    the "in kernel only when nothing is split" policy, and the cp.async / CUDA-core bring-up kernel
    (selected with the debug options)."""
    impl = 0 if request.param == 0 else 1
    try:
        prev = b200._cabi.set_option("decode_impl", impl)
    except b200._cabi.B200NativeError:
        pytest.skip("cross-check kernel not in this build (B200_BUILD_BRINGUP=1)")
    prev_merge = b200._cabi.set_option("decode_fused_combine", {3: 2, 2: 0}.get(request.param, 1))
    yield impl
    b200._cabi.set_option("decode_impl", prev)
    b200._cabi.set_option("decode_fused_combine", prev_merge)


def _check_metadata(md, ref: o_meta.RefMetadata, page_size: int):
    bs = len(ref.cache_seqlens)
    assert np.array_equal(md.cache_seqlens.cpu().numpy(), ref.cache_seqlens)
    assert np.array_equal(md.cu_seqlens_q.cpu().numpy(), ref.cu_seqlens_q)
    assert np.array_equal(md.cu_seqlens_k.cpu().numpy(), ref.cu_seqlens_k)
    assert md.max_seqlen_q == ref.max_seqlen_q and md.max_seqlen_k == ref.max_seqlen_k
    st = md.page_table.cpu().numpy()[:, : ref.max_seqlen_k]
    assert np.array_equal(st, ref.slot_table)
    assert np.array_equal(md.flat_indices().cpu().numpy(), ref.indices_flat)
    assert np.array_equal(md.paged_page_table(page_size).cpu().numpy(), ref.page_table_paged)
    assert np.array_equal(md.get_last_indices(bs).cpu().numpy(), ref.last_indices)
    plan = md.decode_plan.cpu().numpy()
    chunk, total, pbs = int(plan[0]), int(plan[1]), int(plan[2])
    assert pbs == bs and chunk % 128 == 0 and chunk >= 128
    starts = plan[4 : 4 + bs + 1]
    n_chunks = -(-ref.cache_seqlens // chunk)
    assert np.array_equal(np.diff(starts), n_chunks) and starts[0] == 0 and starts[-1] == total
    assert n_chunks.max() <= 16
    # work order: every (request, chunk) exactly once, largest (in 128-token tiles) first
    order = plan[4 + bs + 1 : 4 + bs + 1 + total]
    items = {(int(e) & 0xFFFF, (int(e) >> 16) & 0xF) for e in order}
    assert items == {(r, c) for r in range(bs) for c in range(int(n_chunks[r]))}
    assert all(((int(e) >> 20) & 0x1F) == n_chunks[int(e) & 0xFFFF] for e in order)

    def tiles(e):
        r, c = int(e) & 0xFFFF, (int(e) >> 16) & 0xF
        ln = min(chunk, int(ref.cache_seqlens[r]) - c * chunk) - (1 if c == n_chunks[r] - 1 else 0)
        return -(-ln // 128)

    sizes = [tiles(e) for e in order]
    assert sizes == sorted(sizes, reverse=True)


def _run_case(b200, *, page_size, hq, hkv, lens, phase, seed=0, share_prefix=None, pad_to=None,
              dtype=torch.bfloat16, layer=0, layers=1, max_seq=None):
    max_seq = max_seq or max(d for _, d in lens) + 8
    w = make_world(seed=seed, page_size=page_size, hq=hq, hkv=hkv, layers=layers,
                   max_reqs=max(len(lens), pad_to or 0) + 1, max_seq=max_seq, dtype=dtype)
    add_requests(w, lens, share_prefix_from=share_prefix)
    # every pool row no request owns is poisoned with NaN: unused page tails / free pages hold
    # arbitrary bits in a real engine (torch.empty pool) and must never leak into a result
    used = np.zeros(w.pool_cpu.shape[2], dtype=bool)
    for (t, _, d) in w.reqs:
        used[w.page_table[t, :d]] = True
    gw = GpuWorld(b200, w)
    gw.pool._kv_buffer.view(2, w.layers, -1, hkv, w.d)[:, :, torch.from_numpy(~used).cuda()] = float("nan")
    pool_before = gw.pool._kv_buffer.view(2, w.layers, -1, hkv, w.d)[0, layer].clone()
    batch = gw.batch(phase, pad_to=pad_to)
    triples = list(w.reqs)
    if pad_to:
        dummy_row = w.page_table.shape[0] - 1
        triples += [(dummy_row, 0, 1)] * (pad_to - len(w.reqs))
    ref_md = o_meta.ref_prepare_metadata(w.page_table, triples, page_size)
    # inputs for all padded rows
    w_full = w
    saved = w.reqs
    w.reqs = triples
    qkv, q, k, v = make_inputs(w, seed + 1)
    ref_out, ref_kc, ref_vc = oracle_forward(w, layer, q, k, v, ref_md)
    w.reqs = saved
    qkv_g = qkv.cuda()
    qg, kg, vg = qkv_g.split([hq * w.d, hkv * w.d, hkv * w.d], dim=-1)
    batch.positions = torch.from_numpy(ref_md.positions).cuda()
    batch.out_loc = torch.from_numpy(ref_md.out_loc).cuda()
    gw.backend.prepare_metadata(batch)
    _check_metadata(batch.attn_metadata, ref_md, page_size)
    out = gw.backend.forward(qg.view(-1, hq, w.d), kg, vg, layer, batch)
    torch.cuda.synchronize()
    assert out.shape == (qkv.shape[0], hq, w.d) and out.is_contiguous()
    n_real = sum(d - c for (_, c, d) in saved)
    rel = attn_tolerance_ok(out[:n_real], ref_out[:n_real], f"{phase} ps={page_size} hq={hq} hkv={hkv}")
    # append side effect: pool rows bit-exact (dummy slot excluded: many writers)
    kc, vc = gw.pool_rows(layer)
    real_slots = torch.from_numpy(ref_md.out_loc[:n_real].astype(np.int64))
    assert torch.equal(kc[real_slots].view(torch.int16), ref_kc[real_slots].view(torch.int16))
    assert torch.equal(vc[real_slots].view(torch.int16), ref_vc[real_slots].view(torch.int16))
    # nothing else in the pool moved
    mask = torch.ones(kc.shape[0], dtype=torch.bool)
    mask[torch.from_numpy(ref_md.out_loc.astype(np.int64))] = False
    assert torch.equal(kc[mask].view(torch.int16), pool_before.cpu()[mask].view(torch.int16))
    return rel


DECODE_LENS = {
    "tiny": [(0, 1), (1, 2), (62, 63), (63, 64), (64, 65), (127, 128), (128, 129)],
    "mixed": [(99, 100), (511, 512), (1023, 1024), (256, 257), (700, 701), (64, 65), (1, 2), (1500, 1501)],
    "long": [(4095, 4096), (3000, 3001)],
}


@pytest.mark.parametrize("page_size", [1, 16, 64])
@pytest.mark.parametrize("name", list(DECODE_LENS))
def test_decode_qwen3_0p6b_shape(b200, native_lib, page_size, name, decode_impl):
    _run_case(b200, page_size=page_size, hq=16, hkv=8, lens=DECODE_LENS[name], phase="decode")


@pytest.mark.parametrize("hq,hkv", [(8, 8), (40, 8), (64, 8), (8, 1), (4, 2), (16, 2), (7, 1), (6, 2), (3, 1)])
def test_decode_gqa_groups(b200, native_lib, hq, hkv, decode_impl):
    """Hq/Hkv of every BASELINE model at tp 1/2/4/8 (GQA 1,2,5,8) plus odd group sizes."""
    _run_case(b200, page_size=16, hq=hq, hkv=hkv, lens=DECODE_LENS["mixed"][:5], phase="decode")


def test_decode_padded_dummy_requests(b200, native_lib, decode_impl):
    """Graph-padded batch: dummy requests (kv_len 1, shared dummy slot) ride along (graph.py:160-166)."""
    _run_case(b200, page_size=16, hq=16, hkv=8, lens=DECODE_LENS["mixed"][:3], phase="decode", pad_to=8)


def test_decode_fp16(b200, native_lib, decode_impl):
    _run_case(b200, page_size=1, hq=16, hkv=8, lens=DECODE_LENS["mixed"][:4], phase="decode", dtype=torch.float16)


def test_decode_second_layer_of_pool(b200, native_lib, decode_impl):
    _run_case(b200, page_size=16, hq=16, hkv=8, lens=DECODE_LENS["tiny"], phase="decode", layer=2, layers=3)


@pytest.fixture(params=[1, 2, 0], ids=["tcgen05-fullrow", "tcgen05", "mmasync"])
def prefill_impl(request, b200, native_lib):
    """The tensor-core product kernel (wgmma on sm_90a; the ids keep the variant names the suite has
    always used) with the request-major work order (option prefill_order = 1) and with the size-sorted
    order (default), and the mma.sync bring-up kernel (test builds only)."""
    try:
        prev = b200._cabi.set_option("prefill_impl", 0 if request.param == 0 else 1)
    except b200._cabi.B200NativeError:
        pytest.skip("cross-check kernel not in this build (B200_BUILD_BRINGUP=1)")
    prev_order = b200._cabi.set_option("prefill_order", 1 if request.param == 1 else 0)
    yield request.param
    b200._cabi.set_option("prefill_impl", prev)
    b200._cabi.set_option("prefill_order", prev_order)


PREFILL_LENS = {
    "no_cache": [(0, 1), (0, 17), (0, 64), (0, 65), (0, 200), (0, 333)],
    "single_long": [(0, 1024)],
    "extend": [(64, 200), (128, 129), (256, 700), (0, 50), (320, 321)],
    "chunked": [(512, 1024), (1024, 1100)],
}


@pytest.mark.parametrize("page_size", [1, 16, 64])
@pytest.mark.parametrize("name", list(PREFILL_LENS))
def test_prefill_qwen3_0p6b_shape(b200, native_lib, page_size, name, prefill_impl):
    lens = PREFILL_LENS[name]
    if page_size > 1 and name in ("extend", "chunked"):
        lens = [((c // page_size) * page_size, d) for c, d in lens]  # cached prefixes are page aligned
        lens = [(c, max(d, c + 1)) for c, d in lens]
    _run_case(b200, page_size=page_size, hq=16, hkv=8, lens=lens, phase="prefill")


@pytest.mark.parametrize("hq,hkv", [(40, 8), (8, 1), (64, 8), (4, 4), (6, 2)])
def test_prefill_gqa_groups(b200, native_lib, hq, hkv, prefill_impl):
    _run_case(b200, page_size=16, hq=hq, hkv=hkv, lens=[(0, 130), (64, 300), (0, 7)], phase="prefill")


def test_prefill_radix_shared_prefix_pages(b200, native_lib, prefill_impl):
    """Two requests whose leading page-table entries are identical (radix-shared pages)."""
    # every sharer has the shared pages in its cached range: a prefix only becomes matchable after
    # the forward that produced it (scheduler/cache.py cache_req), so nobody appends into them
    rel = _run_case(b200, page_size=16, hq=16, hkv=8, lens=[(128, 300), (128, 260), (128, 400)],
                    phase="prefill", share_prefix=0)
    assert rel < 3e-3


def test_prefill_with_all_extend_len_one_uses_decode_kernel(b200, native_lib, decode_impl):
    _run_case(b200, page_size=16, hq=16, hkv=8, lens=[(16, 17), (32, 33)], phase="prefill")


def test_forward_rejects_cpu_and_foreign_metadata(b200, native_lib):
    w = make_world(seed=0, page_size=16, hq=16, hkv=8, max_reqs=2, max_seq=64)
    add_requests(w, [(3, 4)])
    gw = GpuWorld(b200, w)
    batch = gw.batch("decode")
    q = torch.zeros(1, 16, 128, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):
        gw.backend.forward(q, q.view(1, -1)[:, :1024], q.view(1, -1)[:, :1024], 0, batch)


def test_cuda_graph_capture_and_replay(b200, native_lib, decode_impl):
    """init_capture_graph / prepare_for_capture / prepare_for_replay drive a captured decode
    (reference engine/graph.py:105-158): replayed output == eager output, pool rows appended."""
    hq, hkv, d, ps = 16, 8, 128, 16
    lens = [(99, 100), (511, 512), (300, 301)]
    w = make_world(seed=4, page_size=ps, hq=hq, hkv=hkv, max_reqs=9, max_seq=1024)
    add_requests(w, lens)
    gw = GpuWorld(b200, w)
    backend = gw.backend
    max_seq_al = w.page_table.shape[1]
    backend.init_capture_graph(max_seq_al, [4, 8])
    dummy_row = w.page_table.shape[0] - 1
    # static buffers owned by the "graph runner"
    bs_cap = 4
    qkv_buf = torch.zeros(bs_cap, (hq + 2 * hkv) * d, dtype=torch.bfloat16, device="cuda")
    out_loc_buf = torch.zeros(bs_cap, dtype=torch.int32, device="cuda")
    out_buf = torch.zeros(bs_cap, hq, d, dtype=torch.bfloat16, device="cuda")
    cap_batch = b200.Batch([b200.Req(table_idx=dummy_row, cached_len=0, device_len=1)] * bs_cap, "decode")
    cap_batch.padded_reqs = cap_batch.reqs
    backend.prepare_for_capture(cap_batch)
    cap_batch.out_loc = out_loc_buf
    out_loc_buf.fill_(int(w.page_table[dummy_row, 0]))

    def run():
        q, k, v = qkv_buf.split([hq * d, hkv * d, hkv * d], dim=-1)
        out_buf.copy_(backend.forward(q.view(-1, hq, d), k, v, 0, cap_batch))

    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        run()  # warm-up outside capture
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            run()
    torch.cuda.synchronize()

    # live batch, padded to 4
    batch = gw.batch("decode", pad_to=bs_cap)
    triples = list(w.reqs) + [(dummy_row, 0, 1)]
    ref_md = o_meta.ref_prepare_metadata(w.page_table, triples, ps)
    saved, w.reqs = w.reqs, triples
    qkv, q, k, v = make_inputs(w, 9)
    ref_out, ref_kc, _ = oracle_forward(w, 0, q, k, v, ref_md)
    w.reqs = saved
    batch.out_loc = torch.from_numpy(ref_md.out_loc).cuda()
    backend.prepare_metadata(batch)
    with torch.cuda.stream(stream):
        qkv_buf.copy_(qkv.cuda())
        out_loc_buf.copy_(batch.out_loc)
        backend.prepare_for_replay(batch)
        graph.replay()
    torch.cuda.synchronize()
    attn_tolerance_ok(out_buf[:3], ref_out[:3], "graph replay")
    kc, _ = gw.pool_rows(0)
    slots = torch.from_numpy(ref_md.out_loc[:3].astype(np.int64))
    assert torch.equal(kc[slots].view(torch.int16), ref_kc[slots].view(torch.int16))


def test_decode_full_size_properties(b200, native_lib, decode_impl):
    """BASELINE cfg1 decode shape (256 seqs, Qwen3-0.6B heads, lens U[100,2048]) -- too big for
    the CPU oracle in seconds, so size-independent properties: (a) appended rows bit-exact,
    (b) a sample of requests matches the oracle, (c) invariance to the split-KV chunking,
    (d) linearity in V."""
    rnd = random.Random(0)
    bs, hq, hkv, d, ps = 256, 16, 8, 128, 64
    lens = [(n - 1, n) for n in (rnd.randint(100, 2048) for _ in range(bs))]
    w = make_world(seed=2, page_size=ps, hq=hq, hkv=hkv, max_reqs=bs, max_seq=2048)
    add_requests(w, lens)
    gw = GpuWorld(b200, w)
    batch = gw.batch("decode")
    ref_md = o_meta.ref_prepare_metadata(w.page_table, w.reqs, ps)
    qkv, q, k, v = make_inputs(w, 3)
    qkv_g = qkv.cuda()
    qg, kg, vg = qkv_g.split([hq * d, hkv * d, hkv * d], dim=-1)
    batch.out_loc = torch.from_numpy(ref_md.out_loc).cuda()
    gw.backend.prepare_metadata(batch)
    out = gw.backend.forward(qg.view(-1, hq, d), kg, vg, 0, batch).clone()
    torch.cuda.synchronize()
    # (a)
    kc, vc = gw.pool_rows(0)
    slots = torch.from_numpy(ref_md.out_loc.astype(np.int64))
    assert torch.equal(kc[slots].view(torch.int16), k.reshape(bs, hkv, d).contiguous().view(torch.int16))
    assert torch.equal(vc[slots].view(torch.int16), v.reshape(bs, hkv, d).contiguous().view(torch.int16))
    # (b) sample
    from oracle.attention import ref_attention_one
    for r in rnd.sample(range(bs), 6):
        n = lens[r][1]
        idx = torch.from_numpy(ref_md.slot_table[r, :n].astype(np.int64))
        ref = ref_attention_one(q[r : r + 1].reshape(1, hq, d), kc[idx], vc[idx], d**-0.5)
        attn_tolerance_ok(out[r : r + 1], ref, f"sample req {r}")
    # (c) different chunking: the default plan keeps 256 requests unsplit; a plan built for a much
    # larger grid splits every request into several chunks (partials + combine)
    md = batch.attn_metadata
    lib = native_lib
    info = torch.tensor([x for t in w.reqs for x in t], dtype=torch.int32).cuda()
    rc = lib.b200_build_metadata(info.data_ptr(), bs, gw.ctx.page_table.data_ptr(), gw.ctx.page_table.stride(0),
                                 md.cache_seqlens.data_ptr(), md.cu_seqlens_q.data_ptr(), md.cu_seqlens_k.data_ptr(),
                                 md.page_table.data_ptr(), md.page_table.stride(0), md.page_table.shape[1],
                                 md.decode_plan.data_ptr(), hkv, 8192, torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    out2 = gw.backend.forward(qg.view(-1, hq, d), kg, vg, 0, batch)
    torch.cuda.synchronize()
    assert int(md.decode_plan[1]) > bs  # really split
    assert (out2.float() - out.float()).abs().max().item() <= 2e-2 * out.float().abs().max().item()
    # (d) linearity in V: attn(V) with V scaled by 2 == 2 * attn(V) up to rounding
    gw.pool._kv_buffer[1].mul_(2)
    out3 = gw.backend.forward(qg.view(-1, hq, d), kg, vg * 2, 0, batch)
    torch.cuda.synchronize()
    assert (out3.float() - 2 * out2.float()).abs().max().item() <= 2e-2 * out3.float().abs().max().item()


@pytest.mark.parametrize("phase", ["decode", "prefill"])
def test_attention_against_flashinfer_golden(b200, native_lib, phase):
    """Product path vs the outputs FlashInfer (fa2 wrappers, the reference's parity oracle) produced
    for the same inputs (tests/golden/make_flashinfer_golden.py)."""
    from pathlib import Path

    from helpers import World

    fi = np.load(Path(__file__).parent / "golden" / "flashinfer_golden.npz")
    bf = lambda a: torch.from_numpy(a.view(np.int16).copy()).view(torch.bfloat16)  # noqa: E731
    hq, hkv, d, ps = 4, 2, 128, 16
    reqs = [tuple(r) for r in fi[f"{phase}_reqs"].tolist()]
    pt = fi[f"{phase}_page_table"]
    used = fi[f"{phase}_used_slots"]
    num_pages = (int(pt.max()) // ps) + 1
    pool = torch.zeros((2, 1, (num_pages + 1) * ps, hkv, d), dtype=torch.bfloat16)
    pool[0, 0, torch.from_numpy(used).long()] = bf(fi[f"{phase}_k_rows"])
    pool[1, 0, torch.from_numpy(used).long()] = bf(fi[f"{phase}_v_rows"])
    w = World(ps, num_pages, hq, hkv, d, 1, torch.bfloat16, pt.copy(), [], pool, reqs)
    md = o_meta.ref_prepare_metadata(pt, reqs, ps)
    gw = GpuWorld(b200, w)
    batch = gw.batch(phase)
    loc = torch.from_numpy(md.out_loc.astype(np.int64))
    q = bf(fi[f"{phase}_q"]).cuda()
    k_new = pool[0, 0, loc].reshape(len(loc), -1).cuda()  # the golden pool already holds the appended rows
    v_new = pool[1, 0, loc].reshape(len(loc), -1).cuda()
    batch.out_loc = torch.from_numpy(md.out_loc).cuda()
    batch.positions = torch.from_numpy(md.positions).cuda()
    gw.backend.prepare_metadata(batch)
    out = gw.backend.forward(q, k_new, v_new, 0, batch)
    torch.cuda.synchronize()
    want = bf(fi[f"{phase}_out"]).float()
    got = out.float().cpu()
    scale = want.abs().max().item()
    # both sides are bf16 outputs of bf16-P tensor-core pipelines: 1e-3 relative + one output ulp each
    bound = 1e-3 * scale + 2.0**-7 * want.abs() + 1e-6
    assert ((got - want).abs() <= bound).all(), ((got - want).abs() - bound).max()
    assert ((got - want).norm() / want.norm()).item() < 2.5e-3


@pytest.mark.parametrize("page_size", [1, 16, 64])
def test_prefill_unaligned_cached_boundary(b200, native_lib, page_size, prefill_impl):
    """Chunked prefill leaves cached_len at arbitrary offsets (scheduler/prefill.py:126-151): the
    K/V tile that straddles cached_len mixes pool rows and rows of this forward's k/v inputs."""
    _run_case(b200, page_size=page_size, hq=16, hkv=8, lens=[(100, 300), (37, 200), (129, 130), (1, 140)],
              phase="prefill")


# ------------------------------------------------------------------ fused pre-attention decode
def _fused_vs_unfused(b200, *, page_size, hq, hkv, lens, with_norm=True, pad_to=None, seed=3, dtype=torch.bfloat16,
                      force_split=False):
    """b200_attn_decode_fused (raw q / k in, qk-norm + RoPE + append + attention in ONE launch) must equal
    ops.qknorm_rope_inplace followed by backend.forward BIT FOR BIT: output, appended K/V rows, and the
    raw q / k inputs must stay untouched."""
    from oracle.rope import ref_cos_sin_cache

    max_seq = max(d for _, d in lens) + 8
    w = make_world(seed=seed, page_size=page_size, hq=hq, hkv=hkv, max_reqs=max(len(lens), pad_to or 0) + 1,
                   max_seq=max_seq, dtype=dtype)
    add_requests(w, lens)
    triples = list(w.reqs)
    if pad_to:
        triples += [(w.page_table.shape[0] - 1, 0, 1)] * (pad_to - len(w.reqs))
    ref_md = o_meta.ref_prepare_metadata(w.page_table, triples, page_size)
    saved, w.reqs = w.reqs, triples
    qkv, _, _, _ = make_inputs(w, seed + 1)
    w.reqs = saved
    d = w.d
    cache = ref_cos_sin_cache(d, max(4096, max_seq), 1e6).cuda()
    g = torch.Generator().manual_seed(seed)
    qw = (torch.rand(d, generator=g) + 0.5).to(dtype).cuda() if with_norm else None
    kw = (torch.rand(d, generator=g) + 0.5).to(dtype).cuda() if with_norm else None
    prev = b200._cabi.set_option("decode_plan_nosplit", 0) if force_split else None
    try:
        results = []
        for fused in (False, True):
            gw = GpuWorld(b200, w)
            batch = gw.batch("decode", pad_to=pad_to)
            batch.positions = torch.from_numpy(ref_md.positions).cuda()
            batch.out_loc = torch.from_numpy(ref_md.out_loc).cuda()
            gw.backend.prepare_metadata(batch)
            x = qkv.cuda()
            q, k, v = x.split([hq * d, hkv * d, hkv * d], dim=-1)
            if fused:
                out = gw.backend.forward_decode_fused(q.view(-1, hq, d), k, v, 0, batch, batch.positions, cache, qw, kw, 1e-6)
                torch.cuda.synchronize()
                assert torch.equal(x.cpu().view(torch.int16), qkv.view(torch.int16)), "fused decode modified its raw inputs"
            else:
                b200.ops.qknorm_rope_inplace(batch.positions, q, k, d, cache, qw, kw, 1e-6)
                out = gw.backend.forward(q.view(-1, hq, d), k, v, 0, batch)
                torch.cuda.synchronize()
            kc, vc = gw.pool_rows(0)
            results.append((out.cpu(), kc, vc))
            b200.core.set_global_ctx(None)
    finally:
        if prev is not None:
            b200._cabi.set_option("decode_plan_nosplit", prev)
    (o0, k0, v0), (o1, k1, v1) = results
    n_real = len(lens)
    assert torch.equal(o0[:n_real].view(torch.int16), o1[:n_real].view(torch.int16)), \
        f"fused output differs: max |d| {(o0[:n_real].float() - o1[:n_real].float()).abs().max().item():.3e}"
    slots = torch.from_numpy(ref_md.out_loc[:n_real].astype(np.int64))
    assert torch.equal(k0[slots].view(torch.int16), k1[slots].view(torch.int16))
    assert torch.equal(v0[slots].view(torch.int16), v1[slots].view(torch.int16))
    mask = torch.ones(k0.shape[0], dtype=torch.bool)
    mask[torch.from_numpy(ref_md.out_loc.astype(np.int64))] = False
    assert torch.equal(k0[mask].view(torch.int16), k1[mask].view(torch.int16))


@pytest.mark.parametrize("page_size", [1, 64])
@pytest.mark.parametrize("name", list(DECODE_LENS))
def test_decode_fused_pre_attention_bit_identical(b200, native_lib, page_size, name):
    _fused_vs_unfused(b200, page_size=page_size, hq=16, hkv=8, lens=DECODE_LENS[name])


@pytest.mark.parametrize("hq,hkv", [(8, 8), (40, 8), (8, 1), (2, 1), (7, 1), (6, 2), (3, 1)])
def test_decode_fused_gqa_groups(b200, native_lib, hq, hkv):
    _fused_vs_unfused(b200, page_size=16, hq=hq, hkv=hkv, lens=DECODE_LENS["mixed"][:5])


def test_decode_fused_without_qk_norm_and_padded(b200, native_lib):
    """Llama-style layer (no q/k norm weights) and a graph-padded batch of dummy requests (kv_len 1:
    units that consist of the appended token only)."""
    _fused_vs_unfused(b200, page_size=16, hq=8, hkv=1, lens=DECODE_LENS["mixed"][:3], with_norm=False)
    _fused_vs_unfused(b200, page_size=16, hq=16, hkv=8, lens=DECODE_LENS["mixed"][:3], pad_to=8)


def test_decode_fused_split_kv_and_many_units(b200, native_lib):
    """Split-KV (several chunks per request: only the last chunk owns the new token) and more
    last-chunk units per CTA than ring slots."""
    _fused_vs_unfused(b200, page_size=64, hq=16, hkv=8, lens=DECODE_LENS["long"] + [(700, 701)], force_split=True)
    rnd = random.Random(4)
    lens = [(n - 1, n) for n in (rnd.randint(1, 300) for _ in range(200))]
    _fused_vs_unfused(b200, page_size=16, hq=16, hkv=8, lens=lens)


def test_decode_fused_fp16(b200, native_lib):
    _fused_vs_unfused(b200, page_size=1, hq=16, hkv=8, lens=DECODE_LENS["mixed"][:4], dtype=torch.float16)


# ------------------------------------------------------------------ reference GPU goldens at real shapes
def _gpu_golden():
    from pathlib import Path

    path = Path(__file__).parent / "golden" / "reference_gpu_golden.npz"
    if not path.exists():
        return None, []
    import json

    z = np.load(path)
    return z, json.loads(bytes(z["cases"]).decode())


_GOLD, _GOLD_CASES = _gpu_golden()


@pytest.mark.skipif(_GOLD is None, reason="tests/golden/reference_gpu_golden.npz not generated yet")
@pytest.mark.parametrize("case", _GOLD_CASES, ids=[c["name"] for c in _GOLD_CASES])
def test_attention_against_reference_gpu_goldens(b200, native_lib, case):
    """Product path vs the outputs of the reference's FlashInfer-fa2 path and, where the page size allows,
    its TRT-LLM-gen path (tests/golden/make_reference_gpu_golden.py), at the BASELINE head shapes.  One
    criterion (oracle/tolerance.vs_reference_gpu): |a - b| <= 1e-3 max|b| + one output ulp."""
    import sys
    from pathlib import Path

    sys.path.insert(0, str(Path(__file__).parent / "golden"))
    import helpers
    from make_reference_gpu_golden import build_case
    from oracle import tolerance

    bf = lambda a: torch.from_numpy(a.view(np.int16).copy()).view(torch.bfloat16)  # noqa: E731
    w, md, qkv = build_case(case, helpers, o_meta)
    hq, hkv, d = case["hq"], case["hkv"], 128
    gw = GpuWorld(b200, w)
    batch = gw.batch(case["phase"])
    g = qkv.cuda()
    qg, kg, vg = g.split([hq * d, hkv * d, hkv * d], dim=-1)
    batch.out_loc = torch.from_numpy(md.out_loc).cuda()
    batch.positions = torch.from_numpy(md.positions).cuda()
    gw.backend.prepare_metadata(batch)
    out = gw.backend.forward(qg.view(-1, hq, d), kg, vg, 0, batch)
    torch.cuda.synchronize()
    got = out[:: case["step"]].cpu()
    for ref_name in ("fi", "trtllm"):
        key = f"{case['name']}_{ref_name}"
        if key not in _GOLD:
            continue
        want = bf(_GOLD[key])
        err = tolerance.vs_reference_gpu(got, want)
        assert err <= tolerance.GPU_REL_TOL, f"{key}: excess error {err:.3e} (gate {tolerance.GPU_REL_TOL})"


# ------------------------------------------------------------------ per-CTA unit lists longer than their smem cache
def test_decode_more_units_than_the_smem_unit_cache(b200, native_lib):
    """kMaxUnitsSmem = 96 units per CTA are decoded into shared memory; beyond that the roles decode
    units on the fly (attn_decode_tc.cu unit_at).  2000 short requests x 8 kv heads = 16 000 units > 96 x 132."""
    rnd = random.Random(11)
    lens = [(n - 1, n) for n in (rnd.randint(1, 9) for _ in range(2000))]
    _run_case(b200, page_size=16, hq=16, hkv=8, lens=lens, phase="decode", max_seq=32)


def test_prefill_more_units_than_the_smem_unit_cache(b200, native_lib):
    """Same for the prefill kernel (kMaxUnitsSmem = 64): 1250 two-token extends x 16 query heads = 20 000 units."""
    lens = [(3, 5)] * 1250
    _run_case(b200, page_size=1, hq=16, hkv=8, lens=lens, phase="prefill", max_seq=32)


def test_prefill_q_len_4096(b200, native_lib):
    """One 4096-token prompt at the GQA-8 tp-shard shape (32 query tiles x 32 K/V tiles), a chunked
    continuation on top of a long cached prefix, and a 2048-token prompt at the Qwen3-0.6B shape."""
    _run_case(b200, page_size=64, hq=8, hkv=1, lens=[(0, 4096)], phase="prefill")
    _run_case(b200, page_size=64, hq=8, hkv=1, lens=[(4096, 4352), (2048, 4096)], phase="prefill")
    _run_case(b200, page_size=64, hq=16, hkv=8, lens=[(0, 2048)], phase="prefill")
