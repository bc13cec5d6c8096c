"""GPU parity: store / RMSNorm / RoPE kernels vs the CPU oracle, through the C ABI (ops.py)."""
import pytest
import torch

from oracle import norm as o_norm
from oracle import rope as o_rope
from oracle.index import ref_indexing
from oracle.store import ref_store_kv

pytestmark = pytest.mark.gpu


def _ulp_close(a: torch.Tensor, b: torch.Tensor, ulps: float = 1.0):
    """|a-b| <= ulps * ulp(b) elementwise for 16-bit floats (fp32 reduction-order noise only)."""
    a32, b32 = a.float().cpu(), b.float().cpu()
    eps = 2.0**-8 if a.dtype == torch.bfloat16 else 2.0**-11
    tol = ulps * eps * b32.abs().clamp_min(1e-3) * 2
    bad = (a32 - b32).abs() > tol
    assert not bad.any(), f"{bad.sum().item()} / {bad.numel()} beyond {ulps} ulp; max {((a32-b32).abs()).max()}"


@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64])
def test_store_reference_golden_shape(b200, native_lib, idx_dtype):
    """The reference's own test (tests/kernel/test_store.py:10-34): fp16 cache, k/v = strided
    slices of one [bs, 4*128] buffer, randperm indices, bs = 2^0 .. 2^15, bit exact."""
    HEAD, TOKENS = 128, 1 << 18
    g = torch.Generator(device="cuda").manual_seed(0)
    kv_cache = torch.randn((TOKENS, 2, HEAD), device="cuda", dtype=torch.float16, generator=g)
    k_cache, v_cache = kv_cache[:, 0, :], kv_cache[:, 1, :]
    for bs in [2**n for n in range(0, 16)]:
        indices = torch.randperm(TOKENS, device="cuda", generator=g)[:bs].to(idx_dtype)
        qkv = torch.randn((bs, HEAD * 4), device="cuda", dtype=torch.float16, generator=g)
        k, v = qkv[:, :HEAD], qkv[:, HEAD : HEAD * 2]
        b200.ops.store_cache(k_cache, v_cache, indices, k, v)
        assert torch.all(k_cache[indices.long()] == k), bs
        assert torch.all(v_cache[indices.long()] == v), bs


@pytest.mark.parametrize("hkv,dtype", [(8, torch.bfloat16), (1, torch.bfloat16), (2, torch.float16), (16, torch.bfloat16)])
def test_store_matches_oracle_bitwise(b200, native_lib, hkv, dtype):
    torch.manual_seed(1)
    slots, n, d = 4096, 777, 128
    kc = torch.randn(slots, hkv, d).to(dtype)
    vc = torch.randn(slots, hkv, d).to(dtype)
    qkv = torch.randn(n, (4 + 2 * hkv) * d).to(dtype)
    k = qkv[:, 4 * d : (4 + hkv) * d]
    v = qkv[:, (4 + hkv) * d :]
    idx = torch.randperm(slots)[:n].to(torch.int32)
    kc_g, vc_g = kc.cuda(), vc.cuda()
    qkv_g = qkv.cuda()
    b200.ops.store_cache(kc_g, vc_g, idx.cuda(), qkv_g[:, 4 * d : (4 + hkv) * d], qkv_g[:, (4 + hkv) * d :])
    ref_store_kv(kc, vc, idx, k, v)
    assert torch.equal(kc_g.cpu().view(torch.int16), kc.view(torch.int16))
    assert torch.equal(vc_g.cpu().view(torch.int16), vc.view(torch.int16))


def test_store_rejects_bad_args(b200, native_lib):
    kc = torch.zeros(16, 128, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):
        b200.ops.store_cache(kc, kc, torch.zeros(2, dtype=torch.int16, device="cuda"), kc[:2], kc[:2])
    with pytest.raises(RuntimeError):
        b200.ops.store_cache(kc.cpu(), kc.cpu(), torch.zeros(2, dtype=torch.int32), kc[:2].cpu(), kc[:2].cpu())


def test_indexing_reference_golden_shape(b200, native_lib):
    """The reference's own tests (tests/kernel/test_index.py:32-99): fp16 table with 4096-wide rows,
    int32 indices, bs = 2^0 .. 2^15, plain and masked to the vocabulary shard of rank 1 of 4."""
    import torch.nn.functional as F

    EMBED, TOKENS, TP = 4096, 32768, 4
    g = torch.Generator(device="cuda").manual_seed(0)
    weights = torch.randn((TOKENS, EMBED), device="cuda", dtype=torch.float16, generator=g)
    shard = TOKENS // TP
    for bs in [2**n for n in range(0, 16)]:
        indices = torch.randint(0, TOKENS, (bs,), device="cuda", dtype=torch.int32, generator=g)
        assert torch.all(b200.ops.indexing(weights, indices) == F.embedding(indices.long(), weights)), bs
        got = b200.ops.indexing(weights[:shard], indices, vocab_range=(shard, shard))
        pos = indices.long() - shard
        mask = (pos < 0) | (pos >= shard)
        want = F.embedding(pos.masked_fill(mask, 0), weights[:shard])
        want[mask] = 0
        assert torch.all(got == want), bs


@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("dim,dtype", [(1024, torch.bfloat16), (128, torch.bfloat16), (5120, torch.float16), (8, torch.bfloat16)])
def test_indexing_matches_oracle_bitwise(b200, native_lib, idx_dtype, dim, dtype):
    """Bit-exact vs the oracle: plain, masked (incl. ids below the shard start, which wrap as unsigned),
    empty input, caller-provided output, row-strided table, and the last-token gather use."""
    torch.manual_seed(2)
    vocab = 3001
    w = torch.randn(vocab, dim).to(dtype)
    wg = w.cuda()
    bits = torch.int16
    for n in (0, 1, 33, 2500):
        idx = torch.randint(0, vocab, (n,), dtype=idx_dtype)
        got = b200.ops.indexing(wg, idx.cuda())
        assert got.shape == (n, dim)
        assert torch.equal(got.cpu().view(bits), ref_indexing(w, idx).view(bits))
        for rng in ((1000, 750), (0, vocab), (2900, 101)):
            shard = w[rng[0] : rng[0] + rng[1]]
            out = torch.full((n, dim), 7.0, dtype=dtype, device="cuda")
            ret = b200.ops.indexing(wg[rng[0] : rng[0] + rng[1]], idx.cuda(), output=out, vocab_range=rng)
            assert ret.data_ptr() == out.data_ptr()
            assert torch.equal(out.cpu().view(bits), ref_indexing(shard, idx, rng).view(bits))
    # row-strided table (a column slice of a wider matrix) and the LM-head gather x[last_indices]
    if dim >= 16:
        wide = torch.randn(257, 2 * dim).to(dtype)
        idx = torch.randint(0, 257, (64,), dtype=idx_dtype)
        got = b200.ops.indexing(wide.cuda()[:, dim:], idx.cuda())
        assert torch.equal(got.cpu().view(bits), wide[:, dim:][idx.long()].contiguous().view(bits))


def test_indexing_rejects_bad_args(b200, native_lib):
    w = torch.zeros(16, 128, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):
        b200.ops.indexing(w, torch.zeros(2, dtype=torch.int16, device="cuda"))
    with pytest.raises(RuntimeError):
        b200.ops.indexing(w, torch.zeros(2, dtype=torch.int32, device="cuda"), output=torch.zeros(3, 128, device="cuda", dtype=torch.bfloat16))
    with pytest.raises(RuntimeError):
        b200.ops.indexing(w.cpu(), torch.zeros(2, dtype=torch.int32))
    with pytest.raises(RuntimeError):  # rows of 4 * 2 = 8 bytes: not a multiple of 16
        b200.ops.indexing(torch.zeros(16, 4, device="cuda", dtype=torch.bfloat16), torch.zeros(2, dtype=torch.int32, device="cuda"))


@pytest.mark.parametrize("rows,dim", [(1, 1024), (37, 1024), (256, 5120), (19, 8192), (5, 4096), (3, 2048 + 64)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_rmsnorm_rows(b200, native_lib, rows, dim, dtype):
    torch.manual_seed(rows * dim)
    x = (torch.randn(rows, dim) * 3).to(dtype)
    w = (torch.randn(dim) * 0.5 + 1).to(dtype)
    ref = o_norm.ref_rmsnorm(x, w, 1e-6)
    out = b200.ops.rmsnorm(x.cuda(), w.cuda(), 1e-6)
    _ulp_close(out, ref)
    xg = x.cuda()
    b200.ops.rmsnorm(xg, w.cuda(), 1e-6, out=xg)  # in place (forward_inplace)
    _ulp_close(xg, ref)


@pytest.mark.parametrize("heads,d", [(16, 128), (8, 128), (5, 64), (2, 256)])
def test_rmsnorm_per_head_strided(b200, native_lib, heads, d):
    """q/k norm: 3-D view of a slice of the fused qkv buffer, in place (layers/attention.py:50-53)."""
    torch.manual_seed(7)
    nnz, width = 53, heads * d + 2 * 64
    buf = torch.randn(nnz, width).to(torch.bfloat16)
    w = (torch.rand(d) + 0.5).to(torch.bfloat16)
    ref = o_norm.ref_rmsnorm(buf[:, : heads * d].reshape(nnz, heads, d), w, 1e-6)
    bg = buf.cuda()
    view = bg[:, : heads * d].view(nnz, heads, d)
    b200.ops.rmsnorm(view, w.cuda(), 1e-6, out=view)
    _ulp_close(view, ref)
    assert torch.equal(bg[:, heads * d :].cpu(), buf[:, heads * d :])  # neighbours untouched


@pytest.mark.parametrize("rows,dim", [(1, 1024), (64, 1024), (33, 5120), (7, 8192)])
def test_fused_add_rmsnorm(b200, native_lib, rows, dim):
    torch.manual_seed(3)
    x = torch.randn(rows, dim).to(torch.bfloat16)
    res = (torch.randn(rows, dim) * 2).to(torch.bfloat16)
    w = (torch.rand(dim) + 0.5).to(torch.bfloat16)
    ref_x, ref_res = o_norm.ref_fused_add_rmsnorm(x, res, w, 1e-6)
    xg, rg = x.cuda(), res.cuda()
    b200.ops.fused_add_rmsnorm(xg, rg, w.cuda(), 1e-6)
    assert torch.equal(rg.cpu().view(torch.int16), ref_res.view(torch.int16))  # residual: exact
    _ulp_close(xg, ref_x)


@pytest.mark.parametrize("pos_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("hq,hkv,d", [(16, 8, 128), (8, 1, 128), (40, 8, 128), (4, 4, 64)])
def test_rope_neox(b200, native_lib, pos_dtype, hq, hkv, d):
    torch.manual_seed(11)
    nnz, max_pos = 97, 4096
    cache = o_rope.ref_cos_sin_cache(d, max_pos, 1e6)
    qkv = torch.randn(nnz, (hq + 2 * hkv) * d).to(torch.bfloat16)
    pos = torch.randint(0, max_pos, (nnz,), dtype=pos_dtype)
    q, k = qkv[:, : hq * d], qkv[:, hq * d : (hq + hkv) * d]
    ref_q = o_rope.ref_apply_rope_neox(pos, q, d, cache)
    ref_k = o_rope.ref_apply_rope_neox(pos, k, d, cache)
    g = qkv.cuda()
    b200.ops.apply_rope_with_cos_sin_cache_inplace(
        positions=pos.cuda(), query=g[:, : hq * d], key=g[:, hq * d : (hq + hkv) * d],
        head_size=d, cos_sin_cache=cache.cuda())
    _ulp_close(g[:, : hq * d], ref_q)
    _ulp_close(g[:, hq * d : (hq + hkv) * d], ref_k)
    assert torch.equal(g[:, (hq + hkv) * d :].cpu(), qkv[:, (hq + hkv) * d :])  # v untouched


def test_rope_llama3_and_yarn_cache_match_oracle(b200):
    sc = {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
          "original_max_position_embeddings": 8192}
    a = b200.layers.RotaryEmbedding(128, 128, 2048, 500000.0, sc)._cos_sin_cache
    assert torch.equal(a, o_rope.ref_cos_sin_cache(128, 2048, 500000.0, sc))
    sc = {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 4096}
    a = b200.layers.RotaryEmbedding(128, 128, 2048, 10000.0, sc)._cos_sin_cache
    assert torch.equal(a, o_rope.ref_cos_sin_cache(128, 2048, 10000.0, sc))


@pytest.mark.parametrize("with_norm", [True, False])
def test_fused_qknorm_rope_equals_three_launches(b200, native_lib, with_norm):
    """The fused pre-attention launch must be bit-identical to norm -> norm -> rope."""
    torch.manual_seed(5)
    nnz, hq, hkv, d = 130, 16, 8, 128
    cache = o_rope.ref_cos_sin_cache(d, 4096, 1e6).cuda()
    qkv = torch.randn(nnz, (hq + 2 * hkv) * d).to(torch.bfloat16).cuda()
    pos = torch.randint(0, 4096, (nnz,), dtype=torch.int32).cuda()
    qw = (torch.rand(d) + 0.5).to(torch.bfloat16).cuda() if with_norm else None
    kw = (torch.rand(d) + 0.5).to(torch.bfloat16).cuda() if with_norm else None
    a, b = qkv.clone(), qkv.clone()
    qa, ka = a[:, : hq * d], a[:, hq * d : (hq + hkv) * d]
    if with_norm:
        b200.ops.rmsnorm(qa.view(nnz, hq, d), qw, 1e-6, out=qa.view(nnz, hq, d))
        b200.ops.rmsnorm(ka.view(nnz, hkv, d), kw, 1e-6, out=ka.view(nnz, hkv, d))
    b200.ops.apply_rope_with_cos_sin_cache_inplace(pos, qa, ka, d, cache)
    b200.ops.qknorm_rope_inplace(pos, b[:, : hq * d], b[:, hq * d : (hq + hkv) * d], d, cache, qw, kw, 1e-6)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("which", ["q_only", "k_only"])
@pytest.mark.parametrize("d", [64, 128])
def test_fused_qknorm_rope_mixed_weights(b200, native_lib, which, d):
    """Only one of q_weight / k_weight given: a warp then holds normed and un-normed head groups side
    by side (2 groups per warp at D=128, 4 at D=64) -- the group reduction must not diverge."""
    torch.manual_seed(6)
    nnz, hq, hkv = 37, 3, 1  # odd head counts: q and k groups share warps
    cache = o_rope.ref_cos_sin_cache(d, 512, 1e6).cuda()
    qkv = torch.randn(nnz, (hq + 2 * hkv) * d).to(torch.bfloat16).cuda()
    pos = torch.randint(0, 512, (nnz,), dtype=torch.int32).cuda()
    qw = (torch.rand(d) + 0.5).to(torch.bfloat16).cuda() if which == "q_only" else None
    kw = (torch.rand(d) + 0.5).to(torch.bfloat16).cuda() if which == "k_only" else None
    a, b = qkv.clone(), qkv.clone()
    qa, ka = a[:, : hq * d], a[:, hq * d : (hq + hkv) * d]
    if qw is not None:
        b200.ops.rmsnorm(qa.view(nnz, hq, d), qw, 1e-6, out=qa.view(nnz, hq, d))
    if kw is not None:
        b200.ops.rmsnorm(ka.view(nnz, hkv, d), kw, 1e-6, out=ka.view(nnz, hkv, d))
    b200.ops.apply_rope_with_cos_sin_cache_inplace(pos, qa, ka, d, cache)
    b200.ops.qknorm_rope_inplace(pos, b[:, : hq * d], b[:, hq * d : (hq + hkv) * d], d, cache, qw, kw, 1e-6)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


# ------------------------------------------------------------------ against FlashInfer itself
def _fi():
    import numpy as np
    from pathlib import Path

    return np.load(Path(__file__).parent / "golden" / "flashinfer_golden.npz")


def _bf(a):
    import numpy as np

    return torch.from_numpy(a.view(np.int16).copy()).view(torch.bfloat16).cuda()


def test_rope_and_norms_bit_identical_to_flashinfer(b200, native_lib):
    """Golden outputs of the FlashInfer ops the reference binds (layers/rotary.py:45, norm.py:16-38):
    the project's kernels reproduce them bit for bit."""
    fi = _fi()
    hq, hkv, d = 4, 2, 128
    x = _bf(fi["rope_x"])
    pos = torch.from_numpy(fi["rope_pos"]).cuda()
    from oracle.rope import ref_cos_sin_cache

    b200.ops.apply_rope_with_cos_sin_cache_inplace(pos, x[:, : hq * d], x[:, hq * d : (hq + hkv) * d], d,
                                                   ref_cos_sin_cache(d, 1024, 1e6).cuda())
    assert torch.equal(x.view(torch.int16), _bf(fi["rope_out"]).view(torch.int16))
    y = b200.ops.rmsnorm(_bf(fi["norm_x"]), _bf(fi["norm_w"]), 1e-6)
    assert torch.equal(y.view(torch.int16), _bf(fi["norm_out"]).view(torch.int16))
    xh = _bf(fi["qknorm_x"])
    b200.ops.rmsnorm(xh, _bf(fi["qknorm_w"]), 1e-6, out=xh)
    assert torch.equal(xh.view(torch.int16), _bf(fi["qknorm_out"]).view(torch.int16))
    xf, rf = _bf(fi["fused_x"]), _bf(fi["fused_res"])
    b200.ops.fused_add_rmsnorm(xf, rf, _bf(fi["norm_w"]), 1e-6)
    assert torch.equal(xf.view(torch.int16), _bf(fi["fused_x_out"]).view(torch.int16))
    assert torch.equal(rf.view(torch.int16), _bf(fi["fused_res_out"]).view(torch.int16))
