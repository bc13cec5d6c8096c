"""CPU: pin the oracle's integer functions against golden vectors produced by the reference's own
Python code (tests/golden/make_metadata_golden.py), and cross-check the oracle's internals."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import attention as o_attn
from oracle import metadata as o_meta
from oracle import norm as o_norm
from oracle import rope as o_rope
from oracle.index import ref_indexing
from oracle.store import ref_store_kv, ref_store_kv_bytes

GOLDEN = json.loads((Path(__file__).parent / "golden" / "metadata_golden.json").read_text())


@pytest.mark.parametrize("case", GOLDEN["cases"], ids=lambda c: c["name"])
def test_metadata_oracle_matches_reference(case):
    pt = np.array(case["page_table"], dtype=np.int32)
    reqs = [tuple(r) for r in case["reqs"]]
    ps = case["page_size"]
    md = o_meta.ref_prepare_metadata(pt, reqs, ps)
    assert md.positions.tolist() == case["positions"]
    assert md.out_loc.tolist() == case["out_loc"]
    assert md.cu_seqlens_q.tolist() == case["fa_cu_seqlens_q"] == case["fi_cu_seqlens_q"]
    assert md.cu_seqlens_k.tolist() == case["fa_cu_seqlens_k"] == case["fi_cu_seqlens_k"]
    assert md.cache_seqlens.tolist() == case["fa_cache_seqlens"] == case["fi_seq_lens"]
    assert md.max_seqlen_q == case["fa_max_seqlen_q"] and md.max_seqlen_k == case["fa_max_seqlen_k"]
    assert md.page_table_paged.tolist() == case["fa_page_table"]
    assert md.indices_flat.tolist() == case["fi_indices"]
    assert md.last_indices.tolist() == case["last_indices"] == case["fi_last_indices"]
    for a in (md.cu_seqlens_q, md.cu_seqlens_k, md.cache_seqlens, md.out_loc, md.positions,
              md.page_table_paged, md.indices_flat, md.slot_table, md.last_indices):
        assert a.dtype == np.int32


@pytest.mark.parametrize("case", GOLDEN["cases"], ids=lambda c: c["name"])
def test_allocation_oracle_matches_reference(case):
    """ref_allocate_paged reproduces the page table CacheManager.allocate_paged wrote."""
    gold = np.array(case["page_table"], dtype=np.int32)
    ps = case["page_size"]
    table = np.zeros_like(gold)
    table[-1, :] = gold[-1, 0]  # dummy row
    free = list(case["free_slots_before"])
    real = [tuple(r) for r in case["reqs"] if r[0] != gold.shape[0] - 1]
    pre = [(t, 0, c) for (t, c, d) in real if c > 0]
    o_meta.ref_allocate_paged(table, free, pre, ps)
    o_meta.ref_allocate_paged(table, free, real, ps)
    assert np.array_equal(table, gold)


def test_store_oracle_is_a_byte_scatter():
    torch.manual_seed(0)
    kc = torch.randn(64, 2, 128).to(torch.bfloat16)
    vc = torch.randn(64, 2, 128).to(torch.bfloat16)
    qkv = torch.randn(9, 1024).to(torch.bfloat16)
    k, v = qkv[:, 256:512], qkv[:, 512:768]
    idx = torch.randperm(64)[:9].to(torch.int32)
    kb = kc.view(64, -1).view(torch.uint8).numpy().copy()
    ref_store_kv(kc, vc, idx, k, v)
    want = ref_store_kv_bytes(kb, idx.numpy(), k.contiguous().view(torch.uint8).numpy())
    assert np.array_equal(kc.view(64, -1).view(torch.uint8).numpy(), want)
    assert torch.equal(vc[idx.long()].view(9, -1), v)


def _reference_known_answer_indexing(weights, indices, vocab_range=None):
    """The reference's own checker for its index kernel (tests/kernel/test_index.py:13-29)."""
    import torch.nn.functional as F

    if vocab_range is None:
        return F.embedding(indices, weights)
    start, length = vocab_range
    indices = indices - start
    mask = (indices < 0) | (indices >= length)
    indices = indices.masked_fill(mask, 0)
    result = F.embedding(indices, weights)
    result[mask] = 0
    return result


@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("vocab_range", [None, (1000, 1000), (0, 4000), (3000, 1000)])
def test_index_oracle_matches_reference_known_answer(idx_dtype, vocab_range):
    torch.manual_seed(5)
    vocab, dim = 4000, 256
    rows = vocab if vocab_range is None else vocab_range[1]
    w = torch.randn(rows, dim).to(torch.float16)
    for n in (1, 7, 512):
        idx = torch.randint(0, vocab, (n,), dtype=idx_dtype)
        got = ref_indexing(w, idx, vocab_range)
        want = _reference_known_answer_indexing(w, idx.long(), vocab_range)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16))


def test_attention_oracle_against_naive_loops():
    """SDPA restatement vs a literal per-element softmax (small case, pure loops)."""
    torch.manual_seed(1)
    q_len, kv_len, hq, hkv, d = 3, 7, 4, 2, 16
    q = torch.randn(q_len, hq, d).to(torch.bfloat16)
    k = torch.randn(kv_len, hkv, d).to(torch.bfloat16)
    v = torch.randn(kv_len, hkv, d).to(torch.bfloat16)
    out = o_attn.ref_attention_one(q, k, v, d**-0.5)
    for i in range(q_len):
        for h in range(hq):
            hk = h // (hq // hkv)
            lim = kv_len - q_len + i
            s = torch.tensor([float(q[i, h].float() @ k[j, hk].float()) * d**-0.5 for j in range(lim + 1)])
            p = torch.softmax(s, 0)
            want = sum(p[j] * v[j, hk].float() for j in range(lim + 1))
            assert torch.allclose(out[i, h], want, atol=1e-5, rtol=1e-5)


def test_attention_flops_formula():
    assert o_attn.attention_flops([1], [10], 2, 8) == 4 * 2 * 8 * (9 + 1)
    assert o_attn.attention_flops([4], [4], 1, 1) == 4 * 10


def test_rope_oracle_properties():
    d = 128
    cache = o_rope.ref_cos_sin_cache(d, 64, 1e6)
    assert cache.shape == (64, d) and cache.dtype == torch.float32
    x = torch.randn(5, 3 * d).to(torch.bfloat16)
    same = o_rope.ref_apply_rope_neox(torch.zeros(5, dtype=torch.int32), x, d, cache)
    assert torch.equal(same, x)  # position 0 is the identity
    y = o_rope.ref_apply_rope_neox(torch.arange(5), x.float(), d, cache)
    assert torch.allclose(y.reshape(5, 3, d).norm(dim=-1), x.float().reshape(5, 3, d).norm(dim=-1), rtol=1e-4)


def test_norm_oracle_properties():
    x = torch.randn(4, 256).to(torch.bfloat16)
    w = torch.ones(256, dtype=torch.bfloat16)
    y = o_norm.ref_rmsnorm(x, w, 0.0).float()
    assert torch.allclose(y.pow(2).mean(-1), torch.ones(4), atol=2e-2)
    nx, nr = o_norm.ref_fused_add_rmsnorm(x, x, w, 1e-6)
    assert torch.equal(nr, (x.float() * 2).to(torch.bfloat16))
    assert torch.allclose(nx.float(), o_norm.ref_rmsnorm((x.float() * 2), w.float(), 1e-6), atol=2e-2)


# ------------------------------------------------------------------ floating-point side
# tests/golden/flashinfer_golden.npz: inputs + outputs of FlashInfer 0.6.11.post2 called exactly as
# the reference's call sites do, produced by tests/golden/make_flashinfer_golden.py.
FI = np.load(Path(__file__).parent / "golden" / "flashinfer_golden.npz")


def _bf16(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(a.view(np.int16).copy()).view(torch.bfloat16)


@pytest.mark.parametrize("phase", ["decode", "prefill"])
def test_attention_oracle_matches_flashinfer(phase):
    reqs = [tuple(r) for r in FI[f"{phase}_reqs"].tolist()]
    pt = FI[f"{phase}_page_table"]
    q = _bf16(FI[f"{phase}_q"])
    used = FI[f"{phase}_used_slots"]
    k_rows, v_rows = _bf16(FI[f"{phase}_k_rows"]), _bf16(FI[f"{phase}_v_rows"])
    remap = {int(s): i for i, s in enumerate(used)}
    want = _bf16(FI[f"{phase}_out"]).float()
    off = 0
    for (t, c, d) in reqs:
        rows = torch.tensor([remap[int(s)] for s in pt[t, :d]])
        ql = d - c
        got = o_attn.ref_attention_one(q[off : off + ql], k_rows[rows], v_rows[rows], 128**-0.5)
        ref = want[off : off + ql]
        scale = ref.abs().max().item()
        # FlashInfer output is bf16 (half an ulp <= 2^-8 |x|) and rounds P to bf16 before PV
        bound = 2e-3 * scale + 2.0**-8 * ref.abs() + 1e-6
        assert ((got - ref).abs() <= bound).all(), ((got - ref).abs() - bound).max()
        off += ql


def test_rope_oracle_matches_flashinfer():
    x, pos = _bf16(FI["rope_x"]), torch.from_numpy(FI["rope_pos"])
    cache = o_rope.ref_cos_sin_cache(128, 1024, 1e6)
    hq, hkv, d = 4, 2, 128
    got = x.clone()
    got[:, : hq * d] = o_rope.ref_apply_rope_neox(pos, x[:, : hq * d], d, cache)
    got[:, hq * d : (hq + hkv) * d] = o_rope.ref_apply_rope_neox(pos, x[:, hq * d : (hq + hkv) * d], d, cache)
    want = _bf16(FI["rope_out"])
    diff = (got.float() - want.float()).abs()
    assert (diff <= 2.0**-7 * want.float().abs() + 1e-6).all()  # <= 1 bf16 ulp (FMA contraction)
    assert (got.view(torch.int16) == want.view(torch.int16)).float().mean() > 0.99


def test_norm_oracle_matches_flashinfer():
    for xk, wk, ok in (("norm_x", "norm_w", "norm_out"), ("qknorm_x", "qknorm_w", "qknorm_out")):
        got = o_norm.ref_rmsnorm(_bf16(FI[xk]), _bf16(FI[wk]), 1e-6)
        want = _bf16(FI[ok])
        assert ((got.float() - want.float()).abs() <= 2.0**-7 * want.float().abs() + 1e-6).all()
    gx, gr = o_norm.ref_fused_add_rmsnorm(_bf16(FI["fused_x"]), _bf16(FI["fused_res"]), _bf16(FI["norm_w"]), 1e-6)
    assert torch.equal(gr.view(torch.int16), _bf16(FI["fused_res_out"]).view(torch.int16))  # residual: exact
    wx = _bf16(FI["fused_x_out"])
    assert ((gx.float() - wx.float()).abs() <= 2.0**-7 * wx.float().abs() + 1e-6).all()


def test_tolerance_criteria_on_an_emulated_16bit_p_kernel():
    """oracle/tolerance.py on a CPU emulation of what every tensor-core backend does (online softmax over
    128-key tiles, P rounded to bf16 before PV, l from the unrounded P, one bf16 output rounding): inside the
    2e-3 budget and inside the element-wise 16-bit-P bound; a result that is wrong by 1 % of one V row is not."""
    from oracle import tolerance

    g = torch.Generator().manual_seed(3)
    hq, hkv, d = 8, 2, 128
    lens = [1, 2, 5, 17, 128, 129, 400, 1000]
    n_slots = sum(lens)
    kc = torch.randn((n_slots, hkv, d), generator=g).to(torch.bfloat16)
    vc = torch.randn((n_slots, hkv, d), generator=g).to(torch.bfloat16)
    q = torch.randn((len(lens), hq, d), generator=g).to(torch.bfloat16)
    rows, off = [], 0
    for n in lens:
        rows.append(torch.arange(off, off + n))
        off += n
    ref = o_attn.ref_paged_attention(q, kc, vc, rows, [1] * len(lens), exact=True)
    assert ref.dtype == torch.float32
    rounded = o_attn.ref_paged_attention(q, kc, vc, rows, [1] * len(lens))
    assert rounded.dtype == torch.bfloat16 and torch.equal(rounded, ref.to(torch.bfloat16))
    absref = o_attn.ref_paged_attention(q, kc, vc.abs(), rows, [1] * len(lens), exact=True)
    def emulate(tile):
        outs = []
        for i, r in enumerate(rows):
            outs.append(emulate_one(i, r, tile))
        return torch.stack(outs)

    def emulate_one(i, r, tile):
        kk = kc[r].float().repeat_interleave(hq // hkv, dim=1)
        vv = vc[r].float().repeat_interleave(hq // hkv, dim=1)
        s = torch.einsum("hd,nhd->hn", q[i].float(), kk) * (d**-0.5) * 1.4426950408889634
        m = torch.full((hq,), -float("inf"))
        l = torch.zeros(hq)
        o = torch.zeros(hq, d)
        for t0 in range(0, len(r), tile):
            st = s[:, t0 : t0 + tile]
            mn = torch.maximum(m, st.max(dim=1).values)
            alpha = torch.where(torch.isinf(m), torch.zeros_like(m), torch.exp2(m - mn))
            p = torch.exp2(st - mn[:, None])
            l = l * alpha + p.sum(1)
            o = o * alpha[:, None] + torch.einsum("hn,nhd->hd", p.to(torch.bfloat16).float(), vv[t0 : t0 + tile])
            m = mn
        return (o / l[:, None]).to(torch.bfloat16)

    out = emulate(128)
    assert tolerance.vs_exact_oracle(out, ref) <= tolerance.ORACLE_REL_TOL
    assert tolerance.p16_bound_excess(out, ref, absref) <= tolerance.P16_EXCESS_TOL
    assert tolerance.vs_exact_oracle(rounded, ref) == 0.0  # the exact result, rounded once: nothing beyond half an ulp
    # a second kernel with another tile size (different running maxima, different P roundings): the pair bound
    other = emulate(64)
    assert tolerance.pair_p16_bound_excess(out, other, absref) <= tolerance.P16_EXCESS_TOL
    bad = out.clone()
    bad[4] = (out[4].float() + 0.01 * vc[rows[4][0], 0].float()).to(torch.bfloat16)
    assert tolerance.p16_bound_excess(bad, ref, absref) > tolerance.P16_EXCESS_TOL
    assert tolerance.vs_exact_oracle(bad, ref) > tolerance.ORACLE_REL_TOL
    assert tolerance.pair_p16_bound_excess(bad, other, absref) > tolerance.P16_EXCESS_TOL
