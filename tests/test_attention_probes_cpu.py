"""CPU self-test of the attention probes (tests/test_gpu_attention_probes.py): the probe arithmetic is exact
in fp32, the probe positions cover the boundaries they are meant to, an emulation of the kernels' flash
algorithm (128-key tiles, fp32 online softmax, P rounded to the 16-bit type including fp16 subnormals, split-KV
merge, the decode token appended on CUDA cores) stays within the fp64 reference's bound in every adversarial
regime, and mutants of that emulation fail the exact probes."""
import math

import pytest
import torch

from oracle import probes as P

D = 128
DTYPES = [torch.bfloat16, torch.float16]
SL2 = torch.tensor(P.scale_log2(D), dtype=torch.float32)


# ------------------------------------------------------------------------------------------- emulation
def emulate(q, k, v, dtype, *, chunk=None, n_visible=None, append_last=False, mutant=None, mutant_key=None, tile=128):
    """Flash attention as the kernels compute it.  q [m, d] query rows; k, v [n, d]; row i sees keys
    [0, n_visible[i]) (all when None).  Decode (append_last): the last key is the token appended by the launch,
    scored on CUDA cores with an unrounded P in the last chunk.  chunk: split-KV chunk size (None: one chunk).
    mutant: None | "drop" | "dup" (key mutant_key) | "l_not_rescaled" | "merge_weight" | "causal_off_by_one" |
    "alpha_half0" (row 8 + r of a 16-row block rescaled with the alpha of row r).  Returns fp32 [m, d]
    rounded to `dtype`."""
    n, m = k.shape[0], q.shape[0]
    s_all = (q.float() @ k.float().T) * SL2
    vf = v.float()
    vis = torch.full((m,), n) if n_visible is None else n_visible
    lim = vis + 1 if mutant == "causal_off_by_one" else vis
    chunk = chunk or n
    parts = []
    for c0 in range(0, n, chunk):
        c1 = min(n, c0 + chunk)
        last = c1 == n
        tc_end = c1 - 1 if (append_last and last) else c1
        m_run = torch.full((m,), -math.inf)
        l_run = torch.zeros(m)
        acc = torch.zeros(m, k.shape[1])
        for t0 in range(c0, tc_end, tile):
            keys = list(range(t0, min(t0 + tile, tc_end)))
            if mutant == "drop" and mutant_key in keys:
                keys.remove(mutant_key)
            if mutant == "dup" and mutant_key in keys:
                keys.append(mutant_key)
            idx = torch.tensor(keys)
            s = s_all[:, idx].masked_fill(idx[None, :] >= lim[:, None], -math.inf)
            m_new = torch.maximum(m_run, s.max(1).values)
            m_use = torch.where(m_new == -math.inf, torch.zeros_like(m_new), m_new)
            alpha = torch.exp2(m_run - m_use)
            p = torch.exp2(s - m_use[:, None])
            p16 = p.to(dtype).float()  # fp16 subnormals kept, as the kernels' conversions do
            a_o = alpha.clone()
            if mutant == "alpha_half0":
                rows = torch.arange(m)
                hi = (rows >> 3) & 1 == 1
                a_o[hi] = alpha[rows[hi] - 8]
            acc = acc * a_o[:, None] + p16 @ vf[idx]
            l_run = (l_run if mutant == "l_not_rescaled" else l_run * alpha) + p.sum(1)
            m_run = m_new
        if append_last and last:
            s_new = s_all[:, n - 1]
            m_new = torch.maximum(m_run, s_new)
            a = torch.exp2(m_run - m_new)
            pn = torch.exp2(s_new - m_new)
            acc = acc * a[:, None] + pn[:, None] * vf[n - 1][None, :]
            l_run = l_run * a + pn
            m_run = m_new
        parts.append((m_run, l_run, acc))
    if len(parts) == 1:
        m_, l_, acc = parts[0]
        return (acc / l_[:, None]).to(dtype).float()
    mx = torch.stack([p_[0] for p_ in parts]).max(0).values
    o = torch.zeros_like(parts[0][2])
    l_tot = torch.zeros_like(parts[0][1])
    for m_c, l_c, a_c in parts:
        w = torch.ones_like(m_c) if mutant == "merge_weight" else torch.exp2(m_c - mx)
        o = o + w[:, None] * a_c
        l_tot = l_tot + w * l_c
    return (o / l_tot[:, None]).to(dtype).float()


# ------------------------------------------------------------------------------------------- probe builders
def decode_needles(n, positions, dtype, seed=0, g=3):
    """One query head (slot g) over n keys with (tied) needles at `positions` -> q [1, d], k, v [n, d],
    expected [d] (the exact mean of the needles' V rows)."""
    gen = torch.Generator().manual_seed(seed)
    k = P.probe_keys(gen, n, 1, dtype)
    for p in positions:
        P.plant_needle(k, p, 0, g)
    v = P.integer_values(gen, n, 1, dtype)
    want = v[positions, 0].double().mean(0)
    return P.needle_query(g).to(dtype)[None], k[:, 0], v[:, 0], want


def prefill_ramp(cached, q_len, dtype, seed=0):
    """Query rows of an extend [cached, cached + q_len): rows with (i >> 3) & 1 == 0 ramp up (expect their own
    position), the others ramp down (expect key 0)."""
    n = cached + q_len
    gen = torch.Generator().manual_seed(seed)
    k = P.probe_keys(gen, n, 1, dtype)[:, 0]
    v = P.integer_values(gen, n, 1, dtype)[:, 0]
    rising = [(i >> 3) & 1 == 0 for i in range(q_len)]
    q = torch.stack([P.ramp_query(dtype, r) for r in rising]).to(dtype)
    vis = torch.arange(cached + 1, n + 1)
    want = torch.stack([v[cached + i] if r else v[0] for i, r in enumerate(rising)]).double()
    return q, k, v, vis, want


def exact(got, want):
    return torch.equal(got.double(), want.double())


# ------------------------------------------------------------------------------------------- probe arithmetic
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_needle_arithmetic_is_exact(dtype):
    n = 2048
    for g in range(16):  # every slot of a GQA group of up to 16 query heads
        q, k, v, _ = decode_needles(n, [777], dtype, g=g)
        s = P.scores_fp32(q[0], k)
        assert s[777].item() == float(torch.tensor(2048.0) * SL2)  # q, k exact in dtype; one product
        others = torch.cat([s[:777], s[778:]])
        assert (others == 0).all()
        assert s[777].item() - others.max().item() >= P.MIN_GAP
        assert (torch.exp2(others - s[777]) == 0).all()  # every other P is exactly 0
        assert torch.exp2(s[777] - s[777]).item() == 1.0
    # tied needles: their mean is exactly representable
    for ties in ([5, 900], [0, 127, 128, 2046]):
        _, _, v, want = decode_needles(n, ties, dtype)
        assert exact(want.to(dtype), want)


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_ramp_arithmetic_is_exact(dtype):
    n = 8192 if dtype == torch.bfloat16 else P.RAMP_FP16_MAX
    j = torch.arange(n)
    kd = P.ramp_key_dims(j, dtype)
    assert exact(kd.to(dtype), kd)
    for rising in (True, False):
        q = P.ramp_query(dtype, rising)
        assert exact(q.to(dtype), q)
        raw = kd[:, 0].double() * q[8].double() + kd[:, 1].double() * q[9].double()
        assert torch.equal(raw, (2.0**11 if rising else -(2.0**11)) * j.double())  # the score is 2^11 j
        assert raw.abs().max() < 2**24  # exact in fp32
        s = raw.float() * SL2
        gaps = (s[1:] - s[:-1]).abs()
        assert gaps.min().item() >= P.MIN_GAP


@pytest.mark.parametrize("page_size", [1, 8, 16, 64, 256])
def test_needle_positions_cover_every_boundary(page_size):
    """Whatever chunk size the plan picks (a multiple of 128 keys), the decode probe requests have a needle on
    both sides of every tile, chunk and page-boundary kind, on the first, last cached and appended key."""
    lens = [2, 3, 129, 257, 385, 513, 1025, 1500, 2048]
    reqs = P.assign_needles(lens, page_size, hq=16)
    for n in lens:
        got = set()
        for n_, pos in reqs:
            assert len(pos) == 16 and all(0 <= x < n_ for x in pos)
            if n_ == n:
                assert len(set(pos)) == min(16, n_)  # distinct heads where the length allows
                got |= set(pos)
        want = {0, n - 2, n - 1} | {x for t in range(128, n, 128) for x in (t - 1, t)}
        for chunk in (128, 256, 512, 1024):
            want |= {x for c in range(chunk, n, chunk) for x in (c - 1, c)}
        for b in list(range(page_size, n, page_size))[:2]:
            want |= {b - 1, b}
        assert want <= got | {-1}, f"n={n}: missing {sorted(want - got)}"


# ------------------------------------------------------------------------------------------- emulation vs bound
def _emulated_regime(name, dtype, mode):
    """Excess over the bound of the emulation on one regime; mode: unsplit | split | prefill."""
    gen = torch.Generator().manual_seed(7)
    if mode == "prefill":
        cached, q_len = 256, 300
        n = cached + q_len
        q, k, v = P.regime_request(name, gen, n, q_len, 1, 1, dtype)
        vis = torch.arange(cached + 1, n + 1)
        got = emulate(q[:, 0], k[:, 0], v[:, 0], dtype, n_visible=vis)
        out, p, bound = P.ref_with_bound(q[:, 0], k[:, 0], v[:, 0], dtype, vis)
    else:
        n = 1100
        q, k, v = P.regime_request(name, gen, n, 1, 1, 1, dtype)
        got = emulate(q[:, 0], k[:, 0], v[:, 0], dtype, chunk=128 if mode == "split" else None, append_last=True)
        out, p, bound = P.ref_with_bound(q[:, 0], k[:, 0], v[:, 0], dtype)
    return P.bound_excess(got, out, bound), p


@pytest.mark.parametrize("mode", ["unsplit", "split", "prefill"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("name", P.REGIMES)
def test_emulated_kernel_within_bound(name, dtype, mode):
    excess, p = _emulated_regime(name, dtype, mode)
    assert excess <= P.P16_EXCESS_TOL, f"{name} {mode}: excess {excess:.3e}"
    if name == "temp0":  # a uniform softmax: P = 1 on every visible key
        assert ((p == 1) | (p == 0)).all() and (p[-1] == 1).all()
    if name == "temp16" and dtype == torch.float16:  # the peaked fp16 regime: many P in fp16 subnormals
        assert ((p > 0) & (p < 2.0**-14)).sum() > 100


# ------------------------------------------------------------------------------------------- mutants fail the probes
def _decode_probe_fails(dtype, n, positions, chunk, **mut):
    q, k, v, want = decode_needles(n, positions, dtype)
    ok = exact(emulate(q, k, v, dtype, chunk=chunk, append_last=True)[0], want)
    assert ok, "the faithful emulation must pass the probe"
    return not exact(emulate(q, k, v, dtype, chunk=chunk, append_last=True, **mut)[0], want)


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_emulation_mutants_fail_the_probes(dtype):
    n = 1025  # 1024 cached keys (8 tiles, 8 chunks of 128) and the appended token (a chunk of its own)
    # a dropped key: a needle there is lost
    for key in (0, 127, 128, 511, 512, 1023):
        assert _decode_probe_fails(dtype, n, [key], 128, mutant="drop", mutant_key=key)
    # a duplicated key: with two tied needles the mean moves
    for key in (127, 128, 1023):
        assert _decode_probe_fails(dtype, n, [key, 700 if key != 700 else 5], 128, mutant="dup", mutant_key=key)
    # l not rescaled: a needle past the first tile
    assert _decode_probe_fails(dtype, n, [300], None, mutant="l_not_rescaled")
    # merge weight ignored: a needle in any chunk but the one with the largest sum
    assert _decode_probe_fails(dtype, n, [600], 128, mutant="merge_weight")
    assert _decode_probe_fails(dtype, n, [1024], 128, mutant="merge_weight")  # the appended token alone
    # prefill: causal mask one past the diagonal, alpha of row half 0 applied to row half 1
    for mut in ("causal_off_by_one", "alpha_half0"):
        q, k, v, vis, want = prefill_ramp(100, 300, dtype)
        assert exact(emulate(q, k, v, dtype, n_visible=vis), want)
        got = emulate(q, k, v, dtype, n_visible=vis, mutant=mut)
        assert not exact(got, want), mut
