"""CPU self-test of the long-context attention harness (tests/test_gpu_attention_long.py): the sampled-row fp64
oracle is the full causal oracle restricted to those rows, the needle positions drawn from a plan cover every
chunk boundary and the first and last tile, and the emulated flash kernel (tests/test_attention_probes_cpu.py)
stays within the fp64 reference's bound over 40 960 keys in the regimes the GPU tests run."""
import random

import pytest
import torch

from oracle import probes as P
from oracle.attention import ref_attention_one
from test_attention_probes_cpu import emulate

D = 128
LONG_LENS = [8193, 16256, 16257, 16384 + 129, 32768, 40960]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("cached,q_len", [(0, 300), (37, 700), (1000, 1)])
def test_sampled_rows_equal_the_full_oracle(cached, q_len, dtype):
    n = cached + q_len
    gen = torch.Generator().manual_seed(cached + q_len)
    q, k, v = P.regime_request("temp1", gen, n, q_len, 1, 1, dtype)
    q, k, v = q[:, 0], k[:, 0], v[:, 0]
    rows = P.sampled_rows(q_len, random.Random(0), n_random=16)
    assert rows == sorted(set(rows)) and all(0 <= r < q_len for r in rows)
    want = {0, 1, 127, 128, 129, q_len - 1} | set(range(max(0, q_len - 130), q_len))
    assert want & set(range(q_len)) <= set(rows)
    idx = torch.tensor(rows)
    full_out, full_p, full_bound = P.ref_with_bound(q, k, v, dtype, torch.arange(cached + 1, n + 1))
    out, p, bound = P.ref_with_bound(q[idx], k, v, dtype, cached + idx + 1)
    torch.testing.assert_close(out, full_out[idx], rtol=1e-12, atol=0)
    torch.testing.assert_close(p, full_p[idx], rtol=1e-12, atol=0)
    torch.testing.assert_close(bound, full_bound[idx], rtol=1e-12, atol=0)
    # and the full oracle is the causal attention of the fp32 SDPA oracle (bottom-right aligned)
    sdpa = ref_attention_one(q[:, None], k[:, None], v[:, None], D**-0.5)[:, 0]
    torch.testing.assert_close(full_out.float(), sdpa, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("hq", [8, 16, 128])
@pytest.mark.parametrize("chunk", [128, 2560, 5120, 40960])
def test_plan_needles_cover_every_chunk_boundary(hq, chunk):
    """For the chunk size a plan picks, the decode needles sit on both sides of every chunk boundary (a multiple
    of the 128-key tile), on the first tile's edges, on both sides of the last tile's start, on the last cached
    key and on the appended key -- with 8 query heads by spreading a length over two requests."""
    copies = -(-(8 + 2 * 15 + 8) // (hq * 4))
    lens = [n for n in LONG_LENS for _ in range(copies)]
    if max(-(-n // chunk) for n in lens) > 16:
        pytest.skip("the plan never cuts a request into more than 16 chunks")
    reqs = P.assign_plan_needles(lens, chunk, hq, seed=1)
    assert [n for n, _ in reqs] == lens
    for n in LONG_LENS:
        got = [p for n_, pos in reqs if n_ == n for head in pos for p in head]
        for n_, pos in reqs:
            assert len(pos) == hq and all(len(set(h)) == len(h) == 4 for h in pos)
        assert len(got) == len(set(got)) == copies * hq * 4  # distinct across heads and requests
        last_tile = (n - 2) // 128 * 128
        want = {0, 127, 128, last_tile - 1, last_tile, n - 2, n - 1}
        want |= {x for c in range(chunk, n, chunk) for x in (c - 1, c)}
        assert all(c % 128 == 0 for c in range(chunk, n, chunk))
        assert want <= set(got), f"n={n} chunk={chunk}: missing {sorted(want - set(got))}"


def test_plan_needles_short_requests():
    """Requests shorter than their needle slots (the short ones of a mixed batch) get one position per head,
    still with the last cached and the appended key among them."""
    lens = [2, 3, 17, 40960, 100]
    for n, pos in P.assign_plan_needles(lens, 40960, 16, seed=2):
        flat = [p for h in pos for p in h]
        assert all(0 <= p < n for p in flat)
        assert {n - 2, n - 1} - {-1} <= set(flat)
        assert all(len(h) == (4 if n >= 64 else 1) for h in pos)


@pytest.mark.parametrize("mode", ["unsplit", "split"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("name", ["temp0", "temp16", "drift_up", "drift_down", "chunk_maxima"])
def test_emulated_kernel_within_bound_at_40960_keys(name, dtype, mode):
    """fp32 sums of l and P.V over 40 960 keys (320 tiles, or 16 chunks of 2560) stay inside the bound: its 2%
    slack on the P rounding term covers the fp32 accumulation, which grows with the number of tiles."""
    n, chunk = 40960, 2560
    gen = torch.Generator().manual_seed(3)
    q, k, v = P.regime_request(name, gen, n, 1, 1, 1, dtype, block=chunk if mode == "split" else 128)
    got = emulate(q[:, 0], k[:, 0], v[:, 0], dtype, chunk=chunk if mode == "split" else None, append_last=True)
    out, _, bound = P.ref_with_bound(q[:, 0], k[:, 0], v[:, 0], dtype)
    assert P.bound_excess(got, out, bound) <= P.P16_EXCESS_TOL
