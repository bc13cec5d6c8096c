"""Exact-answer probes of the attention kernels and an fp64 softmax reference with an element-wise error
bound (TEST INFRASTRUCTURE ONLY: imported by tests/).

Needle.  Query head (h, g) (kv head h, slot g < 16 of its GQA group) has q[needle_dim(g)] = 32 and zeros in
every other dim (needle_dim: dims 0-7 for slots 0-7, dims 10-17 for slots 8-15); its chosen key p has
K[p, h, needle_dim(g)] = 64 and every other key has zeros in dims 0-17.  The needle scores
2048 * D^-0.5 * log2(e) ~ 261 log2 units, every other key exactly 0, so every other P underflows to 0 and
the output is V[p] bit for bit (or the exact mean of 2 or 4 tied needles).

Ramp.  Dims 8-9 of the keys hold the position j (bf16: j >> 8 and j & 255; fp16: j in dim 8 alone) and q
weighs them so that the score is 2^11 * j exactly: adjacent keys are 261 log2 units apart.  A rising ramp
makes every query row pick the last key it may see (its own position), a falling one key 0.

Bound.  For scores s_i (log2 units), p_i = 2^(s_i - max s), L = sum p_i and ref = sum p_i v_i / L, a kernel
that rounds P to 16 bits (unit roundoff u; fp16 subnormal half-spacing h), accumulates the scores in fp32 and
rounds the output to 16 bits is within
    1.02 sum_i max(u p_i, h) |v_i| / L  +  sum_i p_i eps_i |v_i| / L  +  eps_max |ref|  +  ulp(ref) / 2
with eps_i = ln2 * scale_log2 * 128 * 2^-24 * sum_d |q_d k_id| the fp32 score-accumulation error carried
into p_i.  The reported number is the excess over that bound relative to max|ref|; the pass mark is
oracle.tolerance.P16_EXCESS_TOL.
"""
from __future__ import annotations

import math
import random
from typing import List, Optional, Sequence, Tuple

import torch

from .tolerance import P16_EXCESS_TOL  # noqa: F401  (the pass mark of bound_excess)

LOG2E = 1.4426950408889634
NEEDLE_Q = 32.0
NEEDLE_K = 64.0
V_MAX = 32            # V entries of the needle probes are integers in [-V_MAX, V_MAX]
PROBE_DIMS = 18       # dims 0-7 and 10-17: needles (one per GQA slot), 8-9: ramp
MIN_GAP = 160.0       # log2 units every probe maximum must beat the runner-up by
RAMP_FP16_MAX = 2048  # fp16 ramp: positions must stay exact integers


def scale_log2(d: int = 128) -> float:
    """The kernels' fp32 score scale: fp32(fp32(D^-0.5) * fp32(log2 e))."""
    return (torch.tensor(d**-0.5, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)).item()


def p_unit_roundoff(dtype: torch.dtype) -> float:
    return 2.0**-9 if dtype == torch.bfloat16 else 2.0**-12


def p_subnormal_half_spacing(dtype: torch.dtype) -> float:
    return 0.0 if dtype == torch.bfloat16 else 2.0**-25


def out_ulp(dtype: torch.dtype) -> float:
    return 2.0**-7 if dtype == torch.bfloat16 else 2.0**-10


# ------------------------------------------------------------------------------------------- probe values
def needle_dim(g: int) -> int:
    """The dim that carries the needle of GQA slot g (0..15); dims 8-9 belong to the ramp."""
    assert 0 <= g < 16, "needle probes cover GQA groups of up to 16 query heads"
    return g if g < 8 else g + 2


def needle_query(g: int, d: int = 128) -> torch.Tensor:
    q = torch.zeros(d)
    q[needle_dim(g)] = NEEDLE_Q
    return q


def ramp_query(dtype: torch.dtype, rising: bool = True, d: int = 128) -> torch.Tensor:
    q = torch.zeros(d)
    sign = 1.0 if rising else -1.0
    if dtype == torch.bfloat16:
        q[8], q[9] = sign * 2.0**19, sign * 2.0**11
    else:
        q[8] = sign * 2.0**11
    return q


def ramp_key_dims(positions: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Values of dims 8-9 of the keys at `positions` (int64 [n]) -> float [n, 2]; exact in `dtype`."""
    j = positions.to(torch.int64)
    if dtype == torch.bfloat16:
        return torch.stack([(j >> 8).float(), (j & 255).float()], -1)
    assert int(j.max()) < RAMP_FP16_MAX, "fp16 ramp positions must stay below 2048"
    return torch.stack([j.float(), torch.zeros_like(j, dtype=torch.float32)], -1)


def probe_keys(gen: torch.Generator, n: int, hkv: int, dtype: torch.dtype, d: int = 128,
               ramp: bool = True) -> torch.Tensor:
    """Keys [n, hkv, d]: random in dims >= 18 (queries are zero there), the needle dims zero, dims 8-9 the ramp."""
    k = torch.randn((n, hkv, d), generator=gen)
    k[..., :PROBE_DIMS] = 0
    if ramp and n:
        k[..., 8:10] = ramp_key_dims(torch.arange(n), dtype)[:, None, :]
    return k.to(dtype)


def plant_needle(k: torch.Tensor, pos: int, h: int, g: int) -> None:
    k[pos, h, needle_dim(g)] = NEEDLE_K


def integer_values(gen: torch.Generator, n: int, hkv: int, dtype: torch.dtype, d: int = 128) -> torch.Tensor:
    """V [n, hkv, d] of integers in [-32, 32]; every row (over positions and kv heads) distinct."""
    v = torch.randint(-V_MAX, V_MAX + 1, (n, hkv, d), generator=gen).to(dtype)
    rows = v.reshape(-1, d).view(torch.int16)
    assert torch.unique(rows, dim=0).shape[0] == rows.shape[0], "probe V rows must be distinct"
    return v


def scores_fp32(q: torch.Tensor, k: torch.Tensor, sl2: Optional[float] = None) -> torch.Tensor:
    """Scores in log2 units as the kernels form them: 16-bit operands, fp32 products and sums, fp32 scale.
    q [d], k [n, d] -> [n].  Exact for the probes (at most two non-zero products per key)."""
    sl2 = scale_log2(q.shape[-1]) if sl2 is None else sl2
    s = (k.float() * q.float()).sum(-1)
    return s * torch.tensor(sl2, dtype=torch.float32)


def diagnose(row: torch.Tensor, v_rows: torch.Tensor) -> str:
    """Which key a returned output row is: v_rows [n, hkv, d] of the request."""
    bits = row.reshape(-1).view(torch.int16)
    hit = (v_rows.view(torch.int16) == bits).all(-1).nonzero().tolist()
    if hit:
        return "attended to " + ", ".join(f"position {p} of kv head {h}" for p, h in hit)
    r = row.float().reshape(-1)
    if torch.isnan(r).any():
        return "NaN in the output"
    if (r == 0).all():
        return "a zero row"
    return f"a mixture (not any V row; max |out| {r.abs().max().item():.3g})"


# ------------------------------------------------------------------------------------------- fp64 reference
def ref_with_bound(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, dtype: torch.dtype,
                   n_visible: Optional[torch.Tensor] = None):
    """Query rows q [m, d] (or [d]) against keys k [n, d] and values v [n, d], all the stored 16-bit values;
    row i sees keys [0, n_visible[i]) (all keys when None).  Returns (out [m, d], p [m, n], bound [m, d]) in
    float64, p relative to each row's maximum (0 for keys a row does not see)."""
    q64 = q.double().reshape(-1, q.shape[-1])
    k64, v64 = k.double(), v.double()
    sl2 = scale_log2(q.shape[-1])
    s = (q64 @ k64.T) * sl2
    vis = torch.ones_like(s, dtype=torch.bool)
    if n_visible is not None:
        vis = torch.arange(k.shape[0])[None, :] < n_visible.reshape(-1, 1)
    s = s.masked_fill(~vis, -math.inf)
    p = torch.exp2(s - s.max(-1, keepdim=True).values)
    L = p.sum(-1, keepdim=True)
    out = (p @ v64) / L
    u, h = p_unit_roundoff(dtype), p_subnormal_half_spacing(dtype)
    eps = (math.log(2.0) * sl2 * 128 * 2.0**-24) * (q64.abs() @ k64.abs().T) * vis
    av = v64.abs()
    p_err = torch.clamp(u * p, min=h) * vis
    bound = (1.02 * (p_err @ av) + ((p * eps) @ av)) / L + eps.max(-1, keepdim=True).values * out.abs()
    bound = bound + 0.5 * out_ulp(dtype) * out.abs() + (2.0**-25 if dtype == torch.float16 else 0.0)
    return out, p, bound


def bound_excess(got: torch.Tensor, out: torch.Tensor, bound: torch.Tensor) -> float:
    """max(|got - out| - bound)^+ / max|out| over any matching shapes (pass: <= P16_EXCESS_TOL)."""
    g = got.double().cpu()
    if torch.isnan(g).any() or torch.isinf(g).any():
        return float("inf")
    return ((g - out).abs() - bound).clamp_min(0).max().item() / max(out.abs().max().item(), 1e-300)


def boundary_positions(n: int, page_size: int, tile: int = 128) -> List[int]:
    """Decode needle positions of a request of kv_len n (keys 0..n-2 cached, n-1 appended this step): the
    first key, the last cached key and the appended one, both sides of every tile boundary (keys 127 / 128,
    the last key of every tile; chunk sizes are multiples of the tile, so this includes the last key of every
    non-last chunk and the first key of the next), and both sides of the first two page boundaries, of the
    last two and of the first page boundary at or after every tile boundary."""
    want = {0, n - 2, n - 1}
    for t in range(tile, n, tile):
        want |= {t - 1, t}
    pages = list(range(page_size, n, page_size))
    near = set(pages[:2]) | set(pages[-2:]) | {b for b in pages if b % tile < page_size}
    for b in near:
        want |= {b - 1, b}
    return sorted(x for x in want if 0 <= x < n)


def assign_needles(kv_lens: Sequence[int], page_size: int, hq: int, seed: int = 0) -> List[Tuple[int, List[int]]]:
    """Decode requests that between them put a needle on every boundary position of every length: each
    length is repeated until its positions are used up, a request's query heads get distinct positions where
    the length allows (so a wrong head mapping picks a different V row).  Returns [(kv_len, [pos per query
    head])]."""
    rnd = random.Random(seed)
    reqs = []
    for n in kv_lens:
        cand = boundary_positions(n, page_size)
        rnd.shuffle(cand)
        for i in range(0, len(cand), hq):
            pos = cand[i : i + hq]
            free = [x for x in range(n) if x not in pos]
            rnd.shuffle(free)
            while len(pos) < hq:
                pos.append(free.pop() if free else rnd.randrange(n))
            reqs.append((n, pos))
    return reqs


# ------------------------------------------------------------------------------------------- long contexts
def plan_positions(n: int, chunk: int, tile: int = 128) -> List[int]:
    """Decode needle positions of a request of kv_len n under a plan of `chunk`-key chunks (keys 0..n-2 cached
    and streamed in 128-key tiles, n-1 appended by the launch): both sides of every chunk boundary, the first
    and the last tile of the streamed range, the last cached key and the appended one.  A few dozen positions
    at any length (at most 16 chunks), where boundary_positions names every tile boundary."""
    last_tile = (n - 2) // tile * tile if n >= 2 else 0
    want = {0, 1, tile - 1, tile, last_tile - 1, last_tile, n - 2, n - 1}
    for c in range(chunk, n, chunk):
        want |= {c - 1, c}
    return sorted(x for x in want if 0 <= x < n)


def spread_positions(n: int, required: Sequence[int], slots: int, n_random: int, rnd: random.Random) -> List[int]:
    """`slots` distinct positions below n: every required one, n_random random others, and random positions
    for the rest; shuffled (so a position lands on an arbitrary query head and tie group)."""
    pos = list(dict.fromkeys(required))
    assert len(pos) + n_random <= slots <= n, (len(pos), n_random, slots, n)
    taken = set(pos)
    while len(pos) < slots:
        x = rnd.randrange(n)
        if x not in taken:
            taken.add(x)
            pos.append(x)
    rnd.shuffle(pos)
    return pos


def assign_plan_needles(lens: Sequence[int], chunk: int, hq: int, seed: int = 0, ties: int = 4,
                        n_random: int = 8) -> List[Tuple[int, List[List[int]]]]:
    """Needles of decode requests of kv_len `lens` under a plan of `chunk`-key chunks: [(kv_len, [tied positions
    per query head])] in the order of lens.  The requests of one length share out plan_positions(n, chunk),
    n_random random positions and random fill, `ties` distinct positions per query head (one where the length
    is shorter than the requests' slots; positions then repeat across heads)."""
    rnd = random.Random(seed)
    groups = {}
    for n in sorted(set(lens)):
        copies = lens.count(n)
        t = ties if n >= copies * hq * ties else 1
        slots = copies * hq * t
        required = plan_positions(n, chunk)
        assert len(required) <= slots, f"kv_len {n}: {len(required)} plan positions for {slots} needles"
        if slots <= n:
            pos = spread_positions(n, required, slots, min(n_random, slots - len(required)), rnd)
        else:
            pos = required + [rnd.randrange(n) for _ in range(slots - len(required))]
            rnd.shuffle(pos)
        groups[n] = [[pos[(c * hq + h) * t : (c * hq + h + 1) * t] for h in range(hq)] for c in range(copies)]
    return [(n, groups[n].pop(0)) for n in lens]


def sampled_rows(q_len: int, rnd: random.Random, n_random: int = 64, tile: int = 128) -> List[int]:
    """Query rows of a long extend to check against the fp64 reference: rows 0, 1, 127, 128 and 129, both sides
    of every 128-row query tile edge in the first and the last query tile, the last 130 rows and n_random
    random rows."""
    last = (q_len - 1) // tile * tile
    want = {0, 1, tile - 1, tile, tile + 1, last - 1, last, last + 1, q_len - 1}
    want |= set(range(max(0, q_len - 130), q_len))
    want |= {rnd.randrange(q_len) for _ in range(n_random)}
    return sorted(x for x in want if 0 <= x < q_len)


# ------------------------------------------------------------------------------------------- adversarial regimes
REGIMES = ["temp0", "temp0.25", "temp1", "temp4", "temp16", "drift_up", "drift_down", "chunk_maxima", "magnitude"]
CHUNK_OFFSETS = [0.0, 40.0, -40.0, -135.0, 40.0, -20.0, 10.0, -60.0]  # log2 units per block of keys


def regime_request(name: str, gen: torch.Generator, n: int, n_q: int, hq: int, hkv: int, dtype: torch.dtype,
                   d: int = 128, block: int = 128):
    """One request's q [n_q, hq, d], k [n, hkv, d], v [n, hkv, d] (16-bit) for an adversarial softmax regime:
    temperature T (score std T natural units, T = 0 a uniform softmax), a score drift of 8 log2 units per 128
    keys rising or falling, per-block (of `block` keys: the split-KV chunk) score offsets of up to +-40 log2
    units with one block 175 below
    the maximum (its merge weight underflows) and two blocks tied at it, large V (bf16 200 + N(0, 1), fp16
    +-2e4)."""
    temp = float(name[4:]) if name.startswith("temp") else 1.0
    dev = gen.device  # the tensors are made where the generator lives (a CUDA generator: long contexts)
    q = torch.randn((n_q, hq, d), generator=gen, device=dev) * temp
    k = torch.randn((n, hkv, d), generator=gen, device=dev)
    v = torch.randn((n, hkv, d), generator=gen, device=dev)
    j = torch.arange(n, dtype=torch.float64, device=dev)
    off = None  # per-key score offset in log2 units, carried by dim 0 (q[0] = 16)
    if name == "drift_up":
        off = j * (8.0 / 128)
    elif name == "drift_down":
        off = (n - 1 - j) * (8.0 / 128)
    elif name == "chunk_maxima":
        off = torch.tensor(CHUNK_OFFSETS, dtype=torch.float64, device=dev)[(j.long() // block) % len(CHUNK_OFFSETS)]
    if off is not None:
        q[..., 0] = 16.0
        k[..., 0] = (off * math.log(2.0) * math.sqrt(d) / 16.0).float()[:, None]
    if name == "magnitude":
        v = 200.0 + v if dtype == torch.bfloat16 else 2e4 * (2 * torch.rand((n, hkv, d), generator=gen, device=dev) - 1)
    return q.to(dtype), k.to(dtype), v.to(dtype)
