"""Shared builders for the parity tests: a paged world (page table + pool + requests) on CPU,
mirrored onto the GPU for the product path."""
from __future__ import annotations

import contextlib
import importlib
import math
import random
from dataclasses import dataclass
from types import SimpleNamespace
from typing import List, Optional, Sequence, Tuple

import numpy as np
import pytest
import torch

from oracle import attention as o_attn
from oracle import metadata as o_meta


@contextlib.contextmanager
def options(b200, **opts):
    """Sets b200_set_option knobs for the duration of the block, then restores their previous values.  Skips the
    test when a knob is refused: the bring-up kernels (decode_impl / prefill_impl = 0) are only in
    B200_BUILD_BRINGUP=1 builds."""
    prev = []
    try:
        for name, val in opts.items():
            try:
                prev.append((name, b200._cabi.set_option(name, val)))
            except b200._cabi.B200NativeError:
                pytest.skip(f"option {name}={val}: cross-check kernel not in this build (B200_BUILD_BRINGUP=1)")
        yield
    finally:
        for name, val in reversed(prev):
            b200._cabi.set_option(name, val)


# options(b200, **SPLIT_PLAN): every decode request split into 128-key chunks, as many as the plan allows
SPLIT_PLAN = {"decode_plan_nosplit": 0, "decode_plan_target": 16}


def table_align(page_size: int) -> int:
    """Page-table width granule: a multiple of 64 columns and of the page size (the allocator writes whole pages;
    24, 48 and 96 do not divide 64)."""
    return math.lcm(64, page_size)


@dataclass
class World:
    page_size: int
    num_pages: int
    hq: int
    hkv: int
    d: int
    layers: int
    dtype: torch.dtype
    page_table: np.ndarray  # int32 [max_req + 1, max_seq_aligned]
    free_pages: List[int]
    pool_cpu: torch.Tensor  # [2, L, slots, hkv, d]
    reqs: List[Tuple[int, int, int]]  # (table_idx, cached_len, device_len)

    @property
    def slots(self) -> int:
        return self.num_pages * self.page_size


def make_world(
    *,
    seed: int,
    page_size: int,
    hq: int,
    hkv: int,
    d: int = 128,
    layers: int = 1,
    max_reqs: int = 8,
    max_seq: int = 512,
    num_pages: Optional[int] = None,
    dtype: torch.dtype = torch.bfloat16,
    shuffle_pages: bool = True,
) -> World:
    g = torch.Generator().manual_seed(seed)
    al = table_align(page_size)
    max_seq_al = (max_seq + al - 1) // al * al  # whole pages are written by the allocator
    if num_pages is None:
        num_pages = (max_reqs * max_seq_al) // page_size + 8
    slots = (num_pages + 1) * page_size  # +1 dummy page, like the engine
    pool = torch.randn((2, layers, slots, hkv, d), generator=g, dtype=torch.float32).to(dtype)
    table = np.zeros((max_reqs + 1, max_seq_al), dtype=np.int32)
    table[max_reqs, :] = num_pages * page_size  # dummy request row -> dummy page
    free = [p * page_size for p in range(num_pages)]
    if shuffle_pages:
        random.Random(seed).shuffle(free)
    return World(page_size, num_pages, hq, hkv, d, layers, dtype, table, free, pool, [])


def add_requests(w: World, lens: Sequence[Tuple[int, int]], share_prefix_from: Optional[int] = None):
    """lens: (cached_len, device_len) per request; allocates pages for [0, device_len) like the
    scheduler (cached part first, as if an earlier forward had filled it)."""
    for i, (c, dl) in enumerate(lens):
        t = len(w.reqs)
        if share_prefix_from is not None and i > 0 and c > 0:
            src = w.reqs[share_prefix_from][0]
            n = (c // w.page_size) * w.page_size  # radix matches are page aligned
            w.page_table[t, :n] = w.page_table[src, :n]
            o_meta.ref_allocate_paged(w.page_table, w.free_pages, [(t, n, dl)], w.page_size)
        else:
            o_meta.ref_allocate_paged(w.page_table, w.free_pages, [(t, 0, dl)], w.page_size)
        w.reqs.append((t, c, dl))


def padded_reqs(w: World, pad_to: Optional[int] = None) -> List[Tuple[int, int, int]]:
    """w.reqs followed by dummy requests up to pad_to, as a graph-padded batch has them (GpuWorld.batch): the
    page table's last row, kv_len 1, all appending to the dummy page's first slot."""
    return list(w.reqs) + [(w.page_table.shape[0] - 1, 0, 1)] * ((pad_to or 0) - len(w.reqs))


def poison_unowned(w: World) -> None:
    """NaN in every CPU pool row no request owns, before GpuWorld mirrors the pool: unused page tails and free
    pages hold arbitrary bits in a real engine (torch.empty pool) and must never leak into a result."""
    used = np.zeros(w.pool_cpu.shape[2], dtype=bool)
    for (t, _, d) in w.reqs:
        used[w.page_table[t, :d]] = True
    w.pool_cpu[:, :, torch.from_numpy(~used)] = float("nan")


def make_inputs(w: World, seed: int, reqs: Optional[Sequence[Tuple[int, int, int]]] = None):
    """q/k/v for the new tokens of `reqs` (default w.reqs) as row-strided views of one qkv buffer
    (layers/attention.py:49)."""
    g = torch.Generator().manual_seed(seed)
    nnz = sum(d - c for (_, c, d) in (w.reqs if reqs is None else reqs))
    width = (w.hq + 2 * w.hkv) * w.d
    qkv = torch.randn((nnz, width), generator=g, dtype=torch.float32).to(w.dtype)
    q, k, v = qkv.split([w.hq * w.d, w.hkv * w.d, w.hkv * w.d], dim=-1)
    return qkv, q, k, v


# ------------------------------------------------------------------ operand layouts
# A layout takes the dense qkv rows [nnz, q_w + k_w + v_w] and the three widths and returns (q, k, v) as 2-D
# row-strided views holding the same values.  Every element of the buffers behind the views that no view covers
# is NaN (layout_padding), so a kernel that reads with the wrong row stride sees NaN or another operand's rows.
def padded_rows(x: torch.Tensor, pad: int) -> torch.Tensor:
    """x copied into the leading columns of a NaN buffer `pad` elements wider: row stride x.shape[1] + pad."""
    buf = torch.full((x.shape[0], x.shape[1] + pad), float("nan"), dtype=x.dtype, device=x.device)
    buf[:, : x.shape[1]] = x
    return buf[:, : x.shape[1]]


def _layout_split(qkv, widths):
    return qkv.split(list(widths), dim=-1)


def _layout_separate(qkv, widths):
    return tuple(x.contiguous() for x in qkv.split(list(widths), dim=-1))


def _layout_kv_pair(qkv, widths):
    q, k, v = qkv.split(list(widths), dim=-1)
    kv = torch.cat([k, v], dim=-1)
    return q.contiguous(), kv[:, : widths[1]], kv[:, widths[1] :]


def _layout_padded(qkv, widths, pads=(64, 128, 192)):
    return tuple(padded_rows(x, p) for x, p in zip(qkv.split(list(widths), dim=-1), pads))


def _layout_padded_shared_kv(qkv, widths):
    return _layout_padded(qkv, widths, pads=(64, 128, 128))


LAYOUTS = {
    "split": _layout_split,  # slices of one qkv row: q_rs == k_rs == v_rs (the engine's layout)
    "separate": _layout_separate,  # three contiguous tensors: q_rs = hq d, k_rs = v_rs = hkv d
    "kv_pair": _layout_kv_pair,  # separate q projection, fused kv projection: k_rs == v_rs = 2 hkv d
    "padded": _layout_padded,  # three wider buffers: q_rs, k_rs, v_rs pairwise distinct, none a dense width
    "padded_shared_kv": _layout_padded_shared_kv,  # padded, but k and v buffers of one row stride (prefill)
}


def layout_padding(views: Sequence[torch.Tensor]) -> torch.Tensor:
    """The elements of the buffers behind `views` that none of the views covers, flattened (empty for dense
    layouts).  Every buffer must be contiguous (the layouts allocate them so)."""
    bases, covered = {}, {}
    for t in views:
        b = t if t._base is None else t._base
        assert b.is_contiguous()
        bases[id(b)] = b
        m = covered.setdefault(id(b), torch.zeros(b.numel(), dtype=torch.bool, device=b.device))
        m.as_strided(t.shape, t.stride(), t.storage_offset() - b.storage_offset()).fill_(True)
    return torch.cat([bases[i].reshape(-1)[~covered[i]] for i in bases]) if bases else torch.empty(0)


def assert_all_nan_bits(x: torch.Tensor, what: str) -> None:
    """Every element of x holds exactly the bits the layouts filled the padding with."""
    nan = torch.tensor(float("nan"), dtype=x.dtype).view(torch.int16).item()
    bits = x.cpu().view(torch.int16)
    assert bool((bits == nan).all()), f"{what}: {(bits != nan).sum().item()} of {bits.numel()} padding elements written"


def ulp_close(a: torch.Tensor, b: torch.Tensor, ulps: float = 1.0, scale: Optional[torch.Tensor] = None):
    """|a-b| <= ulps * ulp(scale) elementwise for 16-bit floats (fp32 reduction-order noise only); scale
    defaults to |b|, the result itself.  A NaN in a or b fails."""
    a32, b32 = a.float().cpu(), b.float().cpu()
    eps = 2.0**-8 if a.dtype == torch.bfloat16 else 2.0**-11
    s = b32.abs() if scale is None else scale.float().cpu()
    tol = ulps * eps * s.clamp_min(1e-3) * 2
    bad = ~((a32 - b32).abs() <= tol)  # a NaN compares false, so it counts as bad
    assert not bad.any(), f"{bad.sum().item()} / {bad.numel()} beyond {ulps} ulp; max {((a32-b32).abs()).max()}"


def assert_pre_attention_close(q: Optional[torch.Tensor], k: Optional[torch.Tensor], qkv: torch.Tensor,
                               positions: torch.Tensor, hq: int, hkv: int, d: int, cos_sin_cache: torch.Tensor,
                               q_weight=None, k_weight=None, eps: float = 1e-6) -> None:
    """q [nnz, hq*d] and k [nnz, hkv*d] (any device, any row stride; None = not checked) against
    oracle.layer.ref_pre_attention of the raw rows qkv (q-norm, k-norm, neox RoPE).  Without a norm weight the
    rows are within one ulp of the oracle.  With one, the normed value is rounded before RoPE reads it, and that
    rounding may differ by one ulp between kernel and oracle; RoPE carries it into the output as up to one ulp of
    each rotated term, so the bound is one ulp of |out| + |x1 cos| + |x2 sin| (x = the oracle's normed row), which
    a cancellation cannot shrink."""
    from oracle.layer import ref_pre_attention
    from oracle.norm import ref_rmsnorm

    qkv, positions, cos_sin_cache = qkv.cpu(), positions.cpu(), cos_sin_cache.cpu()
    weights = [None if x is None else x.cpu() for x in (q_weight, k_weight)]
    ref_q, ref_k, _ = ref_pre_attention(qkv, positions, hq, hkv, d, cos_sin_cache, *weights, eps)
    nnz, half = qkv.shape[0], d // 2
    cs = cos_sin_cache[positions.to(torch.int64)].abs().unsqueeze(1)  # [nnz, 1, d]
    for got, ref, x, wt, heads in ((q, ref_q, qkv[:, : hq * d], weights[0], hq),
                                   (k, ref_k, qkv[:, hq * d : (hq + hkv) * d], weights[1], hkv)):
        if got is None:
            continue
        ref = ref.reshape(nnz, heads * d)
        if wt is None:
            ulp_close(got, ref)
            continue
        xn = ref_rmsnorm(x.reshape(nnz, heads, d), wt, eps).float().abs()
        x1, x2, c, s = xn[..., :half], xn[..., half:], cs[..., :half], cs[..., half:]
        terms = torch.cat((x1 * c + x2 * s, x2 * c + x1 * s), dim=-1).reshape(nnz, heads * d)
        ulp_close(got, ref, scale=ref.float().abs() + terms)


def oracle_forward(w: World, layer: int, q, k, v, md: o_meta.RefMetadata, fp32: bool = True,
                   reqs: Optional[Sequence[Tuple[int, int, int]]] = None):
    """Runs store + attention of `reqs` (default w.reqs) on CPU copies; returns (out, k_cache_after, v_cache_after)."""
    reqs = w.reqs if reqs is None else reqs
    kc = w.pool_cpu[0, layer].clone()
    vc = w.pool_cpu[1, layer].clone()
    nnz = q.shape[0]
    rows = [torch.from_numpy(md.slot_table[i, : md.cache_seqlens[i]].copy()) for i in range(len(reqs))]
    q_lens = [d - c for (_, c, d) in reqs]
    from oracle.store import ref_store_kv

    ref_store_kv(kc, vc, torch.from_numpy(md.out_loc.copy()), k.reshape(nnz, -1), v.reshape(nnz, -1))
    q3 = q.reshape(nnz, w.hq, w.d)
    out = torch.empty((nnz, w.hq, w.d), dtype=torch.float32)
    off = 0
    for r, ql in zip(rows, q_lens):
        idx = r.to(torch.int64)
        out[off : off + ql] = o_attn.ref_attention_one(q3[off : off + ql], kc[idx], vc[idx], w.d**-0.5)
        off += ql
    return (out if fp32 else out.to(w.dtype)), kc, vc


def attn_tolerance_ok(ours: torch.Tensor, ref32: torch.Tensor, what: str = ""):
    """Tolerance vs the exact-fp32 oracle: the single formula of oracle/tolerance.vs_exact_oracle
    (|err| <= 2e-3 * max|ref| + half an output ulp, element-wise) plus a relative Frobenius bound
    (3e-3 bf16 / 1e-3 fp16; bf16 rounding noise alone is ~1.6e-3).  Returns the relative Frobenius error."""
    from oracle import tolerance

    ours32 = ours.float().cpu()
    assert not torch.isnan(ours32).any(), f"{what}: NaN in output"
    err = tolerance.vs_exact_oracle(ours, ref32)
    rel_fro = ((ours32 - ref32).norm() / ref32.norm()).item()
    assert err <= tolerance.ORACLE_REL_TOL, f"{what}: excess error {err:.3e} > {tolerance.ORACLE_REL_TOL} (rel_fro {rel_fro:.3e})"
    assert rel_fro <= (3e-3 if ours.dtype == torch.bfloat16 else 1e-3), f"{what}: rel_fro {rel_fro:.3e}"
    return rel_fro


def assert_bits_equal(a: torch.Tensor, b: torch.Tensor, what: str):
    """a and b (16-bit, on any device) hold the same bits; a failure reports the largest difference."""
    a, b = a.cpu(), b.cpu()
    assert a.shape == b.shape, f"{what}: shapes {tuple(a.shape)} vs {tuple(b.shape)}"
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)), \
        f"{what}: bits differ, max |a - b| {(a.float() - b.float()).abs().max().item():.3e}"


ORDER_CLAMP_TILES = 127  # metadata.cu kOrderBins - 1: the decode plan's counting sort puts bigger items in one bin
PREFILL_CLAMP_TILES = 1023  # metadata.cu kPrefillBins - 1, the same for the prefill plan


def check_decode_plan(plan: np.ndarray, kv_lens: Sequence[int], max_splits: int = 16) -> None:
    """The split-KV decode plan {chunk, total, bs, 0, chunk_start[bs + 1], order[total]} of requests with
    kv_lens: every (request, chunk) item exactly once, chunk_start the running chunk count, and the work order
    descending in min(tiles, 127), tiles = the item's 128-key tiles (its last chunk without the appended key).
    The counting sort has 128 bins, so items of 127 tiles or more (kv_len >= 16 256 unsplit) share the last bin
    and come out in arbitrary order among themselves: a balance question, not a correctness one."""
    kv_lens = np.asarray(kv_lens, dtype=np.int64)
    bs = len(kv_lens)
    chunk, total, pbs = int(plan[0]), int(plan[1]), int(plan[2])
    assert pbs == bs and chunk % 128 == 0 and chunk >= 128
    starts = plan[4 : 4 + bs + 1]
    n_chunks = -(-kv_lens // chunk)
    assert np.array_equal(np.diff(starts), n_chunks) and starts[0] == 0 and starts[-1] == total
    assert n_chunks.max() <= max_splits
    order = plan[4 + bs + 1 : 4 + bs + 1 + total]
    items = [(int(e) & 0xFFFF, (int(e) >> 16) & 0xF) for e in order]
    assert len(set(items)) == total and set(items) == {(r, c) for r in range(bs) for c in range(int(n_chunks[r]))}
    assert all(((int(e) >> 20) & 0x1F) == n_chunks[int(e) & 0xFFFF] for e in order)

    def tiles(r, c):
        ln = min(chunk, int(kv_lens[r]) - c * chunk) - (1 if c == n_chunks[r] - 1 else 0)
        return min(-(-ln // 128), ORDER_CLAMP_TILES)

    sizes = [tiles(r, c) for r, c in items]
    assert sizes == sorted(sizes, reverse=True), "decode work order is not descending in min(tiles, 127)"


def check_prefill_plan(plan: np.ndarray, reqs: Sequence[Tuple[int, int, int]], request_major: bool) -> None:
    """The prefill plan {n_items, 0, 0, 0, item[n_items]} (item = r | q_tile << 16) of reqs (table_idx, cached,
    kv_len): one item per (request, 128-row query tile), each exactly once; size-sorted: descending in the
    tile's K/V tiles under the causal mask, min(ceil(kv_hi / 128), 1023); request-major: requests in batch order,
    the query tiles of a request adjacent, last tile first."""
    q_tiles = [-(-(d - c) // 128) for (_, c, d) in reqs]
    n = int(plan[0])
    assert n == sum(q_tiles), (n, sum(q_tiles))
    items = [(int(e) & 0xFFFF, (int(e) >> 16) & 0xFFFF) for e in plan[4 : 4 + n]]
    assert len(set(items)) == n and set(items) == {(r, t) for r, nq in enumerate(q_tiles) for t in range(nq)}
    if request_major:
        assert items == [(r, t) for r, nq in enumerate(q_tiles) for t in reversed(range(nq))]
        return

    def work(r, t):
        _, c, d = reqs[r]
        kv_hi = min(d, c + min(d - c, (t + 1) * 128))
        return min(-(-kv_hi // 128), PREFILL_CLAMP_TILES)

    sizes = [work(r, t) for r, t in items]
    assert sizes == sorted(sizes, reverse=True), "prefill work order is not descending in min(kv tiles, 1023)"


def box_rows(page_size: int) -> int:
    """Rows per tiled TMA box of the decode K/V loads (box_rows_for in csrc/attn.cuh): the largest power of two
    from 8 to 64 that divides the page size, 0 = row mode."""
    rows = 64
    while rows > 8 and page_size % rows:
        rows >>= 1
    return rows if page_size % rows == 0 else 0


def tail_range_ends(page_size: int) -> List[int]:
    """Streamed range lengths n (kv_len - 1) whose end falls at every offset of interest in the last page of a
    box-mode page size (>= 8): n mod page_size in {0, 1, 7, 8, 9, box_rows - 1, page_size - 1}, sorted."""
    rb = box_rows(page_size)
    return sorted({k * page_size + r for k in (2, 5) for r in (0, 1, 7, 8, 9, rb - 1, page_size - 1)})


class GpuWorld:
    """Device-side mirror of a World wired into the product's Context / pool / backend."""

    def __init__(self, b200, w: World, device="cuda"):
        self.b200, self.w = b200, w
        dev = torch.device(device)
        ctx = b200.Context(w.page_size)
        b200.core.set_global_ctx(None)
        b200.set_global_ctx(ctx)
        pool = b200.MHAKVCache(w.hkv, w.layers, w.d, w.num_pages + 1, w.page_size, w.dtype, dev)
        pool._kv_buffer.view(2, w.layers, -1, w.hkv, w.d).copy_(w.pool_cpu.to(dev))
        ctx.kv_cache = pool
        ctx.page_table = torch.from_numpy(w.page_table.copy()).to(dev)
        cfg = SimpleNamespace(num_qo_heads=w.hq, num_kv_heads=w.hkv, head_dim=w.d)
        self.backend = b200.create_attention_backend("b200", cfg)
        ctx.attn_backend = self.backend
        self.ctx, self.pool, self.dev = ctx, pool, dev

    def batch(self, phase: str, pad_to: Optional[int] = None, md: Optional[o_meta.RefMetadata] = None):
        """A batch of w.reqs, padded with dummy requests to pad_to; md: out_loc and positions from the oracle's
        metadata of the padded requests."""
        b200 = self.b200
        reqs = [b200.Req(table_idx=t, cached_len=c, device_len=d) for (t, c, d) in self.w.reqs]
        batch = b200.Batch(reqs, phase)
        if pad_to is not None and pad_to > len(reqs):
            dummy = b200.Req(table_idx=self.w.page_table.shape[0] - 1, cached_len=0, device_len=1)
            batch.padded_reqs = reqs + [dummy] * (pad_to - len(reqs))
        if md is not None:
            batch.out_loc = torch.from_numpy(md.out_loc).to(self.dev)
            batch.positions = torch.from_numpy(md.positions).to(self.dev)
        return batch

    def pool_rows(self, layer: int):
        """K and V rows [slots, hkv, d] of one pool layer, on the device."""
        kc = self.pool.k_cache(layer).reshape(-1, self.w.hkv, self.w.d)
        vc = self.pool.v_cache(layer).reshape(-1, self.w.hkv, self.w.d)
        return kc, vc


def run_attention(gw: GpuWorld, batch, qkv: torch.Tensor, *, layer: int = 0, fused: Optional[tuple] = None,
                  graph: bool = False, prepare: bool = True, layout=_layout_split):
    """One attention launch of `batch` on the device rows `qkv` [nnz, (hq + 2 hkv) d], as the engine runs it:
    prepare_metadata (unless the caller ran it already: prepare=False), then `forward`, or for a decode batch
    with fused = (cos_sin_cache, q_weight, k_weight, eps) `forward_decode_fused` on the raw q / k rows.  layout
    (one of LAYOUTS) lays q, k and v out from `qkv`; the default slices one qkv row, as the engine does.  graph:
    the decode launch is captured into a CUDA graph on a dummy batch of the same size and replayed on `batch`
    after prepare_for_replay, like the engine's graph runner; its static q / k / v buffers come from the same
    layout, so the captured launch sees the same strides.  Synchronises.  Returns (out, decode plan, pool K
    rows, pool V rows of the layer), all on the device."""
    w, backend = gw.w, gw.backend
    widths = (w.hq * w.d, w.hkv * w.d, w.hkv * w.d)

    def launch(qkv_views, b):
        q, k, v = qkv_views
        if fused is None:
            return backend.forward(q.view(-1, w.hq, w.d), k, v, layer, b)
        return backend.forward_decode_fused(q.view(-1, w.hq, w.d), k, v, layer, b, b.positions, *fused)

    if not graph:
        if prepare:
            backend.prepare_metadata(batch)
        out = launch(layout(qkv, widths), batch)
    else:
        # static buffers of the "graph runner", captured on a batch of dummy requests of the same size
        bs = batch.padded_size
        backend.init_capture_graph(w.page_table.shape[1], [bs])
        dummy = gw.b200.Req(table_idx=w.page_table.shape[0] - 1, cached_len=0, device_len=1)
        cap = gw.b200.Batch([dummy] * bs, "decode")
        cap.padded_reqs = cap.reqs
        backend.prepare_for_capture(cap)
        static = layout(torch.zeros_like(qkv), widths)
        cap.positions = torch.zeros(bs, dtype=torch.int32, device=gw.dev)
        cap.out_loc = torch.full((bs,), int(w.page_table[-1, 0]), dtype=torch.int32, device=gw.dev)
        out = torch.zeros(bs, w.hq, w.d, dtype=qkv.dtype, device=gw.dev)
        stream = torch.cuda.Stream()
        with torch.cuda.stream(stream):
            out.copy_(launch(static, cap))  # warm-up outside the capture
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                out.copy_(launch(static, cap))
        torch.cuda.synchronize()
        if prepare:
            backend.prepare_metadata(batch)
        stream.wait_stream(torch.cuda.current_stream())  # the live metadata is built on the current stream
        with torch.cuda.stream(stream):
            for dst, src in zip(static, qkv.split(list(widths), dim=-1)):
                dst.copy_(src)
            cap.positions.copy_(batch.positions)
            cap.out_loc.copy_(batch.out_loc)
            backend.prepare_for_replay(batch)
            g.replay()
    torch.cuda.synchronize()
    return (out, batch.attn_metadata.decode_plan) + gw.pool_rows(layer)


def replan(gw: GpuWorld, batch, num_ctas: int) -> None:
    """Rebuilds the prepared metadata of `batch` in place, with the decode plan made for a grid of num_ctas CTAs
    instead of the device's (a much larger grid splits every request into several chunks)."""
    md, pt, b200 = batch.attn_metadata, gw.ctx.page_table, gw.b200
    flat, _, _ = b200.attention.backend.host_req_info(batch.padded_reqs)
    info = torch.tensor(flat, dtype=torch.int32, device=gw.dev)
    b200._cabi.check(gw.backend._lib.b200_build_metadata(
        info.data_ptr(), md.bs, pt.data_ptr(), pt.stride(0), md.cache_seqlens.data_ptr(), md.cu_seqlens_q.data_ptr(),
        md.cu_seqlens_k.data_ptr(), md.page_table.data_ptr(), md.page_table.stride(0), md.page_table.shape[1],
        md.decode_plan.data_ptr(), gw.w.hkv, num_ctas, torch.cuda.current_stream().cuda_stream), "b200_build_metadata")
