"""Shared builders for the parity tests: a paged world (page table + pool + requests) on CPU,
mirrored onto the GPU for the product path."""
from __future__ import annotations

import contextlib
import importlib
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
    al = max(64, page_size)
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


def make_inputs(w: World, seed: int, strided: bool = True):
    """q/k/v for the new tokens as row-strided views of one qkv buffer (layers/attention.py:49)."""
    g = torch.Generator().manual_seed(seed)
    nnz = sum(d - c for (_, c, d) in w.reqs)
    width = (w.hq + 2 * w.hkv) * w.d
    qkv = torch.randn((nnz, width), generator=g, dtype=torch.float32).to(w.dtype)
    if not strided:
        q, k, v = [x.contiguous() for x in qkv.split([w.hq * w.d, w.hkv * w.d, w.hkv * w.d], -1)]
    else:
        q, k, v = qkv.split([w.hq * w.d, w.hkv * w.d, w.hkv * w.d], dim=-1)
    return qkv, q, k, v


def oracle_forward(w: World, layer: int, q, k, v, md: o_meta.RefMetadata, fp32: bool = True):
    """Runs store + attention on CPU copies; returns (out, k_cache_after, v_cache_after)."""
    kc = w.pool_cpu[0, layer].clone()
    vc = w.pool_cpu[1, layer].clone()
    nnz = q.shape[0]
    rows = [torch.from_numpy(md.slot_table[i, : md.cache_seqlens[i]].copy()) for i in range(len(w.reqs))]
    q_lens = [d - c for (_, c, d) in w.reqs]
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

    def batch(self, phase: str, pad_to: Optional[int] = None):
        b200 = self.b200
        reqs = [b200.Req(table_idx=t, cached_len=c, device_len=d) for (t, c, d) in self.w.reqs]
        batch = b200.Batch(reqs, phase)
        if pad_to is not None and pad_to > len(reqs):
            dummy = b200.Req(table_idx=self.w.page_table.shape[0] - 1, cached_len=0, device_len=1)
            batch.padded_reqs = reqs + [dummy] * (pad_to - len(reqs))
        return batch

    def pool_rows(self, layer: int):
        kc = self.pool.k_cache(layer).reshape(-1, self.w.hkv, self.w.d).cpu()
        vc = self.pool.v_cache(layer).reshape(-1, self.w.hkv, self.w.d).cpu()
        return kc, vc
