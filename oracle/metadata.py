"""Oracle: integer metadata of the attention boundary (TEST INFRASTRUCTURE ONLY).

Restates, in numpy, what the reference computes on the host before every forward:

* ``positions`` / ``out_loc``      -- ``python/minisgl/scheduler/scheduler.py:204-249``
* ``prepare_metadata`` (fa/trtllm) -- ``python/minisgl/attention/fa.py:67-105``
                                      (identical in ``trtllm.py:91-129``)
* ``prepare_metadata`` (fi)        -- ``python/minisgl/attention/fi.py:190-225``
* ``get_last_indices``             -- ``python/minisgl/attention/fa.py:32-33``

All results are int32 and must be matched **bit-exactly** by the product.
A request is the triple ``(table_idx, cached_len, device_len)`` -- the only ``Req``
fields the boundary reads (``python/minisgl/core.py:29-54``).
"""

from __future__ import annotations

from dataclasses import dataclass
from typing import List, Sequence, Tuple

import numpy as np

ReqTriple = Tuple[int, int, int]  # (table_idx, cached_len, device_len)


@dataclass
class RefMetadata:
    cu_seqlens_q: np.ndarray  # int32 [bs+1]
    cu_seqlens_k: np.ndarray  # int32 [bs+1]
    cache_seqlens: np.ndarray  # int32 [bs]
    max_seqlen_q: int
    max_seqlen_k: int
    positions: np.ndarray  # int32 [nnz]
    out_loc: np.ndarray  # int32 [nnz]
    page_table_paged: np.ndarray  # int32 [bs, ceil(max_k / page)]  (fa / trtllm dialect)
    indices_flat: np.ndarray  # int32 [sum kv_len]               (fi dialect, page_size == 1 view)
    slot_table: np.ndarray  # int32 [bs, max_k] token-granular slots (columns >= kv_len: raw table)
    last_indices: np.ndarray  # int32 [bs]


def ref_positions(reqs: Sequence[ReqTriple]) -> np.ndarray:
    """scheduler.py:236-249 -- concat of arange(cached_len, device_len)."""
    parts = [np.arange(c, d, dtype=np.int32) for (_, c, d) in reqs]
    return np.concatenate(parts) if parts else np.zeros(0, np.int32)


def ref_out_loc(page_table: np.ndarray, reqs: Sequence[ReqTriple]) -> np.ndarray:
    """scheduler.py:207-210,252-259 -- page_table[table_idx, position] per new token."""
    parts = [page_table[t, c:d] for (t, c, d) in reqs]
    return np.concatenate(parts).astype(np.int32) if parts else np.zeros(0, np.int32)


def ref_cu_seqlens(reqs: Sequence[ReqTriple]) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """fa.py:70-90 -- the three branches (decode arange / no-cache alias / cumsum) all
    produce cumsum(extend_len); values are what matters at the boundary."""
    seqlens_q = np.array([d - c for (_, c, d) in reqs], dtype=np.int64)
    seqlens_k = np.array([d for (_, _, d) in reqs], dtype=np.int64)
    cu_k = np.concatenate([[0], np.cumsum(seqlens_k)]).astype(np.int32)
    max_q = int(seqlens_q.max())
    if max_q == 1:
        cu_q = np.arange(0, len(reqs) + 1, dtype=np.int32)
    elif all(c == 0 for (_, c, _) in reqs):
        cu_q = cu_k.copy()
    else:
        cu_q = np.concatenate([[0], np.cumsum(seqlens_q)]).astype(np.int32)
    return cu_q, cu_k, seqlens_k.astype(np.int32)


def ref_page_table_paged(
    page_table: np.ndarray, reqs: Sequence[ReqTriple], page_size: int
) -> np.ndarray:
    """fa.py:92-97 -- every ``page_size``-th column of the token-granular table, floor-divided."""
    max_k = max(d for (_, _, d) in reqs)
    rows = np.stack([page_table[t, :max_k:page_size] for (t, _, _) in reqs])
    if page_size > 1:
        rows = rows // page_size
    return rows.astype(np.int32)


def ref_indices_flat(page_table: np.ndarray, reqs: Sequence[ReqTriple]) -> np.ndarray:
    """fi.py:215 -- cat(page_table[table_idx, :device_len])."""
    return np.concatenate([page_table[t, :d] for (t, _, d) in reqs]).astype(np.int32)


def ref_slot_table(page_table: np.ndarray, reqs: Sequence[ReqTriple]) -> np.ndarray:
    """Token-granular snapshot ``page_table[table_idx, :max_k]`` (the page_size==1 case of
    fa.py:92-94); this is the dialect the project's kernels consume."""
    max_k = max(d for (_, _, d) in reqs)
    return np.stack([page_table[t, :max_k] for (t, _, _) in reqs]).astype(np.int32)


def ref_last_indices(cu_seqlens_q: np.ndarray, bs: int) -> np.ndarray:
    """fa.py:32-33 -- cu_seqlens_q[1:1+bs] - 1."""
    return (cu_seqlens_q[1 : 1 + bs] - 1).astype(np.int32)


def ref_prepare_metadata(
    page_table: np.ndarray, reqs: Sequence[ReqTriple], page_size: int
) -> RefMetadata:
    reqs = list(reqs)
    cu_q, cu_k, seqlens_k = ref_cu_seqlens(reqs)
    return RefMetadata(
        cu_seqlens_q=cu_q,
        cu_seqlens_k=cu_k,
        cache_seqlens=seqlens_k,
        max_seqlen_q=max(d - c for (_, c, d) in reqs),
        max_seqlen_k=max(d for (_, _, d) in reqs),
        positions=ref_positions(reqs),
        out_loc=ref_out_loc(page_table, reqs),
        page_table_paged=ref_page_table_paged(page_table, reqs, page_size),
        indices_flat=ref_indices_flat(page_table, reqs),
        slot_table=ref_slot_table(page_table, reqs),
        last_indices=ref_last_indices(cu_q, len(reqs)),
    )


def ref_allocate_paged(
    page_table: np.ndarray,
    free_pages: List[int],
    reqs: Sequence[ReqTriple],
    page_size: int,
) -> None:
    """Page allocation as the scheduler does it (``python/minisgl/scheduler/cache.py:42-53,
    119-146``): pop page-aligned slots off the free list and write token-slot ids
    ``page*page_size + offset`` for pages ``[ceil(cached/ps), ceil(device/ps))``."""
    for (t, c, d) in reqs:
        first = -(-c // page_size)
        last = -(-d // page_size)
        for p in range(first, last):
            base = free_pages.pop(0)
            lo, hi = p * page_size, (p + 1) * page_size
            page_table[t, lo:hi] = base + np.arange(page_size, dtype=np.int32)
