"""``B200AttnBackend`` -- the drop-in ``BaseAttnBackend`` (reference ``python/minisgl/attention/
base.py:18-34``) whose ``forward`` runs the hand-written sm_90a kernels of libb200attn.

Contract kept from the reference backends (fi.py:80-271, fa.py:36-136, trtllm.py:35-162):

* constructed by ``BackendCreator(config)`` after ``ctx.kv_cache`` and ``ctx.page_table`` exist
  (engine/engine.py:55-78); borrows both, owns its workspace and capture buffers;
* ``prepare_metadata`` runs on the scheduler stream one step ahead and sets
  ``batch.attn_metadata`` (fresh buffers per batch, nothing an in-flight forward reads);
* ``forward`` appends ``k, v`` at ``batch.out_loc`` (bit-exact rows) and returns a fresh contiguous
  ``[nnz, Hq_local, D]``; never synchronises; capturable in a CUDA graph for decode;
* ``init_capture_graph / prepare_for_capture / prepare_for_replay`` follow fa.py:107-136 (static
  buffers refreshed with device-to-device copies at replay).

What differs: the per-step host loops + ``torch.cat`` / ``torch.stack`` of ``bs`` row slices are one
device kernel (``b200_build_metadata``), the page-table dialect is a token-granular slot snapshot
``[bs, max_k]`` (valid for every ``page_size``, including the default 1), and the decode append is
fused into the attention launch.
"""

from __future__ import annotations

import os
import time
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import torch

from .. import _cabi
from ..core import get_global_ctx
from ..utils import div_even, get_tp_info
from .base import BaseAttnBackend, BaseAttnMetadata

_DEBUG_CHECKS = os.environ.get("B200_DEBUG_CHECKS", "0") not in ("", "0")
_PLAN_HEADER = 4
_DTYPE_CODE = {torch.bfloat16: 0, torch.float16: 1}


def _align(x: int, a: int) -> int:
    return (x + a - 1) // a * a


def host_req_info(reqs: Sequence) -> Tuple[List[int], int, int]:
    """Pure host part of ``prepare_metadata``: flatten ``(table_idx, cached_len, device_len)`` of
    every padded request (the only ``Req`` fields read, reference fa.py:70-74) and the two maxima."""
    flat: List[int] = []
    max_q = 0
    max_k = 0
    for r in reqs:
        c, d = r.cached_len, r.device_len
        flat += (r.table_idx, c, d)
        if d - c > max_q:
            max_q = d - c
        if d > max_k:
            max_k = d
    return flat, max_q, max_k


_MAX_SPLITS = 16


def plan_ints(bs: int) -> int:
    """Size of the split-KV decode plan (``b200_decode_plan_ints``): header, chunk_start[bs+1],
    size-sorted work order (at most 16 chunks per request)."""
    return _PLAN_HEADER + bs + 1 + _MAX_SPLITS * bs


def small_block_layout(bs: int) -> Tuple[int, int, int, int, int]:
    """Offsets (in int32) of seq_lens | cu_q | cu_k | plan inside the per-batch small block; each
    section 16-byte aligned.  Returns (off_seq, off_cuq, off_cuk, off_plan, total)."""
    off_seq = 0
    off_cuq = _align(bs, 4)
    off_cuk = off_cuq + _align(bs + 1, 4)
    off_plan = off_cuk + _align(bs + 1, 4)
    total = off_plan + _align(plan_ints(bs), 4)
    return off_seq, off_cuq, off_cuk, off_plan, total


@dataclass
class B200Metadata(BaseAttnMetadata):
    """Field names follow ``FAMetadata`` (reference fa.py:22-33)."""

    cu_seqlens_k: torch.Tensor  # int32 [bs+1]
    cu_seqlens_q: torch.Tensor  # int32 [bs+1]
    cache_seqlens: torch.Tensor  # int32 [bs]   kv length incl. the tokens of this forward
    max_seqlen_k: int
    max_seqlen_q: int
    page_table: torch.Tensor  # int32 [bs, >= max_seqlen_k] token-granular slot snapshot
    decode_plan: torch.Tensor  # int32 [4 + bs + 1 + 16 bs] split-KV plan (see include/b200attn.h)
    small_block: torch.Tensor  # the contiguous buffer the four small tensors are views of
    bs: int
    prefill_plan: Optional[torch.Tensor] = None  # int32 work list of the prefill kernel (q_len > 1)

    def get_last_indices(self, bs: int) -> torch.Tensor:
        return self.cu_seqlens_q[1 : 1 + bs] - 1

    # --- dialect helpers: what the reference backends would have handed their kernels ---------
    def flat_indices(self) -> torch.Tensor:
        """fi dialect (fi.py:215): ``cat(page_table[table_idx, :device_len])``."""
        lens = self.cache_seqlens.tolist()
        return torch.cat([self.page_table[i, :n] for i, n in enumerate(lens)])

    def paged_page_table(self, page_size: int) -> torch.Tensor:
        """fa / trtllm dialect (fa.py:92-97): every ``page_size``-th column, floor-divided."""
        t = self.page_table[:, : self.max_seqlen_k : page_size]
        return t // page_size if page_size > 1 else t.clone()


@dataclass
class B200CaptureData:
    """Static buffers the captured decode graphs read (reference attention/utils.py:7-23)."""

    small_blocks: dict  # bs -> int32 small block (seq_lens | cu_q | cu_k | plan)
    page_table: torch.Tensor  # int32 [max_bs, max_seq_len]


class B200AttnBackend(BaseAttnBackend):
    def __init__(self, config, *, device: Optional[torch.device] = None) -> None:
        ctx = get_global_ctx()
        self.config = config
        self.kvcache = ctx.kv_cache
        self.page_size = ctx.page_size
        self.device = device if device is not None else self.kvcache.device
        self.head_dim = int(config.head_dim)
        self.scale = self.head_dim**-0.5
        tp = get_tp_info().size
        self.qo_head_local = div_even(config.num_qo_heads, tp)
        self.kv_head_local = div_even(config.num_kv_heads, tp, allow_replicate=True)
        if self.head_dim != 128:
            raise RuntimeError(f"B200AttnBackend supports head_dim 128 only (got {self.head_dim})")
        self.capture: Optional[B200CaptureData] = None
        self.capture_bs: List[int] = []
        self.max_graph_bs = 0
        self._workspace: Optional[torch.Tensor] = None
        self._workspace_bs = 0
        self._retired_workspaces: List[torch.Tensor] = []
        # pinned staging ring for the per-batch (table_idx, cached_len, device_len) triples: re-used, never
        # re-allocated per step; an entry is rewritten only after the copy that read it has completed
        self._info_ring: List[tuple] = []  # (pinned int32 tensor, event of its last copy, numpy view)
        self._layouts: dict = {}
        self._info_next = 0
        self.ring_wait_s = 0.0  # host time spent waiting for a free request-info buffer (GPU back-pressure)
        self._lib = None
        self._sm_count = 0
        if torch.device(self.device).type == "cuda":
            self._lib = _cabi.load()  # raises loudly when the native library is missing
            self._sm_count = torch.cuda.get_device_properties(self.device).multi_processor_count

    # ------------------------------------------------------------------ workspace
    def _get_workspace(self, bs: int) -> torch.Tensor:
        """Split-KV workspace (fp32 partials + arrival counters) of the decode kernel.  Sized ONCE for
        the largest batch the engine can ever hand over -- ``page_table.shape[0]`` rows =
        ``max_running_req + 1`` (engine/engine.py:69-73) -- because captured decode graphs bake its
        address in (partials and the counters at its tail).  Should a larger batch ever show up, a new
        buffer is used for eager launches from then on and the old ones are kept alive, so a captured
        graph never writes into freed memory."""
        if self._workspace is None or bs > self._workspace_bs:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("attention workspace must be sized before graph capture")
            want = max(bs, self.max_graph_bs, int(get_global_ctx().page_table.shape[0]))
            nbytes = self._lib.b200_attn_workspace_bytes(want, self.qo_head_local, self.head_dim)
            if self._workspace is not None:
                self._retired_workspaces.append(self._workspace)
            # zero-filled once: holds the split-KV arrival counters (left at zero by every launch)
            self._workspace = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
            self._workspace_bs = want
        return self._workspace

    # ------------------------------------------------------------------ metadata
    _INFO_RING = 4  # > the scheduler's look-ahead of one batch (overlap scheduling, scheduler.py:83-106)

    def _stage_req_info(self, flat: List[int]) -> Tuple[int, "torch.cuda.Event"]:
        """The request triples are written into one buffer of a small ring of PINNED host buffers and the
        metadata kernels read them from there directly (zero copy: pinned ``cudaHostAlloc`` memory is mapped
        into the device's unified address space) -- no host-to-device copy sits on the critical path of the
        step, where it would queue behind any large upload in the DMA engine.  The reference allocates a fresh pinned
        tensor and issues an H2D copy per step (fa.py:76-90).  Returns (device-visible pointer, event to
        record once the kernels that read it have been enqueued)."""
        n = len(flat)
        if len(self._info_ring) < self._INFO_RING:
            cap = max(3 * int(get_global_ctx().page_table.shape[0]), n)
            host = torch.empty(cap, dtype=torch.int32, pin_memory=True)
            self._info_ring.append((host, torch.cuda.Event(), host.numpy()))
            slot = len(self._info_ring) - 1
        else:
            slot = self._info_next
            self._info_next = (slot + 1) % self._INFO_RING
            t0 = time.perf_counter()
            self._info_ring[slot][1].synchronize()  # the kernels launched 4 batches ago: long done
            self.ring_wait_s += time.perf_counter() - t0
            if self._info_ring[slot][0].numel() < n:
                host = torch.empty(n, dtype=torch.int32, pin_memory=True)
                self._info_ring[slot] = (host, self._info_ring[slot][1], host.numpy())
        host, ev, view = self._info_ring[slot]
        view[:n] = flat  # python ints -> pinned memory, no intermediate tensor
        return host.data_ptr(), ev

    def prepare_metadata(self, batch) -> None:
        reqs = batch.padded_reqs
        bs = len(reqs)
        flat, max_q, max_k = host_req_info(reqs)
        if self._lib is None:
            raise RuntimeError("B200AttnBackend.prepare_metadata needs a CUDA device (no CPU path)")
        dev = self.device
        info_ptr, info_ev = self._stage_req_info(flat)
        lay = self._layouts.get(bs)
        if lay is None:
            lay = self._layouts[bs] = small_block_layout(bs)
        off_seq, off_cuq, off_cuk, off_plan, total = lay
        small = torch.empty(total, dtype=torch.int32, device=dev)
        page_table = get_global_ctx().page_table
        width = min(_align(max_k, 4), page_table.shape[1])
        slot_table = torch.empty((bs, width), dtype=torch.int32, device=dev)
        seq_lens = small[off_seq : off_seq + bs]
        cu_q = small[off_cuq : off_cuq + bs + 1]
        cu_k = small[off_cuk : off_cuk + bs + 1]
        plan = small[off_plan : off_plan + plan_ints(bs)]
        _cabi.check(
            self._lib.b200_build_metadata(
                info_ptr, bs, page_table.data_ptr(), page_table.stride(0),
                seq_lens.data_ptr(), cu_q.data_ptr(), cu_k.data_ptr(), slot_table.data_ptr(),
                slot_table.stride(0), width, plan.data_ptr(), self.kv_head_local,
                2 * self._sm_count, torch.cuda.current_stream(dev).cuda_stream,
            ),
            "b200_build_metadata",
        )
        prefill_plan = None
        if max_q > 1:
            cap = (len(flat) // 3) + sum(r.extend_len for r in reqs) // 128
            prefill_plan = torch.empty(4 + cap, dtype=torch.int32, device=dev)
            _cabi.check(
                self._lib.b200_build_prefill_plan(
                    info_ptr, bs, prefill_plan.data_ptr(), cap,
                    torch.cuda.current_stream(dev).cuda_stream,
                ),
                "b200_build_prefill_plan",
            )
        info_ev.record()  # the pinned triples may be overwritten once these kernels have run
        batch.attn_metadata = B200Metadata(
            cu_seqlens_k=cu_k,
            cu_seqlens_q=cu_q,
            cache_seqlens=seq_lens,
            max_seqlen_k=max_k,
            max_seqlen_q=max_q,
            page_table=slot_table,
            decode_plan=plan,
            small_block=small,
            bs=bs,
            prefill_plan=prefill_plan,
        )

    # ------------------------------------------------------------------ forward
    def _check_inputs(self, q, k, v, layer_id, batch):
        md = batch.attn_metadata
        if not isinstance(md, B200Metadata):
            raise RuntimeError("batch.attn_metadata was not prepared by B200AttnBackend")
        if self._lib is None or not q.is_cuda:
            raise RuntimeError("B200AttnBackend.forward needs CUDA tensors (no CPU fallback)")
        hq, hkv, d = self.qo_head_local, self.kv_head_local, self.head_dim
        nnz = q.shape[0]
        q3 = q.view(nnz, hq, d) if q.dim() == 2 else q
        if q3.stride(2) != 1 or q3.stride(1) != d or k.stride(-1) != 1 or v.stride(-1) != 1:
            raise RuntimeError("attention inputs must have dense heads / contiguous last dim")
        k2 = k.view(nnz, -1) if k.dim() != 2 else k
        v2 = v.view(nnz, -1) if v.dim() != 2 else v
        kc = self.kvcache.k_cache(layer_id)
        vc = self.kvcache.v_cache(layer_id)
        if not (kc.is_contiguous() and vc.is_contiguous()):
            raise RuntimeError("KV pool layer views must be contiguous [pages, page, Hkv, D]")
        dtype = _DTYPE_CODE.get(q.dtype)
        if dtype is None or kc.dtype != q.dtype:
            raise RuntimeError(f"unsupported / mismatched dtypes q={q.dtype} pool={kc.dtype}")
        out_loc = batch.out_loc
        if out_loc.dtype != torch.int32 or not out_loc.is_contiguous():
            raise RuntimeError("batch.out_loc must be a contiguous int32 vector")
        return md, nnz, q3, k2, v2, kc, vc, dtype, out_loc

    def forward(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, layer_id: int, batch):
        md, nnz, q3, k2, v2, kc, vc, dtype, out_loc = self._check_inputs(q, k, v, layer_id, batch)
        hq, hkv, d = self.qo_head_local, self.kv_head_local, self.head_dim
        out = torch.empty((nnz, hq, d), dtype=q.dtype, device=q.device)
        num_slots = kc.numel() // (hkv * d)
        stream = torch.cuda.current_stream(q.device).cuda_stream
        if md.max_seqlen_q == 1:
            if nnz != md.bs:
                raise RuntimeError(f"decode expects one query row per request ({nnz} vs {md.bs})")
            ws = self._get_workspace(md.bs)
            _cabi.check(
                self._lib.b200_attn_decode(
                    q3.data_ptr(), q3.stride(0), k2.data_ptr(), k2.stride(0), v2.data_ptr(),
                    v2.stride(0), kc.data_ptr(), vc.data_ptr(), num_slots, self.page_size,
                    out_loc.data_ptr(),
                    md.page_table.data_ptr(), md.page_table.stride(0), md.cache_seqlens.data_ptr(),
                    md.decode_plan.data_ptr(), md.bs, hq, hkv, d, self.scale, out.data_ptr(),
                    ws.data_ptr(), ws.numel(), dtype, stream,
                ),
                "b200_attn_decode",
            )
        else:
            # Contract of the wgmma prefill kernel: it appends the tile that holds a unit's own tokens
            # at slot_table[r, cached + i] (the metadata snapshot), which equals batch.out_loc by the
            # reference's construction out_loc = page_table[table_idx, cached_len:device_len]
            # (scheduler/scheduler.py:207-210); B200_DEBUG_CHECKS=1 verifies it per call (host sync).
            if _DEBUG_CHECKS:
                self._assert_out_loc_matches_slot_table(md, out_loc)
            _cabi.check(
                self._lib.b200_attn_prefill(
                    q3.data_ptr(), q3.stride(0), k2.data_ptr(), k2.stride(0), v2.data_ptr(),
                    v2.stride(0), kc.data_ptr(), vc.data_ptr(), num_slots, self.page_size,
                    out_loc.data_ptr(),
                    md.page_table.data_ptr(), md.page_table.stride(0), md.cache_seqlens.data_ptr(),
                    md.cu_seqlens_q.data_ptr(),
                    md.prefill_plan.data_ptr() if md.prefill_plan is not None else None,
                    md.bs, nnz, md.max_seqlen_q, hq, hkv, d, self.scale,
                    out.data_ptr(), None, 0, dtype, stream,
                ),
                "b200_attn_prefill",
            )
        return out

    @staticmethod
    def _assert_out_loc_matches_slot_table(md: "B200Metadata", out_loc: torch.Tensor) -> None:
        lens = md.cache_seqlens.tolist()
        cu_q = md.cu_seqlens_q.tolist()
        want = torch.cat([md.page_table[i, n - (cu_q[i + 1] - cu_q[i]) : n] for i, n in enumerate(lens)])
        if not torch.equal(want, out_loc[: want.numel()]):
            raise RuntimeError("batch.out_loc != page_table[table_idx, cached_len:device_len] "
                               "(the fused prefill append relies on the reference's invariant)")

    def forward_decode_fused(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, layer_id: int, batch,
                             positions: torch.Tensor, cos_sin_cache: torch.Tensor,
                             q_weight: Optional[torch.Tensor], k_weight: Optional[torch.Tensor], eps: float):
        """Decode forward with the pre-attention sequence of ``AttentionLayer.forward`` (reference
        layers/attention.py:50-54: q-norm, k-norm, RoPE) folded into the attention launch: ``q`` / ``k``
        are the RAW rows of the qkv projection and stay untouched; the pool receives the normed + roped
        k row.  Bit-identical to ``ops.qknorm_rope_inplace`` followed by :meth:`forward`."""
        md, nnz, q3, k2, v2, kc, vc, dtype, out_loc = self._check_inputs(q, k, v, layer_id, batch)
        if md.max_seqlen_q != 1 or nnz != md.bs:
            raise RuntimeError("forward_decode_fused is for decode batches (one query row per request)")
        if positions.dtype != torch.int32 or positions.numel() != nnz or not positions.is_contiguous():
            raise RuntimeError("forward_decode_fused: positions must be a contiguous int32 [bs] vector")
        if cos_sin_cache.dtype != torch.float32 or cos_sin_cache.shape[-1] != self.head_dim or not cos_sin_cache.is_contiguous():
            raise RuntimeError("forward_decode_fused: cos_sin_cache must be contiguous fp32 [max_pos, head_dim]")
        for w in (q_weight, k_weight):
            if w is not None and (w.dtype != q.dtype or w.shape != (self.head_dim,) or not w.is_contiguous()):
                raise RuntimeError("forward_decode_fused: norm weights must be contiguous [head_dim] of q's dtype")
        hq, hkv, d = self.qo_head_local, self.kv_head_local, self.head_dim
        out = torch.empty((nnz, hq, d), dtype=q.dtype, device=q.device)
        ws = self._get_workspace(md.bs)
        _cabi.check(
            self._lib.b200_attn_decode_fused(
                q3.data_ptr(), q3.stride(0), k2.data_ptr(), k2.stride(0), v2.data_ptr(), v2.stride(0),
                q_weight.data_ptr() if q_weight is not None else None,
                k_weight.data_ptr() if k_weight is not None else None, float(eps),
                positions.data_ptr(), cos_sin_cache.data_ptr(), kc.data_ptr(), vc.data_ptr(),
                kc.numel() // (hkv * d), self.page_size, out_loc.data_ptr(), md.page_table.data_ptr(),
                md.page_table.stride(0), md.cache_seqlens.data_ptr(), md.decode_plan.data_ptr(), md.bs, hq,
                hkv, d, self.scale, out.data_ptr(), ws.data_ptr(), ws.numel(), dtype,
                torch.cuda.current_stream(q.device).cuda_stream,
            ),
            "b200_attn_decode_fused",
        )
        return out

    # ------------------------------------------------------------------ CUDA graphs
    def init_capture_graph(self, max_seq_len: int, bs_list: List[int]) -> None:
        if self.capture is not None:
            raise AssertionError("Capture already initialized.")
        max_bs = max(bs_list)
        dev = self.device
        blocks = {}
        for bs in bs_list:
            off_seq, off_cuq, off_cuk, off_plan, total = small_block_layout(bs)
            blk = torch.zeros(total, dtype=torch.int32, device=dev)
            blk[off_seq : off_seq + bs] = 1
            blk[off_cuq : off_cuq + bs + 1] = torch.arange(bs + 1, dtype=torch.int32, device=dev)
            blk[off_cuk : off_cuk + bs + 1] = torch.arange(bs + 1, dtype=torch.int32, device=dev)
            blocks[bs] = blk
        self.capture = B200CaptureData(
            small_blocks=blocks,
            page_table=torch.zeros((max_bs, max_seq_len), dtype=torch.int32, device=dev),
        )
        self.max_graph_bs = max_bs
        self.capture_bs = sorted(bs_list)
        self._get_workspace(max_bs)

    def _bind_capture(self, bs: int, max_k: int) -> B200Metadata:
        assert self.capture is not None
        blk = self.capture.small_blocks[bs]
        off_seq, off_cuq, off_cuk, off_plan, _ = small_block_layout(bs)
        return B200Metadata(
            cu_seqlens_k=blk[off_cuk : off_cuk + bs + 1],
            cu_seqlens_q=blk[off_cuq : off_cuq + bs + 1],
            cache_seqlens=blk[off_seq : off_seq + bs],
            max_seqlen_k=max_k,
            max_seqlen_q=1,
            page_table=self.capture.page_table[:bs, :],
            decode_plan=blk[off_plan : off_plan + plan_ints(bs)],
            small_block=blk,
            bs=bs,
        )

    def _refresh_capture(self, live: B200Metadata, bs: int) -> None:
        assert self.capture is not None
        self.capture.small_blocks[bs].copy_(live.small_block)
        w = live.page_table.shape[1]
        self.capture.page_table[:bs, :w].copy_(live.page_table)

    def prepare_for_capture(self, batch) -> None:
        bs = batch.size
        if self.capture is None or bs not in self.capture_bs:
            raise AssertionError(f"batch size {bs} was not registered for capture")
        self.prepare_metadata(batch)  # dummy batch: seq_len 1 everywhere
        self._refresh_capture(batch.attn_metadata, bs)
        batch.attn_metadata = self._bind_capture(bs, self.capture.page_table.shape[1])

    def prepare_for_replay(self, batch) -> None:
        md, bs = batch.attn_metadata, batch.padded_size
        if not isinstance(md, B200Metadata) or self.capture is None or bs not in self.capture_bs:
            raise AssertionError("prepare_for_replay: batch was not prepared for a captured size")
        self._refresh_capture(md, bs)
