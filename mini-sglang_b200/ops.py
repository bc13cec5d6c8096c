"""Operator-level host API: the functions the reference's layers call, same names and argument
meaning, backed by the sm_90a kernels through the C ABI.

=====================================================  =====================================
reference call site                                     function here
=====================================================  =====================================
``minisgl.kernel.store_cache`` (kernel/store.py:30)      :func:`store_cache`
``minisgl.kernel.indexing`` (kernel/index.py:32)         :func:`indexing`
``flashinfer.rmsnorm`` (layers/norm.py:10,16-21)         :func:`rmsnorm`
``flashinfer.fused_add_rmsnorm`` (layers/norm.py:25,36)  :func:`fused_add_rmsnorm`
``flashinfer.apply_rope_with_cos_sin_cache_inplace``     :func:`apply_rope_with_cos_sin_cache_inplace`
(layers/rotary.py:35,45-51)
(the three pre-attention launches, attention.py:50-54)   :func:`qknorm_rope_inplace`
``flashinfer.silu_and_mul`` (layers/activation.py:9-13)   :func:`silu_and_mul`
=====================================================  =====================================

Tensors are borrowed (``data_ptr``), work is enqueued on ``torch.cuda.current_stream()`` and
nothing synchronises.  CPU tensors raise -- there is no fallback.
"""

from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import _cabi

_DTYPE_CODE = {torch.bfloat16: 0, torch.float16: 1}


def _stream_ptr(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def _require_cuda(*ts: torch.Tensor) -> None:
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError(
                "mini-sglang_b200 ops need CUDA tensors (sm_90a kernels; no CPU fallback)"
            )


def _dtype_code(t: torch.Tensor) -> int:
    try:
        return _DTYPE_CODE[t.dtype]
    except KeyError:
        raise RuntimeError(f"unsupported dtype {t.dtype}; expected bfloat16 or float16") from None


def store_cache(
    k_cache: torch.Tensor,
    v_cache: torch.Tensor,
    indices: torch.Tensor,
    k: torch.Tensor,
    v: torch.Tensor,
) -> None:
    """``k_cache[indices[t]] = k[t]; v_cache[indices[t]] = v[t]`` (reference kernel/store.py:30-42).

    ``k_cache``/``v_cache``: ``[slots, ...]`` with contiguous rows; ``k``/``v``: ``[n, row]`` row-strided
    views sharing one stride; ``indices``: int32 or int64 ``[n]``."""
    _require_cuda(k_cache, v_cache, indices, k, v)
    slots = k_cache.shape[0]
    kc = k_cache.view(slots, -1)
    vc = v_cache.view(slots, -1)
    n = indices.shape[0]
    k2 = k.view(n, -1) if k.dim() != 2 else k
    v2 = v.view(n, -1) if v.dim() != 2 else v
    if not (kc.stride(1) == 1 and vc.stride(1) == 1 and k2.stride(1) == 1 and v2.stride(1) == 1):
        raise RuntimeError("store_cache: innermost dimension must be contiguous")
    if kc.shape != vc.shape or kc.stride(0) != vc.stride(0):
        raise RuntimeError("store_cache: k_cache / v_cache shape or stride mismatch")
    if k2.shape != v2.shape or k2.stride(0) != v2.stride(0) or k2.shape[1] != kc.shape[1]:
        raise RuntimeError("store_cache: k / v shape or stride mismatch")
    if k2.dtype != kc.dtype or v2.dtype != kc.dtype:
        raise RuntimeError("store_cache: dtype mismatch between inputs and cache")
    if indices.dtype not in (torch.int32, torch.int64) or indices.dim() != 1 or not indices.is_contiguous():
        raise RuntimeError("store_cache: indices must be a contiguous int32/int64 vector")
    es = kc.element_size()
    lib = _cabi.load()
    _cabi.check(
        lib.b200_store_kv(
            kc.data_ptr(),
            vc.data_ptr(),
            kc.stride(0) * es,
            k2.data_ptr(),
            v2.data_ptr(),
            k2.stride(0) * es,
            indices.data_ptr(),
            1 if indices.dtype == torch.int64 else 0,
            n,
            kc.shape[1] * es,
            _stream_ptr(kc),
        ),
        "b200_store_kv",
    )


def indexing(
    weights: torch.Tensor,
    indices: torch.Tensor,
    *,
    output: Optional[torch.Tensor] = None,
    vocab_range: Optional[Tuple[int, int]] = None,  # (start, length)
) -> torch.Tensor:
    """``output[t] = weights[indices[t]]`` -- the reference's ``indexing`` (kernel/index.py:32-53), used
    by ``VocabParallelEmbedding.forward`` (layers/embedding.py:31-41).  With ``vocab_range = (start,
    length)`` rows whose ``indices[t] - start`` falls outside ``[0, length)`` are zero (the TP-sharded
    vocabulary).  ``weights``: ``[rows, dim]`` with contiguous rows (row stride free); ``indices``:
    int32 / int64 ``[n]``.  Also serves the last-token gather ``x[indices].contiguous()``
    (layers/embedding.py:92-94)."""
    _require_cuda(weights, indices, output)
    if weights.dim() != 2 or weights.stride(1) != 1:
        raise RuntimeError("indexing: weights must be 2-D with a contiguous last dimension")
    if indices.dtype not in (torch.int32, torch.int64) or indices.dim() != 1 or not indices.is_contiguous():
        raise RuntimeError("indexing: indices must be a contiguous int32/int64 vector")
    n = indices.shape[0]
    if output is None:
        output = weights.new_empty(n, weights.shape[1])
    if output.shape != (n, weights.shape[1]) or output.dtype != weights.dtype or output.stride(1) != 1:
        raise RuntimeError("indexing: output must be [len(indices), dim] of the weights' dtype")
    es = weights.element_size()
    start, length = (0, -1) if vocab_range is None else (int(vocab_range[0]), int(vocab_range[1]))
    if vocab_range is not None and (length < 0 or length > weights.shape[0]):
        raise RuntimeError("indexing: vocab_range length must lie in [0, rows of weights]")
    _cabi.check(
        _cabi.load().b200_index_rows(
            weights.data_ptr(), weights.stride(0) * es, indices.data_ptr(),
            1 if indices.dtype == torch.int64 else 0, n, weights.shape[1] * es, output.data_ptr(),
            output.stride(0) * es, start, length, _stream_ptr(weights),
        ),
        "b200_index_rows",
    )
    return output


def rmsnorm(
    x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6, out: Optional[torch.Tensor] = None
) -> torch.Tensor:
    """``flashinfer.rmsnorm`` semantics: 2-D ``[rows, dim]`` or 3-D ``[rows, heads, dim]`` (per-head
    norm over the last dim); ``out`` may alias ``x`` (reference layers/norm.py:16-21)."""
    _require_cuda(x, weight, out)
    if out is None:
        out = torch.empty_like(x, memory_format=torch.contiguous_format)
    if x.dim() == 2:
        rows, dim = x.shape
        heads, xhs, ohs = 1, 0, 0
        xrs, ors = x.stride(0), out.stride(0)
    elif x.dim() == 3:
        rows, heads, dim = x.shape
        xrs, xhs = x.stride(0), x.stride(1)
        ors, ohs = out.stride(0), out.stride(1)
    else:
        raise RuntimeError(f"rmsnorm: expected 2-D or 3-D input, got {x.dim()}-D")
    if x.stride(-1) != 1 or out.stride(-1) != 1 or out.shape != x.shape:
        raise RuntimeError("rmsnorm: last dim must be contiguous and out must match x")
    if weight.shape != (dim,) or weight.dtype != x.dtype or not weight.is_contiguous():
        raise RuntimeError("rmsnorm: weight must be a contiguous [dim] tensor of x's dtype")
    lib = _cabi.load()
    _cabi.check(
        lib.b200_rmsnorm(
            out.data_ptr(), x.data_ptr(), weight.data_ptr(), rows, heads, dim, xrs, xhs, ors, ohs,
            float(eps), _dtype_code(x), _stream_ptr(x),
        ),
        "b200_rmsnorm",
    )
    return out


def fused_add_rmsnorm(
    x: torch.Tensor, residual: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6
) -> None:
    """``flashinfer.fused_add_rmsnorm`` semantics, both in place (reference layers/norm.py:32-38)."""
    _require_cuda(x, residual, weight)
    if x.dim() != 2 or residual.shape != x.shape or x.stride(1) != 1 or residual.stride(1) != 1:
        raise RuntimeError("fused_add_rmsnorm: x / residual must be matching 2-D row-major tensors")
    rows, dim = x.shape
    if weight.shape != (dim,) or weight.dtype != x.dtype or residual.dtype != x.dtype:
        raise RuntimeError("fused_add_rmsnorm: dtype / shape mismatch")
    lib = _cabi.load()
    _cabi.check(
        lib.b200_fused_add_rmsnorm(
            x.data_ptr(), residual.data_ptr(), weight.data_ptr(), rows, dim, x.stride(0),
            residual.stride(0), float(eps), _dtype_code(x), _stream_ptr(x),
        ),
        "b200_fused_add_rmsnorm",
    )


def silu_and_mul(
    input: torch.Tensor, out: Optional[torch.Tensor] = None, enable_pdl: Optional[bool] = None
) -> torch.Tensor:
    """``flashinfer.silu_and_mul`` semantics and signature (reference layers/activation.py:9-13):
    ``silu(input[..., :d]) * input[..., d:]`` for ``input`` of shape ``(..., 2d)``, bit for bit what FlashInfer
    computes.  Any ``d >= 1`` and any leading dims whose rows are evenly strided; the last dim must be
    contiguous.  ``out`` (shape ``(..., d)``, same dtype) may be row-strided.  ``enable_pdl`` is accepted for
    signature compatibility: like every kernel of this library, the launch uses programmatic dependent launch
    unless the library option ``use_pdl`` is 0."""
    _require_cuda(input, out)
    if input.dim() < 1 or input.shape[-1] % 2:
        raise RuntimeError(f"silu_and_mul: last dim must be even, got shape {tuple(input.shape)}")
    d = input.shape[-1] // 2
    if out is None:
        out = torch.empty(input.shape[:-1] + (d,), device=input.device, dtype=input.dtype)
    elif out.shape != input.shape[:-1] + (d,) or out.dtype != input.dtype or out.device != input.device:
        raise RuntimeError(f"silu_and_mul: out must be {tuple(input.shape[:-1]) + (d,)} of {input.dtype}")
    if out.numel() == 0:
        return out
    if input.stride(-1) != 1 or out.stride(-1) != 1:
        raise RuntimeError("silu_and_mul: the last dim of input and out must be contiguous")
    try:
        x2, o2 = input.view(-1, 2 * d), out.view(-1, d)
    except RuntimeError:
        raise RuntimeError("silu_and_mul: the leading dims of input / out must collapse to one row stride") from None
    rows = x2.shape[0]
    xrs = x2.stride(0) if rows > 1 else 2 * d  # the stride of a single row is never used
    ors = o2.stride(0) if rows > 1 else d
    _cabi.check(
        _cabi.load().b200_silu_and_mul(
            o2.data_ptr(), ors, x2.data_ptr(), xrs, rows, d, _dtype_code(input), _stream_ptr(input)
        ),
        "b200_silu_and_mul",
    )
    return out


def _qk_views(query: torch.Tensor, key: torch.Tensor, head_size: int):
    nnz = query.shape[0]
    if query.stride(-1) != 1 or key.stride(-1) != 1:
        raise RuntimeError("rope: last dim of query / key must be contiguous")
    q2 = query.reshape(nnz, -1) if query.dim() == 3 and query.stride(1) == head_size else query
    k2 = key.reshape(nnz, -1) if key.dim() == 3 and key.stride(1) == head_size else key
    if q2.dim() != 2 or k2.dim() != 2:
        raise RuntimeError("rope: query / key must be [nnz, H*D] (or [nnz, H, D] with dense heads)")
    if q2.shape[1] % head_size or k2.shape[1] % head_size:
        raise RuntimeError("rope: hidden size not a multiple of head_size")
    return nnz, q2, k2, q2.shape[1] // head_size, k2.shape[1] // head_size


def apply_rope_with_cos_sin_cache_inplace(
    positions: torch.Tensor,
    query: torch.Tensor,
    key: torch.Tensor,
    head_size: int,
    cos_sin_cache: torch.Tensor,
    is_neox: bool = True,
) -> None:
    """Same keyword signature as the FlashInfer op the reference binds (layers/rotary.py:45-51)."""
    if not is_neox:
        raise RuntimeError("only neox-style RoPE is implemented (the reference never uses another)")
    _require_cuda(positions, query, key, cos_sin_cache)
    nnz, q2, k2, hq, hkv = _qk_views(query, key, head_size)
    if cos_sin_cache.dtype != torch.float32 or cos_sin_cache.shape[-1] != head_size:
        raise RuntimeError("rope: cos_sin_cache must be fp32 [max_pos, head_size]")
    if positions.dtype not in (torch.int32, torch.int64) or positions.numel() != nnz:
        raise RuntimeError("rope: positions must be int32/int64 [nnz]")
    lib = _cabi.load()
    _cabi.check(
        lib.b200_rope_neox_inplace(
            q2.data_ptr(), k2.data_ptr(), positions.data_ptr(),
            1 if positions.dtype == torch.int64 else 0, cos_sin_cache.data_ptr(), nnz, hq, hkv,
            head_size, q2.stride(0), k2.stride(0), _dtype_code(q2), _stream_ptr(q2),
        ),
        "b200_rope_neox_inplace",
    )


def qknorm_rope_inplace(
    positions: torch.Tensor,
    query: torch.Tensor,
    key: torch.Tensor,
    head_size: int,
    cos_sin_cache: torch.Tensor,
    q_weight: Optional[torch.Tensor],
    k_weight: Optional[torch.Tensor],
    eps: float,
) -> None:
    """One launch for q-norm + k-norm + RoPE (reference layers/attention.py:50-54, three launches)."""
    _require_cuda(positions, query, key, cos_sin_cache, q_weight, k_weight)
    nnz, q2, k2, hq, hkv = _qk_views(query, key, head_size)
    lib = _cabi.load()
    _cabi.check(
        lib.b200_qknorm_rope_inplace(
            q2.data_ptr(), k2.data_ptr(),
            q_weight.data_ptr() if q_weight is not None else None,
            k_weight.data_ptr() if k_weight is not None else None,
            float(eps), positions.data_ptr(), 1 if positions.dtype == torch.int64 else 0,
            cos_sin_cache.data_ptr(), nnz, hq, hkv, head_size, q2.stride(0), k2.stride(0),
            _dtype_code(q2), _stream_ptr(q2),
        ),
        "b200_qknorm_rope_inplace",
    )
