"""The layers that feed attention, with the reference's class and method names
(``python/minisgl/layers/norm.py``, ``rotary.py``, ``attention.py``), bound to the sm_90a kernels.

Two ways to use them:

* stand-alone (tests, ``bench.py``): construct ``RMSNorm`` / ``RotaryEmbedding`` / ``AttentionLayer``
  directly;
* inside mini-sglang: :func:`patch_minisgl_layers` re-binds the kernel attributes the reference's
  layer objects already hold (``RMSNorm.rmsnorm`` norm.py:14, ``RMSNormFused.{rmsnorm,
  fused_add_rmsnorm}`` norm.py:29-30, ``RotaryEmbedding.apply_rope_with_cos_sin_cache_inplace``
  rotary.py:35-37) -- zero edits to the reference.
"""

from __future__ import annotations

import math
from typing import Any, Callable, Dict, Optional, Tuple

import torch

from . import ops
from .core import get_global_ctx
from .utils import div_even, get_tp_info


class RMSNorm:
    def __init__(self, size: int, eps: float) -> None:
        self.eps = eps
        self.weight = torch.empty(size)
        self.rmsnorm = ops.rmsnorm

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.rmsnorm(x, self.weight, self.eps)

    def forward_inplace(self, x: torch.Tensor) -> None:
        self.rmsnorm(x, self.weight, self.eps, out=x)


class RMSNormFused:
    def __init__(self, size: int, eps: float) -> None:
        self.eps = eps
        self.weight = torch.empty(size)
        self.rmsnorm = ops.rmsnorm
        self.fused_add_rmsnorm = ops.fused_add_rmsnorm

    def forward(
        self, x: torch.Tensor, residual: Optional[torch.Tensor] = None
    ) -> Tuple[torch.Tensor, torch.Tensor]:
        if residual is None:
            return self.rmsnorm(x, self.weight, self.eps), x
        self.fused_add_rmsnorm(x, residual, self.weight, self.eps)
        return x, residual


def make_inv_freq(
    rotary_dim: int, base: float, rope_scaling: Optional[Dict[str, Any]] = None
) -> torch.Tensor:
    """``base**(-2i/D)`` with the llama3 / yarn post-processing of rotary.py:55-114."""
    inv_freq = 1.0 / (base ** (torch.arange(0, rotary_dim, 2, dtype=torch.float) / rotary_dim))
    if rope_scaling is None or rope_scaling.get("rope_type", "default") == "default":
        return inv_freq
    kind = rope_scaling["rope_type"]
    if kind == "llama3":
        factor = rope_scaling["factor"]
        lo, hi = rope_scaling["low_freq_factor"], rope_scaling["high_freq_factor"]
        orig = rope_scaling["original_max_position_embeddings"]
        wave_len = 2 * math.pi / inv_freq
        if lo == hi:
            return torch.where(wave_len < orig / hi, inv_freq, inv_freq / factor)
        smooth = torch.clamp((orig / wave_len - lo) / (hi - lo), 0, 1)
        return ((1 - smooth) / factor + smooth) * inv_freq
    if kind == "yarn":
        factor = rope_scaling["factor"]
        beta_fast = rope_scaling.get("beta_fast", 32.0)
        beta_slow = rope_scaling.get("beta_slow", 1.0)
        orig = rope_scaling["original_max_position_embeddings"]

        def corr(n_rot: float) -> float:
            return rotary_dim * math.log(orig / (n_rot * 2 * math.pi)) / (2 * math.log(base))

        low = max(math.floor(corr(beta_fast)), 0)
        high = min(math.ceil(corr(beta_slow)), rotary_dim // 2 - 1)
        ramp = torch.clamp(
            (torch.arange(rotary_dim // 2, dtype=torch.float32) - low) / max(high - low, 1), 0, 1
        )
        return (inv_freq / factor) * ramp + inv_freq * (1 - ramp)
    raise ValueError(f"Unsupported rope_scaling = {rope_scaling}")


class RotaryEmbedding:
    """fp32 ``[max_pos, D]`` cos|sin cache + in-place neox rotation (rotary.py:12-52)."""

    def __init__(
        self,
        head_size: int,
        rotary_dim: int,
        max_position_embeddings: int,
        base: float,
        rope_scaling: Optional[Dict[str, Any]] = None,
        device: Optional[torch.device] = None,
    ) -> None:
        if rotary_dim != head_size:
            raise AssertionError("partial rotary is not supported (neither in the reference)")
        if head_size not in (64, 128, 256):
            raise AssertionError(f"head_size {head_size} not supported")
        self.head_size = head_size
        inv_freq = make_inv_freq(rotary_dim, base, rope_scaling)
        t = torch.arange(max_position_embeddings, dtype=torch.float)
        freqs = torch.einsum("i,j -> ij", t, inv_freq)
        cache = torch.cat((freqs.cos(), freqs.sin()), dim=-1)
        self._cos_sin_cache = cache.to(device) if device is not None else cache
        self.apply_rope_with_cos_sin_cache_inplace = ops.apply_rope_with_cos_sin_cache_inplace

    def forward(
        self, positions: torch.Tensor, query: torch.Tensor, key: torch.Tensor
    ) -> Tuple[torch.Tensor, torch.Tensor]:
        self.apply_rope_with_cos_sin_cache_inplace(
            positions=positions,
            query=query,
            key=key,
            head_size=self.head_size,
            cos_sin_cache=self._cos_sin_cache,
        )
        return query, key


class AttentionLayer:
    """split -> q/k norm -> RoPE -> ``ctx.attn_backend.forward`` (attention.py:18-57).

    ``fuse_pre_attention=True``: decode batches run norm + RoPE + KV append + attention as ONE launch
    (``b200_attn_decode_fused``); prefill batches run the norm+RoPE sequence as a single fused launch
    (``b200_qknorm_rope_inplace``) in front of the attention launch.  Results are bit-identical to the
    reference's three-launch sequence followed by attention.
    """

    def __init__(
        self,
        layer_id: int,
        num_qo_heads: int,
        num_kv_heads: int,
        head_dim: int,
        rotary: RotaryEmbedding,
        q_norm: Optional[RMSNorm] = None,
        k_norm: Optional[RMSNorm] = None,
        fuse_pre_attention: bool = True,
    ) -> None:
        if num_qo_heads % num_kv_heads != 0:
            raise AssertionError("num_qo_heads must be a multiple of num_kv_heads")
        tp = get_tp_info().size
        self.layer_id = layer_id
        self.head_dim = head_dim
        self.num_qo_heads = div_even(num_qo_heads, tp)
        self.num_kv_heads = div_even(num_kv_heads, tp, allow_replicate=True)
        self.qo_attn_dim = self.num_qo_heads * head_dim
        self.kv_attn_dim = self.num_kv_heads * head_dim
        self.rotary = rotary
        self.q_norm = q_norm
        self.k_norm = k_norm
        self.fuse_pre_attention = fuse_pre_attention

    def forward(self, qkv: torch.Tensor) -> torch.Tensor:
        ctx = get_global_ctx()
        q, k, v = qkv.split([self.qo_attn_dim, self.kv_attn_dim, self.kv_attn_dim], dim=-1)
        eps = self.q_norm.eps if self.q_norm is not None else (
            self.k_norm.eps if self.k_norm is not None else 0.0
        )
        fused_decode = getattr(ctx.attn_backend, "forward_decode_fused", None)
        if (self.fuse_pre_attention and fused_decode is not None and ctx.batch.is_decode
                and ctx.batch.positions.dtype == torch.int32):
            # decode: norm + RoPE + append + attention are ONE launch (q / k stay raw in memory)
            o = fused_decode(
                q.view(-1, self.num_qo_heads, self.head_dim), k, v, self.layer_id, ctx.batch,
                ctx.batch.positions, self.rotary._cos_sin_cache,
                self.q_norm.weight if self.q_norm is not None else None,
                self.k_norm.weight if self.k_norm is not None else None, eps,
            )
            return o.view(-1, self.qo_attn_dim)
        if self.fuse_pre_attention:
            ops.qknorm_rope_inplace(
                ctx.batch.positions, q, k, self.head_dim, self.rotary._cos_sin_cache,
                self.q_norm.weight if self.q_norm is not None else None,
                self.k_norm.weight if self.k_norm is not None else None,
                eps,
            )
        else:
            if self.q_norm is not None:
                self.q_norm.forward_inplace(q.view(-1, self.num_qo_heads, self.head_dim))
            if self.k_norm is not None:
                self.k_norm.forward_inplace(k.view(-1, self.num_kv_heads, self.head_dim))
            q, k = self.rotary.forward(ctx.batch.positions, q, k)
        q = q.view(-1, self.num_qo_heads, self.head_dim)
        o = ctx.attn_backend.forward(q, k, v, self.layer_id, ctx.batch)
        return o.view(-1, self.qo_attn_dim)


def patch_minisgl_layers(model: Any) -> int:
    """Re-bind the kernel attributes of every reference norm / rotary layer found under ``model``
    (any object graph of ``BaseOP``s) to the sm_90a ops.  Returns the number of re-bound layers."""
    seen, count = set(), 0
    stack = [model]
    while stack:
        obj = stack.pop()
        if id(obj) in seen or isinstance(obj, (torch.Tensor, str, bytes, int, float)):
            continue
        seen.add(id(obj))
        hit = False
        if callable(getattr(obj, "fused_add_rmsnorm", None)) and hasattr(obj, "weight"):
            obj.fused_add_rmsnorm = ops.fused_add_rmsnorm
            hit = True
        if callable(getattr(obj, "rmsnorm", None)) and hasattr(obj, "weight"):
            obj.rmsnorm = ops.rmsnorm
            hit = True
        if callable(getattr(obj, "apply_rope_with_cos_sin_cache_inplace", None)) and hasattr(
            obj, "_cos_sin_cache"
        ):
            obj.apply_rope_with_cos_sin_cache_inplace = ops.apply_rope_with_cos_sin_cache_inplace
            hit = True
        count += int(hit)
        children = []
        if isinstance(obj, (list, tuple)):
            children = list(obj)
        elif isinstance(obj, dict):
            children = list(obj.values())
        elif hasattr(obj, "__dict__"):
            children = [c for c in vars(obj).values() if not callable(c) or hasattr(c, "__dict__")]
        stack.extend(children)
    return count


_FLASHINFER_SAVED: Dict[str, Callable] = {}


def patch_flashinfer_entry_points() -> int:
    """Point ``flashinfer.rmsnorm`` / ``fused_add_rmsnorm`` / ``apply_rope_with_cos_sin_cache_inplace``
    at the sm_90a ops.  The reference's layers import these names from the ``flashinfer`` package
    inside ``__init__`` (layers/norm.py:10,25, layers/rotary.py:35), so calling this BEFORE the model is
    built (``LLM(...)`` / ``Engine(...)``) makes every norm / rotary layer bind our kernels -- including
    inside the decode CUDA graphs, which are captured during ``Engine.__init__`` (engine/engine.py:100,
    engine/graph.py:105-141; re-binding layer attributes afterwards only affects eager forwards).
    Returns the number of re-bound names; :func:`restore_flashinfer_entry_points` undoes it."""
    import flashinfer

    table = {
        "rmsnorm": ops.rmsnorm,
        "fused_add_rmsnorm": ops.fused_add_rmsnorm,
        "apply_rope_with_cos_sin_cache_inplace": ops.apply_rope_with_cos_sin_cache_inplace,
    }
    for name, fn in table.items():
        _FLASHINFER_SAVED.setdefault(name, getattr(flashinfer, name))
        setattr(flashinfer, name, fn)
    return len(table)


def install_into_minisgl(norm_rope: bool = True, row_gather: bool = True) -> bool:
    """One call, before ``LLM(...)`` / ``Engine(...)``: makes the reference build its model with the sm_90a
    norm / RoPE kernels and use the sm_90a row gather, with zero edits to the reference.

    ``Engine.__init__`` asserts that CUDA is not initialised yet (engine/engine.py:31) and importing
    ``flashinfer`` initialises it, so the FlashInfer names cannot be re-bound up front.  Instead the module
    attribute ``minisgl.engine.engine.create_model`` (engine.py:12, called at engine.py:50-51 after the device
    is set and before the decode graphs are captured at engine.py:100) is wrapped: the wrapper re-binds the
    FlashInfer entry points (:func:`patch_flashinfer_entry_points`) and then calls the reference's own
    ``create_model``.  Returns False when the reference is not importable."""
    try:
        import minisgl.engine.engine as ref_engine
    except ImportError:
        return False
    if row_gather:
        patch_minisgl_kernels()
    if norm_rope and not getattr(ref_engine.create_model, "_b200_wrapped", False):
        real_create_model = ref_engine.create_model

        def create_model_with_b200_layers(*args, **kwargs):
            patch_flashinfer_entry_points()
            return real_create_model(*args, **kwargs)

        create_model_with_b200_layers._b200_wrapped = True  # type: ignore[attr-defined]
        ref_engine.create_model = create_model_with_b200_layers
    return True


def restore_flashinfer_entry_points() -> None:
    import flashinfer

    for name, fn in _FLASHINFER_SAVED.items():
        setattr(flashinfer, name, fn)
    _FLASHINFER_SAVED.clear()


def patch_minisgl_kernels() -> bool:
    """Point ``minisgl.kernel.indexing`` at the sm_90a row gather.  ``VocabParallelEmbedding.forward``
    imports the function from ``minisgl.kernel`` at call time (reference layers/embedding.py:32-34),
    so re-binding the package attribute is enough; no reference edit.  Returns False when the
    reference package is not importable (nothing to patch)."""
    try:
        import minisgl.kernel as ref_kernel
    except ImportError:
        return False
    ref_kernel.indexing = ops.indexing
    return True
