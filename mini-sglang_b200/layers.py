"""The layers that feed attention, with the reference's class and method names
(``python/minisgl/layers/norm.py``, ``rotary.py``, ``attention.py``), bound to the sm_90a kernels.

Two ways to use them:

* stand-alone (tests, ``bench.py``): construct ``RMSNorm`` / ``RotaryEmbedding`` / ``AttentionLayer``
  directly;
* inside mini-sglang: :func:`patch_minisgl_layers` re-binds the kernel attributes the reference's
  layer objects already hold (``RMSNorm.rmsnorm`` norm.py:14, ``RMSNormFused.{rmsnorm,
  fused_add_rmsnorm}`` norm.py:29-30, ``RotaryEmbedding.apply_rope_with_cos_sin_cache_inplace``
  rotary.py:35-37), and :func:`patch_minisgl_attention` re-binds ``forward`` of the reference's
  ``AttentionLayer`` to :func:`attention_forward`, the same code our ``AttentionLayer`` runs -- zero
  edits to the reference.
"""

from __future__ import annotations

import functools
import math
from typing import Any, Callable, Dict, Optional, Tuple

import torch

from . import ops
from .attention.backend import B200AttnBackend
from .attention.base import HybridBackend
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

    ``fuse_pre_attention=True`` runs :func:`attention_forward`: decode batches run norm + RoPE + KV append +
    attention as ONE launch (``b200_attn_decode_fused``); prefill batches run the norm+RoPE sequence as a
    single fused launch (``b200_qknorm_rope_inplace``) in front of the attention launch.  Results are
    bit-identical to the reference's three-launch sequence followed by attention.
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
        if self.fuse_pre_attention:
            return attention_forward(self, qkv)
        ctx = get_global_ctx()
        q, k, v = qkv.split([self.qo_attn_dim, self.kv_attn_dim, self.kv_attn_dim], dim=-1)
        if self.q_norm is not None:
            self.q_norm.forward_inplace(q.view(-1, self.num_qo_heads, self.head_dim))
        if self.k_norm is not None:
            self.k_norm.forward_inplace(k.view(-1, self.num_kv_heads, self.head_dim))
        q, k = self.rotary.forward(ctx.batch.positions, q, k)
        q = q.view(-1, self.num_qo_heads, self.head_dim)
        o = ctx.attn_backend.forward(q, k, v, self.layer_id, ctx.batch)
        return o.view(-1, self.qo_attn_dim)


def serving_attn_backend(backend: Any, batch: Any) -> Any:
    """The backend that runs ``batch``: a ``HybridBackend`` (``--attn p,d``) hands prefill batches to its
    ``prefill_backend`` and every other batch to its ``decode_backend`` (reference attention/base.py:45-50)."""
    if isinstance(backend, HybridBackend):
        return backend.prefill_backend if batch.is_prefill else backend.decode_backend
    return backend


def attention_forward(
    layer: Any, qkv: torch.Tensor, unfused: Optional[Callable[[torch.Tensor], torch.Tensor]] = None
) -> torch.Tensor:
    """``AttentionLayer.forward`` with the pre-attention work fused into the sm_90a launches, for our
    :class:`AttentionLayer` and for the reference's (``layer`` needs ``layer_id``, ``head_dim``,
    ``num_qo_heads``, ``num_kv_heads``, ``qo_attn_dim``, ``kv_attn_dim``, ``rotary._cos_sin_cache`` and
    ``q_norm`` / ``k_norm`` with ``.weight`` and ``.eps``, or None).

    When the backend serving this batch is a :class:`B200AttnBackend`, a decode batch with int32 positions
    runs q-norm + k-norm + RoPE + KV append + attention as ONE launch (``forward_decode_fused``) and every
    other batch runs ``ops.qknorm_rope_inplace`` (one launch) and then the backend's ``forward``.  Results are
    bit-identical to the reference's three-launch sequence followed by attention.  With any other backend
    ``unfused(qkv)`` is returned when given; without it the fused norm + RoPE launch feeds that backend."""
    ctx = get_global_ctx()
    batch = ctx.batch
    backend = serving_attn_backend(ctx.attn_backend, batch)
    is_b200 = isinstance(backend, B200AttnBackend)
    if unfused is not None and not is_b200:
        return unfused(qkv)
    q, k, v = qkv.split([layer.qo_attn_dim, layer.kv_attn_dim, layer.kv_attn_dim], dim=-1)
    q_norm, k_norm = layer.q_norm, layer.k_norm
    eps = q_norm.eps if q_norm is not None else (k_norm.eps if k_norm is not None else 0.0)
    q_weight = q_norm.weight if q_norm is not None else None
    k_weight = k_norm.weight if k_norm is not None else None
    cos_sin_cache = layer.rotary._cos_sin_cache
    if is_b200 and batch.is_decode and batch.positions.dtype == torch.int32:
        # decode: norm + RoPE + append + attention are ONE launch (q / k stay raw in memory)
        o = backend.forward_decode_fused(
            q.view(-1, layer.num_qo_heads, layer.head_dim), k, v, layer.layer_id, batch, batch.positions,
            cos_sin_cache, q_weight, k_weight, eps,
        )
        return o.view(-1, layer.qo_attn_dim)
    ops.qknorm_rope_inplace(batch.positions, q, k, layer.head_dim, cos_sin_cache, q_weight, k_weight, eps)
    o = backend.forward(q.view(-1, layer.num_qo_heads, layer.head_dim), k, v, layer.layer_id, batch)
    return o.view(-1, layer.qo_attn_dim)


def _walk(model: Any):
    """Every object reachable from ``model`` (any object graph of ``BaseOP``s), each once; the children of an
    object are read after the caller has seen it."""
    seen = set()
    stack = [model]
    while stack:
        obj = stack.pop()
        if id(obj) in seen or isinstance(obj, (torch.Tensor, str, bytes, int, float)):
            continue
        seen.add(id(obj))
        yield obj
        children = []
        if isinstance(obj, (list, tuple)):
            children = list(obj)
        elif isinstance(obj, dict):
            children = list(obj.values())
        elif hasattr(obj, "__dict__"):
            children = [c for c in vars(obj).values() if not callable(c) or hasattr(c, "__dict__")]
        stack.extend(children)


def patch_minisgl_layers(model: Any) -> int:
    """Re-bind the kernel attributes of every reference norm / rotary layer found under ``model``
    (any object graph of ``BaseOP``s) to the sm_90a ops.  Returns the number of re-bound layers."""
    count = 0
    for obj in _walk(model):
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
    return count


def patch_minisgl_attention(model: Any) -> int:
    """Re-bind ``forward`` of every reference ``minisgl.layers.attention.AttentionLayer`` found under ``model``
    to :func:`attention_forward`, so that with ``attention_backend="b200"`` (alone or as either half of a
    hybrid) a decode step is ONE launch per layer (q-norm, k-norm, RoPE, KV append, attention) and a prefill
    forward two (fused q/k-norm + RoPE, attention) instead of four and three.  Batches served by any other
    backend go to the layer's original ``forward``, unchanged.  Zero edits to the reference: the original bound
    method is kept on the instance as ``_b200_unfused_forward``.  Idempotent.  Returns the number of attention
    layers that run :func:`attention_forward` afterwards (0 when the reference is not importable).

    Patch before the decode graphs are captured (``install_into_minisgl`` does); on an engine that already
    exists, only eager forwards change."""
    try:
        from minisgl.layers.attention import AttentionLayer as RefAttentionLayer
    except ImportError:
        return 0
    count = 0
    for obj in _walk(model):
        if not isinstance(obj, RefAttentionLayer):
            continue
        if "_b200_unfused_forward" not in vars(obj):
            unfused = obj.forward
            obj._b200_unfused_forward = unfused
            obj.forward = functools.partial(attention_forward, obj, unfused=unfused)
        count += 1
    return count


_FLASHINFER_SAVED: Dict[str, Callable] = {}


def patch_flashinfer_entry_points() -> int:
    """Point the FlashInfer elementwise entry points ``flashinfer.rmsnorm`` / ``fused_add_rmsnorm`` /
    ``apply_rope_with_cos_sin_cache_inplace`` / ``silu_and_mul`` at the sm_90a ops.  The reference's layers
    import the norm / rotary names from the ``flashinfer`` package inside ``__init__`` (layers/norm.py:10,25,
    layers/rotary.py:35) and ``silu_and_mul`` at every call (layers/activation.py:9-13, the gated MLP of every
    dense model), so calling this BEFORE the model is built (``LLM(...)`` / ``Engine(...)``) makes every norm /
    rotary layer and every MLP activation run our kernels -- including inside the decode CUDA graphs, which are
    captured during ``Engine.__init__`` (engine/engine.py:100, engine/graph.py:105-141; re-binding layer
    attributes afterwards only affects eager forwards).  Returns the number of re-bound names;
    :func:`restore_flashinfer_entry_points` undoes it."""
    import flashinfer

    table = {
        "rmsnorm": ops.rmsnorm,
        "fused_add_rmsnorm": ops.fused_add_rmsnorm,
        "apply_rope_with_cos_sin_cache_inplace": ops.apply_rope_with_cos_sin_cache_inplace,
        "silu_and_mul": ops.silu_and_mul,
    }
    for name, fn in table.items():
        _FLASHINFER_SAVED.setdefault(name, getattr(flashinfer, name))
        setattr(flashinfer, name, fn)
    return len(table)


def install_into_minisgl(norm_rope: bool = True, row_gather: bool = True, attention: bool = True) -> bool:
    """One call, before ``LLM(...)`` / ``Engine(...)``: makes the reference build its model with the sm_90a
    norm / RoPE / MLP-activation kernels, fuse the pre-attention work of its attention layers into the b200
    launches and use the sm_90a row gather, with zero edits to the reference.

    ``Engine.__init__`` asserts that CUDA is not initialised yet (engine/engine.py:31) and importing
    ``flashinfer`` initialises it, so the FlashInfer names cannot be re-bound up front.  Instead the module
    attribute ``minisgl.engine.engine.create_model`` (engine.py:12, called at engine.py:50-51 after the device
    is set and before the decode graphs are captured at engine.py:100) is wrapped: the wrapper re-binds the
    FlashInfer elementwise entry points (:func:`patch_flashinfer_entry_points`, ``norm_rope``: RMSNorm, RoPE
    and the gated MLP's SiLU-and-mul; with ``norm_rope=False`` all of them stay FlashInfer's), calls the
    reference's own ``create_model`` and re-binds ``forward`` of the model's attention layers (:func:`patch_minisgl_attention`,
    ``attention``).  So with ``attention_backend="b200"`` every decode step inside the engine's CUDA graphs is
    ONE launch per layer (q-norm + k-norm + RoPE + KV append + attention); layers whose batch another backend
    serves keep their own forward.  Returns False when the reference is not importable."""
    try:
        import minisgl.engine.engine as ref_engine
    except ImportError:
        return False
    if row_gather:
        patch_minisgl_kernels()
    if (norm_rope or attention) and not getattr(ref_engine.create_model, "_b200_wrapped", False):
        real_create_model = ref_engine.create_model

        def create_model_with_b200_layers(*args, **kwargs):
            if norm_rope:
                patch_flashinfer_entry_points()
            model = real_create_model(*args, **kwargs)
            if attention:
                patch_minisgl_attention(model)
            return model

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
