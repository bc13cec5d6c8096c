"""mini-sglang_b200 -- H100-native (sm_90a) paged-attention backend for mini-sglang.

Holds only what the attention hot path needs (SURVEY.md section 8):

* ``csrc/``       hand-written CUDA kernels + the C ABI (``include/b200attn.h``) -> libb200attn.so
* ``_cabi``       ctypes binding (fails loudly if the library is missing; no CPU fallback)
* ``ops``         operator-level host API (store_cache, rmsnorm, fused_add_rmsnorm, rope, ...)
* ``attention``   ``B200AttnBackend`` behind the reference's ``BaseAttnBackend`` interface
* ``distributed`` one-shot NVLink all-reduce behind the reference's ``DistributedCommunicator`` plug-in point
* ``kvcache`` / ``layers`` / ``core`` / ``utils``  interface mirrors of the reference types the
  boundary touches, for use where the reference is not installed

The directory name is not a Python identifier: import it with
``importlib.import_module("mini-sglang_b200")`` or through the ``minisgl_b200`` shim package.
"""

from . import _cabi, attention, core, distributed, kvcache, layers, ops, utils  # noqa: F401
from .attention import (  # noqa: F401
    BACKEND_NAME,
    SUPPORTED_ATTENTION_BACKENDS,
    create_attention_backend,
)
from .attention.backend import B200AttnBackend, B200Metadata  # noqa: F401
from .build import build as build_native  # noqa: F401
from .core import Batch, Context, Req, get_global_ctx, set_global_ctx  # noqa: F401
from .kvcache import MHAKVCache  # noqa: F401

__all__ = [
    "B200AttnBackend",
    "B200Metadata",
    "BACKEND_NAME",
    "Batch",
    "Context",
    "MHAKVCache",
    "Req",
    "SUPPORTED_ATTENTION_BACKENDS",
    "attention",
    "build_native",
    "core",
    "create_attention_backend",
    "distributed",
    "get_global_ctx",
    "kvcache",
    "layers",
    "ops",
    "set_global_ctx",
    "utils",
]
