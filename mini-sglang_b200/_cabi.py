"""ctypes binding of libb200attn.so (the C ABI declared in ``include/b200attn.h``).

The product path fails loudly when the native library is missing or the device is not
sm_90: there is no CPU or PyTorch fallback anywhere below this module.
"""

from __future__ import annotations

import ctypes as C
import os
from pathlib import Path
from typing import Optional

_LIB: Optional[C.CDLL] = None
LIB_PATH = Path(__file__).resolve().parent / "libb200attn.so"

ABI_VERSION = 9

_i32, _i64, _f32, _vp, _sz = C.c_int, C.c_int64, C.c_float, C.c_void_p, C.c_size_t

# name -> (restype, argtypes); mirrors include/b200attn.h one to one
SIGNATURES = {
    "b200_abi_version": (_i32, []),
    "b200_build_digest": (C.c_char_p, []),
    "b200_last_error": (C.c_char_p, []),
    "b200_launch_count": (C.c_uint64, []),
    "b200_device_supported": (_i32, []),
    "b200_set_option": (_i32, [C.c_char_p, _i32]),
    "b200_store_kv": (_i32, [_vp, _vp, _i64, _vp, _vp, _i64, _vp, _i32, _i64, _i64, _vp]),
    "b200_index_rows": (_i32, [_vp, _i64, _vp, _i32, _i64, _i64, _vp, _i64, _i64, _i64, _vp]),
    "b200_rmsnorm": (
        _i32,
        [_vp, _vp, _vp, _i64, _i32, _i32, _i64, _i64, _i64, _i64, _f32, _i32, _vp],
    ),
    "b200_fused_add_rmsnorm": (_i32, [_vp, _vp, _vp, _i64, _i32, _i64, _i64, _f32, _i32, _vp]),
    "b200_rope_neox_inplace": (
        _i32,
        [_vp, _vp, _vp, _i32, _vp, _i64, _i32, _i32, _i32, _i64, _i64, _i32, _vp],
    ),
    "b200_qknorm_rope_inplace": (
        _i32,
        [_vp, _vp, _vp, _vp, _f32, _vp, _i32, _vp, _i64, _i32, _i32, _i32, _i64, _i64, _i32, _vp],
    ),
    "b200_silu_and_mul": (_i32, [_vp, _i64, _vp, _i64, _i64, _i32, _i32, _vp]),
    "b200_decode_plan_ints": (_sz, [_i32]),
    "b200_build_prefill_plan": (_i32, [_vp, _i32, _vp, _i32, _vp]),
    "b200_build_metadata": (
        _i32,
        [_vp, _i32, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _i32, _vp, _i32, _i32, _vp],
    ),
    "b200_attn_workspace_bytes": (_sz, [_i32, _i32, _i32]),
    "b200_attn_decode": (
        _i32,
        [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _i64, _i32, _vp, _vp, _i64, _vp, _vp]
        + [_i32, _i32, _i32, _i32, _f32, _vp, _vp, _sz, _i32, _vp],
    ),
    "b200_attn_decode_fused": (
        _i32,
        [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _f32, _vp, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _i64, _vp, _vp]
        + [_i32, _i32, _i32, _i32, _f32, _vp, _vp, _sz, _i32, _vp],
    ),
    "b200_attn_prefill": (
        _i32,
        [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _i64, _i32, _vp, _vp, _i64, _vp, _vp, _vp]
        + [_i32, _i64, _i32, _i32, _i32, _i32, _f32, _vp, _vp, _sz, _i32, _vp],
    ),
    "b200_attn_trace_set": (_i32, [_vp, _sz, _i32]),
    "b200_attn_trace_launch_bytes": (_sz, [_i32, _i32]),
    "b200_attn_trace_launches": (_i32, [C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "b200_ar_region_bytes": (_sz, [_i32, _sz]),
    "b200_ar_alloc": (_i32, [_sz, C.POINTER(_vp)]),
    "b200_ar_ipc_handle": (_i32, [_vp, _vp]),
    "b200_ar_ipc_open": (_i32, [_vp, C.POINTER(_vp)]),
    "b200_ar_create": (_i32, [_i32, _i32, C.POINTER(_vp), C.POINTER(_i32), _sz, C.POINTER(_vp)]),
    "b200_ar_destroy": (_i32, [_vp, _i32]),
    "b200_ar_max_bytes": (_sz, [_vp]),
    "b200_ar_allreduce": (_i32, [_vp, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _f32, _i32, _vp]),
}


class B200NativeError(RuntimeError):
    """Raised for every non-zero return of the C ABI (reference: PanicError -> RuntimeError)."""


def load(path: Optional[os.PathLike] = None) -> C.CDLL:
    """dlopen the library (once) and attach prototypes. Raises if it has not been built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    p = Path(path) if path is not None else LIB_PATH
    if not p.exists():
        raise B200NativeError(
            f"{p} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback for the attention path)"
        )
    lib = C.CDLL(str(p))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here == missing export
        fn.restype = res
        fn.argtypes = args
    got = lib.b200_abi_version()
    if got != ABI_VERSION:
        raise B200NativeError(f"libb200attn ABI {got} != expected {ABI_VERSION}; rebuild")
    _LIB = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().b200_last_error().decode(errors="replace")
        raise B200NativeError(f"{what} failed (rc={rc}): {msg}")


def set_option(name: str, value: int) -> int:
    """Debug knob, e.g. set_option("decode_impl", 0) selects the cp.async decode kernel."""
    prev = load().b200_set_option(name.encode(), int(value))
    if prev < 0:
        raise B200NativeError(f"unknown option {name!r}")
    return prev


def launch_count() -> int:
    return int(load().b200_launch_count())
