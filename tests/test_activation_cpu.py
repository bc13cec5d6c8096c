"""The gated-MLP activation (``b200_silu_and_mul`` / ``ops.silu_and_mul``) without a GPU: every bad argument is
refused before anything is launched, and ``flashinfer.silu_and_mul`` is re-bound and restored with the other
FlashInfer elementwise entry points (the GPU tests pin the bits)."""
import ctypes
import sys
from types import ModuleType

import pytest
import torch

from refsite import minisgl_ref  # noqa: F401  (fixture)

BF16, FP16 = 0, 1


@pytest.fixture
def buf():
    raw = (ctypes.c_char * 4096)()
    return ctypes.addressof(raw) // 16 * 16 + 16, raw  # 16-byte aligned host address (never dereferenced)


@pytest.mark.parametrize(
    "case, args, msg",
    [
        ("dtype", dict(dtype=2), b"bad dtype"),
        ("d = 0", dict(d=0), b"[1, 2^30]"),
        ("d too large", dict(d=(1 << 30) + 1, x_rs=1 << 32, o_rs=1 << 31), b"[1, 2^30]"),
        ("negative rows", dict(rows=-1), b"negative row count"),
        ("x stride < 2d", dict(x_rs=63), b"row strides"),
        ("out stride < d", dict(o_rs=31), b"row strides"),
        ("odd out pointer", dict(out_off=1), b"aligned"),
        ("odd x pointer", dict(x_off=1), b"aligned"),
    ],
)
def test_abi_refuses_before_any_launch(native_lib, buf, case, args, msg):
    p, _ = buf
    a = dict(dtype=BF16, d=32, rows=4, x_rs=64, o_rs=32, out_off=0, x_off=0)
    a.update(args)
    before = native_lib.b200_launch_count()
    rc = native_lib.b200_silu_and_mul(p + a["out_off"], a["o_rs"], p + a["x_off"], a["x_rs"], a["rows"], a["d"],
                                      a["dtype"], None)
    assert rc != 0, case
    assert msg in native_lib.b200_last_error(), (case, native_lib.b200_last_error())
    assert native_lib.b200_launch_count() == before, case


def test_abi_zero_rows_launch_nothing(native_lib, buf):
    p, _ = buf
    before = native_lib.b200_launch_count()
    for d, off in ((8, 0), (7, 2)):  # vector and scalar shapes alike
        assert native_lib.b200_silu_and_mul(p + off, d, p, 2 * d, 0, d, FP16, None) == 0
    assert native_lib.b200_launch_count() == before


def test_op_refusals(b200, native_lib):
    x = torch.zeros(4, 64, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        b200.ops.silu_and_mul(x)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        b200.ops.silu_and_mul(x, out=torch.empty(4, 32, dtype=torch.bfloat16))


def _flashinfer_stub(monkeypatch):
    fi = ModuleType("flashinfer")
    for name in ("rmsnorm", "fused_add_rmsnorm", "apply_rope_with_cos_sin_cache_inplace", "silu_and_mul",
                 "gelu_and_mul"):
        setattr(fi, name, lambda *a, _n=name, **k: ("flashinfer", _n))
    monkeypatch.setitem(sys.modules, "flashinfer", fi)
    return fi


def test_patch_and_restore_round_trip(b200, monkeypatch):
    fi = _flashinfer_stub(monkeypatch)
    originals = dict(vars(fi))
    assert b200.layers.patch_flashinfer_entry_points() == 4
    assert fi.silu_and_mul is b200.ops.silu_and_mul
    assert fi.rmsnorm is b200.ops.rmsnorm
    assert fi.gelu_and_mul is originals["gelu_and_mul"]  # no registered model uses it: left alone
    assert b200.layers.patch_flashinfer_entry_points() == 4  # a second patch keeps the true originals
    b200.layers.restore_flashinfer_entry_points()
    assert {k: v for k, v in vars(fi).items()} == originals


def test_the_reference_mlp_activation_reaches_the_patched_name(b200, minisgl_ref, monkeypatch):
    """``minisgl.layers.activation.silu_and_mul`` imports ``flashinfer.silu_and_mul`` at every call, so the
    gated MLP runs whatever the name is bound to at that moment."""
    fi = _flashinfer_stub(monkeypatch)
    from minisgl.layers.activation import silu_and_mul as ref_silu_and_mul

    seen = []
    monkeypatch.setattr(b200.ops, "silu_and_mul", lambda x, out=None, enable_pdl=None: seen.append((x, out)) or "ours")
    x = torch.zeros(2, 8)
    assert ref_silu_and_mul(x) == ("flashinfer", "silu_and_mul")
    b200.layers.patch_flashinfer_entry_points()
    try:
        assert ref_silu_and_mul(x) == "ours" and seen == [(x, None)]
    finally:
        b200.layers.restore_flashinfer_entry_points()
    assert ref_silu_and_mul(x) == ("flashinfer", "silu_and_mul")


@pytest.mark.parametrize("norm_rope", [True, False])
def test_install_binds_the_activation_with_norm_rope(b200, minisgl_ref, monkeypatch, norm_rope):
    fi = _flashinfer_stub(monkeypatch)
    original = fi.silu_and_mul
    import minisgl.engine.engine as ref_engine

    ref_engine.create_model = lambda config: object()  # the module is dropped after the test
    try:
        assert b200.layers.install_into_minisgl(norm_rope=norm_rope, row_gather=False, attention=True)
        ref_engine.create_model(None)
        assert (fi.silu_and_mul is b200.ops.silu_and_mul) == norm_rope
        assert (fi.silu_and_mul is original) != norm_rope
    finally:
        b200.layers.restore_flashinfer_entry_points()
    assert fi.silu_and_mul is original
