"""CPU-only tests of the host side: the C-ABI library loads and exports every symbol the header
declares (no compute calls without a GPU), argument validation surfaces as RuntimeError, the
registry / factory / interface mirrors behave like the reference's, and the pure-host part of
prepare_metadata is correct."""
import ctypes
import re
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent


def _header_symbols():
    text = (ROOT / "include" / "b200attn.h").read_text()
    return sorted(set(re.findall(r"B200_API\s+[\w\s\*]+?\b(b200_\w+)\s*\(", text)))


def test_library_exports_every_declared_symbol(b200, native_lib):
    declared = _header_symbols()
    assert len(declared) >= 15
    for name in declared:
        assert hasattr(native_lib, name), f"{name} declared in include/b200attn.h but not exported"
    # the ctypes prototypes cover exactly the header
    assert sorted(b200._cabi.SIGNATURES) == declared


def test_abi_version_and_helpers(b200, native_lib):
    assert native_lib.b200_abi_version() == b200._cabi.ABI_VERSION
    assert native_lib.b200_decode_plan_ints(256) == 4 + 257 + 16 * 256
    assert native_lib.b200_attn_workspace_bytes(256, 16, 128) > 256 * 16 * 16 * 128 * 4
    assert native_lib.b200_launch_count() == 0  # nothing was launched on this CPU box
    prev = b200._cabi.set_option("decode_plan_target", 3)
    assert b200._cabi.set_option("decode_plan_target", prev) == 3
    # the cross-check kernels (cp.async decode, mma.sync prefill) are not in the product build
    import os

    if os.environ.get("B200_BUILD_BRINGUP", "0") in ("", "0"):
        for name in ("decode_impl", "prefill_impl"):
            with pytest.raises(RuntimeError):
                b200._cabi.set_option(name, 0)
            assert b200._cabi.set_option(name, 1) == 1
    with pytest.raises(RuntimeError):
        b200._cabi.set_option("no_such_option", 1)


def test_workspace_counters_never_overlap_partials(native_lib):
    """ADVICE r1: with odd bs*hq the arrival counters (placed at floor256(size) - ceil256(bs*hq*4) by
    b200_attn_decode) used to overlap the last (m, l) partials.  Both regions are now 256-aligned."""
    for bs, hq in [(257, 7), (1, 1), (3, 5), (255, 3), (256, 16), (129, 9)]:
        total = native_lib.b200_attn_workspace_bytes(bs, hq, 128)
        items = bs * 16 * hq
        partials_end = items * 128 * 4 + items * 2 * 4
        counters_start = total // 256 * 256 - (bs * hq * 4 + 255) // 256 * 256
        assert counters_start >= partials_end, (bs, hq, counters_start, partials_end)


def test_build_digest_is_embedded(b200, native_lib):
    from importlib import import_module

    build = import_module("mini-sglang_b200.build")
    assert native_lib.b200_build_digest().decode() == build.built_digest() != ""


def test_allreduce_host_api_validates(b200, native_lib):
    """Set-up half of the all-reduce ABI needs no GPU: region sizing and communicator creation."""
    assert native_lib.b200_ar_region_bytes(8, 1 << 20) >= 2 * 8 * (1 << 20) + 8 * 128 * 4
    bases = (ctypes.c_void_p * 2)(0x1000, 0x2000)
    opened = (ctypes.c_int * 2)(0, 0)
    comm = ctypes.c_void_p()
    assert native_lib.b200_ar_create(0, 2, bases, opened, 1000, ctypes.byref(comm)) == 0
    assert native_lib.b200_ar_max_bytes(comm) == 1024  # rounded up to 256
    # message larger than the slot, NULL communicator, residual without weight: rejected before any launch
    buf = (ctypes.c_char * 64)()
    p = ctypes.addressof(buf) // 16 * 16
    assert native_lib.b200_ar_allreduce(comm, p, 1024, p, 1024, None, 0, None, 4, 1024, 0.0, 0, None) != 0
    assert b"exceeds" in native_lib.b200_last_error()
    assert native_lib.b200_ar_allreduce(None, p, 8, p, 8, None, 0, None, 1, 8, 0.0, 0, None) != 0
    assert native_lib.b200_ar_allreduce(comm, p, 8, p, 8, p, 8, None, 1, 8, 0.0, 0, None) != 0
    assert native_lib.b200_ar_destroy(comm, 0) == 0
    assert native_lib.b200_ar_create(2, 2, bases, opened, 1000, ctypes.byref(comm)) != 0
    assert native_lib.b200_ar_create(0, 9, bases, opened, 1000, ctypes.byref(comm)) != 0


def test_argument_validation_returns_error_not_crash(b200, native_lib):
    """Bad arguments are rejected before any CUDA call (mirrors TensorMatcher -> RuntimeError)."""
    buf = (ctypes.c_char * 64)()
    p = ctypes.addressof(buf)
    rc = native_lib.b200_store_kv(p, p, 32, p, p, 32, p, 0, 1, 24, None)  # row_bytes not /16
    assert rc != 0 and b"multiple of 16" in native_lib.b200_last_error()
    with pytest.raises(b200._cabi.B200NativeError, match="multiple of 16"):
        b200._cabi.check(rc, "b200_store_kv")
    rc = native_lib.b200_rmsnorm(p, p, p, 1, 1, 12, 16, 0, 16, 0, 1e-6, 0, None)  # dim % 8
    assert rc != 0
    rc = native_lib.b200_attn_decode(p, 8, p, 8, p, 8, p, p, 16, 1, p, p, 8, p, p, 1, 16, 8, 64, 0.1, p, p, 0, 0, None)
    assert rc != 0 and b"head_dim" in native_lib.b200_last_error()


def test_ops_refuse_cpu_tensors(b200, native_lib):
    x = torch.zeros(4, 128, dtype=torch.bfloat16)
    w = torch.ones(128, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        b200.ops.rmsnorm(x, w, 1e-6)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        b200.ops.store_cache(x, x, torch.zeros(1, dtype=torch.int32), x[:1], x[:1])


def test_backend_has_no_cpu_path(b200):
    ctx = b200.Context(16)
    b200.set_global_ctx(ctx)
    ctx.kv_cache = SimpleNamespace(device=torch.device("cpu"), dtype=torch.bfloat16)
    ctx.page_table = torch.zeros((2, 64), dtype=torch.int32)
    cfg = SimpleNamespace(num_qo_heads=16, num_kv_heads=8, head_dim=128)
    backend = b200.create_attention_backend("b200", cfg)
    batch = b200.Batch([b200.Req(table_idx=0, cached_len=3, device_len=4)], "decode")
    with pytest.raises(RuntimeError, match="no CPU path"):
        backend.prepare_metadata(batch)
    with pytest.raises(RuntimeError):
        backend.forward(torch.zeros(1, 16, 128), torch.zeros(1, 1024), torch.zeros(1, 1024), 0, batch)
    with pytest.raises(RuntimeError, match="head_dim 128"):
        b200.create_attention_backend("b200", SimpleNamespace(num_qo_heads=8, num_kv_heads=8, head_dim=64))


def test_registry_and_factory_follow_the_reference(b200):
    reg = b200.SUPPORTED_ATTENTION_BACKENDS
    assert "b200" in reg.supported_names()
    with pytest.raises(KeyError):
        reg.register("b200")(lambda cfg: None)  # duplicate name (utils/registry.py:11-13)
    with pytest.raises(Exception):
        b200.attention.validate_attn_backend("nope")
    with pytest.raises(AssertionError):
        b200.attention.validate_attn_backend("auto", allow_auto=False)
    ctx = b200.Context(1)
    b200.set_global_ctx(ctx)
    ctx.kv_cache = SimpleNamespace(device=torch.device("cpu"), dtype=torch.bfloat16)
    cfg = SimpleNamespace(num_qo_heads=16, num_kv_heads=8, head_dim=128)
    single = b200.create_attention_backend("b200,b200", cfg)  # same name twice -> single backend
    assert isinstance(single, b200.B200AttnBackend)
    with pytest.raises(AssertionError):
        b200.create_attention_backend("b200,b200,b200", cfg)


def test_hybrid_backend_routes_by_phase(b200):
    calls = []

    class Fake(b200.attention.BaseAttnBackend):
        def __init__(self, name):
            self.name = name

        def forward(self, q, k, v, layer_id, batch):
            calls.append((self.name, "forward"))

        def prepare_metadata(self, batch):
            calls.append((self.name, "meta"))

        def init_capture_graph(self, max_seq_len, bs_list):
            calls.append((self.name, "init"))

        def prepare_for_capture(self, batch):
            calls.append((self.name, "cap"))

        def prepare_for_replay(self, batch):
            calls.append((self.name, "replay"))

    h = b200.attention.HybridBackend(Fake("p"), Fake("d"))
    pre = b200.Batch([b200.Req(table_idx=0, cached_len=0, device_len=4)], "prefill")
    dec = b200.Batch([b200.Req(table_idx=0, cached_len=4, device_len=5)], "decode")
    h.prepare_metadata(pre), h.forward(None, None, None, 0, pre)
    h.prepare_metadata(dec), h.forward(None, None, None, 0, dec)
    h.init_capture_graph(64, [1]), h.prepare_for_capture(dec), h.prepare_for_replay(dec)
    assert calls == [("p", "meta"), ("p", "forward"), ("d", "meta"), ("d", "forward"),
                     ("d", "init"), ("d", "cap"), ("d", "replay")]


def test_req_batch_context_invariants(b200):
    with pytest.raises(ValueError):
        b200.Req(table_idx=0, cached_len=4, device_len=4)  # cached_len < device_len (core.py:42)
    r = b200.Req(table_idx=3, cached_len=0, device_len=7, max_device_len=9)
    assert r.extend_len == 7 and r.remain_len == 2 and r.can_decode
    r.complete_one()
    assert (r.cached_len, r.device_len, r.extend_len) == (7, 8, 1)
    b = b200.Batch([r], "decode")
    assert b.is_decode and not b.is_prefill and b.size == b.padded_size == 1
    with pytest.raises(ValueError):
        b200.Batch([r], "train")
    ctx = b200.Context(16)
    with pytest.raises(AssertionError):
        _ = ctx.batch
    with ctx.forward_batch(b):
        assert ctx.batch is b
        with pytest.raises(AssertionError):
            with ctx.forward_batch(b):
                pass
    b200.set_global_ctx(ctx)
    with pytest.raises(AssertionError):
        b200.set_global_ctx(b200.Context(1))  # already set (core.py:128-131)


def test_div_even_and_tp_info(b200):
    u = b200.utils
    assert u.div_even(16, 4) == 4 and u.div_even(8, 16, allow_replicate=True) == 1
    with pytest.raises(AssertionError):
        u.div_even(8, 16)
    with pytest.raises(AssertionError):
        u.div_even(8, 3)
    assert u.get_tp_info().size == 1
    u.set_tp_info(1, 4)
    try:
        assert u.get_tp_info().rank == 1 and not u.get_tp_info().is_primary()
    finally:
        u.set_tp_info(0, 1)


def test_host_req_info_and_block_layout(b200):
    be = b200.attention.backend
    reqs = [b200.Req(table_idx=5, cached_len=0, device_len=9), b200.Req(table_idx=2, cached_len=30, device_len=31)]
    flat, max_q, max_k = be.host_req_info(reqs)
    assert flat == [5, 0, 9, 2, 30, 31] and (max_q, max_k) == (9, 31)
    for bs in (1, 3, 8, 255, 256):
        o_seq, o_q, o_k, o_plan, total = be.small_block_layout(bs)
        assert o_seq == 0 and o_q >= bs and o_k >= o_q + bs + 1 and o_plan >= o_k + bs + 1
        assert all(x % 4 == 0 for x in (o_q, o_k, o_plan, total))  # 16-byte aligned sections
        assert total >= o_plan + be.plan_ints(bs)


def test_rotary_cache_matches_oracle(b200):
    from oracle import rope as o_rope

    emb = b200.layers.RotaryEmbedding(128, 128, 512, 1e6)
    assert torch.equal(emb._cos_sin_cache, o_rope.ref_cos_sin_cache(128, 512, 1e6))
    with pytest.raises(AssertionError):
        b200.layers.RotaryEmbedding(128, 64, 512, 1e6)
