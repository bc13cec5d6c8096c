"""Argument validation of the three attention entry points (b200_attn_decode, b200_attn_decode_fused,
b200_attn_prefill) and the option table, through the C ABI with fake device addresses.

Every malformed call must return non-zero before it reaches the GPU, with an error that names the problem.
Without a device a call whose arguments all pass fails later with some other error (the tensor map or launch
cannot be made), so a check that went missing shows up here as a wrong message.  With a device the fake
addresses could reach a kernel, so the file only runs where there is none."""
import os

import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="fake device pointers: CPU-only test")

BRINGUP = os.environ.get("B200_BUILD_BRINGUP", "0") not in ("", "0")
BS, HQ, HKV, D = 4, 16, 8, 128
QKV_RS = (HQ + 2 * HKV) * D  # q / k / v as row-strided views of one qkv buffer


def _addr(i):
    """Distinct 16-byte aligned fake device addresses; the library never dereferences them on the host."""
    return (1 << 32) + i * (1 << 20)


def _decode_args(native_lib, fused):
    a = dict(q=_addr(0), q_rs=QKV_RS, k=_addr(1), k_rs=QKV_RS, v=_addr(2), v_rs=QKV_RS,
             k_cache=_addr(3), v_cache=_addr(4), num_slots=4096, page_size=16, out_loc=_addr(5),
             slot_table=_addr(6), st_stride=256, seq_lens=_addr(7), plan=_addr(8), bs=BS, hq=HQ, hkv=HKV,
             head_dim=D, scale=D ** -0.5, out=_addr(9), workspace=_addr(10),
             ws_bytes=native_lib.b200_attn_workspace_bytes(BS, HQ, D), dtype=0, stream=None)
    if fused:
        a.update(qw=_addr(11), kw=_addr(12), eps=1e-6, positions=_addr(13), cos_sin=_addr(14))
    return a


def _prefill_args(native_lib):
    return dict(q=_addr(0), q_rs=QKV_RS, k=_addr(1), k_rs=QKV_RS, v=_addr(2), v_rs=QKV_RS, k_cache=_addr(3),
                v_cache=_addr(4), num_slots=4096, page_size=16, out_loc=_addr(5), slot_table=_addr(6),
                st_stride=256, seq_lens=_addr(7), cu_q=_addr(8), plan=_addr(9), bs=BS, nnz=64, max_q=16, hq=HQ,
                hkv=HKV, head_dim=D, scale=D ** -0.5, out=_addr(10), workspace=None, ws_bytes=0, dtype=0,
                stream=None)


def _call(native_lib, phase, a):
    if phase == "decode":
        return native_lib.b200_attn_decode(
            a["q"], a["q_rs"], a["k"], a["k_rs"], a["v"], a["v_rs"], a["k_cache"], a["v_cache"], a["num_slots"],
            a["page_size"], a["out_loc"], a["slot_table"], a["st_stride"], a["seq_lens"], a["plan"], a["bs"],
            a["hq"], a["hkv"], a["head_dim"], a["scale"], a["out"], a["workspace"], a["ws_bytes"], a["dtype"],
            a["stream"])
    if phase == "fused":
        return native_lib.b200_attn_decode_fused(
            a["q"], a["q_rs"], a["k"], a["k_rs"], a["v"], a["v_rs"], a["qw"], a["kw"], a["eps"], a["positions"],
            a["cos_sin"], a["k_cache"], a["v_cache"], a["num_slots"], a["page_size"], a["out_loc"],
            a["slot_table"], a["st_stride"], a["seq_lens"], a["plan"], a["bs"], a["hq"], a["hkv"], a["head_dim"],
            a["scale"], a["out"], a["workspace"], a["ws_bytes"], a["dtype"], a["stream"])
    return native_lib.b200_attn_prefill(
        a["q"], a["q_rs"], a["k"], a["k_rs"], a["v"], a["v_rs"], a["k_cache"], a["v_cache"], a["num_slots"],
        a["page_size"], a["out_loc"], a["slot_table"], a["st_stride"], a["seq_lens"], a["cu_q"], a["plan"],
        a["bs"], a["nnz"], a["max_q"], a["hq"], a["hkv"], a["head_dim"], a["scale"], a["out"], a["workspace"],
        a["ws_bytes"], a["dtype"], a["stream"])


def _args(native_lib, phase):
    return _prefill_args(native_lib) if phase == "prefill" else _decode_args(native_lib, phase == "fused")


# (change to the well-formed call, words the error must contain)
COMMON = {
    "head_dim": ({"head_dim": 64}, "head_dim must be 128"),
    "hq_not_multiple_of_hkv": ({"hkv": 6}, "bad bs/hq/hkv"),
    "bs_zero": ({"bs": 0}, "bad bs/hq/hkv"),
    "q_stride": ({"q_rs": QKV_RS + 4}, "multiples of 8"),
    "k_stride": ({"k_rs": QKV_RS + 4, "v_rs": QKV_RS + 4}, "multiples of 8"),
    **{f"misaligned_{n}": ({n: _addr(20) + 8}, "16-byte aligned") for n in ("q", "k", "v", "k_cache", "v_cache", "out")},
    "num_slots_zero": ({"num_slots": 0}, "num_slots"),
    "num_slots_2p31": ({"num_slots": 1 << 31}, "num_slots"),
    "slot_table_stride": ({"st_stride": 258}, "slot table rows"),
    "slot_table_misaligned": ({"slot_table": _addr(20) + 4}, "slot table rows"),
    "dtype": ({"dtype": 2}, "bad dtype"),
}
DECODE = {
    "workspace_too_small": ({"ws_bytes": "short"}, "workspace too small"),
    "null_plan": ({"plan": None}, "decode_plan is NULL"),
    "page_size_zero": ({"page_size": 0}, "page_size"),
}
FUSED = {
    "null_positions": ({"positions": None}, "must not be NULL"),
    "null_cos_sin": ({"cos_sin": None}, "must not be NULL"),
    "misaligned_q_weight": ({"qw": _addr(20) + 2}, "16-byte aligned"),
    "misaligned_k_weight": ({"kw": _addr(20) + 2}, "16-byte aligned"),
    "misaligned_cos_sin": ({"cos_sin": _addr(20) + 4}, "16-byte aligned"),
}
PREFILL = {
    "k_v_strides_differ": ({"v_rs": QKV_RS + 8}, "share a row stride"),
    "nnz_below_bs": ({"nnz": BS - 1}, "max_seqlen_q/nnz"),
    "max_q_zero": ({"max_q": 0}, "max_seqlen_q/nnz"),
}
CASES = ([("decode", n, *c) for n, c in {**COMMON, **DECODE}.items()]
         + [("fused", n, *c) for n, c in {**COMMON, **DECODE, **FUSED}.items()]
         + [("prefill", n, *c) for n, c in {**COMMON, **PREFILL}.items()])
ALL_WORDS = sorted({w for *_, w in CASES} | {"prefill_plan", "attn_decode:", "attn_prefill:"})


@pytest.mark.parametrize("phase,name,change,words", CASES, ids=[f"{p}-{n}" for p, n, *_ in CASES])
def test_malformed_call_is_rejected(b200, native_lib, phase, name, change, words):
    a = _args(native_lib, phase)
    a.update(change)
    if a.get("ws_bytes") == "short":
        a["ws_bytes"] = native_lib.b200_attn_workspace_bytes(BS, HQ, D) - 1
    launches = native_lib.b200_launch_count()
    assert _call(native_lib, phase, a) != 0
    err = native_lib.b200_last_error().decode()
    assert words in err, f"{name}: {err!r}"
    assert native_lib.b200_launch_count() == launches


def test_prefill_without_plan_is_refused_in_a_product_build(b200, native_lib):
    if BRINGUP:
        pytest.skip("a NULL plan selects the mma.sync bring-up kernel in this build")
    a = _args(native_lib, "prefill")
    a["plan"] = None
    assert _call(native_lib, "prefill", a) != 0
    assert "prefill_plan" in native_lib.b200_last_error().decode()
    assert native_lib.b200_launch_count() == 0


@pytest.mark.parametrize("phase", ["decode", "fused", "prefill"])
def test_well_formed_call_passes_every_check(b200, native_lib, phase):
    """The reference call of the cases above is accepted by every argument check; only the missing device stops
    it, so each case above fails because of its own change."""
    assert _call(native_lib, phase, _args(native_lib, phase)) != 0
    err = native_lib.b200_last_error().decode()
    assert not any(w in err for w in ALL_WORDS), err
    assert native_lib.b200_launch_count() == 0


OPTION_DEFAULTS = {
    "use_pdl": 1, "decode_impl": 1, "prefill_impl": 1, "prefill_order": 0, "prefill_skip_append": 0,
    "decode_plan_target": 2, "decode_plan_nosplit": 75, "decode_fused_combine": 1, "decode_early_kv": 1,
    "decode_exact_tail": 1,
}


def test_every_option_round_trips_its_default(b200, native_lib):
    for name, default in OPTION_DEFAULTS.items():
        assert native_lib.b200_set_option(name.encode(), default) == default, name
        assert native_lib.b200_set_option(name.encode(), default + 7) == default, name
        assert native_lib.b200_set_option(name.encode(), default) == default + 7, name
    assert native_lib.b200_set_option(b"no_such_option", 1) == -1
    assert native_lib.b200_set_option(None, 1) == -1
    assert native_lib.b200_set_option(b"use_pdl_", 1) == -1
    if not BRINGUP:
        for name in ("decode_impl", "prefill_impl"):
            assert native_lib.b200_set_option(name.encode(), 0) == -1
            assert native_lib.b200_set_option(name.encode(), 1) == 1
