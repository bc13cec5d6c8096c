"""The attention event trace without a GPU: decoding of hand-built trace buffers (header, counts, overflow, several
launches), every summary quantity on a timeline with known answers, the Chrome / Perfetto export, and the
argument checks of b200_attn_trace_set through the C ABI with fake device addresses."""
import ctypes as C
import importlib
import json

import numpy as np
import pytest
import torch

tr = importlib.import_module("mini-sglang_b200.trace")


def _region(phase, grid, warps, epw, events, counts=None, seq=0, box_rows=64, flags=0):
    """One region as the kernels write it; events: {(cta, warp): [(ns, code, arg), ...]}."""
    hdr = dict(magic=tr.MAGIC, version=tr.VERSION, phase=phase, grid=grid, threads=warps * 32, warps=warps, bs=3,
               hq=16, hkv=8, group=2, page_size=64, box_rows=box_rows, events_per_warp=epw, plan_kind=0, seq=seq,
               flags=flags)
    buf = bytearray(tr.region_bytes(grid, warps, epw))
    buf[:64] = np.array([hdr[f] for f in tr.HEADER_FIELDS], dtype="<u4").tobytes()
    cnt = np.zeros((grid, warps), dtype="<u4")
    recs = np.zeros((grid, warps, epw), dtype=tr.RECORD_DTYPE)
    for (c, w), evs in events.items():
        cnt[c, w] = len(evs)
        for i, (ns, code, arg) in enumerate(evs[:epw]):
            recs[c, w, i] = (ns, ns * 2 & 0xFFFFFFFF, code, w, arg)
    if counts is not None:
        for k, v in counts.items():
            cnt[k] = v
    buf[64:64 + cnt.nbytes] = cnt.tobytes()
    off = 64 + (grid * warps * 4 + 15) // 16 * 16
    buf[off:off + recs.nbytes] = recs.tobytes()
    return bytes(buf)


def _decode_timeline():
    """Two CTAs of a box-mode decode launch (10 warps) with known waits, tiles and units:
    CTA 0 on SM 7: begin 0, K producer issues tiles at 100 and 300 (waited 50 for the second), consumer warp 4 runs
    one unit of two tiles (K-full waits of 60 and 40, V-full waits of 10 and 20, last PV at 420), end 500.
    CTA 1 on SM 9: begin 10, one tile issued at 150, PV at 200, end 300."""
    ev = {
        (0, 0): [(0, tr.BEGIN, 7), (20, tr.UNIT_BEGIN, 0), (40, tr.EMPTY_WAIT, 0), (40, tr.EMPTY_DONE, 0),
                 (100, tr.ISSUED, 0), (200, tr.EMPTY_WAIT, 1), (250, tr.EMPTY_DONE, 1), (300, tr.ISSUED, 1),
                 (310, tr.UNIT_END, 0), (500, tr.END, 0)],
        (0, 4): [(5, tr.BEGIN, 7), (100, tr.UNIT_BEGIN, 0), (160, tr.K_FULL, 0), (170, tr.QK, 0),
                 (180, tr.SOFTMAX, 0), (190, tr.V_FULL, 0), (200, tr.PV, 0), (240, tr.K_FULL, 1), (250, tr.QK, 1),
                 (260, tr.SOFTMAX, 1), (280, tr.V_FULL, 1), (420, tr.PV, 1), (430, tr.EPI_BEGIN, 0),
                 (440, tr.EPI_END, 0), (450, tr.UNIT_END, 0), (499, tr.END, 0)],
        (1, 0): [(10, tr.BEGIN, 9), (20, tr.UNIT_BEGIN, 0), (30, tr.EMPTY_WAIT, 0), (30, tr.EMPTY_DONE, 0),
                 (150, tr.ISSUED, 0), (160, tr.UNIT_END, 0), (300, tr.END, 0)],
        (1, 4): [(10, tr.BEGIN, 9), (20, tr.UNIT_BEGIN, 0), (160, tr.K_FULL, 0), (170, tr.QK, 0),
                 (180, tr.SOFTMAX, 0), (190, tr.V_FULL, 0), (200, tr.PV, 0), (210, tr.UNIT_END, 0), (290, tr.END, 0)],
    }
    return _region(0, 2, 10, 32, ev)


def test_decode_header_counts_and_events():
    (launch,) = tr.decode_buffer(_decode_timeline())
    assert launch.phase == "decode" and launch.header["grid"] == 2 and launch.header["warps"] == 10
    assert launch.header["events_per_warp"] == 32 and not launch.overflow
    assert launch.counts[0, 4] == 16 and launch.counts[1, 0] == 7 and launch.counts[0, 9] == 0
    w = launch.warp_events(0, 4)
    assert w["ns"].tolist()[:3] == [5, 100, 160] and w["code"][0] == tr.BEGIN and w["arg"][0] == 7
    assert (w["warp"] == 4).all() and (w["cta"] == 0).all()
    assert len(launch.events) == 10 + 16 + 7 + 9


def test_overflow_is_counted_not_recorded():
    evs = {(0, 1): [(i, tr.ISSUED, i) for i in range(10)]}
    (launch,) = tr.decode_buffer(_region(1, 1, 12, 4, evs))
    assert launch.phase == "prefill" and launch.overflow
    assert launch.counts[0, 1] == 10
    assert launch.warp_events(0, 1)["arg"].tolist() == [0, 1, 2, 3]


def test_several_launches_then_an_unwritten_region():
    a = _region(0, 2, 10, 8, {(0, 0): [(1, tr.BEGIN, 3)]}, seq=0)
    b = _region(1, 3, 12, 16, {(2, 5): [(2, tr.BEGIN, 4), (3, tr.END, 0)]}, seq=1)
    unwritten = bytes(len(a))
    launches = tr.decode_buffer(a + b + unwritten)
    assert [l.phase for l in launches] == ["decode", "prefill"]
    assert [l.header["seq"] for l in launches] == [0, 1]
    assert launches[1].warp_events(2, 5)["ns"].tolist() == [2, 3]
    assert tr.decode_buffer(a + b + unwritten, max_launches=1)[0].header["seq"] == 0


def test_bad_version_and_truncated_region_are_errors():
    a = bytearray(_region(0, 1, 10, 4, {}))
    a[4:8] = np.array([99], dtype="<u4").tobytes()
    with pytest.raises(ValueError, match="version"):
        tr.decode_buffer(bytes(a))
    with pytest.raises(ValueError, match="past the buffer"):
        tr.decode_buffer(_region(0, 1, 10, 4, {})[:-16])


def test_summary_on_a_known_timeline():
    (launch,) = tr.decode_buffer(_decode_timeline())
    s = tr.summarise(launch, alg_bytes=1000.0, flops=500.0)
    assert s["span_ns"] == 500
    assert s["cta_busy_ns"] == [500, 290]
    assert s["cta_end_ns"] == [500, 300]
    assert s["cta_idle_end_ns"] == [0, 200]
    assert s["imbalance"] == pytest.approx(500 / 400)
    assert s["prologue_ns"] == [100, 140]
    assert s["drain_ns"] == [500 - 420, 300 - 200]
    assert s["tiles_per_cta"] == [2, 1] and s["units_per_cta"] == [1, 1]
    # producer K: busy 500 + 290 ns, waited 50 ns for an empty slot
    assert s["wait_fraction"]["producer_k"]["empty"] == pytest.approx(50 / 790)
    # consumer: busy 494 + 280; K-full waits 60 + 40 + 140, V-full 10 + 20 + 10
    c = s["wait_fraction"]["consumer"]
    assert c["k_full"] == pytest.approx(240 / 774) and c["v_full"] == pytest.approx(40 / 774)
    assert s["bytes_per_s"] == pytest.approx(1000 / 500e-9) and s["flop_per_s"] == pytest.approx(500 / 500e-9)
    assert not s["overflow"] and s["phase"] == "decode"


def test_roles_of_warps():
    box = {"phase": 0, "box_rows": 64}
    row = {"phase": 0, "box_rows": 0}
    assert [tr.role_of(box, w) for w in range(10)] == ["producer_k", "producer_v", "idle", "idle"] + ["consumer"] * 4 + [
        "q_loader", "combiner"]
    assert [tr.role_of(row, w) for w in range(4)] == ["producer_k"] * 2 + ["producer_v"] * 2
    pf = {"phase": 1, "box_rows": 64}
    assert [tr.role_of(pf, w) for w in range(12)] == ["producer_kq", "producer_v", "idle", "idle"] + [
        "consumer_wg0"] * 4 + ["consumer_wg1"] * 4


def test_chrome_trace_export(tmp_path):
    launches = tr.decode_buffer(_decode_timeline())
    path = tmp_path / "t.json"
    tr.to_chrome_trace(launches, path)
    obj = json.loads(path.read_text())
    evs = obj["traceEvents"]
    procs = {e["args"]["name"] for e in evs if e["ph"] == "M" and e["name"] == "process_name"}
    assert procs == {"SM 7", "SM 9"}
    threads = {(e["pid"], e["args"]["name"]) for e in evs if e["ph"] == "M" and e["name"] == "thread_name"}
    assert threads == {(7, "warp 0 producer_k"), (7, "warp 4 consumer"), (9, "warp 0 producer_k"),
                       (9, "warp 4 consumer")}
    slices = [e for e in evs if e["ph"] == "X"]
    unit = [e for e in slices if e["name"] == "unit 0" and e["pid"] == 7 and e["tid"] == 4]
    assert len(unit) == 1 and unit[0]["ts"] == pytest.approx(0.1) and unit[0]["dur"] == pytest.approx(0.35)
    waits = [e for e in slices if e["name"].startswith("wait empty") and e["pid"] == 7]
    assert [w["dur"] for w in waits] == [pytest.approx(0.0), pytest.approx(0.05)]
    assert all(e["ts"] >= 0 for e in evs if "ts" in e)


# ------------------------------------------------------------------------------------------ C ABI checks
cpu_only = pytest.mark.skipif(torch.cuda.is_available(), reason="fake device pointers: CPU-only test")
FAKE = 1 << 32  # 16-byte aligned, never dereferenced by the host


@cpu_only
@pytest.mark.parametrize("ptr,nbytes,epw,words", [
    (FAKE, 1 << 30, 0, "events_per_warp must be > 0"),
    (FAKE, 1 << 30, -3, "events_per_warp must be > 0"),
    (FAKE + 8, 1 << 30, 64, "16-byte aligned"),
    (FAKE, "short", 64, "smaller than one launch region"),
])
def test_trace_set_rejects_bad_arguments(b200, native_lib, ptr, nbytes, epw, words):
    if nbytes == "short":
        nbytes = native_lib.b200_attn_trace_launch_bytes(0, epw) - 1
    launches = native_lib.b200_launch_count()
    assert native_lib.b200_attn_trace_set(ptr, nbytes, epw) != 0
    assert words in native_lib.b200_last_error().decode()
    assert native_lib.b200_launch_count() == launches


@cpu_only
def test_trace_set_register_and_unregister(b200, native_lib):
    one = native_lib.b200_attn_trace_launch_bytes(0, 64)
    try:
        assert native_lib.b200_attn_trace_set(FAKE, one, 64) == 0
        t, u = C.c_uint64(7), C.c_uint64(7)
        assert native_lib.b200_attn_trace_launches(C.byref(t), C.byref(u)) == 0
        assert (t.value, u.value) == (0, 0)
    finally:
        assert native_lib.b200_attn_trace_set(None, 0, 0) == 0
    assert native_lib.b200_attn_trace_launches(None, None) != 0


def test_launch_bytes_match_the_python_layout(b200, native_lib):
    for phase, warps in ((0, 10), (1, 12)):
        nb = native_lib.b200_attn_trace_launch_bytes(phase, 100)
        grid = None  # the device's SM count: recovered from the size
        for g in range(1, 1025):
            if tr.region_bytes(g, warps, 100) == nb:
                grid = g
                break
        assert grid is not None, (phase, nb)
        assert native_lib.b200_attn_trace_launch_bytes(phase, 200) == tr.region_bytes(grid, warps, 200)
    assert native_lib.b200_attn_trace_launch_bytes(2, 100) == 0
    assert native_lib.b200_attn_trace_launch_bytes(0, 0) == 0
