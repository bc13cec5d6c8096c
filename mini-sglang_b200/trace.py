"""Event timelines of the decode and prefill attention kernels, recorded inside the launches.

``AttentionTrace`` registers a zeroed device buffer with ``b200_attn_trace_set``; while it is registered every
attention launch runs the instrumented instantiation of its kernel, whose warps record timestamped events
(``%globaltimer`` ns, comparable across SMs, and the SM's ``%clock``) into one region of the buffer per launch.
Outputs and launch counts are those of an untraced launch.  ``summarise`` turns one launch into per-CTA and
per-role numbers, ``to_chrome_trace`` writes a timeline that Perfetto or chrome://tracing opens.

A timeline shows when each warp waited and issued work, not what DRAM or the tensor pipe did: a wait share says
how long a role stood at a barrier, not why.  The buffer layout (``csrc/attn.cuh``) is mirrored here.
"""
from __future__ import annotations

import ctypes as C
import json
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import _cabi

MAGIC = 0x52545441
VERSION = 1
PHASES = {0: "decode", 1: "prefill"}
PHASE_IDS = {v: k for k, v in PHASES.items()}
HEADER_FIELDS = ("magic", "version", "phase", "grid", "threads", "warps", "bs", "hq", "hkv", "group", "page_size",
                 "box_rows", "events_per_warp", "plan_kind", "seq", "flags")
HEADER_BYTES = 64
FLAG_FUSED, FLAG_IN_KERNEL_COMBINE, FLAG_EARLY_KV = 1, 2, 4

# event codes (attn.cuh TraceCode)
BEGIN, PDL_WAIT, UNIT_BEGIN, UNIT_END = 1, 2, 3, 4
EMPTY_WAIT, EMPTY_DONE, ISSUED, Q_ISSUED, APPEND = 5, 6, 7, 8, 9
Q_READY, K_FULL, QK, SOFTMAX, V_FULL, PV, SKIP, EPI_BEGIN, EPI_END = 10, 11, 12, 13, 14, 15, 16, 17, 18
ARRIVE, ARRIVE_LAST, MERGE_BEGIN, MERGE_END = 19, 20, 21, 22
END = 31
CODE_NAMES = {BEGIN: "begin", PDL_WAIT: "pdl_wait", UNIT_BEGIN: "unit_begin", UNIT_END: "unit_end",
              EMPTY_WAIT: "empty_wait", EMPTY_DONE: "empty_done", ISSUED: "issued", Q_ISSUED: "q_issued",
              APPEND: "append", Q_READY: "q_ready", K_FULL: "k_full", QK: "qk", SOFTMAX: "softmax",
              V_FULL: "v_full", PV: "pv", SKIP: "skip", EPI_BEGIN: "epilogue_begin", EPI_END: "epilogue_end",
              ARRIVE: "arrive", ARRIVE_LAST: "arrive_last", MERGE_BEGIN: "merge_begin", MERGE_END: "merge_end",
              END: "end"}

RECORD_DTYPE = np.dtype([("ns", "<u8"), ("clock", "<u4"), ("code", "u1"), ("warp", "u1"), ("arg", "<u2")])
EVENT_DTYPE = np.dtype([("cta", "<i4"), ("warp", "<i4"), ("ns", "<u8"), ("clock", "<u4"), ("code", "u1"),
                        ("arg", "<u2")])

# Barrier waits of a consumer: the wait ends at the event, it began at the warp's previous event (so a unit's Q wait
# also holds the unit-start loads issued after its unit_begin).
_CONSUMER_WAITS = {K_FULL: "k_full", V_FULL: "v_full", Q_READY: "q_full"}


def region_bytes(grid: int, warps: int, events_per_warp: int) -> int:
    """Bytes of one launch's region (attn.cuh trace_region_bytes)."""
    return HEADER_BYTES + (grid * warps * 4 + 15) // 16 * 16 + grid * warps * events_per_warp * RECORD_DTYPE.itemsize


def role_of(header: Dict[str, int], warp: int) -> str:
    """The role a warp plays in the launch `header` describes ("idle" for a warp with no role)."""
    if header["phase"] == PHASE_IDS["decode"]:
        if warp < 4:
            if header["box_rows"] > 0:
                return ("producer_k", "producer_v", "idle", "idle")[warp]
            return "producer_k" if warp < 2 else "producer_v"
        if warp < 8:
            return "consumer"
        return "q_loader" if warp == 8 else "combiner"
    if warp < 4:
        return ("producer_kq", "producer_v", "idle", "idle")[warp]
    return "consumer_wg0" if warp < 8 else "consumer_wg1"


@dataclass
class TraceLaunch:
    """One traced launch: its header, the event count of every warp ([grid, warps]; a count above
    events_per_warp means the warp overflowed and its later events are lost) and the recorded events, ordered by
    (cta, warp, recording order)."""
    header: Dict[str, int]
    counts: np.ndarray
    events: np.ndarray
    phase: str = field(init=False)

    def __post_init__(self):
        self.phase = PHASES.get(self.header["phase"], "?")

    @property
    def overflow(self) -> bool:
        return bool((self.counts > self.header["events_per_warp"]).any())

    def warp_events(self, cta: int, warp: int) -> np.ndarray:
        e = self.events
        return e[(e["cta"] == cta) & (e["warp"] == warp)]


def decode_buffer(buf: bytes, max_launches: Optional[int] = None) -> List[TraceLaunch]:
    """Decodes the regions of a trace buffer, front to back, up to the first one without a valid header (a region
    handed to a launch that has not run, or none)."""
    mv = memoryview(buf)
    off, out = 0, []
    while off + HEADER_BYTES <= len(mv) and (max_launches is None or len(out) < max_launches):
        hdr = dict(zip(HEADER_FIELDS, np.frombuffer(mv[off:off + HEADER_BYTES], dtype="<u4").tolist()))
        if hdr["magic"] != MAGIC:
            break
        if hdr["version"] != VERSION:
            raise ValueError(f"trace region at {off}: format version {hdr['version']}, expected {VERSION}")
        grid, warps, epw = hdr["grid"], hdr["warps"], hdr["events_per_warp"]
        size = region_bytes(grid, warps, epw)
        if off + size > len(mv):
            raise ValueError(f"trace region at {off} ({size} bytes) runs past the buffer ({len(mv)} bytes)")
        cnt_off = off + HEADER_BYTES
        counts = np.frombuffer(mv[cnt_off:cnt_off + grid * warps * 4], dtype="<u4").reshape(grid, warps).copy()
        rec_off = cnt_off + (grid * warps * 4 + 15) // 16 * 16
        recs = np.frombuffer(mv[rec_off:rec_off + grid * warps * epw * 16], dtype=RECORD_DTYPE).reshape(grid, warps, epw)
        n = np.minimum(counts, epw)
        parts = []
        for c in range(grid):
            for w in range(warps):
                r = recs[c, w, : n[c, w]]
                ev = np.empty(len(r), dtype=EVENT_DTYPE)
                ev["cta"], ev["warp"] = c, w
                for f in ("ns", "clock", "code", "arg"):
                    ev[f] = r[f]
                parts.append(ev)
        events = np.concatenate(parts) if parts else np.empty(0, dtype=EVENT_DTYPE)
        out.append(TraceLaunch(hdr, counts, events))
        off += size
    return out


class AttentionTrace:
    """Context manager: a zeroed device buffer for `launches` traced launches of up to `events_per_warp` events per
    warp, registered on entry and always unregistered on exit.  Launches past `launches` run untraced.

    A launch captured into a CUDA graph inside the block keeps the region it was given: every replay of that graph
    writes it again, also after the block has ended.  Keep this object, which owns the buffer, alive for as long as
    such a graph may be replayed; once the buffer is freed, a replay would write into whatever reuses its memory.

        with AttentionTrace(4, 4096) as t:
            backend.forward(...)
        for launch in t.launches():
            print(summarise(launch))
    """

    def __init__(self, launches: int, events_per_warp: int, device=None):
        import torch

        if launches <= 0 or events_per_warp <= 0:
            raise ValueError("launches and events_per_warp must be positive")
        self._lib = _cabi.load()
        self.events_per_warp = events_per_warp
        per = max(int(self._lib.b200_attn_trace_launch_bytes(p, events_per_warp)) for p in PHASES)
        self.buffer = torch.zeros(launches * per, dtype=torch.uint8,
                                  device=device if device is not None else torch.device("cuda"))
        self._counts = (0, 0)

    def __enter__(self) -> "AttentionTrace":
        import torch

        torch.cuda.synchronize(self.buffer.device)  # the zero fill is complete before a kernel writes the buffer
        _cabi.check(self._lib.b200_attn_trace_set(self.buffer.data_ptr(), self.buffer.numel(), self.events_per_warp),
                    "b200_attn_trace_set")
        return self

    def __exit__(self, *exc) -> None:
        self._counts = self.counts()
        _cabi.check(self._lib.b200_attn_trace_set(None, 0, 0), "b200_attn_trace_set(NULL)")

    def counts(self) -> tuple:
        """(launches traced, launches that ran untraced because the buffer was full) since registration."""
        t, u = C.c_uint64(), C.c_uint64()
        _cabi.check(self._lib.b200_attn_trace_launches(C.byref(t), C.byref(u)), "b200_attn_trace_launches")
        return int(t.value), int(u.value)

    def launches(self) -> List[TraceLaunch]:
        """Every launch recorded so far (synchronises the buffer's device)."""
        import torch

        torch.cuda.synchronize(self.buffer.device)
        return decode_buffer(self.buffer.cpu().numpy().tobytes())


def _warp_spans(launch: TraceLaunch):
    """{(cta, warp): events of that warp} in recording order."""
    e = launch.events
    order = np.lexsort((np.arange(len(e)), e["warp"], e["cta"]))
    e = e[order]
    keys = e["cta"].astype(np.int64) * 256 + e["warp"]
    cuts = np.flatnonzero(np.diff(keys)) + 1
    return {(int(g["cta"][0]), int(g["warp"][0])): g for g in np.split(e, cuts) if len(g)}


def summarise(launch: TraceLaunch, alg_bytes: Optional[float] = None, flops: Optional[float] = None) -> dict:
    """The numbers of one traced launch, times in ns of %globaltimer:

    span_ns                launch begin (first CTA begin) to launch end (last CTA end)
    cta_busy_ns[c]         CTA c's end minus its begin (first / last event of any of its warps)
    cta_idle_end_ns[c]     launch end minus CTA c's end
    imbalance              max CTA end over mean CTA end, both from launch begin
    wait_fraction[role]    per barrier, the role's time spent waiting there over its warps' busy time: a producer's
                           wait runs from its empty_wait to its empty_done event; a consumer's K / V / Q wait from
                           its previous event to the wait's end (an upper bound: it includes the bookkeeping after
                           that previous event)
    prologue_ns            per CTA, CTA begin to the first tile issued by a producer
    drain_ns               per CTA, the last PV complete to CTA end
    tiles_per_cta          K tiles issued by the K producer warp 0, units_per_cta the units its consumers began
    bytes_per_s / flop_per_s  alg_bytes / flops over span_ns, when given
    """
    hdr = launch.header
    grid = hdr["grid"]
    spans = _warp_spans(launch)
    begin = np.full(grid, np.iinfo(np.int64).max, dtype=np.int64)
    end = np.zeros(grid, dtype=np.int64)
    first_issue = np.full(grid, -1, dtype=np.int64)
    last_pv = np.full(grid, -1, dtype=np.int64)
    tiles = np.zeros(grid, dtype=np.int64)
    units = np.zeros(grid, dtype=np.int64)
    role_busy: Dict[str, float] = {}
    role_wait: Dict[str, Dict[str, float]] = {}
    consumer_unit_warp = 4  # first consumer warp, both phases
    for (c, w), ev in spans.items():
        ns = ev["ns"].astype(np.int64)
        code = ev["code"]
        begin[c] = min(begin[c], int(ns.min()))
        end[c] = max(end[c], int(ns.max()))
        role = role_of(hdr, w)
        role_busy[role] = role_busy.get(role, 0.0) + float(ns.max() - ns.min())
        waits = role_wait.setdefault(role, {})
        if role.startswith("producer"):
            starts = ns[code == EMPTY_WAIT]
            stops = ns[code == EMPTY_DONE]
            k = min(len(starts), len(stops))
            waits["empty"] = waits.get("empty", 0.0) + float((stops[:k] - starts[:k]).sum())
            iss = ns[code == ISSUED]
            if len(iss):
                first_issue[c] = iss.min() if first_issue[c] < 0 else min(first_issue[c], iss.min())
            if w == 0:
                tiles[c] = int((code == ISSUED).sum())
        if role.startswith("consumer"):
            for cd, name in _CONSUMER_WAITS.items():
                idx = np.flatnonzero(code[1:] == cd) + 1
                waits[name] = waits.get(name, 0.0) + float((ns[idx] - ns[idx - 1]).sum())
            pv = ns[code == PV]
            if len(pv):
                last_pv[c] = max(last_pv[c], int(pv.max()))
            if w == consumer_unit_warp:
                units[c] = int((code == UNIT_BEGIN).sum())
    live = end > 0
    t0, t1 = int(begin[live].min()), int(end[live].max())
    cta_end_rel = (end - t0)[live]
    out = {
        "phase": launch.phase,
        "header": dict(hdr),
        "overflow": launch.overflow,
        "span_ns": t1 - t0,
        "cta_busy_ns": (end - begin)[live].tolist(),
        "cta_idle_end_ns": (t1 - end)[live].tolist(),
        "cta_end_ns": cta_end_rel.tolist(),
        "imbalance": float(cta_end_rel.max() / cta_end_rel.mean()),
        "wait_fraction": {r: {b: (v / role_busy[r] if role_busy[r] > 0 else 0.0) for b, v in ws.items()}
                          for r, ws in role_wait.items() if ws},
        "prologue_ns": [int(first_issue[c] - begin[c]) if first_issue[c] >= 0 else None for c in range(grid) if live[c]],
        "drain_ns": [int(end[c] - last_pv[c]) if last_pv[c] >= 0 else None for c in range(grid) if live[c]],
        "tiles_per_cta": tiles[live].tolist(),
        "units_per_cta": units[live].tolist(),
    }
    if alg_bytes is not None:
        out["bytes_per_s"] = alg_bytes / (out["span_ns"] * 1e-9)
    if flops is not None:
        out["flop_per_s"] = flops / (out["span_ns"] * 1e-9)
    return out


_SPANS = {EMPTY_DONE: (EMPTY_WAIT, "wait empty"), UNIT_END: (UNIT_BEGIN, "unit"), EPI_END: (EPI_BEGIN, "epilogue"),
          MERGE_END: (MERGE_BEGIN, "merge")}


def to_chrome_trace(launches: Sequence[TraceLaunch], path) -> dict:
    """Writes the launches as Chrome trace-event JSON (Perfetto, chrome://tracing): one process per SM, one thread
    per (warp, role).  Units, producer waits, epilogues and merges are slices; a consumer's barrier wait is the
    slice from its previous event to the wait's end; every other event is an instant.  Times in us from the first
    event.  Returns the written object."""
    t0 = min((int(l.events["ns"].min()) for l in launches if len(l.events)), default=0)
    out: List[dict] = []
    named = set()
    for li, launch in enumerate(launches):
        for (c, w), ev in _warp_spans(launch).items():
            sm = int(ev["arg"][0]) if ev["code"][0] == BEGIN else 1000 + c
            role = role_of(launch.header, w)
            tid = w
            if (sm, tid) not in named:
                if (sm, -1) not in named:
                    out.append({"ph": "M", "name": "process_name", "pid": sm, "args": {"name": f"SM {sm}"}})
                    named.add((sm, -1))
                out.append({"ph": "M", "name": "thread_name", "pid": sm, "tid": tid,
                            "args": {"name": f"warp {w} {role}"}})
                named.add((sm, tid))
            ns = ev["ns"].astype(np.int64)
            open_at: Dict[int, int] = {}
            for i, (code, arg) in enumerate(zip(ev["code"].tolist(), ev["arg"].tolist())):
                ts = (int(ns[i]) - t0) / 1e3
                base = {"pid": sm, "tid": tid, "args": {"launch": li, "cta": c, "arg": arg}}
                if code in (UNIT_BEGIN, EMPTY_WAIT, EPI_BEGIN, MERGE_BEGIN):
                    open_at[code] = i
                elif code in _SPANS and _SPANS[code][0] in open_at:
                    j = open_at.pop(_SPANS[code][0])
                    out.append({**base, "ph": "X", "name": f"{_SPANS[code][1]} {arg}", "ts": (int(ns[j]) - t0) / 1e3,
                                "dur": (int(ns[i]) - int(ns[j])) / 1e3})
                elif code in _CONSUMER_WAITS and role.startswith("consumer") and i > 0:
                    out.append({**base, "ph": "X", "name": f"wait {_CONSUMER_WAITS[code]}",
                                "ts": (int(ns[i - 1]) - t0) / 1e3, "dur": (int(ns[i]) - int(ns[i - 1])) / 1e3})
                else:
                    out.append({**base, "ph": "i", "s": "t", "name": CODE_NAMES.get(code, str(code)), "ts": ts})
    obj = {"traceEvents": out, "displayTimeUnit": "ns"}
    with open(path, "w") as f:
        json.dump(obj, f)
    return obj
