#!/usr/bin/env python
"""Event timelines of the attention kernels on the bench workloads: one decode or prefill launch traced from inside
the kernel (mini-sglang_b200/trace.py), summarised, and written as a Perfetto / chrome://tracing timeline.

    python tools/attn_trace.py decode --out attn_trace/ --iter 500                  # cfg1, page size 64
    python tools/attn_trace.py decode --out attn_trace/ --page-size 1
    python tools/attn_trace.py prefill --out attn_trace/

Writes under --out: <what>_summary.json (summary, per-call times traced and untraced, the smallest %globaltimer step
seen, the card and its power limit) and <what>_trace.json (the timeline).  Times are CUDA events around windows of
--calls back-to-back calls on the same inputs, traced and untraced windows alternated, so the tracing overhead is
stated beside every number the trace gives; host_enqueue_ms_per_call below call_ms_untraced (gpu_bound) means the
GPU never waited for the host, so a window's time over its calls is the kernel time.  The summary and the timeline
are those of the launch in the middle of the last traced window.  The batch is built the way tools/microbench.py
builds it.
"""
import argparse
import importlib
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402


def card() -> dict:
    """Name and power limit of GPU 0 (read-only nvidia-smi query)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        name, power = [x.strip() for x in out.split(",")[:2]]
        return {"name": name, "power_limit": power}
    except (OSError, ValueError, subprocess.SubprocessError) as e:
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e.__class__.__name__})"}


def timer_step_ns(launches) -> int:
    """Smallest nonzero difference between consecutive %globaltimer stamps of one warp."""
    best = 0
    for l in launches:
        e = l.events
        order = np.lexsort((np.arange(len(e)), e["warp"], e["cta"]))
        e = e[order]
        d = np.diff(e["ns"].astype(np.int64))
        same = (np.diff(e["cta"]) == 0) & (np.diff(e["warp"]) == 0)
        d = d[same & (d > 0)]
        if len(d):
            best = int(d.min()) if best == 0 else min(best, int(d.min()))
    return best


def time_windows(fn, trace, calls: int, epw: int, reps: int):
    """Per-call ms of `calls` back-to-back calls of fn, untraced and traced (a buffer with a region for every call of
    the window), windows alternated, medians over reps; plus the host's enqueue ms per call (when it is below the
    per-call time the GPU never ran dry, so the window times the kernels) and the launches of the last traced window."""
    untraced, traced, host = [], [], []
    launches = []
    for _ in range(reps):
        for on in (False, True):
            t = trace.AttentionTrace(calls, epw) if on else None
            if t is not None:
                t.__enter__()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            h0 = time.perf_counter()
            for _ in range(calls):
                fn()
            host.append((time.perf_counter() - h0) * 1e3 / calls)
            e1.record()
            e1.synchronize()
            (traced if on else untraced).append(e0.elapsed_time(e1) / calls)
            if t is not None:
                launches = t.launches()
                t.__exit__(None, None, None)
    return float(np.median(untraced)), float(np.median(traced)), float(np.median(host)), launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("what", choices=["decode", "prefill"])
    ap.add_argument("--out", required=True)
    ap.add_argument("--config", default="cfg1", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--iter", type=int, default=500, help="decode: the schedule iteration whose batch is traced")
    ap.add_argument("--page-size", type=int, default=64)
    ap.add_argument("--hq", type=int, default=0, help="override the (local) q heads of the config")
    ap.add_argument("--hkv", type=int, default=0)
    ap.add_argument("--events-per-warp", type=int, default=16384)
    ap.add_argument("--calls", type=int, default=50, help="back-to-back calls per timed window")
    ap.add_argument("--reps", type=int, default=10, help="alternated traced / untraced windows")
    args = ap.parse_args()
    bench.set_workload(args.config)
    bench.L = 1
    if args.hq:
        bench.HQ, bench.HKV = args.hq, args.hkv or bench.HKV
    pkg = importlib.import_module("mini-sglang_b200")
    pkg.build_native()
    trace = pkg.trace
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    sched = bench.Schedule()
    r = bench.AttentionPathRunner(pkg, sched, bench.HQ, bench.HKV, args.page_size, dev)
    hq, hkv, D = r.hq, r.hkv, bench.D
    out_dir = Path(args.out)
    out_dir.mkdir(parents=True, exist_ok=True)
    with torch.cuda.stream(r.stream):
        if args.what == "decode":
            tr = sched.live(args.iter)
            batch = r.make_batch(tr, "decode")
            bs = batch.padded_size
            pos_h, loc_h = r.host_inputs(batch)
            batch.positions, batch.out_loc = pos_h.to(dev), loc_h.to(dev)
            r.backend.prepare_metadata(batch)
            q, k, v = r.qkv_views(0, bs)
            triples = [(x.table_idx, x.cached_len, x.device_len) for x in batch.padded_reqs]
            work = {"alg_bytes": float(bench.decode_bytes_per_layer(triples, hq, hkv))}
            fn = lambda: r.backend.forward(q.view(bs, hq, D), k, v, 0, batch)  # noqa: E731
            shape = {"bs": bs, "sum_kv": int(sum(x[2] for x in triples))}
        else:
            tr = sched.prefill_batches()[0]
            batch = r.make_batch(tr, "prefill")
            pos_h, loc_h = r.host_inputs(batch)
            nnz = pos_h.numel()
            batch.positions, batch.out_loc = pos_h.to(dev), loc_h.to(dev)
            r.backend.prepare_metadata(batch)
            qkv = torch.randn((nnz, r.width), device=dev, dtype=torch.bfloat16)
            q, k, v = qkv.split([hq * D, hkv * D, hkv * D], dim=-1)
            work = {"flops": float(bench.prefill_flops_per_layer(tr, hq))}
            fn = lambda: r.backend.forward(q.view(nnz, hq, D), k, v, 0, batch)  # noqa: E731
            shape = {"nnz": nnz, "reqs": len(tr)}
        for _ in range(3):  # warm-up: module load, tensor maps, both instantiations
            fn()
            with trace.AttentionTrace(1, args.events_per_warp) as t:
                fn()
                probe = t.launches()[0]
        torch.cuda.synchronize()
        # the timed windows' buffer: room for the most events a warp recorded in the probe launch, plus a margin
        epw = int(probe.counts.max()) * 5 // 4 + 64
        untraced_ms, traced_ms, host_ms, launches = time_windows(fn, trace, args.calls, epw, args.reps)
    # the launch in the middle of the last traced window: it ran back to back with its neighbours, as in a step
    mid = launches[len(launches) // 2]
    spans = [trace.summarise(l)["span_ns"] / 1e6 for l in launches]
    window_overflow = any(l.overflow for l in launches)
    launches = [mid]
    summary = trace.summarise(mid, **work)
    cta_end = np.array(summary["cta_end_ns"], dtype=np.float64)
    prologue = [x for x in summary["prologue_ns"] if x is not None]
    drain = [x for x in summary["drain_ns"] if x is not None]
    res = {
        "what": args.what, "config": args.config, "page_size": args.page_size, "hq": hq, "hkv": hkv, **shape,
        "card": card(),
        "calls_per_window": args.calls, "call_ms_untraced": untraced_ms, "call_ms_traced": traced_ms,
        "tracing_overhead": traced_ms / untraced_ms - 1.0, "host_enqueue_ms_per_call": host_ms,
        "gpu_bound": host_ms < untraced_ms, "traced_span_ms_median": float(np.median(spans)),
        "overflow_in_window": window_overflow,
        "globaltimer_min_step_ns": timer_step_ns(launches),
        "cta_end_spread_ns": {"min": float(cta_end.min()), "median": float(np.median(cta_end)), "max": float(cta_end.max())},
        "prologue_share": float(np.mean(prologue) / summary["span_ns"]) if prologue else None,
        "drain_share": float(np.mean(drain) / summary["span_ns"]) if drain else None,
        "summary": summary,
    }
    (out_dir / f"{args.what}_summary.json").write_text(json.dumps(res, indent=1))
    trace.to_chrome_trace(launches, out_dir / f"{args.what}_trace.json")
    brief = {k: v for k, v in res.items() if k != "summary"}
    brief.update({k: summary[k] for k in ("span_ns", "imbalance", "wait_fraction", "overflow")})
    print(json.dumps(brief))


if __name__ == "__main__":
    main()
