#!/usr/bin/env python
"""A/B of the decode kernel's exact-tail K/V loads (option decode_exact_tail) on a bench.py workload.

    python tools/decode_tail_ab.py [--pairs 3] [--out DIR] [-- <extra bench.py arguments>]

Runs `bench.py --skip-prefill --skip-cpu --skip-ref-gpu` once per arm in alternation (option at 1, 0, 1, 0, ...;
one process per run, so neither arm inherits the other's warm state), prints every run's `value`,
`roofline.achieved` and `roofline.per_step_bs_us_frac` with the card's name and power limit, and checks that the
`--dump-outputs` of the first run of each arm (attention outputs, appended K and V rows) are bitwise equal.

It also prints the modelled K/V rows the kernel reads from HBM over the rows the algorithm needs, for both arms,
from the same schedule bench.py times: `tile_loads` below restates, per 128-key tile, the TMA loads the box-mode
producer of attn_decode_tc.cu issues and the transaction bytes it announces (tests/test_decode_tail_cpu.py checks
that restatement).  The byte saving the model predicts can be set against the measured speed-up.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path
from typing import List, Tuple

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
TILE = 128  # keys per tile (kTileN)
ROW_BYTES = 128  # one 64-column half of a 16-bit K or V row
TAIL_BOX = 8  # rows of the boxes the piece holding the end of a range is loaded with


def box_rows_for(page_size: int) -> int:
    """Rows per tiled TMA box at this page size (box_rows_for in csrc/attn.cuh): the largest power of two
    <= min(page size, 64) that divides the page size, 0 = row mode (page sizes below 8)."""
    if page_size < 8:
        return 0
    rb = 64
    while rb > 8 and page_size % rb:
        rb >>= 1
    return rb if page_size % rb == 0 else 0


def tile_loads(rb: int, tile_begin: int, kv_end: int, exact: bool) -> Tuple[List[Tuple[int, int, int, int]], int]:
    """The loads of one tile at positions [tile_begin, tile_begin + 128) of a range ending at kv_end, as the box-mode
    producer warp issues them: lane = (box, half), `rows` per lane, one rb-row box when rows == rb, otherwise rows / 8
    eight-row boxes.  Returns ([(half, first smem row, rows, first position)], announced transaction bytes); the bytes
    are summed from the same per-lane `rows` the loads are issued from, as in the kernel."""
    loads, total_rows = [], 0
    n_instr = (TILE // rb) * 2
    for lane in range(32):
        box, half = lane >> 1, lane & 1
        pb = tile_begin + box * rb
        left = kv_end - pb
        rows = 0
        if lane < n_instr:
            rows = rb if not exact else (0 if left <= 0 else min(rb, (left + 7) & ~7))
        total_rows += rows
        if rows == rb:
            loads.append((half, box * rb, rb, pb))
        else:
            for r in range(0, rows, TAIL_BOX):
                loads.append((half, box * rb + r, TAIL_BOX, pb + r))
    return loads, total_rows * ROW_BYTES


def range_rows_read(rb: int, kv_begin: int, kv_end: int, exact: bool) -> int:
    """Pool rows one half of one unit reads from HBM for the keys [kv_begin, kv_end): rows of loads that start
    inside the range (a box wholly past the end is out-of-range rows in the old mode: zero filled, not read)."""
    n = 0
    for t0 in range(kv_begin, kv_end, TILE):
        loads, _ = tile_loads(rb, t0, kv_end, exact)
        n += sum(rows for (half, _, rows, pos) in loads if half == 0 and pos < kv_end)
    return n


def modelled_read_over_need(page_size: int, config: str, steps: int) -> dict:
    """Rows read / rows needed over the timed steps of bench.py's schedule.  Every request contributes the range
    [0, kv_len - 1) (the appended token is not streamed); split-KV chunks end on 128-key tile boundaries except the
    last one, so a split plan reads the same rows."""
    sys.path.insert(0, str(ROOT))
    import bench

    wl = bench.set_workload(config)
    sched = bench.Schedule(wl)
    rb = box_rows_for(page_size)
    if rb == 0:
        return {"page_size": page_size, "box_rows": 0, "note": "row mode: one load per valid row in both arms"}
    need = read_new = read_old = 0
    for it in sched.sample_iters(steps):
        for (_, _, d) in sched.live(it):
            n = d - 1
            need += n
            read_new += range_rows_read(rb, 0, n, True)
            read_old += range_rows_read(rb, 0, n, False)
    return {"page_size": page_size, "box_rows": rb, "exact_tail_1": round(read_new / need, 4),
            "exact_tail_0": round(read_old / need, 4), "predicted_saving": round(1 - read_new / read_old, 4)}


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # the measurement stands without the label; say why it is missing
        return f"unknown ({type(e).__name__})"


def run_bench(arm: int, bench_args: List[str], dump: str | None) -> dict:
    cmd = [sys.executable, str(ROOT / "bench.py"), "--skip-prefill", "--skip-cpu", "--skip-ref-gpu",
           "--opt", f"decode_exact_tail={arm}", *bench_args]
    if dump:
        cmd += ["--dump-outputs", dump]
    res = subprocess.run(cmd, capture_output=True, text=True)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    if res.returncode != 0 or not lines:
        sys.stderr.write(res.stdout[-4000:] + res.stderr[-4000:])
        raise SystemExit(f"bench.py failed (exit {res.returncode}): {' '.join(cmd)}")
    return json.loads(lines[-1])


def dumps_equal(a: str, b: str) -> dict:
    out = {}
    for name in ("attn_out", "k_appended", "v_appended", "rows"):
        x, y = np.load(Path(a) / f"{name}.npy"), np.load(Path(b) / f"{name}.npy")
        out[name] = bool(x.shape == y.shape and x.tobytes() == y.tobytes())
    return out


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--pairs", type=int, default=3, help="runs per arm (alternating 1, 0, 1, 0, ...)")
    ap.add_argument("--out", default=None, help="directory for the dumps and summary.json (default: a temp dir)")
    ap.add_argument("bench_args", nargs=argparse.REMAINDER, help="after --: passed to bench.py")
    args = ap.parse_args()
    bench_args = [a for a in args.bench_args if a != "--"]
    bap = argparse.ArgumentParser(add_help=False)
    bap.add_argument("--page-size", type=int, default=64)
    bap.add_argument("--config", default="cfg1")
    bap.add_argument("--steps", type=int, default=40)
    known, _ = bap.parse_known_args(bench_args)
    out = Path(args.out or tempfile.mkdtemp(prefix="decode_tail_ab_"))
    out.mkdir(parents=True, exist_ok=True)

    model = modelled_read_over_need(known.page_size, known.config, known.steps)
    print(f"card: {card()}", flush=True)
    print(f"bench args: {' '.join(bench_args) or '(defaults)'}", flush=True)
    print(f"modelled K/V rows read / rows needed: {json.dumps(model)}", flush=True)
    runs = {1: [], 0: []}
    for i in range(args.pairs):
        for arm in (1, 0):
            r = run_bench(arm, bench_args, str(out / f"dump_{arm}") if i == 0 else None)
            rf = r["roofline"]
            runs[arm].append({"value": r["value"], "achieved": rf["achieved"], "frac_of_hbm_roofline": r["frac_of_hbm_roofline"],
                              "alg_bytes_per_launch": rf["alg_bytes_per_launch"], "us_per_launch": rf["us_per_launch"],
                              "per_step_bs_us_frac": rf["per_step_bs_us_frac"], "clocks": r.get("clocks")})
            print(f"decode_exact_tail={arm} run {i}: value {r['value']} tok/s, roofline.achieved {rf['achieved']} GB/s, "
                  f"us_per_launch {rf['us_per_launch']}, alg_bytes_per_launch {rf['alg_bytes_per_launch']}, "
                  f"frac_of_hbm_roofline {r['frac_of_hbm_roofline']}", flush=True)
            print(f"  per_step_bs_us_frac {json.dumps(rf['per_step_bs_us_frac'])}", flush=True)
    eq = dumps_equal(str(out / "dump_1"), str(out / "dump_0"))
    v1, v0 = [r["value"] for r in runs[1]], [r["value"] for r in runs[0]]
    summary = {
        "card": card(), "bench_args": bench_args, "model": model, "runs": {str(k): v for k, v in runs.items()},
        "dumps_bitwise_equal": eq,
        "value_exact_tail_1": {"min": min(v1), "max": max(v1), "mean": round(float(np.mean(v1)), 1)},
        "value_exact_tail_0": {"min": min(v0), "max": max(v0), "mean": round(float(np.mean(v0)), 1)},
        "gain_mean": round(float(np.mean(v1)) / float(np.mean(v0)) - 1, 4),
        "every_1_beats_every_0": min(v1) > max(v0),
        "alg_bytes_per_launch_equal": len({r["alg_bytes_per_launch"] for r in runs[1] + runs[0]}) == 1,
    }
    (out / "summary.json").write_text(json.dumps(summary, indent=1))
    print(json.dumps({k: summary[k] for k in summary if k != "runs"}))
    if not all(eq.values()):
        raise SystemExit("the two arms' outputs differ")


if __name__ == "__main__":
    main()
