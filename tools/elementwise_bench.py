#!/usr/bin/env python
"""HBM-bound elementwise kernels of the path at PREFILL sizes (one cfg1 prompt batch: 16 384 tokens,
Qwen3-0.6B shape): achieved GB/s = algorithmic bytes (rows read + written, weights once) / CUDA-event
time, against the measured HBM peak.  Inputs are rotated over buffers larger than L2 so every launch is
cold.  Run plain for the timing JSON, or under
  ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none
for the per-launch DRAM traffic.

The gated MLP's SiLU-and-mul follows, ours next to flashinfer.silu_and_mul in the same process, at decode
rows (1, 64, 256) and one 8192-row prefill chunk, for the MLP widths of Qwen3-0.6B (3072), Qwen3-14B (17408)
and Llama-3.1-70B at tp8 (3584).  Kernel time is the replay of a CUDA graph of back-to-back launches (how
the engine runs decode); the two are timed in alternation, `--trials` times each, and the median with the
min..max spread is reported, next to the per-call time of an eager Python loop (host-bound at small sizes).
Bytes = rows * d * 3 * 2 (gate and up read, product written).

    python tools/elementwise_bench.py [--out elementwise.json] [--reps 20] [--trials 5]
"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--nnz", type=int, default=16384)
    ap.add_argument("--trials", type=int, default=5)
    args = ap.parse_args()
    pkg = importlib.import_module("mini-sglang_b200")
    pkg.build_native()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    peaks = bench.load_peaks()
    nnz, hq, hkv, D, hidden = args.nnz, 16, 8, 128, 1024
    width = (hq + 2 * hkv) * D
    n_buf = 6  # 6 x 128 MB of qkv rows > 126 MB L2
    qkv = [torch.randn((nnz, width), device=dev, dtype=torch.bfloat16) for _ in range(n_buf)]
    hid = [torch.randn((nnz, hidden), device=dev, dtype=torch.bfloat16) for _ in range(n_buf * 4)]
    res = [torch.randn((nnz, hidden), device=dev, dtype=torch.bfloat16) for _ in range(n_buf * 4)]
    w_h = torch.ones(hidden, device=dev, dtype=torch.bfloat16)
    w_d = torch.ones(D, device=dev, dtype=torch.bfloat16)
    pos = torch.randint(0, 4096, (nnz,), device=dev, dtype=torch.int32)
    cache = pkg.layers.RotaryEmbedding(D, D, 4096, 1e6, device=dev)._cos_sin_cache
    slots = nnz * 2
    kc = [torch.empty((slots, hkv * D), device=dev, dtype=torch.bfloat16) for _ in range(n_buf)]
    vc = [torch.empty((slots, hkv * D), device=dev, dtype=torch.bfloat16) for _ in range(n_buf)]
    loc = torch.randperm(slots, device=dev)[:nnz].to(torch.int32)
    table = torch.randn((151936, hidden), device=dev, dtype=torch.bfloat16)
    ids = torch.randint(0, table.shape[0], (nnz,), device=dev, dtype=torch.int32)
    outb = [torch.empty((nnz, hidden), device=dev, dtype=torch.bfloat16) for _ in range(4)]

    def split(i):
        return qkv[i % n_buf].split([hq * D, hkv * D, hkv * D], dim=-1)

    cases = {
        "qknorm_rope_kernel (q-norm + k-norm + RoPE, one launch)": (
            lambda i: pkg.ops.qknorm_rope_inplace(pos, split(i)[0], split(i)[1], D, cache, w_d, w_d, 1e-6),
            2 * nnz * (hq + hkv) * D * 2),
        "qknorm_rope_kernel<no norm> (RoPE only)": (
            lambda i: pkg.ops.apply_rope_with_cos_sin_cache_inplace(pos, split(i)[0], split(i)[1], D, cache),
            2 * nnz * (hq + hkv) * D * 2),
        "rmsnorm_group_kernel (per-head q-norm, in place)": (
            lambda i: pkg.ops.rmsnorm(split(i)[0].view(nnz, hq, D), w_d, 1e-6, out=split(i)[0].view(nnz, hq, D)),
            2 * nnz * hq * D * 2),
        "rmsnorm_row_kernel (hidden 1024)": (
            lambda i: pkg.ops.rmsnorm(hid[i % len(hid)], w_h, 1e-6, out=outb[i % 4]), 2 * nnz * hidden * 2),
        "rmsnorm_row_kernel<fused add> (hidden 1024)": (
            lambda i: pkg.ops.fused_add_rmsnorm(hid[i % len(hid)], res[i % len(res)], w_h, 1e-6), 4 * nnz * hidden * 2),
        "store_kv_kernel (KV append, 2 KiB rows)": (
            lambda i: pkg.ops.store_cache(kc[i % n_buf], vc[i % n_buf], loc, split(i)[1], split(i)[2]),
            2 * 2 * nnz * hkv * D * 2 + nnz * 4),
        "index_rows_kernel (embedding gather, 2 KiB rows)": (
            lambda i: pkg.ops.indexing(table, ids, output=outb[i % 4]), 2 * nnz * hidden * 2 + nnz * 4),
    }
    out = {"nnz": nnz, "peak_GBs": peaks["hbm_gbs"], "peak_source": peaks["source"], "kernels": {}}
    for name, (fn, nbytes) in cases.items():
        for i in range(3):
            fn(i)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.reps):
            fn(i)
        e1.record()
        e1.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / args.reps
        gbs = nbytes / us / 1e3
        out["kernels"][name] = {"us": round(us, 2), "alg_bytes": nbytes, "GBs": round(gbs, 1), "frac_of_hbm_peak": round(gbs / peaks["hbm_gbs"], 3)}
        print(f"{name:64s} {us:8.2f} us  {gbs:8.1f} GB/s  {gbs / peaks['hbm_gbs']:.3f}", flush=True)
    del qkv, hid, res, kc, vc, table, outb
    torch.cuda.empty_cache()
    out["silu_and_mul"] = silu_and_mul_rows(pkg, dev, args)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(out, indent=1))


def card() -> dict:
    """Name and power limit of the card the numbers were measured on."""
    info = {"name": torch.cuda.get_device_name(0), "power_limit": "unknown"}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=30, text=True)
        if q.returncode == 0 and q.stdout.strip():
            limit, sm_clock = (x.strip() for x in q.stdout.strip().split(","))
            info.update(power_limit=limit, max_sm_clock=sm_clock)
    except (OSError, subprocess.SubprocessError):
        pass
    return info


def _graph(fn, n_buf, reps):
    """reps launches captured into one CUDA graph: replaying it times the kernels, not the Python that issues them."""
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(reps):
            fn(i % n_buf)
    return g


def _event_us(work, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    work()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


def silu_and_mul_rows(pkg, dev, args) -> dict:
    os.environ.setdefault("FLASHINFER_WORKSPACE_BASE", bench.flashinfer_workspace())
    try:
        import flashinfer

        fi = flashinfer.silu_and_mul
    except Exception as e:  # noqa: BLE001
        fi, why = None, f"{type(e).__name__}: {e}"
    res = {"card": card(), "peak_GBs": 3350.0, "peak_source": "H100 SXM data sheet (HBM3 3.35 TB/s)",
           "trials": args.trials, "shapes": {}}
    if fi is None:
        res["flashinfer"] = f"not measured ({why})"
    print(f"silu_and_mul on {res['card']}", flush=True)
    for d, model in ((3072, "Qwen3-0.6B"), (17408, "Qwen3-14B"), (3584, "Llama-3.1-70B tp8")):
        for rows in (1, 64, 256, 8192):
            nbytes = rows * d * 3 * 2
            n_buf = max(1, min(64, -(-256 * 2**20 // nbytes)))  # > 126 MB of inputs, so big shapes run cold
            xs = [torch.randn((rows, 2 * d), device=dev, dtype=torch.bfloat16) for _ in range(n_buf)]
            outs = [torch.empty((rows, d), device=dev, dtype=torch.bfloat16) for _ in range(min(n_buf, 4))]
            impls = {"ours": lambda i: pkg.ops.silu_and_mul(xs[i], out=outs[i % len(outs)])}
            if fi is not None:
                impls["flashinfer"] = lambda i: fi(xs[i], out=outs[i % len(outs)])
            times = {k: [] for k in impls}
            eager = {k: [] for k in impls}
            for fn in impls.values():
                for i in range(3):
                    fn(i % n_buf)
            torch.cuda.synchronize()
            reps = max(args.reps, 200 if rows < 8192 else args.reps)
            graphs = {name: _graph(fn, n_buf, reps) for name, fn in impls.items()}
            for g in graphs.values():
                g.replay()
            for _ in range(args.trials):
                for name, fn in impls.items():  # alternate, so drift hits both alike
                    times[name].append(_event_us(graphs[name].replay, reps))
                    eager[name].append(_event_us(lambda: [fn(i % n_buf) for i in range(reps)], reps))
            row = {"model": model, "rows": rows, "d": d, "alg_bytes": nbytes}
            for name, ts in times.items():
                us = statistics.median(ts)
                gbs = nbytes / us / 1e3
                row[name] = {"us": round(us, 2), "us_min": round(min(ts), 2), "us_max": round(max(ts), 2),
                             "GBs": round(gbs, 1), "frac_of_3350_GBs": round(gbs / 3350.0, 3),
                             "eager_call_us": round(statistics.median(eager[name]), 2)}
            if "flashinfer" in row:
                row["ours_over_flashinfer"] = round(row["ours"]["us"] / row["flashinfer"]["us"], 3)
            res["shapes"][f"{rows}x{d}"] = row
            line = "  ".join(f"{k} {v['us']:8.2f} us [{v['us_min']:.2f}..{v['us_max']:.2f}] {v['GBs']:7.1f} GB/s "
                             f"{v['frac_of_3350_GBs']:.3f} (eager {v['eager_call_us']:.1f} us/call)"
                             for k, v in row.items() if isinstance(v, dict))
            print(f"silu_and_mul {rows:5d} x {d:5d}  {line}", flush=True)
            del xs, outs, graphs
    return res


if __name__ == "__main__":
    main()
