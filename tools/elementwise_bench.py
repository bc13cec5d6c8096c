#!/usr/bin/env python
"""HBM-bound elementwise kernels of the path at PREFILL sizes (one cfg1 prompt batch: 16 384 tokens,
Qwen3-0.6B shape): achieved GB/s = algorithmic bytes (rows read + written, weights once) / CUDA-event
time, against the measured HBM peak.  Inputs are rotated over buffers larger than L2 so every launch is
cold.  Run plain for the timing JSON, or under
  ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none
for the per-launch DRAM traffic.

    python tools/elementwise_bench.py [--out gpurun_out/elementwise.json] [--reps 20]
"""
import argparse
import importlib
import json
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
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
