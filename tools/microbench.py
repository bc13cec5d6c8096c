#!/usr/bin/env python
"""Kernel-level micro-benchmark on the bench workload (one decode iteration of cfg1, a few layers):
used under ncu for per-kernel captures and stand-alone for quick timing.

    python tools/microbench.py decode --iter 500 --layers 4 --reps 5
    python tools/microbench.py prefill --layers 2
    python tools/microbench.py prefill --config cfg4 --layers 4            # 2 x 4096-token prompts, GQA 8
    python tools/microbench.py prefill --lens 0:8192 --hq 8 --hkv 1        # custom (cached:total,...) prompts
"""
import argparse
import importlib
import sys
from pathlib import Path
from types import SimpleNamespace

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("what", choices=["decode", "prefill", "elementwise"])
    ap.add_argument("--iter", type=int, default=500)
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--page-size", type=int, default=64)
    ap.add_argument("--config", default="cfg1", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--hq", type=int, default=0, help="override the (local) q heads of the config")
    ap.add_argument("--hkv", type=int, default=0)
    ap.add_argument("--lens", default="", help="prefill: comma list of cached:total prompt lengths instead of the schedule's batches")
    ap.add_argument("--batches", type=int, default=2)
    ap.add_argument("--opt", action="append", default=[], help="name=value for b200_set_option")
    args = ap.parse_args()
    bench.set_workload(args.config)
    bench.L = args.layers
    if args.hq:
        bench.HQ, bench.HKV = args.hq, args.hkv or bench.HKV
    args.hq, args.hkv = bench.HQ, bench.HKV
    pkg = importlib.import_module("mini-sglang_b200")
    pkg.build_native()
    for o in args.opt:
        k, v = o.split("=")
        pkg._cabi.set_option(k, int(v))
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    sched = bench.Schedule()
    r = bench.AttentionPathRunner(pkg, sched, args.hq, args.hkv, args.page_size, dev)
    hq, hkv, D = r.hq, r.hkv, bench.D
    peaks = bench.load_peaks()
    with torch.cuda.stream(r.stream):
        if args.what in ("decode", "elementwise"):
            tr = sched.live(args.iter)
            batch = r.make_batch(tr, "decode")
            bs = batch.padded_size
            pos_h, loc_h = r.host_inputs(batch)
            batch.positions, batch.out_loc = pos_h.to(dev), loc_h.to(dev)
            r.backend.prepare_metadata(batch)
            qs = [r.qkv_views(l, bs) for l in range(args.layers)]
            nbytes = bench.decode_bytes_per_layer([(x.table_idx, x.cached_len, x.device_len) for x in batch.padded_reqs], hq, hkv)
            times = []
            for rep in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for l in range(args.layers):
                    q, k, v = qs[l]
                    if args.what == "elementwise":
                        pkg.ops.qknorm_rope_inplace(batch.positions, q, k, D, r.rotary._cos_sin_cache, r.qw, r.kw, 1e-6)
                    else:
                        r.backend.forward(q.view(bs, hq, D), k, v, l, batch)
                e1.record()
                e1.synchronize()
                us = e0.elapsed_time(e1) * 1e3 / args.layers
                times.append(us)
                if rep < args.reps - 1:
                    continue
                us = sorted(times)[len(times) // 2]
                if args.what == "decode":
                    print(f"decode bs={bs} sum_kv={sum(x[2] for x in tr)} : {us:.1f} us/layer, {nbytes / us / 1e3:.0f} GB/s "
                          f"({nbytes / us / 1e3 / peaks['hbm_gbs']:.3f} of {peaks['source']} HBM peak; min {min(times):.1f} us) opts={args.opt} plan={batch.attn_metadata.decode_plan[:3].tolist()}")
                else:
                    eb = bs * (hq + hkv) * D * 2 * 2
                    print(f"qknorm_rope bs={bs}: {us:.1f} us/layer, {eb / us / 1e3:.0f} GB/s")
        else:
            batches = sched.prefill_batches()[: args.batches]
            if args.lens:
                batches = [[(i, int(x.split(":")[0]), int(x.split(":")[1])) for i, x in enumerate(args.lens.split(","))]]
            for tr in batches:
                batch = r.make_batch(tr, "prefill")
                pos_h, loc_h = r.host_inputs(batch)
                nnz = pos_h.numel()
                batch.positions, batch.out_loc = pos_h.to(dev), loc_h.to(dev)
                r.backend.prepare_metadata(batch)
                qkv = torch.randn((nnz, r.width), device=dev, dtype=torch.bfloat16)
                q, k, v = qkv.split([hq * D, hkv * D, hkv * D], dim=-1)
                for rep in range(args.reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for l in range(args.layers):
                        r.backend.forward(q.view(nnz, hq, D), k, v, l, batch)
                    e1.record()
                    e1.synchronize()
                    ms = e0.elapsed_time(e1) / args.layers
                    fl = bench.prefill_flops_per_layer(tr, hq)
                    print(f"prefill nnz={nnz} reqs={len(tr)}: {ms:.3f} ms/layer, {fl / ms / 1e9:.1f} TFLOP/s "
                          f"({fl / ms / 1e9 / peaks['bf16_tflops']:.3f} of bf16 peak)")


if __name__ == "__main__":
    main()
