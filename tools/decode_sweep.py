#!/usr/bin/env python
"""Sweep of the split-KV plan policy (b200_set_option decode_plan_target / decode_plan_nosplit /
decode_fused_combine) over decode iterations of cfg1 with different live batch sizes, one process.

    python tools/decode_sweep.py --iters 100,500,800,900,980,1015 --targets 1,2,4 --nosplit 0,50,75,100 --fused 0,1,2
    python tools/decode_sweep.py --graph --layers 28 --opts "decode_fused_combine=0;decode_fused_combine=1"
"""
import argparse
import importlib
import itertools
import json
import os
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", default="100,500,800,900,980,1015")
    ap.add_argument("--targets", default="2", help="decode_plan_target values, e.g. 1,2,4")
    ap.add_argument("--nosplit", default="75", help="decode_plan_nosplit values (percent of the CTA hint; 0 = always split)")
    ap.add_argument("--fused", default="2", help="decode_fused_combine values (2 = auto)")
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--hq", type=int, default=bench.HQ)
    ap.add_argument("--hkv", type=int, default=bench.HKV)
    ap.add_argument("--graph", action="store_true",
                    help="time a captured graph of --layers launches (what the engine replays) instead of eager "
                         "launches, which are host-bound below ~30 us per layer")
    ap.add_argument("--out", default="gpurun_out/decode_sweep.json")
    ap.add_argument("--opts", default="", help="extra option sets to cross with the sweep: 'a=1,b=2;a=0' (';' separates sets)")
    args = ap.parse_args()
    bench.L = args.layers
    bench.HQ, bench.HKV = args.hq, args.hkv
    pkg = importlib.import_module("mini-sglang_b200")
    pkg.build_native()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    sched = bench.Schedule()
    r = bench.AttentionPathRunner(pkg, sched, args.hq, args.hkv, 64, dev)
    hq, hkv, D = r.hq, r.hkv, bench.D
    peaks = bench.load_peaks()
    rows = []
    with torch.cuda.stream(r.stream):
        for it in [int(x) for x in args.iters.split(",")]:
            tr = sched.live(it)
            batch = r.make_batch(tr, "decode")
            bs = batch.padded_size
            pos_h, loc_h = r.host_inputs(batch)
            batch.positions, batch.out_loc = pos_h.to(dev), loc_h.to(dev)
            qs = [r.qkv_views(l, bs) for l in range(args.layers)]
            nbytes = bench.decode_bytes_per_layer([(x.table_idx, x.cached_len, x.device_len) for x in batch.padded_reqs], hq, hkv)
            best = None
            extra_sets = [dict(kv.split("=") for kv in es.split(",") if kv) for es in args.opts.split(";")] if args.opts else [{}]
            for extra, (tg, ns, fu) in itertools.product(extra_sets, itertools.product([int(x) for x in args.targets.split(",")], [int(x) for x in args.nosplit.split(",")],
                                                [int(x) for x in args.fused.split(",")])):
                prev = {k: pkg._cabi.set_option(k, int(v)) for k, v in extra.items()}
                pkg._cabi.set_option("decode_plan_target", tg)
                pkg._cabi.set_option("decode_plan_nosplit", ns)
                pkg._cabi.set_option("decode_fused_combine", fu)
                r.backend.prepare_metadata(batch)
                plan = batch.attn_metadata.decode_plan[:2].tolist()
                ts = []

                def run_layers():
                    for l in range(args.layers):
                        q, k, v = qs[l]
                        r.backend.forward(q.view(bs, hq, D), k, v, l, batch)

                graph = None
                if args.graph:
                    run_layers()
                    r.stream.synchronize()
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph, stream=r.stream):
                        run_layers()
                    graph.replay()
                for rep in range(args.reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    if graph is not None:
                        graph.replay()
                    else:
                        run_layers()
                    e1.record()
                    e1.synchronize()
                    ts.append(e0.elapsed_time(e1) * 1e3 / args.layers)
                us = float(np.median(ts))
                for k, v in prev.items():
                    pkg._cabi.set_option(k, v)
                del graph
                row = dict(iter=it, bs=bs, live=len(tr), **extra, target=tg, nosplit=ns, fused=fu, chunk=plan[0], items=plan[1], us=round(us, 1),
                           frac=round(nbytes / us / 1e3 / peaks["hbm_gbs"], 3))
                rows.append(row)
                if best is None or us < best["us"]:
                    best = row
            print("BEST", json.dumps(best), flush=True)
    out = ROOT / args.out
    out.parent.mkdir(parents=True, exist_ok=True)
    out.write_text(json.dumps(rows))
    for row in rows:
        print(json.dumps(row))


if __name__ == "__main__":
    main()
