#!/usr/bin/env python
"""Same-box comparison with the reference's two GPU attention paths on the bench workload
(BASELINE.md section 2): R-fi = FlashInfer fa2 wrappers with page_size 1 (python/minisgl/attention/
fi.py), R-trtllm = FlashInfer's TRT-LLM-gen sm100a FMHA cubins with page_size 64
(python/minisgl/attention/trtllm.py; what the reference auto-selects on sm_100).  FlashInfer is called
with exactly the keyword usage of those files; the reference's own tvm-ffi store kernel cannot be
built here, so the KV append in front of the FlashInfer calls uses our store kernel (same bytes).

Per layer and step: [KV append +] attention, layers on distinct pool slices (L2-cold), CUDA events,
median over repetitions.  Also prints output differences (ours vs fi vs trtllm) on layer 0.

    FLASHINFER_WORKSPACE_BASE=oracle/_ref/flashinfer_ws python tools/flashinfer_compare.py
"""
import argparse
import importlib
import json
import os
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
os.environ.setdefault("FLASHINFER_WORKSPACE_BASE", str(ROOT / "oracle" / "_ref" / "flashinfer_ws"))
import bench  # noqa: E402


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def relerr(a, b):
    a, b = a.float(), b.float()
    return (a - b).abs().max().item() / b.abs().max().item(), ((a - b).norm() / b.norm()).item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=8)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iter", type=int, default=500)
    args = ap.parse_args()
    import flashinfer
    from flashinfer.decode import trtllm_batch_decode_with_kv_cache
    from flashinfer.prefill import trtllm_batch_context_with_kv_cache

    bench.L = args.layers
    L = args.layers
    pkg = importlib.import_module("mini-sglang_b200")
    pkg.build_native()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    sched = bench.Schedule()
    PS = 64
    r = bench.AttentionPathRunner(pkg, sched, bench.HQ, bench.HKV, PS, dev)
    hq, hkv, D = r.hq, r.hkv, bench.D
    scale = D**-0.5
    peaks = bench.load_peaks()
    res = {"flashinfer": flashinfer.__version__, "layers": L, "page_size": PS}
    ws_fi = torch.empty(128 * 1024 * 1024, dtype=torch.uint8, device=dev)
    ws_trt = torch.zeros(128 * 1024 * 1024, dtype=torch.uint8, device=dev)

    def pool(l):
        return r.pool.k_cache(l), r.pool.v_cache(l)

    with torch.cuda.stream(r.stream):
        # ------------------------------------------------------------------ decode
        tr = sched.live(args.iter)
        batch = r.make_batch(tr, "decode", pad=False)
        bs = len(tr)
        pos_h, loc_h = r.host_inputs(batch)
        batch.positions, batch.out_loc = pos_h.to(dev), loc_h.to(dev)
        r.backend.prepare_metadata(batch)
        md = batch.attn_metadata
        qs = [r.qkv_views(l, bs) for l in range(L)]
        nbytes = bench.decode_bytes_per_layer(tr, hq, hkv)

        def ours_decode():
            for l in range(L):
                q, k, v = qs[l]
                ours_decode.out = r.backend.forward(q.view(bs, hq, D), k, v, l, batch)

        # R-fi: page_size 1 view, flat indices, plan once per batch (fi.py:123-166)
        seq_cpu = md.cache_seqlens.cpu()
        cu_k_cpu = md.cu_seqlens_k.cpu()
        indices = md.flat_indices()
        dec = flashinfer.BatchDecodeWithPagedKVCacheWrapper(ws_fi, kv_layout="NHD", use_tensor_cores=False, backend="fa2")
        dec.plan(indptr=cu_k_cpu, indices=indices, last_page_len=torch.ones(bs, dtype=torch.int32), num_qo_heads=hq,
                 num_kv_heads=hkv, head_dim=D, page_size=1, pos_encoding_mode="NONE", seq_lens=seq_cpu,
                 data_type=torch.bfloat16, q_data_type=torch.bfloat16, kv_data_type=torch.bfloat16, non_blocking=True)

        def fi_decode():
            for l in range(L):
                q, k, v = qs[l]
                r.pool.store_kv(k, v, batch.out_loc, l)
                kc, vc = pool(l)
                fi_decode.out = dec.run(q=q.reshape(bs, hq, D), paged_kv_cache=(kc.view(-1, 1, hkv, D), vc.view(-1, 1, hkv, D)))

        # R-trtllm: real pages, block table = every 64th slot // 64 (trtllm.py:117-122)
        block_tables = md.paged_page_table(PS).contiguous()

        def trt_decode():
            for l in range(L):
                q, k, v = qs[l]
                r.pool.store_kv(k, v, batch.out_loc, l)
                trt_decode.out = trtllm_batch_decode_with_kv_cache(
                    query=q.reshape(bs, hq, D), kv_cache=pool(l), workspace_buffer=ws_trt, block_tables=block_tables,
                    seq_lens=md.cache_seqlens, max_seq_len=md.max_seqlen_k, bmm1_scale=scale, bmm2_scale=1.0,
                    kv_layout="NHD", out_dtype=torch.bfloat16)

        for name, fn in (("b200", ours_decode), ("fi", fi_decode), ("trtllm", trt_decode)):
            try:
                fn()
                torch.cuda.synchronize()
                ms = timed(fn, args.reps) / L
                res[f"decode_{name}_us_per_layer"] = round(ms * 1e3, 1)
                res[f"decode_{name}_GBs"] = round(nbytes / ms / 1e6, 0)
                res[f"decode_{name}_frac_hbm"] = round(nbytes / ms / 1e6 / peaks["hbm_gbs"], 3)
            except Exception as e:  # keep going: one missing path must not hide the others
                res[f"decode_{name}_error"] = f"{type(e).__name__}: {str(e)[:200]}"
        # outputs of the last layer, same inputs (append is idempotent)
        try:
            res["decode_b200_vs_fi"] = relerr(ours_decode.out, fi_decode.out)
            res["decode_b200_vs_trtllm"] = relerr(ours_decode.out, trt_decode.out)
            res["decode_fi_vs_trtllm"] = relerr(fi_decode.out, trt_decode.out)
        except Exception as e:
            res["decode_cmp_error"] = str(e)[:200]
        print(json.dumps(res), flush=True)

        # ------------------------------------------------------------------ prefill (first prompt batch)
        trp = sched.prefill_batches()[1]
        pb = r.make_batch(trp, "prefill")
        pos_h, loc_h = r.host_inputs(pb)
        nnz = pos_h.numel()
        pb.positions, pb.out_loc = pos_h.to(dev), loc_h.to(dev)
        r.backend.prepare_metadata(pb)
        pmd = pb.attn_metadata
        qkv = torch.randn((nnz, r.width), device=dev, dtype=torch.bfloat16)
        q, k, v = qkv.split([hq * D, hkv * D, hkv * D], dim=-1)
        flops = bench.prefill_flops_per_layer(trp, hq)

        def ours_prefill():
            for l in range(L):
                ours_prefill.out = r.backend.forward(q.view(nnz, hq, D), k, v, l, pb)

        pre = flashinfer.BatchPrefillWithPagedKVCacheWrapper(ws_fi, kv_layout="NHD", backend="fa2")
        pre.plan(qo_indptr=pmd.cu_seqlens_q.cpu(), paged_kv_indptr=pmd.cu_seqlens_k.cpu(), paged_kv_indices=pmd.flat_indices(),
                 paged_kv_last_page_len=torch.ones(len(trp), dtype=torch.int32), num_qo_heads=hq, num_kv_heads=hkv,
                 head_dim_qk=D, page_size=1, pos_encoding_mode="NONE", seq_lens=pmd.cache_seqlens.cpu(),
                 q_data_type=torch.bfloat16, kv_data_type=torch.bfloat16, non_blocking=True, causal=True)
        qc = q.reshape(nnz, hq, D).contiguous()

        def fi_prefill():
            for l in range(L):
                r.pool.store_kv(k, v, pb.out_loc, l)
                kc, vc = pool(l)
                fi_prefill.out = pre.run(q=qc, paged_kv_cache=(kc.view(-1, 1, hkv, D), vc.view(-1, 1, hkv, D)))

        pbt = pmd.paged_page_table(PS).contiguous()

        def trt_prefill():
            for l in range(L):
                r.pool.store_kv(k, v, pb.out_loc, l)
                trt_prefill.out = trtllm_batch_context_with_kv_cache(
                    query=qc, kv_cache=pool(l), workspace_buffer=ws_trt, block_tables=pbt, seq_lens=pmd.cache_seqlens,
                    max_q_len=pmd.max_seqlen_q, max_kv_len=pmd.max_seqlen_k, bmm1_scale=scale, bmm2_scale=1.0,
                    cum_seq_lens_q=pmd.cu_seqlens_q, cum_seq_lens_kv=pmd.cu_seqlens_k, kv_layout="NHD",
                    batch_size=len(trp), out_dtype=torch.bfloat16)

        for name, fn in (("b200", ours_prefill), ("fi", fi_prefill), ("trtllm", trt_prefill)):
            try:
                fn()
                torch.cuda.synchronize()
                ms = timed(fn, args.reps) / L
                res[f"prefill_{name}_ms_per_layer"] = round(ms, 4)
                res[f"prefill_{name}_TFs"] = round(flops / ms / 1e9, 1)
            except Exception as e:
                res[f"prefill_{name}_error"] = f"{type(e).__name__}: {str(e)[:200]}"
        try:
            res["prefill_b200_vs_fi"] = relerr(ours_prefill.out, fi_prefill.out)
            res["prefill_b200_vs_trtllm"] = relerr(ours_prefill.out, trt_prefill.out)
            res["prefill_fi_vs_trtllm"] = relerr(fi_prefill.out, trt_prefill.out)
        except Exception as e:
            res["prefill_cmp_error"] = str(e)[:200]
    print(json.dumps(res))
    os.makedirs(ROOT / "gpurun_out", exist_ok=True)
    (ROOT / "gpurun_out" / "flashinfer_compare.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
