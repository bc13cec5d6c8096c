#!/usr/bin/env python
"""Golden outputs of the reference's TWO GPU attention paths at the BASELINE head shapes, produced on the
GPU by calling FlashInfer exactly as the reference's backends do:

  * "fi":     BatchDecode / BatchPrefillWithPagedKVCacheWrapper, backend "fa2", page_size-1 view
              (python/minisgl/attention/fi.py:93-103,134-165,185-188; use_tensor_cores = GQA >= 4, fi.py:235-241)
  * "trtllm": trtllm_batch_decode / context_with_kv_cache on real pages
              (python/minisgl/attention/trtllm.py:57-89; page table = every page_size-th slot // page_size,
              trtllm.py:117-122)

Inputs are NOT stored: every case is rebuilt from its seed by tests/helpers.make_world / make_inputs (torch
CPU generators), so the file holds only the case table and the 16-bit reference outputs.  Shapes: Qwen3-0.6B
(Hq 16 / Hkv 8) with page 1 and 64, a GQA-5 shape (Qwen3-14B's ratio) and the GQA-8 tp-shard shape of
Llama-3.1-70B (Hq 8 / Hkv 1), decode + prefill (with cached prefixes), and one 4096-row prefill whose
output is stored for every 16th row only.

    FLASHINFER_WORKSPACE_BASE=oracle/_ref/flashinfer_ws python tests/golden/make_reference_gpu_golden.py
    -> gpurun_out/reference_gpu_golden.npz (commit as tests/golden/reference_gpu_golden.npz)
"""
import importlib
import json
import os
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
os.environ.setdefault("FLASHINFER_WORKSPACE_BASE", str(ROOT / "oracle" / "_ref" / "flashinfer_ws"))

D = 128
CASES = [
    # name, phase, hq, hkv, page_size (pool layout), lens [(cached, total)], row_step (store every n-th output row)
    dict(name="dec_q16kv8_p1", phase="decode", hq=16, hkv=8, ps=1, lens=[(69, 70), (199, 200), (332, 333), (0, 1), (1023, 1024)], step=1),
    dict(name="dec_q16kv8_p64", phase="decode", hq=16, hkv=8, ps=64, lens=[(63, 64), (64, 65), (511, 512), (900, 901), (127, 128), (0, 1)], step=1),
    dict(name="dec_q10kv2_p64", phase="decode", hq=10, hkv=2, ps=64, lens=[(99, 100), (700, 701), (256, 257)], step=1),
    dict(name="dec_q8kv1_p64", phase="decode", hq=8, hkv=1, ps=64, lens=[(4096, 4097), (4351, 4352), (130, 131)], step=1),
    dict(name="pre_q16kv8_p1", phase="prefill", hq=16, hkv=8, ps=1, lens=[(0, 70), (37, 150), (0, 1), (5, 6)], step=1),
    dict(name="pre_q16kv8_p64", phase="prefill", hq=16, hkv=8, ps=64, lens=[(0, 129), (64, 200), (128, 129)], step=1),
    dict(name="pre_q10kv2_p64", phase="prefill", hq=10, hkv=2, ps=64, lens=[(0, 200), (64, 130)], step=1),
    dict(name="pre_q8kv1_p64", phase="prefill", hq=8, hkv=1, ps=64, lens=[(0, 300), (192, 260)], step=1),
    dict(name="pre_q8kv1_p64_long", phase="prefill", hq=8, hkv=1, ps=64, lens=[(0, 4096)], step=16),
]


def u16(t):
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def build_case(c, helpers, o_meta):
    """World + inputs of a case, deterministically from its name (shared with the test)."""
    seed = sum(ord(ch) for ch in c["name"])
    w = helpers.make_world(seed=seed, page_size=c["ps"], hq=c["hq"], hkv=c["hkv"], max_reqs=len(c["lens"]),
                           max_seq=max(t for _, t in c["lens"]) + 8)
    helpers.add_requests(w, c["lens"])
    md = o_meta.ref_prepare_metadata(w.page_table, w.reqs, c["ps"])
    qkv, q, k, v = helpers.make_inputs(w, seed + 1)
    return w, md, qkv


def main():
    import flashinfer
    from flashinfer.decode import trtllm_batch_decode_with_kv_cache
    from flashinfer.prefill import trtllm_batch_context_with_kv_cache

    import helpers
    from oracle import metadata as o_meta
    from oracle import tolerance

    pkg = importlib.import_module("mini-sglang_b200")
    pkg.build_native()
    dev = torch.device("cuda")
    out, report = {"cases": np.frombuffer(json.dumps(CASES).encode(), dtype=np.uint8)}, []
    ws = torch.empty(128 * 1024 * 1024, dtype=torch.uint8, device=dev)
    ws_trt = torch.zeros(128 * 1024 * 1024, dtype=torch.uint8, device=dev)
    for c in CASES:
        hq, hkv, ps, phase = c["hq"], c["hkv"], c["ps"], c["phase"]
        w, md, qkv = build_case(c, helpers, o_meta)
        gw = helpers.GpuWorld(pkg, w)
        g = qkv.to(dev)
        qg, kg, vg = g.split([hq * D, hkv * D, hkv * D], dim=-1)
        nnz = g.shape[0]
        # reference order: store_kv, then attention over the pool (fi.py:185-188)
        kc = gw.pool.k_cache(0).reshape(-1, hkv, D).clone()
        vc = gw.pool.v_cache(0).reshape(-1, hkv, D).clone()
        loc = torch.from_numpy(md.out_loc).to(dev).long()
        kc[loc] = kg.reshape(-1, hkv, D)
        vc[loc] = vg.reshape(-1, hkv, D)
        q3 = qg.reshape(nnz, hq, D).contiguous()
        cu_k, cu_q = torch.from_numpy(md.cu_seqlens_k), torch.from_numpy(md.cu_seqlens_q)
        seq = torch.from_numpy(md.cache_seqlens)
        ones = torch.ones(len(w.reqs), dtype=torch.int32)
        kv1 = (kc.view(-1, 1, hkv, D), vc.view(-1, 1, hkv, D))
        if phase == "decode":
            wr = flashinfer.BatchDecodeWithPagedKVCacheWrapper(ws, kv_layout="NHD", use_tensor_cores=(hq // hkv) >= 4, backend="fa2")
            wr.plan(indptr=cu_k, indices=torch.from_numpy(md.indices_flat).to(dev), last_page_len=ones, num_qo_heads=hq,
                    num_kv_heads=hkv, head_dim=D, page_size=1, pos_encoding_mode="NONE", seq_lens=seq, data_type=torch.bfloat16,
                    q_data_type=torch.bfloat16, kv_data_type=torch.bfloat16, non_blocking=True)
        else:
            wr = flashinfer.BatchPrefillWithPagedKVCacheWrapper(ws, kv_layout="NHD", backend="fa2")
            wr.plan(qo_indptr=cu_q, paged_kv_indptr=cu_k, paged_kv_indices=torch.from_numpy(md.indices_flat).to(dev),
                    paged_kv_last_page_len=ones, num_qo_heads=hq, num_kv_heads=hkv, head_dim_qk=D, page_size=1,
                    pos_encoding_mode="NONE", seq_lens=seq, q_data_type=torch.bfloat16, kv_data_type=torch.bfloat16,
                    non_blocking=True, causal=True)
        fi_out = wr.run(q=q3, paged_kv_cache=kv1)
        trt_out = None
        if ps in (16, 32, 64):
            kvp = (kc.view(-1, ps, hkv, D), vc.view(-1, ps, hkv, D))
            bt = torch.from_numpy(md.page_table_paged).to(dev).contiguous()
            seq_d = seq.to(dev)
            try:
                if phase == "decode":
                    trt_out = trtllm_batch_decode_with_kv_cache(
                        query=q3, kv_cache=kvp, workspace_buffer=ws_trt, block_tables=bt, seq_lens=seq_d,
                        max_seq_len=int(md.max_seqlen_k), bmm1_scale=D**-0.5, bmm2_scale=1.0, kv_layout="NHD",
                        out_dtype=torch.bfloat16)
                else:
                    trt_out = trtllm_batch_context_with_kv_cache(
                        query=q3, kv_cache=kvp, workspace_buffer=ws_trt, block_tables=bt, seq_lens=seq_d,
                        max_q_len=int(md.max_seqlen_q), max_kv_len=int(md.max_seqlen_k), bmm1_scale=D**-0.5, bmm2_scale=1.0,
                        cum_seq_lens_q=cu_q.to(dev), cum_seq_lens_kv=cu_k.to(dev), kv_layout="NHD",
                        batch_size=len(w.reqs), out_dtype=torch.bfloat16)
            except Exception as e:  # record, keep going
                report.append(f"{c['name']}: trtllm failed: {type(e).__name__}: {str(e)[:160]}")
        # ours on the same inputs, for the record
        batch = gw.batch(phase)
        batch.out_loc = torch.from_numpy(md.out_loc).to(dev)
        batch.positions = torch.from_numpy(md.positions).to(dev)
        gw.backend.prepare_metadata(batch)
        ours = gw.backend.forward(qg.view(-1, hq, D), kg, vg, 0, batch)
        torch.cuda.synchronize()
        st = c["step"]
        out[c["name"] + "_fi"] = u16(fi_out[::st])
        line = f"{c['name']}: b200 vs fi {tolerance.vs_reference_gpu(ours, fi_out):.2e}"
        if trt_out is not None:
            out[c["name"] + "_trtllm"] = u16(trt_out[::st])
            line += f", b200 vs trtllm {tolerance.vs_reference_gpu(ours, trt_out):.2e}, trtllm vs fi {tolerance.vs_reference_gpu(trt_out, fi_out):.2e}"
        report.append(line + "   (excess over one output ulp / max|ref|; gate 1e-3)")
        pkg.core.set_global_ctx(None)
    os.makedirs(ROOT / "gpurun_out", exist_ok=True)
    np.savez_compressed(ROOT / "gpurun_out" / "reference_gpu_golden.npz", **out)
    (ROOT / "gpurun_out" / "reference_gpu_parity.txt").write_text("\n".join(report) + "\n")
    print("\n".join(report))
    print("flashinfer", flashinfer.__version__, "wrote gpurun_out/reference_gpu_golden.npz")


if __name__ == "__main__":
    main()
