#!/usr/bin/env python
"""Golden vectors for the FLOATING-POINT side of the boundary, produced on the GPU by calling
FlashInfer exactly the way the reference's call sites do (the reference's arithmetic for this path
lives in flashinfer-python, pinned >=0.5.3 in its pyproject.toml:30; 0.6.11.post2 in this image):

  * decode / prefill attention: BatchDecode/BatchPrefillWithPagedKVCacheWrapper, backend "fa2",
    kv_layout NHD, page_size 1 view of the pool, pos_encoding "NONE", causal
    (python/minisgl/attention/fi.py:82-103,134-165,176-188)
  * RoPE: flashinfer.apply_rope_with_cos_sin_cache_inplace   (python/minisgl/layers/rotary.py:45-51)
  * RMSNorm: flashinfer.rmsnorm (2-D and per-head 3-D), fused_add_rmsnorm (layers/norm.py:16-38)

Run on the GPU box (JIT modules are pre-built by tools/flashinfer_prebuild.py):

    FLASHINFER_WORKSPACE_BASE=oracle/_ref/flashinfer_ws python tests/golden/make_flashinfer_golden.py

Writes gpurun_out/flashinfer_golden.npz (inputs + FlashInfer outputs, bf16 stored as uint16); the
file is then committed as tests/golden/flashinfer_golden.npz and checked by
tests/test_oracle_golden.py (oracle vs FlashInfer) -- and this script prints, for the record, how
the project's kernels compare with FlashInfer on the same inputs.
"""
import importlib
import os
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
os.environ.setdefault("FLASHINFER_WORKSPACE_BASE", str(ROOT / "oracle" / "_ref" / "flashinfer_ws"))

import flashinfer  # noqa: E402

from helpers import GpuWorld, add_requests, make_inputs, make_world  # noqa: E402
from oracle import metadata as o_meta  # noqa: E402

HQ, HKV, D, PS = 4, 2, 128, 16
dev = torch.device("cuda")


def u16(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def fi_attention(phase, w, md, qg, kc, vc):
    """The reference's FlashInferBackend.forward after store_kv: plan once, run."""
    ws = torch.empty(128 * 1024 * 1024, dtype=torch.uint8, device=dev)
    cu_k = torch.from_numpy(md.cu_seqlens_k)
    cu_q = torch.from_numpy(md.cu_seqlens_q)
    indices = torch.from_numpy(md.indices_flat).to(dev)
    ones = torch.ones(len(w.reqs), dtype=torch.int32)
    seq = torch.from_numpy(md.cache_seqlens)
    kv = (kc.view(-1, 1, HKV, D), vc.view(-1, 1, HKV, D))
    if phase == "decode":
        wr = flashinfer.BatchDecodeWithPagedKVCacheWrapper(ws, kv_layout="NHD", use_tensor_cores=False, backend="fa2")
        wr.plan(indptr=cu_k, indices=indices, last_page_len=ones, num_qo_heads=HQ, num_kv_heads=HKV,
                head_dim=D, page_size=1, pos_encoding_mode="NONE", seq_lens=seq, data_type=torch.bfloat16,
                q_data_type=torch.bfloat16, kv_data_type=torch.bfloat16, non_blocking=True)
    else:
        wr = flashinfer.BatchPrefillWithPagedKVCacheWrapper(ws, kv_layout="NHD", backend="fa2")
        wr.plan(qo_indptr=cu_q, paged_kv_indptr=cu_k, paged_kv_indices=indices, paged_kv_last_page_len=ones,
                num_qo_heads=HQ, num_kv_heads=HKV, head_dim_qk=D, page_size=1, pos_encoding_mode="NONE",
                seq_lens=seq, q_data_type=torch.bfloat16, kv_data_type=torch.bfloat16, non_blocking=True,
                causal=True)
    return wr.run(q=qg, paged_kv_cache=kv)


def main():
    pkg = importlib.import_module("mini-sglang_b200")
    pkg.build_native()
    out = {}
    report = []
    cases = {
        "decode": [(69, 70), (199, 200), (332, 333), (0, 1), (63, 64)],
        "prefill": [(0, 150), (64, 200), (0, 1), (32, 33), (0, 129)],
    }
    for phase, lens in cases.items():
        w = make_world(seed=7, page_size=PS, hq=HQ, hkv=HKV, max_reqs=len(lens), max_seq=512)
        add_requests(w, lens)
        md = o_meta.ref_prepare_metadata(w.page_table, w.reqs, PS)
        qkv, q, k, v = make_inputs(w, 8)
        gw = GpuWorld(pkg, w)
        g = qkv.to(dev)
        qg, kg, vg = g.split([HQ * D, HKV * D, HKV * D], dim=-1)
        # ---- reference order: store_kv, then attention over the pool (fi.py:185-188)
        kc = gw.pool.k_cache(0).reshape(-1, HKV, D).clone()
        vc = gw.pool.v_cache(0).reshape(-1, HKV, D).clone()
        loc = torch.from_numpy(md.out_loc).to(dev).long()
        kc[loc] = kg.reshape(-1, HKV, D)
        vc[loc] = vg.reshape(-1, HKV, D)
        fi_out = fi_attention(phase, w, md, qg.reshape(-1, HQ, D).contiguous(), kc, vc)
        # ---- ours on the same inputs
        batch = gw.batch(phase)
        batch.out_loc = torch.from_numpy(md.out_loc).to(dev)
        batch.positions = torch.from_numpy(md.positions).to(dev)
        gw.backend.prepare_metadata(batch)
        ours = gw.backend.forward(qg.view(-1, HQ, D), kg, vg, 0, batch)
        torch.cuda.synchronize()
        a, b = ours.float(), fi_out.float()
        err = (a - b).abs().max().item() / b.abs().max().item()
        fro = ((a - b).norm() / b.norm()).item()
        report.append(f"{phase}: project kernel vs FlashInfer fa2: max|d|/max|ref| = {err:.2e}, rel_fro = {fro:.2e}")
        used = np.unique(np.concatenate([md.slot_table[i, : md.cache_seqlens[i]] for i in range(len(w.reqs))]))
        out[f"{phase}_reqs"] = np.array(w.reqs, dtype=np.int32)
        out[f"{phase}_page_table"] = w.page_table
        out[f"{phase}_q"] = u16(q.reshape(-1, HQ, D))
        out[f"{phase}_used_slots"] = used.astype(np.int32)
        out[f"{phase}_k_rows"] = u16(kc[torch.from_numpy(used).to(dev).long()])
        out[f"{phase}_v_rows"] = u16(vc[torch.from_numpy(used).to(dev).long()])
        out[f"{phase}_out"] = u16(fi_out)
        pkg.core.set_global_ctx(None)

    # ---- RoPE
    torch.manual_seed(3)
    nnz, max_pos = 37, 1024
    from oracle.rope import ref_cos_sin_cache

    cache = ref_cos_sin_cache(D, max_pos, 1e6)
    x = torch.randn(nnz, (HQ + 2 * HKV) * D).to(torch.bfloat16)
    pos = torch.randint(0, max_pos, (nnz,), dtype=torch.int32)
    xg = x.to(dev)
    flashinfer.apply_rope_with_cos_sin_cache_inplace(positions=pos.to(dev), query=xg[:, : HQ * D],
                                                     key=xg[:, HQ * D : (HQ + HKV) * D], head_size=D,
                                                     cos_sin_cache=cache.to(dev))
    mine = x.to(dev)
    pkg.ops.apply_rope_with_cos_sin_cache_inplace(pos.to(dev), mine[:, : HQ * D], mine[:, HQ * D : (HQ + HKV) * D], D, cache.to(dev))
    out["rope_x"], out["rope_pos"], out["rope_out"] = u16(x), pos.numpy(), u16(xg)
    report.append(f"rope: project kernel vs FlashInfer bit-identical = {bool(torch.equal(mine.view(torch.int16), xg.view(torch.int16)))}, "
                  f"max |d| = {(mine.float() - xg.float()).abs().max().item():.3e}")

    # ---- RMSNorm (2-D), per-head (3-D, in place), fused add
    xn = (torch.randn(19, 1024) * 2).to(torch.bfloat16)
    wn = (torch.rand(1024) + 0.5).to(torch.bfloat16)
    yn = flashinfer.rmsnorm(xn.to(dev), wn.to(dev), 1e-6)
    mine = pkg.ops.rmsnorm(xn.to(dev), wn.to(dev), 1e-6)
    report.append(f"rmsnorm: bit-identical = {bool(torch.equal(mine.view(torch.int16), yn.view(torch.int16)))}, max |d| = {(mine.float()-yn.float()).abs().max().item():.3e}")
    xh = torch.randn(23, HQ, D).to(torch.bfloat16)
    wh = (torch.rand(D) + 0.5).to(torch.bfloat16)
    yh = xh.to(dev)
    flashinfer.rmsnorm(yh, wh.to(dev), 1e-6, out=yh)
    xr, rr = torch.randn(11, 1024).to(torch.bfloat16), torch.randn(11, 1024).to(torch.bfloat16)
    xf, rf = xr.to(dev), rr.to(dev)
    flashinfer.fused_add_rmsnorm(xf, rf, wn.to(dev), 1e-6)
    m1, m2 = xr.to(dev), rr.to(dev)
    pkg.ops.fused_add_rmsnorm(m1, m2, wn.to(dev), 1e-6)
    report.append(f"fused_add_rmsnorm: x bit-identical = {bool(torch.equal(m1.view(torch.int16), xf.view(torch.int16)))}, "
                  f"residual bit-identical = {bool(torch.equal(m2.view(torch.int16), rf.view(torch.int16)))}")
    out.update(norm_x=u16(xn), norm_w=u16(wn), norm_out=u16(yn), qknorm_x=u16(xh), qknorm_w=u16(wh), qknorm_out=u16(yh),
               fused_x=u16(xr), fused_res=u16(rr), fused_x_out=u16(xf), fused_res_out=u16(rf))
    os.makedirs(ROOT / "gpurun_out", exist_ok=True)
    np.savez_compressed(ROOT / "gpurun_out" / "flashinfer_golden.npz", **out)
    (ROOT / "gpurun_out" / "flashinfer_parity.txt").write_text("\n".join(report) + "\n")
    print("\n".join(report))
    print("flashinfer", flashinfer.__version__, "wrote gpurun_out/flashinfer_golden.npz")


if __name__ == "__main__":
    main()
