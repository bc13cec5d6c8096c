#!/usr/bin/env python
"""Pre-compile (on the CPU build box, no GPU needed) the FlashInfer JIT modules the reference's
attention path uses, into oracle/_ref/flashinfer_ws -- git-ignored, but shipped to the GPU box with
the snapshot, so that tools/flashinfer_compare.py does not spend GPU-box minutes in nvcc.

Modules = exactly what the reference's call sites instantiate for Qwen3-0.6B / bf16:
  fi.py:93-103  BatchPrefill/BatchDecode wrappers, backend "fa2", NHD, pos_encoding NONE
  trtllm.py:52-53 trtllm_batch_{context,decode}_with_kv_cache  (TRT-LLM-gen launcher; kernels are cubins)
  rotary.py:35  apply_rope_with_cos_sin_cache_inplace ; norm.py:10,25 rmsnorm / fused_add_rmsnorm
  activation.py:10 silu_and_mul (GatedMLP.forward, models/utils.py:48)
The target is the H100 (9.0a) unless FLASHINFER_CUDA_ARCH_LIST says otherwise.
"""
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
WS = ROOT / "oracle" / "_ref" / "flashinfer_ws"
os.environ["FLASHINFER_WORKSPACE_BASE"] = str(WS)
os.environ.setdefault("FLASHINFER_CUDA_ARCH_LIST", "9.0a")
os.environ.setdefault("MAX_JOBS", str(os.cpu_count() or 8))

import torch  # noqa: E402
from flashinfer.jit.activation import gen_act_and_mul_module  # noqa: E402
from flashinfer.jit.attention.modules import gen_batch_decode_module, gen_batch_prefill_module  # noqa: E402
from flashinfer.jit.norm import gen_norm_module  # noqa: E402
from flashinfer.jit.rope import gen_rope_module  # noqa: E402

bf = torch.bfloat16
specs = [
    gen_batch_decode_module(bf, bf, bf, torch.int32, 128, 128, 0, False, False),
    gen_batch_prefill_module("fa2", bf, bf, bf, torch.int32, 128, 128, 0, False, False, False),
    gen_rope_module(),
    gen_norm_module(),
    gen_act_and_mul_module("silu"),
]
try:
    from flashinfer.jit.attention.modules import gen_trtllm_gen_fmha_module

    specs.append(gen_trtllm_gen_fmha_module())
except Exception as e:  # pragma: no cover
    print("trtllm-gen module generator unavailable:", e)

for s in specs:
    print("building", s.name, flush=True)
    try:
        s.build(verbose=False)
        print("  ->", s.get_library_path(), flush=True)
    except Exception as e:
        print("  FAILED:", type(e).__name__, str(e)[:300], flush=True)
