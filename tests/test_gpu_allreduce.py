"""Multi-GPU parity of the one-shot NVLink all-reduce (csrc/allreduce.cu, SURVEY 8(f) rank 4): spawns
tools/ar_check.py under torch.distributed.run with 2 ranks (needs >= 2 GPUs; skipped on a 1-GPU box --
run `python -m pytest tests/test_gpu_allreduce.py -m gpu` on a machine with two).  The checks themselves
(bit-exact rank-order fp32 sum, identical bits on all ranks, == NCCL at world 2, fused residual +
RMSNorm == unfused sequence, CUDA-graph replay, 1500-call stress, the reference's plug-in point) are
documented in tools/ar_check.py."""
import json
import subprocess
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("world", [2])
def test_allreduce_checks(world, native_lib):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", "29517", str(ROOT / "tools" / "ar_check.py"),
           "--skip-timing"]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=str(ROOT))
    out = res.stdout.decode(errors="replace")
    assert res.returncode == 0, out[-4000:]
    line = [l for l in out.splitlines() if l.startswith("{")][-1]
    summary = json.loads(line)
    assert summary["ok_all_ranks"], summary
    assert all(summary["checks"].values()), summary
