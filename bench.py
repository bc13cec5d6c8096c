#!/usr/bin/env python
"""bench.py -- BASELINE.json's metric on BASELINE.json's config, for the attention hot path.

Workload (config.workload = "cfg1"): exactly the token schedule of the reference's
benchmark/offline/bench.py:10-38 replayed from its RNG (random.seed(0); 256 prompts
len~randint(100,1024); max_tokens~randint(100,1024)), Qwen3-0.6B attention shape
(L=28, Hq=16, Hkv=8, D=128, bf16), KV pool + page table laid out as the engine does
(python/minisgl/engine/engine.py:55-73), pages handed out in random order.

A "step" = one decode iteration of the schedule pushed through the hot path for all 28 layers:
    prepare_metadata  ->  per layer: fused qk-norm+RoPE  ->  attention (+ fused KV append)
driven the way the reference's engine drives its backend (static buffers + CUDA-graph replay,
engine/graph.py:105-158).  K timed steps are spread evenly over the 1023 decode iterations.
Each layer has its own pool slice, so one step reads gigabytes, far more than the 50 MB L2 of an H100.

Prints ONE JSON line: value = decode tokens/s (device-timed, inputs
resident), e2e = same through the plugin API with host buffers, roofline for the decode kernel,
cpu_baseline (the oracle on the host cores, bounded sample), prefill TFLOP/s as an extra key.
`--impl reference` times the CPU oracle (the reference has no CPU implementation of this path,
its arithmetic is CUDA-only FlashInfer; see DESIGN.md) on the same workload.
`--dump-outputs DIR` writes what the last timed step computed (see dump_outputs) so that two builds can
be compared output for output; the inputs are seeded, so the same arguments give the same inputs.
"""

from __future__ import annotations

import argparse
import gc
import importlib
import json
import os
import random
import sys
import tempfile
import threading
import time
from pathlib import Path
from types import SimpleNamespace
from typing import List, Tuple

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

# ----------------------------------------------------------------------------- workload
D = 128
EPS = 1e-6


class Workload:
    """One BASELINE.json config made concrete (BASELINE.md section 3).  Head counts are the model's
    global ones; `tp_shard` > 1 means "the configuration is quoted at that TP degree": bench.py then
    runs ONE rank's shard of it per GPU (heads divided by tp_shard), which at N = tp_shard is the real
    thing and at N = 1 is one rank's share (no all-reduce partner)."""

    def __init__(self, name, model, layers, hq, hkv, hidden, num_seqs, max_extend, desc, tp_shard=1,
                 in_out=None, shared_prefix=0):
        self.name, self.model, self.L, self.hq, self.hkv, self.hidden = name, model, layers, hq, hkv, hidden
        self.num_seqs, self.max_extend, self.desc, self.tp_shard = num_seqs, max_extend, desc, tp_shard
        self.in_out, self.shared_prefix = in_out, shared_prefix


WORKLOADS = {
    # benchmark/offline/bench.py:10-38 -- the reference's headline run
    "cfg1": Workload("cfg1", "Qwen3-0.6B", 28, 16, 8, 1024, 256, 16384,
                     "256 seqs in/out U[100,1024] (reference bench.py RNG replay), radix cache off"),
    # same token schedule on the 14B shape, radix cache on: every prompt starts with a 256-token system
    # prefix that is already cached (cached_len = 256 extends), prompts chunked at max_extend_tokens 8192
    "cfg2": Workload("cfg2", "Qwen3-14B", 40, 40, 8, 5120, 256, 8192,
                     "256 seqs in/out U[100,1024] (same RNG replay), radix cache on: shared 256-token prefix "
                     "(page aligned) already cached, chunked prefill at 8192", shared_prefix=256),
    # Llama-3.1-70B shape at tp=8: per GPU Hq 8, Hkv 1 (GQA 8), long-context decode
    "cfg4": Workload("cfg4", "Llama-3.1-70B (random init)", 80, 64, 8, 8192, 64, 8192,
                     "64 seqs in=4096 out=256, tp=8 shard per GPU (Hq_l 8, Hkv_l 1)", tp_shard=8,
                     in_out=(4096, 256)),
}
WL = WORKLOADS["cfg1"]
# module-level views of the active workload (tools/ and tests/ read them)
L, HQ, HKV, HIDDEN = WL.L, WL.hq, WL.hkv, WL.hidden
NUM_SEQS, MAX_IN, MAX_OUT = 256, 1024, 1024
MAX_EXTEND_TOKENS = WL.max_extend


def set_workload(name: str) -> Workload:
    global WL, L, HQ, HKV, HIDDEN, NUM_SEQS, MAX_EXTEND_TOKENS
    WL = WORKLOADS[name]
    L, HQ, HKV, HIDDEN = WL.L, WL.hq // WL.tp_shard, max(1, WL.hkv // WL.tp_shard), WL.hidden
    NUM_SEQS, MAX_EXTEND_TOKENS = WL.num_seqs, WL.max_extend
    return WL


def replay_reference_rng() -> Tuple[List[int], List[int]]:
    """benchmark/offline/bench.py:11-31 -- the prompt token ids are drawn between the two length
    draws, so the RNG stream has to be replayed literally."""
    random.seed(0)
    in_lens = []
    for _ in range(256):
        n = random.randint(100, MAX_IN)
        for _ in range(n):
            random.randint(0, 10000)
        in_lens.append(n)
    out_lens = [random.randint(100, MAX_OUT) for _ in range(256)]
    return in_lens, out_lens


class Schedule:
    """Decode iteration i (0-based): request r is live while i < out_r - 1; its kv length in that
    iteration (including the token being appended) is in_r + i + 1."""

    def __init__(self, wl: "Workload | None" = None) -> None:
        wl = wl or WL
        self.wl = wl
        if wl.in_out is None:
            self.in_lens, self.out_lens = replay_reference_rng()
        else:
            self.in_lens, self.out_lens = [wl.in_out[0]] * wl.num_seqs, [wl.in_out[1]] * wl.num_seqs
        self.n_iters = max(self.out_lens) - 1
        self.decode_token_steps = sum(o - 1 for o in self.out_lens)
        self.sum_kv = sum(
            sum(range(i + 1, i + o)) for i, o in zip(self.in_lens, self.out_lens)
        )  # sum over decode steps of kv_len

    def live(self, it: int) -> List[Tuple[int, int, int]]:
        """(table_idx, cached_len, device_len) of the live requests at decode iteration `it`."""
        return [
            (r, i + it, i + it + 1)
            for r, (i, o) in enumerate(zip(self.in_lens, self.out_lens))
            if it < o - 1
        ]

    def sample_iters(self, k: int) -> List[int]:
        return [min(self.n_iters - 1, int((j + 0.5) * self.n_iters / k)) for j in range(k)]

    def prefill_batches(self) -> List[List[Tuple[int, int, int]]]:
        """Greedy admission under max_extend_tokens with chunk splitting
        (python/minisgl/scheduler/prefill.py:64-90,126-151).  A shared prefix that is already in the
        radix cache makes every request start at cached_len = prefix (page aligned,
        kvcache/radix_cache.py:137); without it cached_len = 0."""
        budget0, prefix = self.wl.max_extend, self.wl.shared_prefix
        batches, cur, budget = [], [], budget0
        for r, n in enumerate(self.in_lens):
            # match_prefix(input_ids[:n-1]), whole pages, and never more than request 0 (the prefix's owner) has
            done = min(prefix, (n - 1) // 64 * 64, (self.in_lens[0] - 1) // 64 * 64) if prefix else 0
            while done < n:
                if budget <= 0:
                    batches.append(cur)
                    cur, budget = [], budget0
                chunk = min(budget, n - done)
                cur.append((r, done, done + chunk))
                budget -= chunk
                done += chunk
        if cur:
            batches.append(cur)
        return batches


def decode_bytes_per_layer(triples, hq=HQ, hkv=HKV) -> int:
    """SURVEY.md 8(d): sum kv_len * 2*Hkv*D*2 + nnz * 2*Hkv*D*2 (append) + nnz * 2*Hq*D*2 (q, o)."""
    kv = sum(d for (_, _, d) in triples)
    n = len(triples)
    return kv * 2 * hkv * D * 2 + n * 2 * hkv * D * 2 + n * 2 * hq * D * 2


def prefill_flops_per_layer(triples, hq=HQ) -> int:
    tot = 0
    for (_, c, d) in triples:
        q = d - c
        tot += q * c + q * (q + 1) // 2
    return 4 * hq * D * tot


def prefill_bytes_per_layer(triples, hq=HQ, hkv=HKV) -> int:
    """Algorithmic HBM bytes of one prefill launch: q read + o written (nnz * 2*Hq*D*2), this forward's
    k, v read and appended (nnz * 2 * 2*Hkv*D*2), cached prefix K/V read once per kv head
    (sum cached * 2*Hkv*D*2).  K/V tiles shared by the q tiles of a request are counted once."""
    nnz = sum(d - c for (_, c, d) in triples)
    cached = sum(c for (_, c, _) in triples)
    return nnz * 2 * hq * D * 2 + nnz * 2 * 2 * hkv * D * 2 + cached * 2 * hkv * D * 2


def graph_bs_list(max_bs: int = 256) -> List[int]:
    return [1, 2, 4] + list(range(8, max_bs + 1, 8))  # engine/graph.py:67


def effective_cpus() -> int:
    """Cores this process may really use: affinity mask capped by the cgroup CPU quota (nproc can
    report the whole host inside a quota-limited container; oversubscribing makes torch crawl)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        txt = Path("/sys/fs/cgroup/cpu.max").read_text().split()
        if txt[0] != "max":
            n = min(n, max(1, int(int(txt[0]) / int(txt[1]))))
    except Exception:
        try:
            q = int(Path("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read_text())
            per = int(Path("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read_text())
            if q > 0:
                n = min(n, max(1, q // per))
        except Exception:
            pass
    return max(1, min(n, 64))


def flashinfer_workspace() -> str:
    """Where FlashInfer JIT-compiles (used when FLASHINFER_WORKSPACE_BASE is unset): the tree's
    oracle/_ref/flashinfer_ws -- the cache tools/flashinfer_prebuild.py fills and the golden / in-situ tools
    use -- when it exists and is writable, otherwise one fixed directory under the system temp dir, so that
    a read-only tree stays untouched and repeated runs reuse their compiled modules."""
    ws = ROOT / "oracle" / "_ref" / "flashinfer_ws"
    if ws.is_dir() and os.access(ws, os.W_OK):
        return str(ws)
    tmp = Path(tempfile.gettempdir()) / f"mini-sglang-flashinfer-ws-{os.getuid()}"
    tmp.mkdir(exist_ok=True)
    return str(tmp)


def load_peaks() -> dict:
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        d = json.loads(p.read_text())
        return {"hbm_gbs": d["hbm_gbs"], "bf16_tflops": d.get("bf16_tflops_sustained", d["bf16_tflops"]),
                "source": "measured"}
    # NVIDIA's data sheet for the H100 SXM (700 W): 3.35 TB/s HBM3, 989 dense BF16 TFLOP/s -- a ceiling to
    # divide by, not a rate any kernel reached
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "source": "H100 SXM data sheet"}


# ----------------------------------------------------------------------------- clocks
class ClockSampler:
    """Samples SM clock / throttle reasons with NVML while the timed region runs."""

    def __init__(self, index: int) -> None:
        self.samples, self.reasons, self.max_mhz = [], set(), None
        self._stop = threading.Event()
        self._thread = None
        try:
            import pynvml

            pynvml.nvmlInit()
            self.nv = pynvml
            self.h = pynvml.nvmlDeviceGetHandleByIndex(index)
            self.max_mhz = pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM)
        except Exception:
            self.nv = None

    def _run(self) -> None:
        nv = self.nv
        names = {
            "hw_slowdown": getattr(nv, "nvmlClocksEventReasonHwSlowdown", 0x8),
            "sw_power_cap": getattr(nv, "nvmlClocksEventReasonSwPowerCap", 0x4),
            "hw_thermal_slowdown": getattr(nv, "nvmlClocksEventReasonHwThermalSlowdown", 0x40),
            "sw_thermal_slowdown": getattr(nv, "nvmlClocksEventReasonSwThermalSlowdown", 0x20),
            "hw_power_brake": getattr(nv, "nvmlClocksEventReasonHwPowerBrakeSlowdown", 0x80),
        }
        while not self._stop.is_set():
            try:
                self.samples.append(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM))
                try:
                    mask = nv.nvmlDeviceGetCurrentClocksEventReasons(self.h)
                except Exception:
                    mask = nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h)
                for k, bit in names.items():
                    if mask & bit:
                        self.reasons.add(k)
            except Exception:
                pass
            time.sleep(0.02)

    def __enter__(self):
        if self.nv is not None:
            self._thread = threading.Thread(target=self._run, daemon=True)
            self._thread.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        if self._thread is not None:
            self._thread.join(timeout=1.0)

    def summary(self) -> dict:
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": self.max_mhz, "reasons": ["unavailable"]}
        return {"sm_mhz": float(np.median(self.samples)), "sm_max_mhz": self.max_mhz,
                "reasons": sorted(self.reasons)}


# ----------------------------------------------------------------------------- our arm
class AttentionPathRunner:
    """Static buffers + captured graphs around the backend, like engine/graph.py does for the
    whole model -- here for the attention path only (everything else is out of scope)."""

    def __init__(self, pkg, sched: Schedule, hq: int, hkv: int, page_size: int, device, world=1, tp_group=None,
                 allreduce: str = "b200", fuse_pre_attention: bool = False):
        # hq / hkv are the heads of this process' configuration; each TP rank owns hq/world, max(1, hkv/world)
        self.pkg, self.sched, self.page_size = pkg, sched, page_size
        self.hq, self.hkv = hq // world, max(1, hkv // world)
        self.dev = device
        self.tp_group = tp_group
        self.n_seqs = len(sched.in_lens)
        # TP all-reduce after o_proj (layers/linear.py:102-106), one per layer:
        #   "b200": the one-shot NVLink push kernel fused with the residual add + RMSNorm that follows
        #           (models/qwen3.py:38-41), launched per layer INSIDE the captured graph;
        #   "nccl": torch.distributed all_reduce issued eagerly behind the graph replay (round-1 behaviour)
        self.allreduce = allreduce if (world > 1 and tp_group is not None) else "none"
        self.ar = None
        if self.allreduce == "b200":
            d_mod = importlib.import_module("mini-sglang_b200.distributed")
            self.ar = d_mod.B200AllReduce(int(os.environ.get("RANK", "0")), world, tp_group, device,
                                          max_bytes=self.n_seqs * HIDDEN * 2)
        self.fuse_pre_attention = fuse_pre_attention
        g = torch.Generator(device=device).manual_seed(42)
        max_len = max(i + o for i, o in zip(sched.in_lens, sched.out_lens))
        self.max_seq = (max_len + 63) // 64 * 64
        pages_per_req = [-(-(i + o) // page_size) for i, o in zip(sched.in_lens, sched.out_lens)]
        self.num_pages = sum(pages_per_req)
        ctx = pkg.Context(page_size)
        pkg.core.set_global_ctx(None)
        pkg.set_global_ctx(ctx)
        self.pool = pkg.MHAKVCache(hkv, L, D, self.num_pages + 1, page_size, torch.bfloat16, device)
        for l in range(L):  # N(0,1) pool contents (SURVEY 8(d) kernel-level inputs)
            self.pool._kv_buffer[0, l].normal_(generator=g)
            self.pool._kv_buffer[1, l].normal_(generator=g)
        ctx.kv_cache = self.pool
        # page table: pages handed out in a random permutation (worst-case scatter)
        perm = np.random.RandomState(0).permutation(self.num_pages).astype(np.int64)
        table = np.zeros((self.n_seqs + 1, self.max_seq), dtype=np.int32)
        off = 0
        for r, n in enumerate(pages_per_req):
            slots = (perm[off : off + n, None] * page_size + np.arange(page_size)[None, :]).reshape(-1)
            table[r, : n * page_size] = slots[: self.max_seq] if n * page_size > self.max_seq else slots
            off += n
        if sched.wl.shared_prefix:
            # radix-shared prefix pages: a request's first pages are request 0's -- as many whole pages as its
            # prompt shares (match_prefix(input_ids[:n-1]), page aligned; prefill_batches() uses the same length),
            # so that no request ever appends into a shared page
            for r, n in enumerate(sched.in_lens):
                share = min(sched.wl.shared_prefix, (n - 1) // 64 * 64, (sched.in_lens[0] - 1) // 64 * 64)
                table[r, :share] = table[0, :share]
        table[self.n_seqs, :] = self.num_pages * page_size
        self.table_np = table
        ctx.page_table = torch.from_numpy(table).to(device)
        cfg = SimpleNamespace(num_qo_heads=hq, num_kv_heads=hkv, head_dim=D)
        self.backend = pkg.create_attention_backend("b200", cfg)
        ctx.attn_backend = self.backend
        self.ctx = ctx
        self.width = (self.hq + 2 * self.hkv) * D
        # static qkv input of the graphs: [request row][layer][q | k | v] -- the rows of a padded batch
        # are one contiguous block, so a step's host inputs arrive with ONE host-to-device copy
        self.qkv = torch.randn((self.n_seqs, L, self.width), device=device, dtype=torch.float32, generator=g).to(torch.bfloat16)
        self.last_out = {}
        self.layer_outs = {}  # padded bs -> the captured graph's attention output of every layer
        self.positions = torch.zeros(self.n_seqs, dtype=torch.int32, device=device)
        self.out_loc = torch.zeros(self.n_seqs, dtype=torch.int32, device=device)
        self.qw = (torch.rand(D, device=device, generator=g) + 0.5).to(torch.bfloat16)
        self.kw = (torch.rand(D, device=device, generator=g) + 0.5).to(torch.bfloat16)
        self.rotary = pkg.layers.RotaryEmbedding(D, D, max(4096, self.max_seq), 1e6, device=device)
        # stand-ins for the o_proj output / residual stream / post-attention norm weight of the layer
        self.hidden = (torch.randn((self.n_seqs, HIDDEN), device=device, generator=g) * 0.01).to(torch.bfloat16)
        self.hidden_out = torch.empty_like(self.hidden)
        self.resid = torch.zeros((self.n_seqs, HIDDEN), device=device, dtype=torch.bfloat16)
        self.norm_w = torch.ones(HIDDEN, device=device, dtype=torch.bfloat16)
        self.graphs = {}
        self.graph_launches = {}
        self.stream = torch.cuda.Stream(device=device)
        self.bs_list = [b for b in graph_bs_list() if b <= max(8, self.n_seqs)]
        self.backend.init_capture_graph(self.max_seq, self.bs_list)
        self.lib = pkg._cabi.load()
        # e2e leg: pipelined host -> device staging
        self.copy_stream = torch.cuda.Stream(device)
        self.staging = None
        self.stg_ready = [torch.cuda.Event() for _ in range(2)]
        self.stg_free = [torch.cuda.Event() for _ in range(2)]
        self._e2e_step = 0
        # host-side cost of a step, by phase (microseconds, accumulated; bench reports the per-step mean)
        self.host_us = {"inputs_h2d": 0.0, "prepare_metadata": 0.0, "prepare_for_replay": 0.0, "graph_replay": 0.0, "steps": 0}

    def pad_bs(self, n: int) -> int:
        return next(b for b in self.bs_list if b >= n)

    # ---- batch objects
    def make_batch(self, triples, phase, pad=True):
        pkg = self.pkg
        reqs = [pkg.Req(table_idx=t, cached_len=c, device_len=d) for (t, c, d) in triples]
        batch = pkg.Batch(reqs, phase)
        if pad and phase == "decode":
            bs = self.pad_bs(len(reqs))
            dummy = pkg.Req(table_idx=self.n_seqs, cached_len=0, device_len=1)
            batch.padded_reqs = reqs + [dummy] * (bs - len(reqs))
        return batch

    def host_inputs(self, batch):
        """positions / out_loc exactly as scheduler.py:204-259 derives them (host ints)."""
        pos, loc = [], []
        for r in batch.padded_reqs:
            pos.extend(range(r.cached_len, r.device_len))
            loc.extend(self.table_np[r.table_idx, r.cached_len : r.device_len].tolist())
        return (torch.tensor(pos, dtype=torch.int32).pin_memory(), torch.tensor(loc, dtype=torch.int32).pin_memory())

    def qkv_views(self, l: int, n: int):
        return self.qkv[:n, l].split([self.hq * D, self.hkv * D, self.hkv * D], dim=-1)

    # ---- one layer of the hot path on rows [0, n) of the static buffers
    def layer(self, l: int, n: int, batch) -> None:
        q, k, v = self.qkv_views(l, n)
        if self.fuse_pre_attention:  # qk-norm + RoPE + append + attention: one launch
            o = self.backend.forward_decode_fused(q.view(n, self.hq, D), k, v, l, batch, batch.positions,
                                                  self.rotary._cos_sin_cache, self.qw, self.kw, EPS)
        else:
            self.pkg.ops.qknorm_rope_inplace(batch.positions, q, k, D, self.rotary._cos_sin_cache, self.qw, self.kw, EPS)
            o = self.backend.forward(q.view(n, self.hq, D), k, v, l, batch)
        self._last_out = o
        if self.ar is not None:
            self.ar.all_reduce(self.hidden[:n], out=self.hidden_out[:n], residual=self.resid[:n],
                               weight=self.norm_w, eps=EPS)

    def capture(self, bs: int) -> None:
        if bs in self.graphs:
            return
        pkg = self.pkg
        dummy = pkg.Req(table_idx=self.n_seqs, cached_len=0, device_len=1)
        batch = pkg.Batch([dummy] * bs, "decode")
        batch.padded_reqs = batch.reqs
        with torch.cuda.stream(self.stream):
            self.backend.prepare_for_capture(batch)
            batch.positions = self.positions[:bs]
            batch.out_loc = self.out_loc[:bs]
            self.out_loc[:bs].fill_(self.num_pages * self.page_size)
            for l in range(L):
                self.layer(l, bs, batch)
            self.stream.synchronize()
            g = torch.cuda.CUDAGraph()
            before = self.lib.b200_launch_count()
            outs = []
            with torch.cuda.graph(g, stream=self.stream):
                for l in range(L):
                    self.layer(l, bs, batch)
                    outs.append(self._last_out)
            self.graph_launches[bs] = self.lib.b200_launch_count() - before
            self.last_out[bs] = self._last_out
            self.layer_outs[bs] = outs
        self.graphs[bs] = g

    def schedule_step(self, triples):
        """What the reference's scheduler hands to the path for one decode iteration (outside the
        timed region, like the scheduler thread): the Batch of Reqs and the pinned host positions /
        out_loc (scheduler.py:204-259)."""
        batch = self.make_batch(triples, "decode")
        pos_h, loc_h = self.host_inputs(batch)
        return batch, pos_h, loc_h, len(triples)

    def decode_step(self, step, host_copy: bool = False, host_bufs=None) -> int:
        """H2D of the step's inputs + prepare_metadata + replay on self.stream. Returns number of real tokens."""
        batch, pos_h, loc_h, n_tokens = step
        bs = batch.padded_size
        with torch.cuda.stream(self.stream):
            if host_copy:
                # The step's host inputs (the qkv rows of all layers: one contiguous block) go up on a copy
                # stream into one of two staging buffers, so the upload of step i+1 overlaps the attention of
                # step i (the engine / scheduler stream split of the reference, scheduler.py:53-55,102); the
                # compute stream moves them into the graph's static buffer with one device-to-device copy.
                qkv_h, out_h = host_bufs
                slot = self._e2e_step % 2
                self._e2e_step += 1
                if self.staging is None:
                    self.staging = [torch.empty_like(self.qkv) for _ in range(2)]
                    self.staging_idx = [torch.empty((2, self.n_seqs), dtype=torch.int32, device=self.dev) for _ in range(2)]
                stg, stg_idx = self.staging[slot], self.staging_idx[slot]
                self.copy_stream.wait_event(self.stg_free[slot])
                with torch.cuda.stream(self.copy_stream):
                    # ALL host inputs of the step travel on the copy stream, the small index vectors first: a small
                    # H2D on the compute stream would queue behind the 29 MB transfer in the DMA engine
                    stg_idx[0, :bs].copy_(pos_h, non_blocking=True)
                    stg_idx[1, :bs].copy_(loc_h, non_blocking=True)
                    stg[:bs].copy_(qkv_h[:bs], non_blocking=True)
                    self.stg_ready[slot].record(self.copy_stream)
                self.stream.wait_event(self.stg_ready[slot])
                self.qkv[:bs].copy_(stg[:bs], non_blocking=True)
                t0 = time.perf_counter()
                self.positions[:bs].copy_(stg_idx[0, :bs], non_blocking=True)
                self.out_loc[:bs].copy_(stg_idx[1, :bs], non_blocking=True)
                self.stg_free[slot].record(self.stream)
            else:
                t0 = time.perf_counter()
                self.positions[:bs].copy_(pos_h, non_blocking=True)
                self.out_loc[:bs].copy_(loc_h, non_blocking=True)
            batch.positions, batch.out_loc = self.positions[:bs], self.out_loc[:bs]
            t1 = time.perf_counter()
            self.backend.prepare_metadata(batch)
            t2 = time.perf_counter()
            self.backend.prepare_for_replay(batch)
            t3 = time.perf_counter()
            self.graphs[bs].replay()
            t4 = time.perf_counter()
            hb = self.host_us
            hb["inputs_h2d"] += (t1 - t0) * 1e6
            hb["prepare_metadata"] += (t2 - t1) * 1e6
            hb["prepare_for_replay"] += (t3 - t2) * 1e6
            hb["graph_replay"] += (t4 - t3) * 1e6
            hb["steps"] += 1
            if self.allreduce == "nccl":
                # the reference's NCCL all-reduce of [nnz, hidden] after o_proj (layers/linear.py:102-106),
                # one per layer; issued eagerly behind the replay
                for _ in range(L):
                    torch.distributed.all_reduce(self.hidden[:bs], group=self.tp_group)
            if host_copy:
                out_h[:bs].copy_(self.last_out[bs].view(bs, -1), non_blocking=True)
            # The step is over for the scheduler: its metadata dies with it, as in the engine, where a Batch does not
            # outlive its forward.  The timed steps are scheduled ahead of the timed region here; left alive, their
            # metadata (slot-table snapshot, 1-2 MB each) would make the caching allocator cudaMalloc fresh segments
            # INSIDE the timed region.
            batch.attn_metadata = None
        return n_tokens


DUMP_MAX_BYTES = 64_000_000  # all files together, headers included (64 MB in either reading)


def dump_outputs(runner: AttentionPathRunner, step, out_dir: str) -> None:
    """What the last timed decode step computed, as a caller of the path receives it, in float32: the attention
    output of every layer (attn_out.npy, [L, n, hq, D]) and the K / V rows the step appended to every layer's
    pool slice (k_appended.npy / v_appended.npy, [L, n, hkv, D]; in the fused path k is the normed + roped row).
    n = the step's real requests; when that would exceed 64 MB in all, a fixed seeded sample of them is written.
    rows.npy lists the step's request rows that were written."""
    batch, _, _, n = step
    bs = batch.padded_size
    torch.cuda.synchronize()
    per_row = L * (runner.hq + 2 * runner.hkv) * D * 4 + 8  # the three arrays' rows + the row index
    budget = DUMP_MAX_BYTES - 4 * 4096  # .npy headers
    rows = np.arange(n)
    if n * per_row > budget:
        rows = np.sort(np.random.RandomState(0).choice(n, budget // per_row, replace=False))
    idx = torch.from_numpy(rows).to(runner.dev)
    loc = runner.out_loc[:bs][idx].long()
    arrays = {
        "attn_out": torch.stack([o.reshape(bs, runner.hq, D)[idx] for o in runner.layer_outs[bs]]),
        "k_appended": torch.stack([runner.pool.k_cache(l).reshape(-1, runner.hkv, D)[loc] for l in range(L)]),
        "v_appended": torch.stack([runner.pool.v_cache(l).reshape(-1, runner.hkv, D)[loc] for l in range(L)]),
    }
    out = Path(out_dir)
    out.mkdir(parents=True, exist_ok=True)
    for name, t in arrays.items():
        np.save(out / f"{name}.npy", t.float().cpu().numpy())
    np.save(out / "rows.npy", rows.astype(np.float64))


def _parity_vs_gpu(a: torch.Tensor, b: torch.Tensor) -> float:
    """THE criterion against a reference GPU backend's output (oracle/tolerance.vs_reference_gpu, the same
    function the GPU tests and smoke() use; bench.py calls into oracle/ only as the checker):
    max_i (|a_i - b_i| - one output ulp)^+ / max|b|, pass <= oracle.tolerance.GPU_REL_TOL (1.5e-3: north_star's
    1e-3 plus the spread the reference's own fa2 / TRT-LLM-gen paths show against each other, printed beside it)."""
    from oracle import tolerance

    return tolerance.vs_reference_gpu(a, b)


def ref_gpu_arms(runner, sched, pkg, peaks, iters, reps: int = 5, layers: int = 8) -> dict:
    """The reference's two GPU attention paths timed beside ours in the same process, on the identical
    pool / page table / q (north_star: "next to the reference's own FlashInfer path on the same box ...
    in the same run"):  R-fi = FlashInfer fa2 wrappers with page_size 1 exactly as attention/fi.py:93-103,
    134-165,185-188 calls them; R-trtllm = the TRT-LLM-gen path exactly as attention/trtllm.py:57-89 calls
    it -- only on compute capability 10.x, the only architecture FlashInfer ships its kernels for (elsewhere
    it is neither timed nor compared, and its spread never enters a gate).  `store_kv`
    in front of both is our store kernel (the reference's tvm-ffi store.cu cannot be built offline; same
    bytes).  Per layer: [append +] attention, eager, layers on distinct pool slices (L2 cold), CUDA events,
    median of `reps`."""
    res: dict = {"layers_timed": layers, "method": "eager launches, CUDA events, median of %d, per layer" % reps,
                 "parity_criterion": "oracle/tolerance.vs_reference_gpu: max (|a - b| - one output ulp)^+ / max|b|, pass <= 1.5e-3 "
                                     "(north_star 1e-3 + the fa2-vs-TRT-LLM-gen spread of the reference itself, keys *_parity_trtllm_vs_fi)"}
    try:
        if "FLASHINFER_WORKSPACE_BASE" not in os.environ:
            os.environ["FLASHINFER_WORKSPACE_BASE"] = flashinfer_workspace()
        import flashinfer
        from flashinfer.decode import trtllm_batch_decode_with_kv_cache
        from flashinfer.prefill import trtllm_batch_context_with_kv_cache
    except Exception as e:  # pragma: no cover
        return {"unavailable": f"flashinfer import failed: {type(e).__name__}: {str(e)[:200]}"}
    dev, hq, hkv, PS = runner.dev, runner.hq, runner.hkv, runner.page_size
    nl = min(layers, L)
    scale = D**-0.5
    res["flashinfer"] = flashinfer.__version__
    with_trtllm = torch.cuda.get_device_capability(dev)[0] == 10
    if not with_trtllm:
        res["trtllm"] = "not run: FlashInfer's TRT-LLM-gen kernels exist for compute capability 10.x only"
    ws_fi = torch.empty(128 * 1024 * 1024, dtype=torch.uint8, device=dev)
    ws_trt = torch.zeros(128 * 1024 * 1024, dtype=torch.uint8, device=dev) if with_trtllm else None

    def timed(fn):
        ts = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return float(np.median(ts)) / nl

    def pool(l):
        return runner.pool.k_cache(l), runner.pool.v_cache(l)

    def run_three(tag, fns, work, unit):
        outs = {}
        for name, fn in fns:
            try:
                fn()
                torch.cuda.synchronize()
                ms = timed(fn)
                res[f"{tag}_{name}_us_per_layer"] = round(ms * 1e3, 1)
                res[f"{tag}_{name}_{unit}"] = round(work / ms / (1e6 if unit == "GBs" else 1e9), 1)
                outs[name] = fn.out
            except Exception as e:  # one missing path must not hide the others
                res[f"{tag}_{name}_error"] = f"{type(e).__name__}: {str(e)[:200]}"
        errs = {}
        for a, b in (("trtllm", "fi"), ("b200", "fi"), ("b200", "trtllm")):
            if a in outs and b in outs:
                errs[(a, b)] = e = _parity_vs_gpu(outs[a], outs[b])
                res[f"{tag}_parity_{a}_vs_{b}"] = float(f"{e:.3e}")
        set_ok(tag, errs)
        return outs, errs

    def set_ok(tag, errs, pair_excess=None):
        """pass / fail of OUR output against each reference arm: the gate of oracle/tolerance (1.5e-3), or -- where the
        reference's own two backends disagree by more than that on this very input (long contexts: 2.5e-3 at kv 4096)
        -- 1.25 x their spread.  The full-batch number is the maximum over ~5e5 elements of the difference of two
        kernels that are each ~1.2e-3 from the exact result, so it scatters around the gate from run to run
        (1.05e-3 .. 1.58e-3 for the same cfg1 batch); where the oracle sample is available the rigorous form decides
        a number between 1x and 2x the gate: |ours - ref| <= 2 * 2^-9 * softmax(S)|V| + one ulp element-wise
        (oracle/tolerance.pair_p16_bound_excess <= 2e-4)."""
        from oracle import tolerance

        spread = errs.get(("trtllm", "fi"), 0.0)
        gate = max(tolerance.GPU_REL_TOL, 1.25 * spread)
        for b in ("fi", "trtllm"):
            if ("b200", b) in errs:
                e = errs[("b200", b)]
                ok = e <= gate
                if not ok and pair_excess is not None and b in pair_excess:
                    ok = e <= 2 * gate and pair_excess[b] <= tolerance.P16_EXCESS_TOL
                res[f"{tag}_parity_b200_vs_{b}_ok"] = bool(ok)

    def vs_oracle(tag, outs, errs, tr, layer, q):
        """All three GPU outputs of the last timed layer against the exact fp32 oracle on a sample of the
        batch's requests (oracle/tolerance.vs_exact_oracle, gate 2e-3): says how much of a backend's distance
        to the oracle is the method's (16-bit P, shared by all three) and how much is its own."""
        from oracle import tolerance
        from oracle.attention import ref_paged_attention

        step = max(1, len(tr) // 24)
        pick = list(range(0, len(tr), step))[:24]
        rows = [torch.from_numpy(runner.table_np[tr[i][0], : tr[i][2]].astype(np.int64)) for i in pick]
        uniq = torch.unique(torch.cat(rows))
        remap = torch.full((int(uniq.max()) + 1,), -1, dtype=torch.int64)
        remap[uniq] = torch.arange(uniq.numel())
        kc = runner.pool.k_cache(layer).reshape(-1, hkv, D)[uniq.to(dev)].cpu()
        vc = runner.pool.v_cache(layer).reshape(-1, hkv, D)[uniq.to(dev)].cpu()
        idx = torch.tensor(pick, device=dev)
        q_s, rows_s = q.reshape(len(tr), hq, D)[idx].cpu(), [remap[r] for r in rows]
        ref = ref_paged_attention(q_s, kc, vc, rows_s, [1] * len(pick), exact=True)
        absref = ref_paged_attention(q_s, kc, vc.abs(), rows_s, [1] * len(pick), exact=True)  # softmax(S) |V|
        for name, o in outs.items():
            o_s = o.reshape(len(tr), hq, D)[idx]
            res[f"{tag}_parity_{name}_vs_oracle"] = float(f"{tolerance.vs_exact_oracle(o_s, ref):.3e}")
            res[f"{tag}_p16_bound_excess_{name}"] = float(f"{tolerance.p16_bound_excess(o_s, ref, absref):.3e}")
        pair = {}
        for b in ("fi", "trtllm"):
            if "b200" in outs and b in outs:
                pair[b] = tolerance.pair_p16_bound_excess(outs["b200"].reshape(len(tr), hq, D)[idx], outs[b].reshape(len(tr), hq, D)[idx], absref)
                res[f"{tag}_pair_p16_bound_excess_b200_vs_{b}"] = float(f"{pair[b]:.3e}")
        set_ok(tag, errs, pair)
        res[f"{tag}_parity_vs_oracle_sample"] = f"{len(pick)} requests, layer {layer}"

    with torch.cuda.stream(runner.stream):
        # ------------------------------------------------------------------ decode
        for it in iters:
            tr = sched.live(it)
            batch = runner.make_batch(tr, "decode", pad=False)
            bs = len(tr)
            pos_h, loc_h = runner.host_inputs(batch)
            batch.positions, batch.out_loc = pos_h.to(dev), loc_h.to(dev)
            runner.backend.prepare_metadata(batch)
            md = batch.attn_metadata
            qs = [runner.qkv_views(l, bs) for l in range(nl)]
            nbytes = decode_bytes_per_layer(tr, hq, hkv)

            def ours():
                for l in range(nl):
                    q, k, v = qs[l]
                    ours.out = runner.backend.forward(q.view(bs, hq, D), k, v, l, batch)

            seq_cpu, cu_k_cpu = md.cache_seqlens.cpu(), md.cu_seqlens_k.cpu()
            dec = flashinfer.BatchDecodeWithPagedKVCacheWrapper(ws_fi, kv_layout="NHD", use_tensor_cores=(hq // hkv) >= 4, backend="fa2")
            dec.plan(indptr=cu_k_cpu, indices=md.flat_indices(), last_page_len=torch.ones(bs, dtype=torch.int32),
                     num_qo_heads=hq, num_kv_heads=hkv, head_dim=D, page_size=1, pos_encoding_mode="NONE", seq_lens=seq_cpu,
                     data_type=torch.bfloat16, q_data_type=torch.bfloat16, kv_data_type=torch.bfloat16, non_blocking=True)

            def fi():
                for l in range(nl):
                    q, k, v = qs[l]
                    runner.pool.store_kv(k, v, batch.out_loc, l)
                    kc, vc = pool(l)
                    fi.out = dec.run(q=q.reshape(bs, hq, D), paged_kv_cache=(kc.view(-1, 1, hkv, D), vc.view(-1, 1, hkv, D)))

            block_tables = md.paged_page_table(PS).contiguous()

            def trtllm():
                for l in range(nl):
                    q, k, v = qs[l]
                    runner.pool.store_kv(k, v, batch.out_loc, l)
                    trtllm.out = trtllm_batch_decode_with_kv_cache(
                        query=q.reshape(bs, hq, D), kv_cache=pool(l), workspace_buffer=ws_trt, block_tables=block_tables,
                        seq_lens=md.cache_seqlens, max_seq_len=md.max_seqlen_k, bmm1_scale=scale, bmm2_scale=1.0,
                        kv_layout="NHD", out_dtype=torch.bfloat16)

            tag = f"decode_it{it}_bs{bs}"
            outs, errs = run_three(tag, (("b200", ours), ("fi", fi)) + ((("trtllm", trtllm),) if with_trtllm else ()),
                                   nbytes, "GBs")
            torch.cuda.synchronize()
            try:
                vs_oracle(tag, outs, errs, tr, nl - 1, qs[nl - 1][0])
            except Exception as e:  # the extra evidence must not take the bench line down
                res[f"{tag}_parity_vs_oracle_error"] = f"{type(e).__name__}: {str(e)[:200]}"
            for name in ("b200", "fi", "trtllm"):
                k = f"{tag}_{name}_GBs"
                if k in res:
                    res[f"{tag}_{name}_frac_hbm"] = round(res[k] / peaks["hbm_gbs"], 3)
        # ------------------------------------------------------------------ prefill (one prompt batch)
        batches = sched.prefill_batches()
        trp = batches[min(1, len(batches) - 1)]
        pb = runner.make_batch(trp, "prefill")
        pos_h, loc_h = runner.host_inputs(pb)
        nnz = pos_h.numel()
        pb.positions, pb.out_loc = pos_h.to(dev), loc_h.to(dev)
        runner.backend.prepare_metadata(pb)
        pmd = pb.attn_metadata
        qkv = torch.randn((nnz, runner.width), device=dev, dtype=torch.bfloat16)
        q, k, v = qkv.split([hq * D, hkv * D, hkv * D], dim=-1)
        flops = prefill_flops_per_layer(trp, hq)
        # cached prefixes must hold the same K/V for all three: they already do (pool contents)

        def ours_p():
            for l in range(nl):
                ours_p.out = runner.backend.forward(q.view(nnz, hq, D), k, v, l, pb)

        pre = flashinfer.BatchPrefillWithPagedKVCacheWrapper(ws_fi, kv_layout="NHD", backend="fa2")
        pre.plan(qo_indptr=pmd.cu_seqlens_q.cpu(), paged_kv_indptr=pmd.cu_seqlens_k.cpu(), paged_kv_indices=pmd.flat_indices(),
                 paged_kv_last_page_len=torch.ones(len(trp), dtype=torch.int32), num_qo_heads=hq, num_kv_heads=hkv,
                 head_dim_qk=D, page_size=1, pos_encoding_mode="NONE", seq_lens=pmd.cache_seqlens.cpu(),
                 q_data_type=torch.bfloat16, kv_data_type=torch.bfloat16, non_blocking=True, causal=True)
        qc = q.reshape(nnz, hq, D).contiguous()

        def fi_p():
            for l in range(nl):
                runner.pool.store_kv(k, v, pb.out_loc, l)
                kc, vc = pool(l)
                fi_p.out = pre.run(q=qc, paged_kv_cache=(kc.view(-1, 1, hkv, D), vc.view(-1, 1, hkv, D)))

        pbt = pmd.paged_page_table(PS).contiguous()

        def trt_p():
            for l in range(nl):
                runner.pool.store_kv(k, v, pb.out_loc, l)
                trt_p.out = trtllm_batch_context_with_kv_cache(
                    query=qc, kv_cache=pool(l), workspace_buffer=ws_trt, block_tables=pbt, seq_lens=pmd.cache_seqlens,
                    max_q_len=pmd.max_seqlen_q, max_kv_len=pmd.max_seqlen_k, bmm1_scale=scale, bmm2_scale=1.0,
                    cum_seq_lens_q=pmd.cu_seqlens_q, cum_seq_lens_kv=pmd.cu_seqlens_k, kv_layout="NHD",
                    batch_size=len(trp), out_dtype=torch.bfloat16)

        tag = f"prefill_nnz{nnz}_reqs{len(trp)}"
        run_three(tag, (("b200", ours_p), ("fi", fi_p)) + ((("trtllm", trt_p),) if with_trtllm else ()), flops, "TFs")
    del ws_fi, ws_trt
    return res


def run_ours(args) -> dict:
    pkg = importlib.import_module("mini-sglang_b200")
    pkg.build_native()
    for o in args.opt:
        name, val = o.split("=")
        if pkg._cabi.set_option(name, int(val)) == -1:
            raise SystemExit(f"unknown option {name}")
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    wl = set_workload(args.config)
    if args.tp_shard > 1:  # run ONE rank's shard of a tp-N job on a single GPU (no all-reduce partner)
        if world != 1:
            raise SystemExit("--tp-shard is for single-GPU runs")
        wl.tp_shard = args.tp_shard
        set_workload(args.config)
    tp_group = None
    if world > 1:
        import faulthandler

        faulthandler.dump_traceback_later(int(os.environ.get("B200_BENCH_WATCHDOG_S", "420")), exit=True)
        torch.distributed.init_process_group("nccl", device_id=dev)
        pkg.utils.set_tp_info(rank, world)
        tp_group = torch.distributed.group.WORLD if not args.no_allreduce else None
    if wl.tp_shard > 1 and world not in (1, wl.tp_shard):
        raise SystemExit(f"{wl.name} is a tp={wl.tp_shard} configuration: run it with --gpus 1 (one rank's shard) or --gpus {wl.tp_shard}")
    # heads of this process: the model's heads divided by the TP degree the config is quoted at, when it
    # is run as one rank's shard (world 1); otherwise the runner divides by world itself
    shard = wl.tp_shard if world == 1 else 1
    g_hq, g_hkv = wl.hq // shard, max(1, wl.hkv // shard)
    hq, hkv = g_hq // world, max(1, g_hkv // world)
    sched = Schedule(wl)
    runner = AttentionPathRunner(pkg, sched, g_hq, g_hkv, args.page_size, dev, world, tp_group, args.allreduce,
                                 fuse_pre_attention=not args.unfused_pre_attention)
    lib = runner.lib
    peaks = load_peaks()

    iters = sched.sample_iters(args.steps)
    warm_iters = sched.sample_iters(max(args.warmup, 1))[: args.warmup]
    step_triples = [sched.live(it) for it in iters]
    for tr in step_triples + [sched.live(it) for it in warm_iters]:
        runner.capture(runner.pad_bs(len(tr)))
    torch.cuda.synchronize()

    def barrier():
        if world > 1:
            torch.distributed.barrier()
        torch.cuda.synchronize()

    by_rank = {}

    def max_over_ranks(ms: float, tag: str = "") -> float:
        if world > 1:
            t = torch.tensor([ms], device=dev)
            parts = [torch.empty_like(t) for _ in range(world)]
            torch.distributed.all_gather(parts, t)
            vals = [round(float(x.item()), 3) for x in parts]
            if tag:
                by_rank[tag] = vals
            return max(vals)
        return ms

    # ---------------- device-timed value
    steps = [runner.schedule_step(tr) for tr in step_triples]
    warm_steps = [runner.schedule_step(sched.live(it)) for it in warm_iters]
    for st in warm_steps:
        runner.decode_step(st)
    # A CUDA graph is uploaded to the device on its FIRST launch (milliseconds, and different on every rank): every
    # distinct captured graph the timed steps replay is launched once here, as a serving engine's graphs are warm
    # after the first seconds (a cold first launch per batch size can cost more than the step itself).
    seen_bs = set()
    for st in steps:
        if st[0].padded_size not in seen_bs:
            seen_bs.add(st[0].padded_size)
            runner.decode_step(st)
    # Python's cyclic collector is parked for the timed legs, as serving engines do after warm-up (gc.freeze): a
    # full collection of a process with torch loaded takes tens of milliseconds and the scheduler thread of this
    # path is at most 4 steps (the pinned request ring) ahead of the GPU.
    if os.environ.get("B200_BENCH_KEEP_GC", "0") == "0":  # =1: A/B of the claim above
        gc.collect()
        gc.freeze()
        gc.disable()
    barrier()
    for k in runner.host_us:
        runner.host_us[k] = 0
    launches0 = lib.b200_launch_count()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    tokens = 0
    with ClockSampler(local_rank) as clocks:
        with torch.cuda.stream(runner.stream):
            ev0.record()
        host_t0 = time.perf_counter()
        step_evs = []
        step_own_ms = []  # host time of each step minus the time it waited for the GPU (request-info ring)
        for st in steps:
            t_s, w_s = time.perf_counter(), runner.backend.ring_wait_s
            tokens += runner.decode_step(st)
            step_own_ms.append(((time.perf_counter() - t_s) - (runner.backend.ring_wait_s - w_s)) * 1e3)
            step_evs.append(torch.cuda.Event(enable_timing=True))
            step_evs[-1].record(runner.stream)
        value_host_ms = (time.perf_counter() - host_t0) * 1e3
        host_breakdown = {k: round(v / max(runner.host_us["steps"], 1), 1) for k, v in runner.host_us.items() if k != "steps"}
        with torch.cuda.stream(runner.stream):
            ev1.record()
        barrier()
    ms = max_over_ranks(ev0.elapsed_time(ev1), "value_ms")
    step_gpu_ms = [a.elapsed_time(b) for a, b in zip([ev0] + step_evs[:-1], step_evs)]
    eager_launches = lib.b200_launch_count() - launches0
    graph_launches = sum(runner.graph_launches[runner.pad_bs(len(tr))] for tr in step_triples)
    value = tokens / (ms * 1e-3)
    if args.dump_outputs and rank == 0:
        dump_outputs(runner, steps[-1], args.dump_outputs)

    # ---------------- host cost of a step with an idle GPU (no back-pressure from the pinned staging ring):
    # what the scheduler thread pays per decode iteration for prepare_metadata / prepare_for_replay / replay
    for k in runner.host_us:
        runner.host_us[k] = 0
    for st in steps[: min(10, len(steps))]:
        torch.cuda.synchronize()
        runner.decode_step(st)
    torch.cuda.synchronize()
    host_unloaded = {k: round(v / max(runner.host_us["steps"], 1), 1) for k, v in runner.host_us.items() if k != "steps"}
    host_unloaded["total"] = round(sum(host_unloaded.values()), 1)

    # ---------------- e2e: host buffers, copies inside the timed region
    qkv_h = torch.empty(tuple(runner.qkv.shape), dtype=torch.bfloat16).pin_memory()
    qkv_h.copy_(runner.qkv.cpu())
    out_h = torch.empty((runner.n_seqs, hq * D), dtype=torch.bfloat16).pin_memory()
    for st in warm_steps[:2]:
        runner.decode_step(st, True, (qkv_h, out_h))
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    h2d = d2h = 0
    with torch.cuda.stream(runner.stream):
        e0.record()
    host_t0 = time.perf_counter()
    for st, tr in zip(steps, step_triples):
        runner.decode_step(st, True, (qkv_h, out_h))
        bs = runner.pad_bs(len(tr))
        h2d += L * bs * runner.width * 2 + bs * 8 + bs * 12
        d2h += bs * hq * D * 2
    host_enqueue_ms = (time.perf_counter() - host_t0) * 1e3  # CPU time to enqueue all steps (GPU runs behind)
    with torch.cuda.stream(runner.stream):
        e1.record()
    barrier()
    e2e_ms = max_over_ranks(e0.elapsed_time(e1), "e2e_ms")
    e2e_value = tokens / (e2e_ms * 1e-3)
    gc.enable()

    # ---------------- roofline of the dominant kernel (decode attention): for every timed step an
    # attention-only CUDA graph (L launches, one per layer, each on its own pool slice => L2 cold)
    # is replayed between two events on the launching stream.
    alg_bytes = 0
    attn_ms = 0.0
    n_launch = 0
    per_step = []  # [padded bs, us per layer, fraction of the HBM peak] of every timed step
    with torch.cuda.stream(runner.stream):
        for tr in step_triples:
            batch = runner.make_batch(tr, "decode")
            bs = batch.padded_size
            pos_h, loc_h = runner.host_inputs(batch)
            runner.positions[:bs].copy_(pos_h)
            runner.out_loc[:bs].copy_(loc_h)
            batch.positions, batch.out_loc = runner.positions[:bs], runner.out_loc[:bs]
            runner.backend.prepare_metadata(batch)
            qs = [runner.qkv_views(l, bs) for l in range(L)]
            runner.stream.synchronize()
            ag = torch.cuda.CUDAGraph()
            with torch.cuda.graph(ag, stream=runner.stream):
                for l in range(L):
                    q, k, v = qs[l]
                    runner.backend.forward(q.view(bs, hq, D), k, v, l, batch)
            a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ag.replay()  # warm
            a0.record()
            ag.replay()
            a1.record()
            a1.synchronize()
            step_ms = a0.elapsed_time(a1)
            step_bytes = L * decode_bytes_per_layer([(r.table_idx, r.cached_len, r.device_len) for r in batch.padded_reqs], hq, hkv)
            attn_ms += step_ms
            alg_bytes += step_bytes
            per_step.append([bs, round(step_ms * 1e3 / L, 1), round(step_bytes / (step_ms * 1e-3) / 1e9 / peaks["hbm_gbs"], 3)])
            n_launch += L
            del ag
    achieved = alg_bytes / (attn_ms * 1e-3) / 1e9
    roofline = {"kernel": "attn_decode_tc_kernel(+combine)", "bound": "hbm", "achieved": round(achieved, 1),
                "peak": peaks["hbm_gbs"], "unit": "GB/s", "frac": round(achieved / peaks["hbm_gbs"], 4),
                "peak_source": peaks["source"],
                "alg_bytes_per_launch": int(alg_bytes / n_launch), "us_per_launch": round(attn_ms * 1e3 / n_launch, 2),
                "per_step_bs_us_frac": per_step}

    # ---------------- prefill TFLOP/s over the schedule's prompt batches
    prefill = None
    if not args.skip_prefill:
        batches = sched.prefill_batches()
        if args.prefill_batches > 0:
            batches = batches[: args.prefill_batches]
        pl = min(L, args.prefill_layers) if args.prefill_layers > 0 else L
        flops = 0
        p_ms = 0.0
        with torch.cuda.stream(runner.stream):
            for rep in range(2):  # first pass = warm-up
                flops, p_ms, p_bytes = 0, 0.0, 0
                for tr in batches:
                    batch = runner.make_batch(tr, "prefill")
                    pos_h, loc_h = runner.host_inputs(batch)
                    nnz = pos_h.numel()
                    batch.positions = pos_h.to(dev, non_blocking=True)
                    batch.out_loc = loc_h.to(dev, non_blocking=True)
                    runner.backend.prepare_metadata(batch)
                    qkv = torch.randn((nnz, runner.width), device=dev, dtype=torch.bfloat16)
                    q, k, v = qkv.split([hq * D, hkv * D, hkv * D], dim=-1)
                    p0, p1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    p0.record()
                    for l in range(pl):
                        runner.backend.forward(q.view(nnz, hq, D), k, v, l, batch)
                    p1.record()
                    p1.synchronize()
                    p_ms += p0.elapsed_time(p1)
                    flops += pl * prefill_flops_per_layer(tr, hq)
                    p_bytes += pl * prefill_bytes_per_layer(tr, hq, hkv)
        tf = flops / (p_ms * 1e-3) / 1e12
        # short prompts (cfg1: avg 558 tokens, GQA 2) are bounded by HBM about as much as by the tensor
        # pipe, so both floors are reported
        t_tensor = flops / (peaks["bf16_tflops"] * 1e12) * 1e3
        t_hbm = p_bytes / (peaks["hbm_gbs"] * 1e9) * 1e3
        prefill = {"tflops": round(tf, 1), "ms": round(p_ms, 2), "flops": flops, "layers_timed": pl,
                   "frac_of_bf16_peak": round(tf / peaks["bf16_tflops"], 4), "peak_tflops": peaks["bf16_tflops"],
                   "alg_bytes": p_bytes, "GBs": round(p_bytes / (p_ms * 1e-3) / 1e9, 1),
                   "tensor_floor_ms": round(t_tensor, 2), "hbm_floor_ms": round(t_hbm, 2),
                   "frac_of_roofline": round(max(t_tensor, t_hbm) / p_ms, 4),
                   "tokens": sum(d - c for b in batches for (_, c, d) in b), "batches": len(batches)}

    # ---------------- the reference's GPU paths beside ours (same process, same inputs)
    ref_gpu = None
    if rank == 0 and world == 1 and not args.skip_ref_gpu:
        ref_gpu = ref_gpu_arms(runner, sched, pkg, peaks, sorted({iters[len(iters) // 8], iters[len(iters) // 2]}))
        if prefill is not None:
            for name in ("fi", "trtllm"):
                ks = [k for k in ref_gpu if k.startswith("prefill_") and k.endswith(f"_{name}_TFs")]
                if ks:
                    prefill[f"ref_{name}_tflops_one_batch"] = ref_gpu[ks[0]]

    # ---------------- row gather (embedding lookup of one prompt batch; table >> L2)
    gather = None
    if not args.skip_prefill:
        with torch.cuda.stream(runner.stream):
            table = torch.randn((151936, 1024), device=dev, dtype=torch.bfloat16)  # Qwen3-0.6B embedding: vocab x hidden
            ids = torch.randint(0, table.shape[0], (16384,), device=dev, dtype=torch.int32)
            outb = torch.empty((ids.numel(), table.shape[1]), device=dev, dtype=torch.bfloat16)
            for _ in range(3):
                pkg.ops.indexing(table, ids, output=outb)
            g0, g1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 20
            g0.record()
            for _ in range(reps):
                pkg.ops.indexing(table, ids, output=outb)
            g1.record()
            g1.synchronize()
            us = g0.elapsed_time(g1) * 1e3 / reps
            gbytes = 2 * outb.numel() * 2 + ids.numel() * 4
            gather = {"kernel": "index_rows_kernel", "rows": ids.numel(), "row_bytes": table.shape[1] * 2, "us": round(us, 2),
                      "GBs": round(gbytes / us / 1e3, 1), "frac_of_hbm_peak": round(gbytes / us / 1e3 / peaks["hbm_gbs"], 3)}
            del table, outb

    # ---------------- CPU baseline (oracle, bounded sample) + parity on the bench workload
    cpu = None
    if rank == 0 and not args.skip_cpu:
        cpu = cpu_baseline_sample(runner, sched, iters[len(iters) // 2], hq, hkv, budget_s=args.cpu_budget)

    ceiling = sched.decode_token_steps / (
        (sched.sum_kv * L * 2 * hkv * D * 2) / (peaks["hbm_gbs"] * 1e9))
    par = f"tp{world}" if world > 1 else ("tp1" if wl.tp_shard == 1 else f"one rank's shard of tp{wl.tp_shard}")
    res = {
        "metric": f"decode tokens/sec (attention hot path, {L} layers) + prefill TFLOPS, {wl.num_seqs}-seq {wl.model} batch",
        "value": round(value, 1), "unit": "tokens/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": round(ms / args.steps, 4), "host_enqueue_ms_per_step": round(value_host_ms / args.steps, 4),
        "host_us_per_step": host_breakdown, "host_us_per_step_gpu_idle": host_unloaded,
        # host time of a timed step NOT spent waiting for the GPU: a spike here is a host-side stall (scheduling, GC)
        "host_step_own_ms": {"median": round(float(np.median(step_own_ms)), 3), "max": round(max(step_own_ms), 3),
                             "argmax": int(np.argmax(step_own_ms))},
        "gpu_step_ms": {"median": round(float(np.median(step_gpu_ms)), 3), "max": round(max(step_gpu_ms), 3),
                        "argmax": int(np.argmax(step_gpu_ms))},
        "timed_ms_by_rank": by_rank or None,
        "higher_is_better": True,
        "scaling": "strong", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
        "config": {"workload": f"{wl.name}: {wl.model} attention path, {wl.desc}, "
                               f"decode iterations sampled evenly over {sched.n_iters}",
                   "layers": L, "hq": wl.hq, "hkv": wl.hkv, "hq_local": hq, "hkv_local": hkv, "head_dim": D,
                   "page_size": args.page_size, "parallelism": par, "cuda_graph": True,
                   "graph_warmup": "every distinct captured graph of the timed steps is replayed once, untimed, after the W warm-up steps",
                   "decode_step": ("per layer ONE launch: qk-norm + RoPE + KV append + attention (b200_attn_decode_fused)"
                                   if runner.fuse_pre_attention else "per layer: qk-norm+RoPE launch, attention(+append) launch"),
                   "allreduce": {"b200": "captured: one-shot NVLink push all-reduce of [bs,%d] bf16 fused with residual add + RMSNorm "
                                         "(csrc/allreduce.cu), one launch per layer inside the decode graph" % HIDDEN,
                                 "nccl": "nccl all-reduce [bs,%d] bf16 x %d per step (eager, behind the graph replay)" % (HIDDEN, L),
                                 "none": "none"}[runner.allreduce],
                   "l2": "each layer reads its own pool slice; one step touches far more than the 50 MB L2",
                   "hbm_roofline_tokens_per_s": round(ceiling, 1)},
        "frac_of_hbm_roofline": round(value / ceiling, 4),
        "e2e": {"value": round(e2e_value, 1), "unit": "tokens/s", "h2d_bytes_per_step": int(h2d / args.steps),
                "d2h_bytes_per_step": int(d2h / args.steps), "ms_per_step": round(e2e_ms / args.steps, 4),
                "frac_of_value": round(e2e_value / value, 3),
                "host_enqueue_ms_per_step": round(host_enqueue_ms / args.steps, 4)},
        "gpu_launches": int(eager_launches + graph_launches),
        "roofline": roofline, "prefill": prefill, "ref_gpu": ref_gpu, "index_rows": gather, "cpu_baseline": cpu,
        "clocks": clocks.summary(),
    }
    if world > 1:
        import faulthandler

        faulthandler.cancel_dump_traceback_later()
        runner.graphs.clear()
        if runner.ar is not None:
            runner.ar.destroy()
        torch.distributed.destroy_process_group()
    return res if rank == 0 else {}


def cpu_baseline_sample(runner, sched, it, hq, hkv, budget_s: float) -> dict:
    """Oracle (torch SDPA on the host cores) on one decode iteration of the same workload; the first
    layer is also compared with the GPU result (parity on the bench workload)."""
    from oracle.attention import ref_paged_attention

    torch.set_num_threads(effective_cpus())
    tr = sched.live(it)
    if len(tr) > 64:  # bounded sample: at most 64 requests of the iteration
        tr = tr[:: max(1, len(tr) // 64)][:64]
    n = len(tr)
    batch = runner.make_batch(tr, "decode", pad=False)
    pos_h, loc_h = runner.host_inputs(batch)
    dev = runner.dev
    with torch.cuda.stream(runner.stream):
        batch.positions, batch.out_loc = pos_h.to(dev), loc_h.to(dev)
        runner.backend.prepare_metadata(batch)
        qkv = runner.qkv[:n, 0].clone()
        q, k, v = qkv.split([hq * D, hkv * D, hkv * D], dim=-1)
        out = runner.backend.forward(q.view(n, hq, D), k, v, 0, batch)
        runner.stream.synchronize()
    kc = runner.pool.k_cache(0).reshape(-1, hkv, D)
    vc = runner.pool.v_cache(0).reshape(-1, hkv, D)
    rows = [torch.from_numpy(runner.table_np[t, :d].astype(np.int64)) for (t, _, d) in tr]
    # gather only the rows the sample needs (the pool is tens of GB)
    uniq = torch.unique(torch.cat(rows))
    remap = torch.full((int(uniq.max()) + 1,), -1, dtype=torch.int64)
    remap[uniq] = torch.arange(uniq.numel())
    kc_cpu = kc[uniq.to(dev)].cpu()
    vc_cpu = vc[uniq.to(dev)].cpu()
    rows_l = [remap[r] for r in rows]
    q_cpu = q.reshape(n, hq, D).cpu()
    t0 = time.perf_counter()
    ref = ref_paged_attention(q_cpu, kc_cpu, vc_cpu, rows_l, [1] * n, exact=True)
    t_layer = time.perf_counter() - t0
    from oracle import tolerance

    err = tolerance.vs_exact_oracle(out, ref)
    absref = ref_paged_attention(q_cpu, kc_cpu, vc_cpu.abs(), rows_l, [1] * n, exact=True)  # softmax(S) |V|
    p16 = tolerance.p16_bound_excess(out, ref, absref)
    reps = int(max(1, min(L - 1, budget_s / max(t_layer, 1e-3))))
    t0 = time.perf_counter()
    for _ in range(reps):
        ref_paged_attention(q_cpu, kc_cpu, vc_cpu, rows_l, [1] * n)
    t_avg = (time.perf_counter() - t0) / reps
    return {"value": round(n / (t_avg * L), 2), "unit": "tokens/s", "cores": torch.get_num_threads(), "kind": "port",
            "sample": f"decode iteration {it}, {n} of its requests, attention of 1 layer timed {reps}x and scaled to {L} layers; "
                      "oracle = torch SDPA fp32 per request",
            "parity_max_rel_err_vs_gpu": float(f"{err:.3e}"),
            "parity_criterion": "oracle/tolerance.vs_exact_oracle: max (|gpu - oracle| - half an output ulp)^+ / max|oracle|, "
                                "oracle = exact fp32 softmax; gate 2e-3 (the same function the GPU tests use)",
            "parity_ok": bool(err <= tolerance.ORACLE_REL_TOL),
            "parity_p16_bound_excess": float(f"{p16:.3e}"),
            "parity_p16_criterion": "oracle/tolerance.p16_bound_excess: max (|gpu - oracle| - 2^-9 * 1.02 * softmax(S)|V| - half an output ulp)^+ "
                                    "/ max|oracle| -- the element-wise bound of rounding P to 16 bits; gate 2e-4",
            "parity_p16_ok": bool(p16 <= tolerance.P16_EXCESS_TOL)}


# ----------------------------------------------------------------------------- reference arm
def run_reference(args) -> dict:
    """The reference has no CPU implementation of this path (its arithmetic is CUDA-only FlashInfer); its
    CPU form is the oracle port (kind "port").  A step is a BOUNDED SAMPLE of one decode iteration of the
    workload: `--ref-reqs` of the iteration's live requests through ALL layers, on the same paged pool
    layout (page_size, random page order, slot table) as our arm.  Nothing is extrapolated:
    value = tokens actually attended / wall time actually spent, ms_per_step = the measured step time."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return {}
    from oracle.attention import ref_paged_attention

    torch.set_num_threads(effective_cpus())
    wl = set_workload(args.config)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    shard = wl.tp_shard if world == 1 else 1
    hq, hkv = wl.hq // shard // world, max(1, wl.hkv // shard // world)
    sched = Schedule(wl)
    g = torch.Generator().manual_seed(0)
    iters = sched.sample_iters(args.steps)
    PS = args.page_size
    n_req = args.ref_reqs

    # per step: the sampled requests' pages are materialised on the CPU in a paged pool of their own
    # (random page order, slots = page * page_size + offset), one pool slice per layer like the engine's
    def make_step(it):
        tr = sched.live(it)
        tr = tr[:: max(1, len(tr) // n_req)][:n_req]
        n = len(tr)
        pages = [-(-d // PS) for (_, _, d) in tr]
        perm = np.random.RandomState(it).permutation(sum(pages))
        rows, off = [], 0
        for (_, _, d), np_ in zip(tr, pages):
            slots = (perm[off : off + np_, None] * PS + np.arange(PS)[None, :]).reshape(-1)[:d]
            rows.append(torch.from_numpy(slots.astype(np.int64)))
            off += np_
        n_slots = sum(pages) * PS
        kc = torch.randn((n_slots, hkv, D), generator=g).to(torch.bfloat16)
        vc = torch.randn((n_slots, hkv, D), generator=g).to(torch.bfloat16)
        q = torch.randn((L, n, hq, D), generator=g).to(torch.bfloat16)
        return n, q, kc, vc, rows

    def run_step(st):
        n, q, kc, vc, rows = st
        for l in range(L):  # all layers (same pool slice re-used: contents do not affect CPU time)
            ref_paged_attention(q[l], kc, vc, rows, [1] * n)
        return n

    for it in sched.sample_iters(max(args.warmup, 1))[: args.warmup]:
        run_step(make_step(it))
    steps = [make_step(it) for it in iters]
    t0 = time.perf_counter()
    tokens = sum(run_step(st) for st in steps)
    dt = time.perf_counter() - t0
    value = tokens / dt
    sample = (f"each step = one decode iteration of {wl.name}, {n_req} of its live requests, ALL {L} layers, "
              f"paged pool (page_size {PS}, random page order); nothing extrapolated")
    return {
        "impl": "reference",
        "metric": f"decode tokens/sec (attention hot path, {L} layers) + prefill TFLOPS, {wl.num_seqs}-seq {wl.model} batch",
        "value": round(value, 2), "unit": "tokens/s", "n_gpus": world,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": round(dt * 1e3 / max(args.steps, 1), 2),
        "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32 over bf16 storage",
        "data": "synthetic",
        "config": {"workload": f"{wl.name}: {wl.model} attention path, {wl.desc}, "
                               f"decode iterations sampled evenly over {sched.n_iters}",
                   "layers": L, "hq": wl.hq, "hkv": wl.hkv, "hq_local": hq, "hkv_local": hkv, "head_dim": D,
                   "page_size": PS, "parallelism": "cpu", "sample": sample},
        "cpu_baseline": {"value": round(value, 2), "unit": "tokens/s", "cores": torch.get_num_threads(), "kind": "port",
                         "sample": sample},
        "e2e": {"value": round(value, 2), "unit": "tokens/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--config", default="cfg1", choices=sorted(WORKLOADS), help="BASELINE.json workload (default: the headline cfg1)")
    ap.add_argument("--page-size", type=int, default=64)
    ap.add_argument("--tp-shard", type=int, default=0, help="single GPU: run one rank's shard of a tp-N job (heads / N)")
    ap.add_argument("--ref-reqs", type=int, default=8, help="--impl reference: requests sampled per step")
    ap.add_argument("--cpu-budget", type=float, default=12.0)
    ap.add_argument("--skip-prefill", action="store_true")
    ap.add_argument("--prefill-batches", type=int, default=0, help="time only the first N prompt batches (0 = all)")
    ap.add_argument("--prefill-layers", type=int, default=0, help="time only N layers per prompt batch (0 = all)")
    ap.add_argument("--skip-cpu", action="store_true")
    ap.add_argument("--unfused-pre-attention", action="store_true",
                    help="decode step = qk-norm+RoPE launch, then attention (round-1 chain) instead of the single fused launch")
    ap.add_argument("--skip-ref-gpu", action="store_true")
    ap.add_argument("--no-allreduce", action="store_true")
    ap.add_argument("--allreduce", default="b200", choices=["b200", "nccl"], help="TP all-reduce implementation (N > 1)")
    ap.add_argument("--opt", action="append", default=[], help="name=value for b200_set_option (A/B experiments)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed step's outputs as DIR/<name>.npy (float32, at most 64 MB)")
    args = ap.parse_args()
    if args.warmup < 3 and args.impl == "b200":
        args.warmup = 3
    res = run_reference(args) if args.impl == "reference" else run_ours(args)
    if res:
        print(json.dumps(res))


if __name__ == "__main__":
    main()
