#!/usr/bin/env python
"""Captured decode-step time of the UNMODIFIED reference engine (Qwen3-0.6B shape, 28 layers, dummy weights,
`attention_backend="b200"`) with the attention layers re-bound by `layers.patch_minisgl_attention` (ONE launch
per layer: q-norm + k-norm + RoPE + KV append + attention) against the same engine without it (q-norm,
k-norm and RoPE as three separate launches of our kernels in front of the attention launch, as
`install_into_minisgl(attention=False)` builds it).

One process per page size (`Engine` asserts a fresh CUDA context).  The engine captures its own decode graphs
with the unpatched layers; the script then patches the layers and captures a second set of graphs on the
engine's own capture buffers, exactly the way `GraphRunner._capture_graphs` does (reference
engine/graph.py:129-144).  Each batch size is timed through `GraphRunner.replay` of a live decode batch
(every request `--ctx` tokens deep), swapping the runner's graph map between the two sets: CUDA events around
`--steps` replays, the two modes alternated for `--rounds` rounds after warm-up; the median round is reported.

    python tools/insitu_decode_time.py [--out result.json] [--bs 1 64 256] [--page-sizes 64 1]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
import insitu  # noqa: E402

ROOT, REF = insitu.ROOT, insitu.REF


def card() -> dict:
    """Name, power limit and max SM clock of GPU 0 (read-only query)."""
    try:
        line = subprocess.run(
            ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
            capture_output=True, text=True, timeout=60, check=True).stdout.strip()
        name, power, clock = [x.strip() for x in line.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except (OSError, subprocess.SubprocessError, ValueError) as e:
        return {"name": "unknown", "error": str(e)}


def child(args) -> None:
    sys.path.insert(0, str(REF))
    sys.path.insert(0, str(ROOT))
    os.environ.setdefault("FLASHINFER_WORKSPACE_BASE", str(ROOT / "oracle" / "_ref" / "flashinfer_ws"))
    import torch

    import minisgl_b200

    b200_layers = minisgl_b200.PACKAGE.layers
    assert b200_layers.install_into_minisgl(norm_rope=True, row_gather=True, attention=False)
    import minisgl.scheduler.scheduler as ref_sched

    ref_sched.load_tokenizer = lambda path: insitu._StubTokenizer()
    from minisgl.core import Batch, Req, get_global_ctx
    from minisgl.llm import LLM

    model_dir = Path(tempfile.mkdtemp(prefix="q3cfg_"))
    (model_dir / "config.json").write_text(json.dumps(insitu.QWEN3_0_6B))
    ps, ctx_len, bs_list = args.page_size, args.ctx, sorted(args.bs)
    max_bs = max(bs_list)
    pages_per_req = -(-(ctx_len + 1) // ps)
    llm = LLM(str(model_dir), attention_backend="b200", page_size=ps, max_seq_len_override=ctx_len + 64,
              max_extend_tokens=4096, cuda_graph_bs=bs_list, use_dummy_weight=True,
              num_page_override=max_bs * pages_per_req + 1, max_running_req=max_bs)
    eng = llm.engine
    runner, backend = eng.graph_runner, eng.attn_backend
    assert type(backend).__name__ == "B200AttnBackend", type(backend)
    graphs = {"unpatched": dict(runner.graph_map)}

    # the fused forward, captured the way GraphRunner._capture_graphs does, on the runner's own buffers
    n = b200_layers.patch_minisgl_attention(eng.model)
    assert n == insitu.QWEN3_0_6B["num_hidden_layers"], n
    fused, pool = {}, None
    for bs in sorted(bs_list, reverse=True):
        g = torch.cuda.CUDAGraph()
        batch = Batch(reqs=[eng.dummy_req] * bs, phase="decode")
        batch.padded_reqs = batch.reqs
        backend.prepare_for_capture(batch)
        runner.buffer.set_batch(batch)
        with get_global_ctx().forward_batch(batch):
            runner.buffer.logits[:bs] = eng.model.forward()
            with torch.cuda.graph(g, pool=pool, stream=runner.stream):
                runner.buffer.logits[:bs] = eng.model.forward()
        pool = pool or g.pool()
        fused[bs] = g
    graphs["patched"] = fused

    # live decode batches: request i owns pages [i * pages_per_req, ...), ctx_len tokens cached, one appended
    gen = torch.Generator().manual_seed(0)
    for i in range(max_bs):
        eng.page_table[i, : ctx_len + 1] = torch.arange(ctx_len + 1, dtype=torch.int32, device=eng.device) \
            + i * pages_per_req * ps
    results = []
    for bs in bs_list:
        reqs = [Req(input_ids=torch.randint(1, 10000, (ctx_len + 1,), generator=gen, dtype=torch.int32),
                    table_idx=i, cached_len=ctx_len, output_len=16, uid=i, sampling_params=None,
                    cache_handle=None) for i in range(bs)]
        batch = Batch(reqs=reqs, phase="decode")
        batch.padded_reqs = reqs
        batch.input_ids = torch.randint(1, 10000, (bs,), generator=gen, dtype=torch.int32).to(eng.device)
        batch.positions = torch.full((bs,), ctx_len, dtype=torch.int32, device=eng.device)
        batch.out_loc = eng.page_table[:bs, ctx_len].clone()
        backend.prepare_metadata(batch)
        torch.cuda.synchronize()
        per_mode = {"unpatched": [], "patched": []}
        order = ["unpatched", "patched"]
        for rd in range(-1, args.rounds):  # round -1 is warm-up
            for mode in (order if rd % 2 == 0 else order[::-1]):
                runner.graph_map = graphs[mode]
                steps = args.warmup if rd < 0 else args.steps
                start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                for _ in range(steps):
                    runner.replay(batch)
                end.record()
                end.synchronize()
                if rd >= 0:
                    per_mode[mode].append(start.elapsed_time(end) * 1e3 / steps)
        # both graph sets compute the same logits bit for bit
        runner.graph_map = graphs["unpatched"]
        a = runner.replay(batch).clone()
        runner.graph_map = graphs["patched"]
        b = runner.replay(batch).clone()
        row = {"page_size": ps, "bs": bs, "ctx": ctx_len,
               "unpatched_us": statistics.median(per_mode["unpatched"]),
               "patched_us": statistics.median(per_mode["patched"]),
               "unpatched_us_rounds": [round(x, 1) for x in per_mode["unpatched"]],
               "patched_us_rounds": [round(x, 1) for x in per_mode["patched"]],
               "logits_bit_identical": bool(torch.equal(a, b))}
        row["saved_us"] = row["unpatched_us"] - row["patched_us"]
        results.append(row)
        print(f"[decode_time] page {ps} bs {bs}: unpatched {row['unpatched_us']:.1f} us, patched "
              f"{row['patched_us']:.1f} us, bits {'same' if row['logits_bit_identical'] else 'DIFFER'}", flush=True)
    runner.graph_map = graphs["unpatched"]
    Path(args.out).write_text(json.dumps(results))
    try:
        llm.shutdown()
    except Exception as e:  # pragma: no cover
        print("[decode_time] shutdown:", e)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--page-size", type=int, default=64, help=argparse.SUPPRESS)
    ap.add_argument("--page-sizes", type=int, nargs="+", default=[64, 1])
    ap.add_argument("--bs", type=int, nargs="+", default=[1, 64, 256])
    ap.add_argument("--ctx", type=int, default=1024, help="cached tokens per request")
    ap.add_argument("--steps", type=int, default=50, help="replays per timed round")
    ap.add_argument("--warmup", type=int, default=20, help="replays per mode before timing")
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not insitu.reference_available():
        raise SystemExit("the reference is not installed: MINISGL_REFERENCE=<reference checkout> python -m oracle.reference_site")
    if args.child:
        return child(args)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        for ps in args.page_sizes:
            out = Path(tmp) / f"p{ps}.json"
            cmd = [sys.executable, str(Path(__file__).resolve()), "--child", "--page-size", str(ps), "--out", str(out),
                   "--ctx", str(args.ctx), "--steps", str(args.steps), "--warmup", str(args.warmup),
                   "--rounds", str(args.rounds), "--bs", *map(str, args.bs)]
            subprocess.run(cmd, check=True, cwd=str(ROOT))
            rows += json.loads(out.read_text())
    summary = {"card": card(), "model": "Qwen3-0.6B shape, 28 layers, dummy weights, bf16, reference engine",
               "unit": "us per captured decode step (median of rounds)", "rows": rows}
    print(json.dumps(summary, indent=1))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(summary, indent=1))


if __name__ == "__main__":
    main()
