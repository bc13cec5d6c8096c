#!/usr/bin/env python
"""In-situ drop-in check: the UNMODIFIED reference (`minisgl`, copied into the git-ignored
oracle/_ref/minisgl_site by build(), see oracle/reference_site.py) drives the attention backend through its own `LLM` -> `Scheduler` -> `Engine` ->
`GraphRunner` -> `CacheManager` stack, once per attention backend, and the bf16 logits of every
forward (prefill, chunked prefill, radix-hit extend, graph-replayed padded decode) are compared.

  child mode (one process per engine -- `Engine` asserts a fresh CUDA context, engine.py:32):
      python tools/insitu.py child --attn b200 --page-size 64 --out /tmp/x.pt [--force /tmp/fi.pt]
             [--patch none|flashinfer|model|fused] [--patch-kernels] [--unfused-attention]
  driver mode (spawns the children, compares, prints + writes a JSON summary):
      python tools/insitu.py run --out insitu_summary.json
  `run_fused()` spawns the children of tests/test_gpu_insitu_fused.py (`--patch fused` against `--patch model`).
  census mode (which kernels one eager prefill forward and one decode graph replay launch, torch.profiler):
      python tools/insitu.py census --out census.json

What the reference is asked to do (reference file:line of the code that runs):
  * `LLM.generate` twice (llm/llm.py:81-98): round A fills the radix cache, round B re-uses two of
    its prefixes => `cached_len > 0` extends (scheduler/prefill.py:39-61, kvcache/radix_cache.py);
  * `max_extend_tokens=256` => the 515-token prompt is chunked (prefill.py:64-90, `ChunkedReq`);
  * decode batches of 3..6 requests are padded to the captured sizes 4 / 8 with the dummy request
    (engine/graph.py:154-166) and replayed (graph.py:147-152) => `prepare_for_replay`;
  * overlap scheduling is on (scheduler.py:83-106): `prepare_metadata` of step i+1 runs on the
    scheduler stream while step i is in flight.
Greedy sampling; every run but the first is teacher-forced with the first run's tokens (the sampler's
argmax is replaced, engine/sample.py:70-75), so all runs see identical batches step by step.

Nothing under the reference is edited: the stub tokenizer and the hooks are module / instance
attributes set from here.
"""
from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
# the unmodified reference, copied by build() into a git-ignored directory (oracle/reference_site.py)
REF = ROOT / "oracle" / "_ref" / "minisgl_site"

QWEN3_0_6B = {  # public HF config of Qwen/Qwen3-0.6B (SURVEY.md section 8)
    "architectures": ["Qwen3ForCausalLM"], "model_type": "qwen3", "hidden_size": 1024,
    "intermediate_size": 3072, "num_hidden_layers": 28, "num_attention_heads": 16,
    "num_key_value_heads": 8, "head_dim": 128, "vocab_size": 151936,
    "max_position_embeddings": 40960, "rms_norm_eps": 1e-06, "rope_theta": 1000000,
    "rope_scaling": None, "hidden_act": "silu", "tie_word_embeddings": True,
    "torch_dtype": "bfloat16", "attention_bias": False,
}


def reference_available() -> bool:
    return (REF / "minisgl" / "core.py").exists()


def workload():
    """Two rounds of (prompt ids, max_tokens).  Round B shares page-aligned prefixes with round A."""
    rnd = random.Random(1234)
    tok = lambda n: [rnd.randrange(1, 10000) for _ in range(n)]  # noqa: E731
    a = [(tok(200), 10), (tok(37), 12), (tok(515), 9), (tok(3), 8), (tok(64), 11), (tok(130), 8)]
    b = [(a[0][0][:192] + tok(50), 9), (a[2][0][:400] + tok(30), 8), (tok(90), 10)]
    return [a, b]


# ------------------------------------------------------------------------------------ census
KERNEL_GROUPS = ("ours", "cublas", "flashinfer", "other")


def kernel_group(name: str) -> str:
    """ours (namespace b200 of libb200attn) / cuBLAS / FlashInfer / other (PyTorch's own kernels, copies)."""
    low = name.lower()
    if "b200::" in name:
        return "ours"
    if "flashinfer" in low:
        return "flashinfer"
    if any(k in low for k in ("cublas", "gemm", "nvjet", "xmma", "cutlass")):
        return "cublas"
    return "other"


def profile_kernels(fn):
    """Run fn() under torch.profiler with CUDA activities; returns (fn's result, {group: {kernel: launches}})."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        result = fn()
        torch.cuda.synchronize()
    groups = {g: {} for g in KERNEL_GROUPS}
    for e in prof.events():
        if str(e.device_type).endswith("CUDA"):
            kinds = groups[kernel_group(e.name)]
            kinds[e.name] = kinds.get(e.name, 0) + 1
    return result, groups


# ------------------------------------------------------------------------------------- child
class _StubTokenizer:
    eos_token_id = -1

    def decode(self, ids, **kw):
        return ""

    def encode(self, text, **kw):
        raise RuntimeError("the in-situ harness feeds token ids only")


def child(args) -> None:
    sys.path.insert(0, str(REF))
    sys.path.insert(0, str(ROOT))
    os.environ.setdefault("FLASHINFER_WORKSPACE_BASE", str(ROOT / "oracle" / "_ref" / "flashinfer_ws"))
    if args.fi_tensor_cores:  # the reference's own switch (env.py FLASHINFER_USE_TENSOR_CORES, fi.py use_tensor_cores)
        os.environ["MINISGL_FLASHINFER_USE_TENSOR_CORES"] = "1"
    import torch

    model_dir = Path(tempfile.mkdtemp(prefix="q3cfg_"))
    cfg = dict(QWEN3_0_6B)
    cfg["num_hidden_layers"] = args.layers
    (model_dir / "config.json").write_text(json.dumps(cfg))

    uses_b200 = "b200" in args.attn
    if uses_b200 or args.patch != "none" or args.patch_kernels:
        import minisgl_b200  # registers "b200" with the reference's registry

        b200_layers = minisgl_b200.PACKAGE.layers
    if args.patch == "flashinfer":  # the documented one-call integration (INTEGRATION.md section 2)
        assert b200_layers.install_into_minisgl(norm_rope=True, row_gather=args.patch_kernels,
                                                attention=not args.unfused_attention)
    import minisgl.scheduler.scheduler as ref_sched

    ref_sched.load_tokenizer = lambda path: _StubTokenizer()  # no tokenizer files offline
    import minisgl.engine.engine as ref_engine
    from minisgl.core import get_global_ctx as ref_ctx

    real_runner = ref_engine.GraphRunner
    forwards = {"prefill": 0, "decode": 0}  # model forwards that launch kernels: eager or being captured
    census = {}

    def launch_count():
        return int(minisgl_b200.PACKAGE._cabi.launch_count()) if "minisgl_b200" in sys.modules else 0

    def runner_with_patched_model(*a, **kw):
        model = kw["model"]
        if args.patch in ("model", "fused"):
            n = b200_layers.patch_minisgl_layers(model)
            print(f"[insitu] patch_minisgl_layers re-bound {n} layers", flush=True)
            assert n > 0
        if args.patch == "fused":
            n = b200_layers.patch_minisgl_attention(model)
            print(f"[insitu] patch_minisgl_attention re-bound {n} layers", flush=True)
            assert n == args.layers
        real_model_forward = model.forward

        def counted_forward(*fa, **fkw):  # graph replays do not call it
            phase = ref_ctx().batch.phase
            forwards[phase] += 1
            if args.census and phase == "prefill" and "prefill_forward" not in census:
                before = launch_count()
                out, census["prefill_forward"] = profile_kernels(lambda: real_model_forward(*fa, **fkw))
                census["prefill_forward_b200_launches"] = launch_count() - before
                return out
            return real_model_forward(*fa, **fkw)

        model.forward = counted_forward
        return real_runner(*a, **kw)

    ref_engine.GraphRunner = runner_with_patched_model
    if args.patch_kernels:
        assert b200_layers.patch_minisgl_kernels()

    from minisgl.core import SamplingParams
    from minisgl.llm import LLM
    from minisgl.scheduler.prefill import ChunkedReq

    tokens_total = 16384
    t0 = time.time()
    llm = LLM(
        str(model_dir), attention_backend=args.attn, page_size=args.page_size, cache_type=args.cache,
        max_seq_len_override=2048, max_extend_tokens=args.max_extend, cuda_graph_bs=[1, 2, 4, 8],
        use_dummy_weight=True, num_page_override=tokens_total // args.page_size, max_running_req=16,
    )
    print(f"[insitu] engine up in {time.time() - t0:.1f}s backend={type(llm.engine.attn_backend).__name__}", flush=True)
    eng = llm.engine
    if uses_b200:
        from minisgl.attention.base import BaseAttnBackend

        be = eng.attn_backend
        assert isinstance(be, BaseAttnBackend), "b200 backend is not a reference BaseAttnBackend"
        assert type(be).__module__.startswith("mini-sglang_b200"), type(be)

    if args.census:
        real_replay, real_sample = eng.graph_runner.replay, eng.sampler.sample

        def replay(batch):
            if "decode_replay" in census:
                return real_replay(batch)
            logits, census["decode_replay"] = profile_kernels(lambda: real_replay(batch))
            census["decode_replay_bs"] = [int(batch.size), int(batch.padded_size)]
            # the engine's own sampler on these logits, outside the forward (its result is not used)
            sargs = eng.sampler.prepare(batch)
            _, census["sampler"] = profile_kernels(lambda: real_sample(logits, sargs))
            return logits

        eng.graph_runner.replay = replay

    forced = torch.load(args.force)["tokens"] if args.force else None
    state = {"round": 0, "count": {}}
    records, tokens_out, appended = [], {}, {}

    real_forward_batch = eng.forward_batch

    def forward_batch(batch, sargs):
        state["batch"] = batch
        state["pre"] = [(int(r.uid), int(r.cached_len), int(r.device_len), isinstance(r, ChunkedReq)) for r in batch.reqs]
        return real_forward_batch(batch, sargs)

    def sample(logits, sargs):
        batch, pre, rd = state["batch"], state["pre"], state["round"]
        out_loc = batch.out_loc.cpu()
        off = 0
        for (uid, c, d, _chunk) in pre:  # slot of every appended (round, uid, position)
            for p in range(c, d):
                appended[(rd, uid, p)] = int(out_loc[off])
                off += 1
        picked = torch.argmax(logits, dim=-1)
        toks = []
        for i, (uid, c, d, chunk) in enumerate(pre):
            if chunk:
                toks.append(0)  # never used (ChunkedReq.append_host raises; scheduler skips it)
                continue
            key = (rd, uid)
            idx = state["count"].get(key, 0)
            state["count"][key] = idx + 1
            t = int(forced[key][idx]) if forced is not None else int(picked[i])
            toks.append(t)
            tokens_out.setdefault(key, []).append(t)
        records.append({"round": rd, "phase": batch.phase, "reqs": pre, "padded": int(batch.padded_size),
                        "graph": bool(eng.graph_runner.can_use_cuda_graph(batch)),
                        "logits": logits.float().cpu()})
        return torch.tensor(toks, dtype=picked.dtype, device=logits.device)

    eng.forward_batch = forward_batch
    eng.sampler.sample = sample

    for rd, reqs in enumerate(workload()):
        state["round"] = rd
        prompts = [p for p, _ in reqs]
        sps = [SamplingParams(temperature=0.0, ignore_eos=True, max_tokens=n) for _, n in reqs]
        llm.generate(prompts, sps)
    torch.cuda.synchronize()

    # K / V rows of every appended token, first and last layer, in canonical (round, uid, pos) order
    keys = sorted(appended)
    slots = torch.tensor([appended[k] for k in keys], dtype=torch.int64, device=eng.device)
    kv = {}
    for name, layer in (("first", 0), ("last", args.layers - 1)):
        kc = eng.kv_cache.k_cache(layer).reshape(-1, eng.kv_cache.k_cache(layer).shape[-2] * 128)
        vc = eng.kv_cache.v_cache(layer).reshape(-1, eng.kv_cache.v_cache(layer).shape[-2] * 128)
        kv[name] = (kc[slots].cpu(), vc[slots].cpu())
    launches = None
    if uses_b200 or args.patch != "none" or args.patch_kernels:
        launches = int(minisgl_b200.PACKAGE._cabi.launch_count())
    torch.save({"records": records, "tokens": tokens_out, "append_keys": keys, "kv": kv,
                "b200_launches": launches, "forwards": forwards, "args": vars(args)}, args.out)
    print(f"[insitu] {len(records)} forwards recorded, b200 kernel launches: {launches}", flush=True)
    if args.census:
        Path(args.census).write_text(json.dumps(census, indent=1))
    try:
        llm.shutdown()
    except Exception as e:  # pragma: no cover
        print("[insitu] shutdown:", e)


# ------------------------------------------------------------------------------------- compare
def logits_rel_err(a, b) -> float:
    """THE logits criterion (north_star: 1e-3 relative for bf16 logits): per request row,
    max|a - b| / max|b| over the vocabulary; the worst row of the forward is returned."""
    import torch

    num = (a - b).abs().amax(dim=-1)
    den = b.abs().amax(dim=-1).clamp_min(1e-12)
    return float((num / den).max())


def compare(path_a: str, path_b: str) -> dict:
    """a = run under test, b = the reference run.  Rows are matched by uid (decode batches are
    `list(set)`, scheduler/decode.py:32-35: any order)."""
    import torch

    A, B = torch.load(path_a), torch.load(path_b)
    ra, rb = A["records"], B["records"]
    assert len(ra) == len(rb), f"forward counts differ: {len(ra)} vs {len(rb)}"
    worst, per_phase, n_graph, n_ext, n_chunk = 0.0, {}, 0, 0, 0
    agree = tot = 0
    for x, y in zip(ra, rb):
        assert x["phase"] == y["phase"] and x["padded"] == y["padded"] and x["round"] == y["round"]
        assert sorted(x["reqs"]) == sorted(y["reqs"]), (x["reqs"], y["reqs"])
        order = [[u for (u, *_rest) in y["reqs"]].index(u) for (u, *_rest) in x["reqs"]]
        lb = y["logits"][order]
        e = logits_rel_err(x["logits"], lb)
        worst = max(worst, e)
        per_phase[x["phase"]] = max(per_phase.get(x["phase"], 0.0), e)
        n_graph += int(x["graph"])
        n_ext += sum(1 for (_, c, _, _) in x["reqs"] if c > 0 and x["phase"] == "prefill")
        n_chunk += sum(1 for (*_r, ch) in x["reqs"] if ch)
        agree += int((x["logits"].argmax(-1) == lb.argmax(-1)).sum())
        tot += lb.shape[0]
    assert A["append_keys"] == B["append_keys"], "the runs appended different (round, uid, position) sets"
    kv = {}
    for name in ("first", "last"):
        for i, which in enumerate("kv"):
            ta, tb = A["kv"][name][i], B["kv"][name][i]
            kv[f"{which}_{name}_bit_exact"] = bool(torch.equal(ta.view(torch.int16), tb.view(torch.int16)))
            kv[f"{which}_{name}_rel"] = float((ta.float() - tb.float()).abs().max() / tb.float().abs().max())
    return {"forwards": len(ra), "graph_replays": n_graph, "extend_reqs_with_cache_hit": n_ext,
            "chunked_reqs": n_chunk, "logits_rel_worst": worst, "logits_rel_by_phase": per_phase,
            "argmax_agree": f"{agree}/{tot}", "appended_tokens": len(A["append_keys"]), **kv,
            "b200_launches": A.get("b200_launches")}


def logits_bit_identical(path_a: str, path_b: str) -> bool:
    import torch

    A, B = torch.load(path_a), torch.load(path_b)
    if len(A["records"]) != len(B["records"]):
        return False
    for x, y in zip(A["records"], B["records"]):
        order = [[u for (u, *_r) in y["reqs"]].index(u) for (u, *_r) in x["reqs"]]
        if not torch.equal(x["logits"], y["logits"][order]):
            return False
    return True


def run_child(tag: str, out_dir: Path, attn: str, page_size: int, force: "str | None", patch: str = "none",
              patch_kernels: bool = False, layers: int = 28, timeout: int = 600, fi_tensor_cores: bool = False,
              unfused_attention: bool = False, census: "str | None" = None) -> str:
    out = out_dir / f"{tag}.pt"
    cmd = [sys.executable, str(Path(__file__).resolve()), "child", "--attn", attn, "--page-size", str(page_size),
           "--out", str(out), "--patch", patch, "--layers", str(layers)]
    if force:
        cmd += ["--force", force]
    if patch_kernels:
        cmd += ["--patch-kernels"]
    if fi_tensor_cores:
        cmd += ["--fi-tensor-cores"]
    if unfused_attention:
        cmd += ["--unfused-attention"]
    if census:
        cmd += ["--census", census]
    t0 = time.time()
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout, cwd=str(ROOT))
    log = res.stdout.decode(errors="replace")
    (out_dir / f"{tag}.log").write_text(log)
    if res.returncode != 0 or not out.exists():
        raise RuntimeError(f"in-situ child {tag} failed (rc={res.returncode}):\n{log[-4000:]}")
    print(f"[insitu] {tag}: ok in {time.time() - t0:.0f}s", flush=True)
    return str(out)


def run(args) -> dict:
    out_dir = Path(tempfile.mkdtemp(prefix="insitu_"))
    L = args.layers
    summary = {"model": f"Qwen3-0.6B shape, {L} layers, dummy weights (engine.py:140-144), bf16",
               "criterion": "per row max|a-b| / max|b| over the vocabulary, worst row of all forwards"}
    # canonical free-running run: the reference's FlashInfer path, page_size 1 (fi.py only knows page 1);
    # every other run is teacher-forced with its tokens.  The reference's second path for the spread it shows
    # against itself is its FlashInfer backend with tensor-core decode (16-bit P, as the reference runs it for
    # GQA >= 4 models, fi.py use_tensor_cores); its TRT-LLM-gen path ships sm_100 kernels only.
    fi1 = run_child("fi_p1", out_dir, "fi", 1, None, layers=L)
    runs, errors = {"fi_p1": fi1}, {}
    plan = [
        ("b200_p1", dict(attn="b200", page_size=1)),
        ("fi_p64", dict(attn="fi", page_size=64)),
        ("fi_tc_p64", dict(attn="fi", page_size=64, fi_tensor_cores=True)),
        ("b200_p64", dict(attn="b200", page_size=64)),
        ("b200_p64_patched", dict(attn="b200", page_size=64, patch="model", patch_kernels=True)),
        ("fi_p64_fipatched", dict(attn="fi", page_size=64, patch="flashinfer", patch_kernels=True)),
    ]
    for tag, kw in plan:
        try:
            runs[tag] = run_child(tag, out_dir, force=fi1, layers=L, **kw)
        except Exception as e:  # keep going: the summary says what is missing
            errors[tag] = str(e)[-1500:]
            print(f"[insitu] {tag} FAILED: {errors[tag]}", flush=True)
    pairs = {
        "b200_vs_fi_page1": ("b200_p1", "fi_p1"),
        "b200_vs_fi_page64": ("b200_p64", "fi_p64"),
        "fi_tc_vs_fi_page64": ("fi_tc_p64", "fi_p64"),
        "b200_vs_fi_tc_page64": ("b200_p64", "fi_tc_p64"),
        "b200_patched_vs_fi_page64": ("b200_p64_patched", "fi_p64"),
        "b200_patched_vs_b200_page64": ("b200_p64_patched", "b200_p64"),
    }
    for name, (a, b) in pairs.items():
        if a in runs and b in runs:
            summary[name] = compare(runs[a], runs[b])
    if "fi_p64_fipatched" in runs and "fi_p64" in runs:
        # the reference's own fi backend with OUR RMSNorm / RoPE / row-gather kernels inside the reference's model
        summary["fi_with_b200_layers_vs_fi_page64"] = compare(runs["fi_p64_fipatched"], runs["fi_p64"])
    if errors:
        summary["errors"] = errors
    summary["log_dir"] = str(out_dir)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(summary, indent=1))
    print(json.dumps(summary, indent=1))
    return summary


def run_fused(args) -> dict:
    """The fused attention forward inside the engine (`patch_minisgl_attention`, `--patch fused`) next to the
    unfused patched model (`--patch model`, our norm / RoPE kernels as separate launches) at page sizes 64 and 1,
    the one-call `install_into_minisgl` with the b200 backend, and with the reference's own fi backend with and
    without the attention patch.  Every run is teacher-forced with the tokens of the free-running fi_p64 run.
    Returns {tag: path of the child's .pt}; the comparisons are the caller's (tests/test_gpu_insitu_fused.py)."""
    out_dir = Path(tempfile.mkdtemp(prefix="insitu_fused_"))
    L = args.layers
    fi64 = run_child("fi_p64", out_dir, "fi", 64, None, layers=L)
    runs = {"fi_p64": fi64}
    plan = [
        ("fi_tc_p64", dict(attn="fi", page_size=64, fi_tensor_cores=True)),
        ("b200_p64_patched", dict(attn="b200", page_size=64, patch="model", patch_kernels=True)),
        ("b200_p64_fused", dict(attn="b200", page_size=64, patch="fused", patch_kernels=True)),
        ("b200_p1_patched", dict(attn="b200", page_size=1, patch="model", patch_kernels=True)),
        ("b200_p1_fused", dict(attn="b200", page_size=1, patch="fused", patch_kernels=True)),
        ("b200_p64_installed", dict(attn="b200", page_size=64, patch="flashinfer", patch_kernels=True)),
        ("fi_p64_installed", dict(attn="fi", page_size=64, patch="flashinfer", patch_kernels=True)),
        ("fi_p64_installed_unfused", dict(attn="fi", page_size=64, patch="flashinfer", patch_kernels=True,
                                          unfused_attention=True)),
    ]
    for tag, kw in plan:
        runs[tag] = run_child(tag, out_dir, force=fi64, layers=L, **kw)
    return runs


def run_census(args) -> dict:
    """Kernel census of the installed engine (`install_into_minisgl()`, b200 attention, page 64): every kernel of
    one eager prefill forward and of one decode graph replay, grouped ours / cuBLAS / FlashInfer / other, and the
    engine's sampler on that step's logits, reported apart (it runs after the forward).  The same engine with the
    model patched layer by layer (`--patch fused`, which leaves `flashinfer.silu_and_mul` bound) is the
    comparison: the installed prefill forward makes exactly one b200 launch more per layer (the MLP activation)."""
    out_dir = Path(tempfile.mkdtemp(prefix="insitu_census_"))
    L = args.layers
    summary = {"model": f"Qwen3-0.6B shape, {L} layers, dummy weights, bf16, attention_backend=b200, page 64"}
    for tag, patch in (("installed", "flashinfer"), ("patched_layers", "fused")):
        path = out_dir / f"{tag}.json"
        run_child(tag, out_dir, "b200", 64, None, patch=patch, patch_kernels=True, layers=L, census=str(path))
        summary[tag] = json.loads(path.read_text())
    inst, ref = summary["installed"], summary["patched_layers"]

    def count(groups, group):
        return sum(groups[group].values())

    summary["checks"] = {
        "installed_forward_flashinfer_kernels": count(inst["prefill_forward"], "flashinfer")
        + count(inst["decode_replay"], "flashinfer"),
        "installed_prefill_b200_launches_minus_patched_layers": inst["prefill_forward_b200_launches"]
        - ref["prefill_forward_b200_launches"],
        "layers": L,
    }
    c = summary["checks"]
    c["ok"] = c["installed_forward_flashinfer_kernels"] == 0 and c[
        "installed_prefill_b200_launches_minus_patched_layers"] == L
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(summary, indent=1))
    print(json.dumps(summary, indent=1))
    return summary


def main() -> None:
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="mode", required=True)
    c = sub.add_parser("child")
    c.add_argument("--attn", required=True)
    c.add_argument("--page-size", type=int, default=64)
    c.add_argument("--cache", default="radix")
    c.add_argument("--max-extend", type=int, default=256)
    c.add_argument("--layers", type=int, default=28)
    c.add_argument("--out", required=True)
    c.add_argument("--force", default=None)
    c.add_argument("--patch", default="none", choices=["none", "flashinfer", "model", "fused"])
    c.add_argument("--unfused-attention", action="store_true",
                   help="--patch flashinfer: install_into_minisgl(attention=False)")
    c.add_argument("--patch-kernels", action="store_true")
    c.add_argument("--fi-tensor-cores", action="store_true")
    c.add_argument("--census", default=None, help="write the kernel census of this engine to this JSON file")
    r = sub.add_parser("run")
    r.add_argument("--out", default=None)
    r.add_argument("--layers", type=int, default=28)
    k = sub.add_parser("census")
    k.add_argument("--out", default=None)
    k.add_argument("--layers", type=int, default=28)
    args = ap.parse_args()
    if not reference_available():
        raise SystemExit("the reference is not installed: MINISGL_REFERENCE=<reference checkout> python -m oracle.reference_site")
    {"child": child, "run": run, "census": run_census}[args.mode](args)


if __name__ == "__main__":
    main()
