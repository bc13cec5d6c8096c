"""Decode with GQA groups of 9 to 16 query heads per kv head (the wgmma decode kernel at N = 16): the shapes of
96 q / 8 kv heads (group 12), 64 / 4 and 128 / 8 heads (group 16) under tensor parallelism, and odd groups, held
to the same checks as the groups of 1 to 8 in test_gpu_attention.py -- fp32 oracle, appended K/V rows bit-exact,
every other row of the NaN-poisoned pool untouched, the fused pre-attention launch bit-identical to the
two-launch sequence -- plus needles that pin every query head to its own key and an end-to-end generation."""
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from helpers import (SPLIT_PLAN, GpuWorld, add_requests, assert_bits_equal, attn_tolerance_ok, make_inputs,
                     make_world, options, oracle_forward, padded_reqs, run_attention)
from oracle import metadata as o_meta
from oracle.cpu_backend import CpuPool, SDPACpuBackend
from plumbing import TinyModel, oracle_pre_attention, run_generation
from test_gpu_attention import DECODE_LENS, _fused_vs_unfused, _run_case
from test_gpu_attention_probes import _check_exact, _run, _world

pytestmark = pytest.mark.gpu

GROUP_SHAPES = [(9, 1), (12, 1), (16, 1), (24, 2), (32, 2), (96, 8), (128, 8)]
SHAPE_IDS = [f"hq{hq}-hkv{hkv}" for hq, hkv in GROUP_SHAPES]


@pytest.fixture(params=[1, 0, 2], ids=["inkernel-merge", "combine-launch", "combine-auto"])
def merge(request, b200, native_lib):
    """The split-KV merge of the wgmma decode kernel: by the last-arriving chunk inside the launch (default), as
    its own launch over all hq heads, and in the launch only when the plan splits nothing."""
    with options(b200, decode_impl=1, decode_fused_combine=request.param):
        yield request.param


@pytest.mark.parametrize("name", list(DECODE_LENS))
@pytest.mark.parametrize("page_size", [1, 16, 64])
@pytest.mark.parametrize("hq,hkv", GROUP_SHAPES, ids=SHAPE_IDS)
def test_decode_large_groups(b200, native_lib, hq, hkv, page_size, name):
    _run_case(b200, page_size=page_size, hq=hq, hkv=hkv, lens=DECODE_LENS[name], phase="decode")


@pytest.mark.parametrize("hq,hkv", GROUP_SHAPES, ids=SHAPE_IDS)
def test_decode_large_groups_long_merge_variants(b200, native_lib, hq, hkv, merge):
    """kv_len 4096 and 3000: the default plan splits these, so every merge variant runs."""
    _run_case(b200, page_size=16, hq=hq, hkv=hkv, lens=DECODE_LENS["long"], phase="decode")


@pytest.mark.parametrize("hq,hkv", [(12, 1), (16, 1), (96, 8), (128, 8)])
def test_decode_large_groups_split_plan(b200, native_lib, hq, hkv, merge):
    """Every request cut into 128-key chunks: multi-chunk merges of 12 and 16 heads per kv head."""
    with options(b200, **SPLIT_PLAN):
        _run_case(b200, page_size=16, hq=hq, hkv=hkv, lens=DECODE_LENS["mixed"][:5] + DECODE_LENS["long"][:1],
                  phase="decode")


@pytest.mark.parametrize("hq,hkv", [(12, 1), (16, 1)])
def test_decode_large_groups_padded_fp16_second_layer(b200, native_lib, hq, hkv):
    _run_case(b200, page_size=16, hq=hq, hkv=hkv, lens=DECODE_LENS["mixed"][:3], phase="decode", pad_to=8)
    _run_case(b200, page_size=1, hq=hq, hkv=hkv, lens=DECODE_LENS["mixed"][:4], phase="decode", dtype=torch.float16)
    _run_case(b200, page_size=16, hq=hq, hkv=hkv, lens=DECODE_LENS["tiny"], phase="decode", layer=1, layers=2)


@pytest.mark.parametrize("hq,hkv", [(12, 1), (16, 1), (96, 8)])
def test_decode_large_groups_graph_replay(b200, native_lib, hq, hkv, merge):
    """A decode launch captured into a CUDA graph on dummy requests and replayed on a live padded batch."""
    ps = 16
    w = make_world(seed=4, page_size=ps, hq=hq, hkv=hkv, max_reqs=9, max_seq=1024)
    add_requests(w, [(99, 100), (511, 512), (300, 301)])
    reqs = padded_reqs(w, 4)
    ref_md = o_meta.ref_prepare_metadata(w.page_table, reqs, ps)
    qkv, q, k, v = make_inputs(w, 9, reqs=reqs)
    ref_out, ref_kc, ref_vc = oracle_forward(w, 0, q, k, v, ref_md, reqs=reqs)
    gw = GpuWorld(b200, w)
    out, _, kc, vc = run_attention(gw, gw.batch("decode", pad_to=4, md=ref_md), qkv.cuda(), graph=True)
    attn_tolerance_ok(out[:3], ref_out[:3], f"graph replay {hq}/{hkv}")
    slots = torch.from_numpy(ref_md.out_loc[:3].astype(np.int64))
    assert_bits_equal(kc[slots], ref_kc[slots], "appended k rows")
    assert_bits_equal(vc[slots], ref_vc[slots], "appended v rows")


@pytest.mark.parametrize("norms", ["both", "none", "q", "k"], ids=["qk-norm", "no-norm", "q-norm", "k-norm"])
@pytest.mark.parametrize("hq,hkv", [(9, 1), (12, 1), (16, 1), (32, 2)])
def test_decode_fused_large_groups_bit_identical(b200, native_lib, hq, hkv, norms):
    """The fused launch (qk-norm + RoPE of up to 16 q rows and the k row in the Q loader) equals
    ops.qknorm_rope_inplace followed by forward, bit for bit, with both norm weights, none, or only one."""
    _fused_vs_unfused(b200, page_size=16, hq=hq, hkv=hkv, lens=DECODE_LENS["mixed"][:5], norms=norms)


@pytest.mark.parametrize("hq,hkv", [(12, 1), (16, 1)])
def test_decode_fused_large_groups_split_padded(b200, native_lib, hq, hkv):
    _fused_vs_unfused(b200, page_size=64, hq=hq, hkv=hkv, lens=DECODE_LENS["long"] + [(700, 701)], force_split=True)
    _fused_vs_unfused(b200, page_size=1, hq=hq, hkv=hkv, lens=DECODE_LENS["tiny"], pad_to=10)


# ------------------------------------------------------------------------------------------- head routing
NEEDLE_Q, NEEDLE_K, V_MAX = 32.0, 64.0, 32


def _routing_build(reqs, hq, hkv, dtype, seed):
    """Needle decode requests [(kv_len, [pos per query head])] for groups up to 16: query head (h, g) has
    q[g] = 32 and zeros elsewhere, its key K[pos, h, g] = 64, and every key is zero in dims 0-15 otherwise, so
    head (h, g) scores 2048 at its needle and exactly 0 at every other key: its output is V[pos, h] bit for bit.
    Heads of a group get distinct positions, so a swapped column or N-half returns another head's V row."""
    G = hq // hkv
    want = torch.empty(len(reqs), hq, 128, dtype=dtype)

    def build(chunk):
        gen = torch.Generator().manual_seed(seed)
        kv, q = [], torch.zeros(len(reqs), hq, 128)
        for r, (n, pos) in enumerate(reqs):
            k = torch.randn((n, hkv, 128), generator=gen)
            k[..., :16] = 0
            v = torch.randint(-V_MAX, V_MAX + 1, (n, hkv, 128), generator=gen).float()
            for head in range(hq):
                h, g = divmod(head, G)
                k[pos[head], h, g] = NEEDLE_K
                q[r, head, g] = NEEDLE_Q
                want[r, head] = v[pos[head], h].to(dtype)
            kv.append((k.to(dtype), v.to(dtype)))
        return kv, q.to(dtype)

    return build, want


@pytest.mark.parametrize("plan,merge", [("unsplit", 1), ("split", 1), ("split", 0), ("split", 2)],
                         ids=["unsplit", "split-inkernel-merge", "split-combine-launch", "split-combine-auto"])
@pytest.mark.parametrize("page_size", [1, 64])
@pytest.mark.parametrize("hq,hkv", [(9, 1), (12, 1), (16, 1), (32, 2), (128, 8)])
def test_decode_head_routing_needles(b200, native_lib, hq, hkv, page_size, plan, merge):
    rnd = random.Random(hq * 1000 + page_size)
    lens = [2, 17, 129, 130, 300, 700, 1025]
    reqs = []
    for n in lens:
        pos = rnd.sample(range(n), min(n, hq))
        reqs.append((n, pos + [rnd.randrange(n) for _ in range(hq - len(pos))]))
    w = _world(page_size=page_size, hq=hq, hkv=hkv, dtype=torch.bfloat16, lens=[(n - 1, n) for n, _ in reqs])
    build, want = _routing_build(reqs, hq, hkv, torch.bfloat16, seed=hq)
    opts = {"decode_impl": 1, "decode_fused_combine": merge,
            **({"decode_plan_nosplit": 1} if plan == "unsplit" else SPLIT_PLAN)}
    out, kv, _, _, batch, _ = _run(b200, w, "decode", build, opts)
    total = int(batch.attn_metadata.decode_plan[1])
    assert (total == len(reqs)) if plan == "unsplit" else (total > len(reqs))
    _check_exact(out, want, kv, reqs, hq, hkv, f"routing ps={page_size} {hq}/{hkv} {plan} merge={merge}")


# ------------------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("page_size", [1, 64])
@pytest.mark.parametrize("hq,hkv", [(24, 2), (16, 1)])
def test_generation_with_large_groups_matches_cpu_oracle_backend(b200, native_lib, hq, hkv, page_size):
    """The tiny model of tests/plumbing.py at groups of 12 and 16: prefill, then 11 decode steps through
    AttentionLayer (fused qk-norm + RoPE decode) and B200AttnBackend, teacher-forced on the CPU oracle backend's
    tokens; the hidden state of every step must agree to bf16 noise."""
    layers, n_seqs, in_len, out_len, hidden, vocab, max_seq, d = 2, 4, 128, 12, 256, 512, 256, 128
    rnd = random.Random(0)
    prompts = [[rnd.randrange(vocab) for _ in range(in_len - 7 * i)] for i in range(n_seqs)]
    num_pages = n_seqs * max_seq // page_size + 4

    def setup(device):
        ctx = b200.Context(page_size)
        b200.core.set_global_ctx(None)
        b200.set_global_ctx(ctx)
        ctx.page_table = torch.zeros((n_seqs + 1, max_seq), dtype=torch.int32, device=device)
        free = [p * page_size for p in range(num_pages)]
        random.Random(page_size).shuffle(free)
        return ctx, free

    ctx, free = setup(torch.device("cpu"))
    ctx.kv_cache = CpuPool(hkv, layers, d, num_pages + 1, page_size, torch.bfloat16)
    cpu_backend = SDPACpuBackend(ctx, hq, hkv, d)
    ctx.attn_backend = cpu_backend
    model = TinyModel(hq, hkv, d, layers, hidden, vocab, torch.device("cpu"))
    ref_trace = []
    ref_ids, _ = run_generation(model, ctx, cpu_backend, b200.Req, b200.Batch, prompts, out_len, page_size,
                                lambda m, l, qkv, batch: oracle_pre_attention(m, l, qkv, batch, cpu_backend), free,
                                hidden_trace=ref_trace)

    dev = torch.device("cuda")
    ctx, free = setup(dev)
    ctx.kv_cache = b200.MHAKVCache(hkv, layers, d, num_pages + 1, page_size, torch.bfloat16, dev)
    ctx.kv_cache._kv_buffer.fill_(float("nan"))
    backend = b200.create_attention_backend("b200", SimpleNamespace(num_qo_heads=hq, num_kv_heads=hkv, head_dim=d))
    ctx.attn_backend = backend
    gmodel = TinyModel(hq, hkv, d, layers, hidden, vocab, dev)
    rotary = b200.layers.RotaryEmbedding(d, d, 4096, 1e6, device=dev)
    attn_layers = []
    for l in range(layers):
        qn, kn = b200.layers.RMSNorm(d, 1e-6), b200.layers.RMSNorm(d, 1e-6)
        qn.weight, kn.weight = gmodel.qw[l], gmodel.kw[l]
        attn_layers.append(b200.layers.AttentionLayer(l, hq, hkv, d, rotary, qn, kn, fuse_pre_attention=True))
    trace = []
    ids, _ = run_generation(gmodel, ctx, backend, b200.Req, b200.Batch, prompts, out_len, page_size,
                            lambda m, l, qkv, batch: attn_layers[l].forward(qkv), free, forced=ref_ids,
                            hidden_trace=trace)
    assert len(trace) == out_len
    for step, (a, b) in enumerate(zip(trace, ref_trace)):
        err = (a - b).abs().max().item() / b.abs().max().item()
        assert err < 3e-2, f"step {step}: hidden states differ by {err:.3e}"
    assert (ids == ref_ids).mean() >= 0.9, (ids, ref_ids)
