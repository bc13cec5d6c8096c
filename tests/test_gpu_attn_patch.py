"""The reference's own `AttentionLayer` (built by its __init__), re-bound by `layers.patch_minisgl_attention`,
captured into a CUDA graph on a padded dummy decode batch and replayed on a live one the way the engine's
GraphRunner does (engine/graph.py:133-158), against our `layers.AttentionLayer` run eagerly on the same batch:
outputs and appended K / V rows bit for bit, and ONE launch per captured forward.  Skipped when build()
found no reference checkout."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from helpers import GpuWorld, add_requests, assert_bits_equal, make_inputs, make_world, padded_reqs
from oracle import metadata as o_meta
from refsite import minisgl_ref  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

HQ, HKV, D = 16, 8, 128
LENS = [(70, 71), (150, 151), (500, 501)]
PAD_TO = 4


@pytest.mark.parametrize("page_size", [1, 64])
def test_patched_reference_layer_in_graph_equals_mirror(b200, native_lib, minisgl_ref, page_size):
    from minisgl.distributed import set_tp_info, try_get_tp_info
    from minisgl.layers.attention import AttentionLayer as RefAttentionLayer

    lib = native_lib
    w = make_world(seed=11, page_size=page_size, hq=HQ, hkv=HKV, max_reqs=PAD_TO + 1, max_seq=512)
    add_requests(w, LENS)
    reqs = padded_reqs(w, PAD_TO)
    md = o_meta.ref_prepare_metadata(w.page_table, reqs, page_size)
    qkv, _, _, _ = make_inputs(w, 12, reqs=reqs)
    x = qkv.cuda()
    g = torch.Generator().manual_seed(13)
    q_norm, k_norm = b200.layers.RMSNorm(D, 1e-6), b200.layers.RMSNorm(D, 1e-6)
    q_norm.weight = (torch.rand(D, generator=g) + 0.5).to(torch.bfloat16).cuda()
    k_norm.weight = (torch.rand(D, generator=g) + 0.5).to(torch.bfloat16).cuda()

    if try_get_tp_info() is None:
        set_tp_info(rank=0, size=1)
    rope = SimpleNamespace(rotary_dim=D, max_position=1024, base=1e6, scaling=None)
    with torch.device("cuda"):
        ref = RefAttentionLayer(0, HQ, HKV, D, rope, q_norm=q_norm, k_norm=k_norm)
    mirror = b200.layers.AttentionLayer(0, HQ, HKV, D, ref.rotary, q_norm, k_norm, fuse_pre_attention=True)

    # our layer, eager
    gw = GpuWorld(b200, w)
    batch = gw.batch("decode", pad_to=PAD_TO, md=md)
    gw.backend.prepare_metadata(batch)
    with gw.ctx.forward_batch(batch):
        before = lib.b200_launch_count()
        want = mirror.forward(x)
        assert lib.b200_launch_count() - before == 1
    torch.cuda.synchronize()
    want_k, want_v = gw.pool_rows(0)

    # the reference's layer, patched, captured on a dummy batch and replayed on the live one
    assert b200.layers.patch_minisgl_attention(SimpleNamespace(self_attn=SimpleNamespace(attn=ref))) == 1
    gw = GpuWorld(b200, w)
    backend = gw.backend
    backend.init_capture_graph(w.page_table.shape[1], [PAD_TO])
    dummy = b200.Req(table_idx=w.page_table.shape[0] - 1, cached_len=0, device_len=1)
    cap = b200.Batch([dummy] * PAD_TO, "decode")
    cap.padded_reqs = cap.reqs
    backend.prepare_for_capture(cap)
    cap.positions = torch.zeros(PAD_TO, dtype=torch.int32, device=gw.dev)
    cap.out_loc = torch.full((PAD_TO,), int(w.page_table[-1, 0]), dtype=torch.int32, device=gw.dev)
    x_buf = torch.zeros_like(x)
    out = torch.zeros(PAD_TO, HQ * D, dtype=x.dtype, device=gw.dev)
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream), gw.ctx.forward_batch(cap):
        out.copy_(ref.forward(x_buf))  # warm-up outside the capture, as the graph runner does
        before = lib.b200_launch_count()
        with torch.cuda.graph(graph, stream=stream):
            out.copy_(ref.forward(x_buf))
        assert lib.b200_launch_count() - before == 1
    torch.cuda.synchronize()
    live = gw.batch("decode", pad_to=PAD_TO, md=md)
    backend.prepare_metadata(live)
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        x_buf.copy_(x)
        cap.positions.copy_(live.positions)
        cap.out_loc.copy_(live.out_loc)
        backend.prepare_for_replay(live)
        graph.replay()
    torch.cuda.synchronize()
    got_k, got_v = gw.pool_rows(0)

    n = len(LENS)
    assert_bits_equal(out[:n], want[:n], "patched reference layer vs our layer: output")
    slots = torch.from_numpy(md.out_loc[:n].astype(np.int64)).to(gw.dev)
    assert_bits_equal(got_k[slots], want_k[slots], "appended k rows")
    assert_bits_equal(got_v[slots], want_v[slots], "appended v rows")
    assert_bits_equal(x_buf, x, "raw qkv rows after the fused decode")
