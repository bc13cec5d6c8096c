"""The attention-layer forward shared by our ``AttentionLayer`` and the reference's patched one
(``layers.attention_forward``), which backend serves a batch (``layers.serving_attn_backend``), and
``layers.patch_minisgl_attention`` / ``install_into_minisgl`` re-binding the reference's layers, on CPU with
stand-in backends and kernels: which calls each kind of batch makes, not what they compute (the GPU tests
pin the bits)."""
import sys
from types import SimpleNamespace

import pytest
import torch

from refsite import minisgl_ref  # noqa: F401  (fixture)

HQ, HKV, D = 4, 2, 8


class _Foreign:
    """A backend that is not ours (fi / fa / trtllm)."""

    def forward(self, q, k, v, layer_id, batch):
        raise AssertionError("the foreign backend must not be reached through the fused path")


def _b200_stub(b200, calls):
    """A ``B200AttnBackend`` whose launches are recorded instead of run."""

    class Stub(b200.B200AttnBackend):
        def __init__(self):  # no device, no library
            pass

        def forward(self, q, k, v, layer_id, batch):
            calls.append(("forward", layer_id, tuple(q.shape)))
            return torch.zeros(q.shape[0], HQ, D)

        def forward_decode_fused(self, q, k, v, layer_id, batch, positions, cos_sin_cache, q_weight, k_weight, eps):
            calls.append(("decode_fused", layer_id, tuple(q.shape), eps))
            return torch.zeros(q.shape[0], HQ, D)

    return Stub()


def _batch(phase, n=3, dtype=torch.int32):
    return SimpleNamespace(is_prefill=phase == "prefill", is_decode=phase == "decode",
                           positions=torch.arange(n, dtype=dtype))


def _set_ctx(b200, backend):
    ctx = b200.Context(1)
    ctx.attn_backend = backend
    b200.set_global_ctx(ctx)
    return ctx


@pytest.fixture
def calls(b200, monkeypatch):
    """Recorded launches; ``ops.qknorm_rope_inplace`` is recorded too."""
    log = []
    monkeypatch.setattr(b200.ops, "qknorm_rope_inplace", lambda *a: log.append(("qknorm_rope",)))
    return log


def _fill_layer(layer, layer_id=5):
    """The attributes attention_forward reads, as the reference's __init__ sets them (attention.py:29-45)."""
    norm = SimpleNamespace(weight=torch.ones(D), eps=1e-6)
    layer.layer_id, layer.head_dim = layer_id, D
    layer.num_qo_heads, layer.num_kv_heads = HQ, HKV
    layer.qo_attn_dim, layer.kv_attn_dim = HQ * D, HKV * D
    layer.rotary = SimpleNamespace(_cos_sin_cache=torch.zeros(16, D))
    layer.q_norm, layer.k_norm = norm, norm
    return layer


def _qkv(n=3):
    return torch.zeros(n, (HQ + 2 * HKV) * D)


# ------------------------------------------------------------------ backend resolution
def test_serving_backend_resolution(b200):
    resolve = b200.layers.serving_attn_backend
    ours, foreign = _b200_stub(b200, []), _Foreign()
    prefill, decode = _batch("prefill"), _batch("decode")
    for batch in (prefill, decode):
        assert resolve(ours, batch) is ours
        assert resolve(foreign, batch) is foreign
    b200_fi = b200.attention.HybridBackend(ours, foreign)  # --attn b200,fi
    assert resolve(b200_fi, prefill) is ours and resolve(b200_fi, decode) is foreign
    fi_b200 = b200.attention.HybridBackend(foreign, ours)  # --attn fi,b200
    assert resolve(fi_b200, prefill) is foreign and resolve(fi_b200, decode) is ours


# ------------------------------------------------------------------ calls per batch
def test_mirror_layer_launches_with_b200_backend(b200, calls):
    """Our AttentionLayer with a plain B200AttnBackend: decode = one fused launch; prefill and int64-position
    decode = the fused norm + RoPE launch, then forward."""
    _set_ctx(b200, _b200_stub(b200, calls))
    layer = _fill_layer(b200.layers.AttentionLayer.__new__(b200.layers.AttentionLayer))
    layer.fuse_pre_attention = True
    ctx = b200.get_global_ctx()
    with ctx.forward_batch(_batch("decode")):
        assert layer.forward(_qkv()).shape == (3, HQ * D)
    assert calls == [("decode_fused", 5, (3, HQ, D), 1e-6)]
    calls.clear()
    with ctx.forward_batch(_batch("prefill", 7)):
        layer.forward(_qkv(7))
    with ctx.forward_batch(_batch("decode", dtype=torch.int64)):
        layer.forward(_qkv())
    assert calls == [("qknorm_rope",), ("forward", 5, (7, HQ, D)), ("qknorm_rope",), ("forward", 5, (3, HQ, D))]


@pytest.mark.parametrize("order", ["b200,fi", "fi,b200"])
def test_hybrid_backend_fuses_only_the_b200_half(b200, calls, order):
    ours, foreign = _b200_stub(b200, calls), _Foreign()
    p, d = (ours, foreign) if order == "b200,fi" else (foreign, ours)
    ctx = _set_ctx(b200, b200.attention.HybridBackend(p, d))
    layer = _fill_layer(SimpleNamespace())
    unfused_calls = []

    def unfused(qkv):
        unfused_calls.append(qkv.shape[0])
        return qkv

    for phase in ("prefill", "decode"):
        with ctx.forward_batch(_batch(phase)):
            b200.layers.attention_forward(layer, _qkv(), unfused=unfused)
    if order == "b200,fi":
        assert calls == [("qknorm_rope",), ("forward", 5, (3, HQ, D))] and unfused_calls == [3]
    else:
        assert calls == [("decode_fused", 5, (3, HQ, D), 1e-6)] and unfused_calls == [3]


def test_foreign_backend_runs_the_unfused_forward(b200, calls):
    ctx = _set_ctx(b200, _Foreign())
    layer = _fill_layer(SimpleNamespace())
    qkv = _qkv()
    for phase in ("prefill", "decode"):
        with ctx.forward_batch(_batch(phase)):
            assert b200.layers.attention_forward(layer, qkv, unfused=lambda x: ("unfused", x))[1] is qkv
    assert calls == []


# ------------------------------------------------------------------ patching the reference's layers
def _ref_layer(cls, layer_id):
    return _fill_layer(cls.__new__(cls), layer_id)


def test_patch_without_reference_returns_zero(b200, monkeypatch):
    monkeypatch.setitem(sys.modules, "minisgl.layers.attention", None)  # import raises ImportError
    assert b200.layers.patch_minisgl_attention(SimpleNamespace(layers=[object()])) == 0


def test_patch_rebinds_exactly_the_reference_attention_layers(b200, minisgl_ref, calls):
    Ref = minisgl_ref.layers.attention.AttentionLayer

    class RefSub(Ref):  # a model's own subclass is still the reference's layer
        pass

    refs = [_ref_layer(Ref, 0), _ref_layer(Ref, 1), _ref_layer(RefSub, 2)]
    mirror = _fill_layer(b200.layers.AttentionLayer.__new__(b200.layers.AttentionLayer), 3)
    mirror.fuse_pre_attention = True
    lookalike = _fill_layer(SimpleNamespace(forward=lambda qkv: "lookalike"), 4)  # same attributes, other class
    model = SimpleNamespace(
        layers=SimpleNamespace(op_list=[SimpleNamespace(self_attn=SimpleNamespace(attn=refs[0])),
                                        SimpleNamespace(self_attn=SimpleNamespace(attn=refs[1]))]),
        extra={"sub": (refs[2], mirror)}, lookalike=lookalike,
    )
    model.layers.parent = model  # cycles are walked once
    before = {id(x): vars(x).get("forward") for x in (mirror, lookalike)}
    assert b200.layers.patch_minisgl_attention(model) == 3
    for r in refs:
        assert "forward" in vars(r) and r._b200_unfused_forward.__func__ is type(r).forward
    assert "forward" not in vars(mirror) and vars(lookalike)["forward"] is before[id(lookalike)]
    assert lookalike.forward(None) == "lookalike"

    # idempotent: a second call finds the same layers and leaves them as they are
    bound = [(r.forward, r._b200_unfused_forward) for r in refs]
    assert b200.layers.patch_minisgl_attention(model) == 3
    assert [(r.forward, r._b200_unfused_forward) for r in refs] == bound

    # the patched forward is attention_forward: one fused launch for a b200 decode batch
    ctx = _set_ctx(b200, _b200_stub(b200, calls))
    with ctx.forward_batch(_batch("decode")):
        refs[1].forward(_qkv())
    assert calls == [("decode_fused", 1, (3, HQ, D), 1e-6)]


def test_patched_layer_calls_its_original_forward_for_foreign_backends(b200, minisgl_ref, calls):
    Ref = minisgl_ref.layers.attention.AttentionLayer
    seen = []

    class Probe(Ref):
        def forward(self, qkv):
            seen.append((self.layer_id, qkv))
            return "original"

    layer = _ref_layer(Probe, 7)
    assert b200.layers.patch_minisgl_attention([layer]) == 1
    qkv = _qkv()
    ctx = _set_ctx(b200, _Foreign())
    for phase in ("prefill", "decode"):
        with ctx.forward_batch(_batch(phase)):
            assert layer.forward(qkv) == "original"
    assert [s[0] for s in seen] == [7, 7] and all(s[1] is qkv for s in seen) and calls == []


def test_install_patches_the_model_create_model_returns(b200, minisgl_ref, calls):
    """install_into_minisgl wraps the engine's create_model: the model it returns has its attention layers
    re-bound before the engine captures any graph."""
    import minisgl.engine.engine as ref_engine

    Ref = minisgl_ref.layers.attention.AttentionLayer
    layers = [_ref_layer(Ref, i) for i in range(3)]
    model = SimpleNamespace(layers=layers)
    ref_engine.create_model = lambda config: model  # the module is dropped after the test
    assert b200.layers.install_into_minisgl(norm_rope=False, row_gather=False)
    assert ref_engine.create_model(None) is model
    assert all("_b200_unfused_forward" in vars(x) for x in layers)
