"""GPU: the gated-MLP activation ``ops.silu_and_mul`` against ``flashinfer.silu_and_mul`` in the same process (bit
identity: every 16-bit gate pattern, every width class, both kernel paths) and against an fp64 oracle (one ulp of
the output type), plus row strides, ``out=`` and CUDA-graph replay.  When FlashInfer cannot load, its comparisons
skip and the oracle checks still run."""
import os
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
TINY = 2.0**-126  # smallest normal fp32


@pytest.fixture(scope="module")
def fi_silu(b200):
    """FlashInfer's own ``silu_and_mul`` (never our re-bound name), JIT-built once for this device."""
    os.environ.setdefault("FLASHINFER_WORKSPACE_BASE", bench.flashinfer_workspace())
    try:
        import flashinfer

        fn = b200.layers._FLASHINFER_SAVED.get("silu_and_mul", flashinfer.silu_and_mul)
        fn(torch.ones(2, 16, device="cuda", dtype=torch.bfloat16))
        torch.cuda.synchronize()
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"flashinfer.silu_and_mul cannot run here ({type(e).__name__}: {str(e)[:200]})")
    return fn


def _bits(t):
    return t.contiguous().view(torch.int16)


def _oracles(x):
    """fp64 silu(gate) * up, exact and with FlashInfer's fast-math flush-to-zero of fp32 subnormals applied to
    the gate, the sigmoid factor 1 / (1 + e^-g) (the reciprocal flushes for g < -87.3), silu(g) and the result."""
    d = x.shape[-1] // 2
    g, u = x[..., :d].double(), x[..., d:].double()
    sig = torch.sigmoid(g)
    flush = lambda t: torch.where(t.abs() < TINY, torch.zeros_like(t), t)  # noqa: E731
    return g * sig * u, flush(flush(flush(g) * flush(sig)) * u)


def _assert_within_one_ulp(got, x, what):
    """|got - oracle| <= one ulp of the output type for one of the two oracles; overflow to +-inf counts as the
    value 2^(emax + 1)."""
    exact, ftz = _oracles(x)
    mant, emin, emax = (7, -126, 127) if got.dtype == torch.bfloat16 else (10, -14, 15)
    nan = torch.isnan(exact)
    assert torch.equal(torch.isnan(got), nan), f"{what}: NaN positions differ"
    cap = 2.0 ** (emax + 1)
    g = got.double()[~nan].clamp(-cap, cap)
    worst = None
    for ref in (exact, ftz):
        r = ref[~nan].clamp(-cap, cap)
        big = torch.maximum(g.abs(), r.abs()).clamp_min(2.0**emin)
        ulps = (g - r).abs() / torch.exp2(torch.floor(torch.log2(big)) - mant)
        worst = ulps if worst is None else torch.minimum(worst, ulps)
    bad = worst > 1
    assert not bad.any(), f"{what}: {int(bad.sum())} values off by more than one ulp, worst {float(worst.max()):.2f}"


def _x(shape, dtype, seed=0):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=gen) * 3).to(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_gate_bit_pattern_matches_flashinfer(b200, native_lib, fi_silu, dtype):
    """All 65 536 gate patterns (±0, subnormals, ±inf, NaN included) against 4 random up rows: the vector path
    (d = 65 536) bit for bit against FlashInfer, and the one-element-per-thread path (d = 12) bit for bit against
    the vector path.  (FlashInfer itself cannot take d = 12: it loads the up half, d elements into the row, with
    16-byte vectors, which needs d % 8 == 0.)"""
    pats = torch.arange(-(1 << 15), 1 << 15, dtype=torch.int32, device="cuda").to(torch.int16).view(dtype)
    n = pats.numel()
    for r in range(4):
        up = _x((n,), dtype, seed=r)
        x = torch.cat([pats, up]).view(1, 2 * n)
        ours = b200.ops.silu_and_mul(x)
        assert torch.equal(_bits(ours), _bits(fi_silu(x))), f"vector path, up row {r}"
        _assert_within_one_ulp(ours, x, f"vector path, up row {r}")
        rows = -(-n // 12)
        g = torch.zeros(rows * 12, dtype=dtype, device="cuda")
        g[:n] = pats
        u = torch.ones(rows * 12, dtype=dtype, device="cuda")
        u[:n] = up
        x12 = torch.cat([g.view(rows, 12), u.view(rows, 12)], dim=1)
        ours12 = b200.ops.silu_and_mul(x12)
        assert torch.equal(_bits(ours12).flatten()[:n], _bits(ours).flatten()), "the two paths differ"


WIDTHS = [1, 7, 8, 3072, 3584, 17408]
ROWS = [1, 3, 8192]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d", WIDTHS)
def test_widths_and_rows(b200, native_lib, fi_silu, dtype, d):
    for rows in ROWS:
        x = _x((rows, 2 * d), dtype, seed=d + rows)
        ours = b200.ops.silu_and_mul(x)
        assert ours.shape == (rows, d) and ours.dtype == dtype
        _assert_within_one_ulp(ours, x, f"d={d} rows={rows}")
        if d % 8 == 0:  # FlashInfer reads both halves with 16-byte vectors: other widths are not its to take
            assert torch.equal(_bits(ours), _bits(fi_silu(x))), f"d={d} rows={rows} vs flashinfer"
    x3 = _x((2, 5, 2 * d), dtype, seed=7)
    ours3 = b200.ops.silu_and_mul(x3)
    assert ours3.shape == (2, 5, d)
    assert torch.equal(_bits(ours3), _bits(b200.ops.silu_and_mul(x3.view(10, 2 * d))).view(2, 5, d))
    _assert_within_one_ulp(ours3, x3, f"3-D d={d}")


def test_oracle_check_without_flashinfer(b200, native_lib):
    """The fp64 oracle alone, so the kernels stay checked where FlashInfer cannot load."""
    for dtype in DTYPES:
        for d in (7, 3072):
            x = _x((64, 2 * d), dtype, seed=d)
            _assert_within_one_ulp(b200.ops.silu_and_mul(x), x, f"{dtype} d={d}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d, x_pad, o_pad", [(3072, 64, 8), (3584, 16, 24), (1024, 3, 0), (1000, 8, 5), (7, 1, 2)])
def test_strided_rows_leave_the_padding_alone(b200, native_lib, dtype, d, x_pad, o_pad):
    """Input and output rows inside wider NaN-filled buffers (aligned pads take the vector path, odd pads the
    scalar one): the result equals the contiguous one bit for bit and every padding element is still NaN."""
    rows = 37
    src = _x((rows, 2 * d), dtype, seed=d)
    xb = torch.full((rows, 2 * d + x_pad), float("nan"), device="cuda", dtype=dtype)
    xb[:, : 2 * d] = src
    ob = torch.full((rows, d + o_pad), float("nan"), device="cuda", dtype=dtype)
    got = b200.ops.silu_and_mul(xb[:, : 2 * d], out=ob[:, :d])
    assert got.data_ptr() == ob.data_ptr()
    assert torch.equal(_bits(ob[:, :d]), _bits(b200.ops.silu_and_mul(src)))
    assert torch.isnan(ob[:, d:]).all() and torch.isnan(xb[:, 2 * d :]).all()


def test_out_argument_and_refusals(b200, native_lib):
    x = _x((5, 2 * 64), torch.bfloat16)
    out = torch.empty(5, 64, device="cuda", dtype=torch.bfloat16)
    assert b200.ops.silu_and_mul(x, out=out, enable_pdl=True) is out
    assert torch.equal(_bits(out), _bits(b200.ops.silu_and_mul(x, enable_pdl=False)))
    empty = b200.ops.silu_and_mul(torch.empty(0, 128, device="cuda", dtype=torch.bfloat16))
    assert empty.shape == (0, 64)
    with pytest.raises(RuntimeError, match="even"):
        b200.ops.silu_and_mul(torch.zeros(3, 7, device="cuda", dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="out must be"):
        b200.ops.silu_and_mul(x, out=torch.empty(5, 63, device="cuda", dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="out must be"):
        b200.ops.silu_and_mul(x, out=torch.empty(5, 64, device="cuda", dtype=torch.float16))
    with pytest.raises(RuntimeError, match="unsupported dtype"):
        b200.ops.silu_and_mul(torch.zeros(3, 8, device="cuda", dtype=torch.float32))
    with pytest.raises(RuntimeError, match="contiguous"):
        b200.ops.silu_and_mul(torch.zeros(16, 3, device="cuda", dtype=torch.bfloat16).t())


def test_cuda_graph_capture_and_replay(b200, native_lib):
    x = _x((64, 2 * 3072), torch.bfloat16)
    out = torch.empty(64, 3072, device="cuda", dtype=torch.bfloat16)
    b200.ops.silu_and_mul(x, out=out)  # warm-up outside capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        b200.ops.silu_and_mul(x, out=out)
    for seed in (1, 2):
        x.copy_(_x(x.shape, x.dtype, seed=seed))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bits(out), _bits(b200.ops.silu_and_mul(x))), seed
