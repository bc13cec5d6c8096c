"""The one-shot push all-reduce (csrc/allreduce.cu) on ONE GPU, with stand-in peers.

All `world` regions of a communicator live in this process as torch tensors.  The region of `rank` is the one
the kernel polls; before every launch the test writes the other senders' payloads into it, in both parities and
over the whole slot, as if the peers had already pushed.  The kernel therefore never waits for anything it does
not store itself (the payloads never hold the sentinel), and a wrong offset shows up as a wrong result, never as
a spin.  The other regions receive the kernel's pushes and are inspected afterwards.  Checked here: the rank-order
fp32 sum bit for bit (the contract of include/b200attn.h), the fused residual add + RMSNorm, the sentinel
re-arm and the epoch / parity state, CUDA-graph replay, and argument checks.  What one GPU cannot show -- NVLink
peer stores, CUDA IPC mappings, equality with NCCL -- is left to tests/test_gpu_allreduce.py (>= 2 GPUs)."""
import ctypes as C
import random
from importlib import import_module

import pytest
import torch

from oracle import norm as o_norm

pytestmark = pytest.mark.gpu

MAX_BYTES = 4 << 20  # slots hold rows > 512 at hidden 1024
SENT = -0x8000  # the sentinel: a 16-bit negative zero, as int16
DTYPES = {torch.bfloat16: 0, torch.float16: 1}


def _a256(n: int) -> int:
    return (n + 255) // 256 * 256


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.int16)


def _sendable(x: torch.Tensor) -> torch.Tensor:
    """What the kernel sends for x: contiguous rows, -0.0 replaced by +0.0 (so a payload is never the sentinel)."""
    b = _bits(x.contiguous())
    return torch.where(b == SENT, torch.zeros_like(b), b).view(x.dtype)


def _ref_sum(payloads, dtype) -> torch.Tensor:
    """round(sum over senders of float32(payload)), accumulated from zero in rank order (on the CPU)."""
    acc = torch.zeros(payloads[0].shape, dtype=torch.float32)
    for p in payloads:
        acc += p.cpu().float()
    return acc.to(dtype)


def _assert_bits(got: torch.Tensor, want: torch.Tensor, what: str) -> None:
    """Bit-exact, except that NaN lanes only have to be NaN (the device's canonical NaN differs from torch's)."""
    got, want = got.cpu(), want.cpu()
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan), f"{what}: NaN lanes differ"
    bad = (_bits(got) != _bits(want)) & ~nan
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} lanes differ, first at {i}: got "
                             f"{got[tuple(i)].item()!r} want {want[tuple(i)].item()!r}")


def _ulp_close(a: torch.Tensor, b: torch.Tensor, what: str) -> None:
    """|a-b| <= 1 ulp(b): the oracle's mean of squares sums in another order than the kernel."""
    a32, b32 = a.float().cpu(), b.float().cpu()
    eps = 2.0**-8 if a.dtype == torch.bfloat16 else 2.0**-11
    bad = (a32 - b32).abs() > eps * b32.abs().clamp_min(1e-3) * 2
    assert not bad.any(), f"{what}: {int(bad.sum())} lanes beyond 1 ulp of the oracle"


class Ring:
    """The `world` regions of one all-reduce group, allocated and initialised like b200_ar_alloc does: every
    32-bit word the sentinel pair except the last 256 bytes, which are zero.  Layout (allreduce.cu):
    data [2 parities][world senders][slot] from offset 0, slot = align256(max_bytes); a reserved area; the epoch
    (u32) at region_bytes - 256 and the CTA count-in counter right after it.  A communicator is created per
    rank on the same regions: rank r polls regions[r], the others stand in for its peers."""

    def __init__(self, lib, world: int, max_bytes: int = MAX_BYTES, seed: int = 0):
        self.lib, self.world = lib, world
        self.slot = _a256(max_bytes)
        self.nbytes = int(lib.b200_ar_region_bytes(world, max_bytes))
        self.regions = []
        for _ in range(world):
            r = torch.empty(self.nbytes, dtype=torch.uint8, device="cuda")
            r[: self.nbytes - 256].view(torch.int32).fill_(-0x7FFF8000)  # 0x80008000
            r[self.nbytes - 256 :].zero_()
            self.regions.append(r)
        self.comms = {}
        bases = (C.c_void_p * world)(*[r.data_ptr() for r in self.regions])
        opened = (C.c_int * world)()
        for rank in range(world):
            c = C.c_void_p()
            assert lib.b200_ar_create(rank, world, bases, opened, max_bytes, C.byref(c)) == 0
            self.comms[rank] = c
        g = torch.Generator(device="cuda").manual_seed(seed)
        # what fills a stand-in sender's slot beyond the message: small positive numbers in both types
        self.filler = [torch.randint(1, 0x3C00, (self.slot // 2,), generator=g, device="cuda", dtype=torch.int16)
                       for _ in range(world)]

    def close(self) -> None:
        torch.cuda.synchronize()
        for c in self.comms.values():
            assert self.lib.b200_ar_destroy(c, 0) == 0  # torch owns the memory
        self.comms = {}

    # ---- views
    def data(self, buf: torch.Tensor, parity: int, sender: int) -> torch.Tensor:
        off = (parity * self.world + sender) * self.slot
        return buf[off : off + self.slot].view(torch.int16)

    def _u32(self, buf: torch.Tensor, i: int) -> torch.Tensor:
        off = self.nbytes - 256 + 4 * i
        return buf[off : off + 4].view(torch.int32)

    def epoch(self, rank: int) -> int:
        return int(self._u32(self.regions[rank], 0).item()) & 0xFFFFFFFF

    def counter(self, rank: int) -> int:
        return int(self._u32(self.regions[rank], 1).item()) & 0xFFFFFFFF

    def set_epoch(self, rank: int, value: int) -> None:
        self._u32(self.regions[rank], 0).fill_(value - (1 << 32) if value >= 1 << 31 else value)

    def where(self, off: int) -> str:
        if off < 2 * self.world * self.slot:
            return f"data[parity {off // (self.world * self.slot)}][sender {off // self.slot % self.world}] + {off % self.slot}"
        if off < self.nbytes - 256:
            return f"reserved area + {off - 2 * self.world * self.slot}"
        return f"epoch / counter + {off - (self.nbytes - 256)}"

    # ---- staging (hang safety: every sender != rank, both parities, the whole slot, never the sentinel)
    def sources(self, rank: int, payloads) -> dict:
        srcs = {}
        for s in range(self.world):
            if s != rank:
                src = self.filler[s].clone()
                p = _bits(payloads[s].contiguous()).reshape(-1)
                assert not (p == SENT).any(), "a stand-in payload must not hold the sentinel"
                src[: p.numel()] = p
                srcs[s] = src
        return srcs

    def refill(self, rank: int, srcs: dict) -> None:
        """Stream-ordered copies, so they can be captured in a CUDA graph."""
        for s, src in srcs.items():
            for parity in (0, 1):
                self.data(self.regions[rank], parity, s).copy_(src)

    # ---- the C ABI
    def launch(self, rank, x, out, residual=None, weight=None, eps=0.0, rows=None, dim=None) -> int:
        return self.lib.b200_ar_allreduce(
            self.comms[rank], x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0),
            None if residual is None else residual.data_ptr(), 0 if residual is None else residual.stride(0),
            None if weight is None else weight.data_ptr(), x.shape[0] if rows is None else rows,
            x.shape[1] if dim is None else dim, float(eps), DTYPES[x.dtype], torch.cuda.current_stream().cuda_stream)

    def run(self, rank, xs, out, residual=None, weight=None, eps=0.0, what="") -> torch.Tensor:
        """One checked launch.  xs[s] is sender s's input; xs[rank] is the kernel's x (may hold -0.0, may be
        row-strided).  Stages the stand-ins, launches, checks every region; returns the reference sum."""
        mine = _sendable(xs[rank])
        pays = [mine if s == rank else _sendable(xs[s]) for s in range(self.world)]
        self.refill(rank, self.sources(rank, pays))
        before = [r.clone() for r in self.regions]
        old = self.epoch(rank)
        rc = self.launch(rank, xs[rank], out, residual, weight, eps)
        assert rc == 0, self.lib.b200_last_error()
        torch.cuda.synchronize()
        self.check_regions(rank, before, old, mine, what)
        return _ref_sum(pays, mine.dtype)

    def check_regions(self, rank, before, old_epoch, mine, what="") -> None:
        """After a launch of epoch old+1: the consumed parity's slots of the own region are re-armed over the
        message, the payload sits in slot[parity][rank] of every stand-in region, the epoch advanced by one,
        the counter is back to 0, and not one other byte changed anywhere."""
        parity, n = (old_epoch + 1) & 1, mine.numel()
        for t in range(self.world):
            exp = before[t].clone()
            if t == rank:
                for s in range(self.world):
                    self.data(exp, parity, s)[:n] = SENT
                new = (old_epoch + 1) & 0xFFFFFFFF
                self._u32(exp, 0).fill_(new - (1 << 32) if new >= 1 << 31 else new)
                self._u32(exp, 1).zero_()
            else:
                self.data(exp, parity, rank)[:n] = _bits(mine).reshape(-1)
            if not torch.equal(self.regions[t], exp):
                off = int((self.regions[t] != exp).nonzero()[0].item())
                role = "own region" if t == rank else f"stand-in region {t}"
                raise AssertionError(f"{what} rank {rank}, epoch {old_epoch} -> parity {parity}: {role} wrong at "
                                     f"{self.where(off)} (got byte {self.regions[t][off].item()}, "
                                     f"want {exp[off].item()})")


def _randn(g, rows, dim, dtype, scale=1.0):
    return (torch.randn(rows, dim, generator=g, device="cuda") * scale).to(dtype)


def _ranks(world):
    return sorted({0, world // 2, world - 1})


@pytest.fixture(scope="module")
def lib(native_lib):
    return native_lib


# (rows, dim): dims 8 .. 8192 incl. a partial last warp (1032), the last one-chunk-per-thread width (4096) and
# the first two-chunk one (4104); rows past the 512 CTAs (several rows per CTA); a message that fills the slot
PLAIN_SHAPES = [(7, 8), (513, 16), (130, 64), (2000, 128), (1, 1024), (513, 1024), (2000, 1024), (512, 1032),
                (130, 4096), (512, 4096), (7, 4104), (1, 5120), (130, 8192), (7, 8192)]
assert 512 * 4096 * 2 == _a256(MAX_BYTES)  # (512, 4096) fills a slot to its last byte


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_plain_sum_and_region_state(lib, world, dtype):
    """out == round(fp32 rank-order sum) bit for bit, at ranks 0, W/2 and W-1; strided x, separate out and
    out aliasing x; after every launch the regions hold exactly what the protocol says (check_regions)."""
    ring = Ring(lib, world)
    g = torch.Generator(device="cuda").manual_seed(world * 10 + DTYPES[dtype])
    try:
        for i, (rows, dim) in enumerate(PLAIN_SHAPES):
            for rank in _ranks(world):
                xs = [_randn(g, rows, dim, dtype, 4.0) for _ in range(world)]
                mode = (i + rank) % 3
                if mode == 1:  # x: rows of a wider buffer (row stride dim + 16)
                    wide = _randn(g, rows, dim + 16, dtype)
                    wide[:, :dim] = xs[rank]
                    xs[rank] = wide[:, :dim]
                out = xs[rank] if mode == 2 else torch.empty(rows, dim, dtype=dtype, device="cuda")
                x_before = xs[rank].clone()
                what = f"plain {rows}x{dim} w{world}"
                want = ring.run(rank, xs, out, what=what)
                _assert_bits(out, want, f"{what} rank {rank}")
                if mode != 2:
                    assert torch.equal(_bits(xs[rank]), _bits(x_before)), f"{what}: x was modified"
    finally:
        ring.close()


def _order_lanes(world, rows, dim, dtype, g):
    """Lane group k (column % world == k): ranks k, k+1, k+2 (mod world) send 1, 2^-24, -1.  In fp32,
    1 + 2^-24 rounds back to 1, so the sum depends on the order; rank order is the contract.  A sum in
    push order (rank + 1, rank + 2, ...) differs from it in some group at every rank but world - 1."""
    xs = [_randn(g, rows, dim, dtype) for _ in range(world)]
    cols = torch.arange(dim, device="cuda") % world
    for k in range(world):
        sel = cols == k
        for s in range(world):
            xs[s][:, sel] = 0.0
        for j, v in enumerate((1.0, 2.0**-24, -1.0)):
            xs[(k + j) % world][:, sel] = v
    for s in range(world):  # odd rows: plain random values
        xs[s][1::2] = _randn(g, rows, dim, dtype)[1::2]
    return xs


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("world", [3, 4, 8])
def test_sum_is_in_rank_order_on_every_rank(lib, world, dtype):
    ring = Ring(lib, world)
    g = torch.Generator(device="cuda").manual_seed(77 + world)
    try:
        for rows, dim in ((6, 1024), (600, 64), (3, 4104)):
            xs = _order_lanes(world, rows, dim, dtype, g)
            outs = []
            for rank in range(world):
                out = torch.empty(rows, dim, dtype=dtype, device="cuda")
                want = ring.run(rank, [x.clone() for x in xs], out, what=f"order {rows}x{dim}")
                _assert_bits(out, want, f"order lanes {rows}x{dim} w{world} rank {rank}")
                outs.append(out)
            for rank in range(1, world):
                assert torch.equal(_bits(outs[rank]), _bits(outs[0])), f"rank {rank} differs from rank 0"
    finally:
        ring.close()


def _adversarial(world, rows, dim, dtype, g):
    """Inputs whose bits the protocol or the arithmetic could get wrong, by column % 12."""
    fp16 = dtype == torch.float16
    sub_hi = 0x03FF if fp16 else 0x007F  # largest subnormal magnitude bits
    big = 0x7BFF if fp16 else 0x7F7F  # largest finite
    nan, inf = (0x7E00, 0x7C00) if fp16 else (0x7FC0, 0x7F80)
    xs = [_bits(_randn(g, rows, dim, dtype, 2.0)).clone() for _ in range(world)]
    col = torch.arange(dim, device="cuda") % 12

    def put(s, cls, bits):
        sel = col == cls
        xs[s][:, sel] = bits if isinstance(bits, int) else bits[:, sel]

    rnd = lambda lo, hi: torch.randint(lo, hi + 1, (rows, dim), generator=g, device="cuda", dtype=torch.int32).to(torch.int16)
    for s in range(world):
        if s % 2 == 0:
            put(s, 0, SENT)  # -0.0 from some ranks
        put(s, 1, SENT)  # -0.0 from every rank: the sum is +0.0
        put(s, 2, -0x7FFF)  # 0x8001, the negative subnormal next to the sentinel
        put(s, 3, rnd(1, sub_hi) | SENT)  # negative subnormals
        put(s, 4, rnd(1, sub_hi))  # positive subnormals (no flush to zero)
        put(s, 5, rnd(1, sub_hi) | (rnd(0, 1) * SENT))  # either sign
        put(s, 10, big)  # the sum of two overflows to inf
        put(s, 11, 0x0400 if fp16 else 0x0080)  # smallest normals, next to largest finite below
    put(0, 6, inf)
    put(world - 1, 7, inf | SENT)
    put(0, 8, inf)
    put(world - 1, 8, inf | SENT)  # +inf + -inf (or just +inf at world 1)
    put(world // 2, 9, nan)
    put(0, 11, big)
    return [x.view(dtype) for x in xs]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_adversarial_bits(lib, world, dtype):
    """-0.0 (sent as +0.0: an all-negative-zero sum is +0.0, unlike NCCL), 0x8001 and other subnormals (never
    taken for the sentinel, never flushed), +-inf, NaN and overflow to inf."""
    ring = Ring(lib, world)
    g = torch.Generator(device="cuda").manual_seed(5 + world)
    try:
        for rows, dim in ((7, 1032), (513, 128)):
            for rank in sorted({0, world - 1}):
                xs = _adversarial(world, rows, dim, dtype, g)
                out = torch.empty(rows, dim, dtype=dtype, device="cuda")
                want = ring.run(rank, xs, out, what=f"adversarial {rows}x{dim} w{world}")
                _assert_bits(out, want, f"adversarial {rows}x{dim} w{world} rank {rank}")
                zero = (torch.arange(dim) % 12 == 1)
                assert (_bits(out.cpu())[:, zero] == 0).all(), "an all -0.0 sum must be +0.0"
    finally:
        ring.close()


FUSED_SHAPES = [(1, 1024), (130, 1032), (513, 1024), (7, 4104), (64, 5120), (3, 8192), (33, 64), (600, 128)]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_fused_add_rmsnorm_epilogue(b200, lib, world, dtype):
    """residual and out equal the plain sum followed by b200_fused_add_rmsnorm bit for bit (the header's
    promise), and are within 1 ulp of the oracle applied to the reference sum (residual exact).  Includes
    out aliasing x, strided residual rows, rows > 512 (red[] reused across rows of a CTA) and zero-sum rows."""
    ring = Ring(lib, world)
    g = torch.Generator(device="cuda").manual_seed(300 + world)
    try:
        for i, (rows, dim) in enumerate(FUSED_SHAPES):
            eps = 1e-6 if i % 2 == 0 else 1e-5
            for rank in sorted({0, world - 1}):
                what = f"fused {rows}x{dim} w{world} rank {rank} eps {eps}"
                xs = [_randn(g, rows, dim, dtype, 3.0) for _ in range(world)]
                for s in range(world):  # row 0: the senders cancel; row 1: zero sum and zero residual
                    xs[s][:2] = 0.0
                if world > 1:
                    xs[0][0] = _randn(g, 1, dim, dtype)[0]
                    xs[1][0] = -xs[0][0]
                w = (torch.rand(dim, generator=g, device="cuda") + 0.5).to(dtype)
                res0 = _randn(g, rows, dim, dtype, 2.0)
                if rows > 1:
                    res0[1] = 0.0
                y = torch.empty(rows, dim, dtype=dtype, device="cuda")
                want = ring.run(rank, [x.clone() for x in xs], y, what=what + " plain")
                _assert_bits(y, want, what + " plain")
                r_ref = res0.clone()
                b200.ops.fused_add_rmsnorm(y, r_ref, w, eps)  # y <- norm, r_ref <- residual
                if i % 2 == 0:  # residual rows of a wider buffer
                    rbuf = _randn(g, rows, dim + 24, dtype)
                    res = rbuf[:, :dim]
                    pad = rbuf[:, dim:].clone()
                else:
                    res, rbuf = res0.clone(), None
                res.copy_(res0)
                out = xs[rank] if i % 3 == 1 else torch.empty(rows, dim, dtype=dtype, device="cuda")
                ring.run(rank, xs, out, residual=res, weight=w, eps=eps, what=what)
                _assert_bits(res, r_ref, what + " residual vs sum + fused_add_rmsnorm")
                _assert_bits(out, y, what + " out vs sum + fused_add_rmsnorm")
                o_out, o_res = o_norm.ref_fused_add_rmsnorm(want, res0.cpu(), w.cpu(), eps)
                _assert_bits(res, o_res, what + " residual vs oracle")
                _ulp_close(out, o_out, what + " out vs oracle")
                if rbuf is not None:
                    assert torch.equal(rbuf[:, dim:], pad), f"{what}: residual row padding written"
                if rows > 1:
                    assert (_bits(out[1]) == 0).all(), f"{what}: a zero row must normalise to zero"
    finally:
        ring.close()


@pytest.mark.parametrize("world", [1, 4])
def test_graph_replay_matches_eager(lib, world):
    """3 fused + 2 plain launches in one graph (an odd count: consecutive replays start at opposite parities),
    with the stand-in refills captured before each launch; 3 replays equal the eager sequence bit for bit."""
    ring = Ring(lib, world)
    rank, rows, dim, n = world // 2, 130, 1024, 5
    dtype = torch.bfloat16
    g = torch.Generator(device="cuda").manual_seed(41)
    try:
        xs = [[_randn(g, rows, dim, dtype, 2.0) for _ in range(world)] for _ in range(n)]
        srcs = [ring.sources(rank, [_sendable(x) for x in xs[l]]) for l in range(n)]
        w = (torch.rand(dim, generator=g, device="cuda") + 0.5).to(dtype)
        res0 = _randn(g, rows, dim, dtype)
        res = res0.clone()
        outs = [torch.empty(rows, dim, dtype=dtype, device="cuda") for _ in range(n)]

        def sequence():
            for l in range(n):
                ring.refill(rank, srcs[l])
                fused = l < 3
                rc = ring.launch(rank, xs[l][rank], outs[l], res if fused else None, w if fused else None, 1e-6)
                assert rc == 0, lib.b200_last_error()

        sequence()
        torch.cuda.synchronize()
        eager_outs, eager_res = [o.clone() for o in outs], res.clone()
        for l in (3, 4):
            _assert_bits(eager_outs[l], _ref_sum([_sendable(x) for x in xs[l]], dtype), f"eager launch {l}")
        graph = torch.cuda.CUDAGraph()
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            with torch.cuda.graph(graph, stream=st):
                sequence()
        torch.cuda.current_stream().wait_stream(st)
        torch.cuda.synchronize()
        for rep in range(3):
            res.copy_(res0)
            for o in outs:
                o.zero_()
            e0 = ring.epoch(rank)
            graph.replay()
            torch.cuda.synchronize()
            assert ring.epoch(rank) == e0 + n and ring.counter(rank) == 0
            for l in range(n):
                assert torch.equal(_bits(outs[l]), _bits(eager_outs[l])), f"replay {rep} (first parity {(e0 + 1) & 1}), launch {l}"
            assert torch.equal(_bits(res), _bits(eager_res)), f"replay {rep}: residual"
        del graph
    finally:
        ring.close()


def test_epoch_wraps_and_parity_alternates(lib):
    """Parity (e + 1) & 1 from the stored epoch e, checked launch by launch by check_regions, so consecutive
    launches alternate; from 0xFFFFFFFF the epoch wraps to 0 and the launch uses parity 0."""
    world, rank = 3, 1
    ring = Ring(lib, world)
    g = torch.Generator(device="cuda").manual_seed(9)
    try:
        for preset in (None, 0xFFFFFFFF, 0x7FFFFFFF):
            if preset is not None:
                ring.set_epoch(rank, preset)
            start = ring.epoch(rank)
            for k in range(3):
                xs = [_randn(g, 9, 256, torch.bfloat16) for _ in range(world)]
                out = torch.empty(9, 256, dtype=torch.bfloat16, device="cuda")
                want = ring.run(rank, xs, out, what=f"epoch {start:#x} + {k}")
                _assert_bits(out, want, f"epoch {start:#x} + {k}")
                if preset == 0xFFFFFFFF and k == 0:
                    assert ring.epoch(rank) == 0  # wrapped; check_regions saw parity 0 consumed
            assert ring.epoch(rank) == (start + 3) & 0xFFFFFFFF
    finally:
        ring.close()


def test_many_calls_world1(b200, lib):
    """300 back-to-back launches with changing row counts.  At world 1 every launch re-arms exactly what it
    stored, so the whole data area must still be the sentinel whenever it is looked at."""
    ring = Ring(lib, 1)
    rnd = random.Random(3)
    g = torch.Generator(device="cuda").manual_seed(3)
    base = _randn(g, 2000, 1024, torch.bfloat16, 8.0)
    want = _sendable(base)
    buf = torch.empty_like(base)
    try:
        for it in range(1, 301):
            n = rnd.choice([1, 2, 3, 8, 31, 64, 129, 200, 512, 513, 1000, 2000])
            assert ring.launch(0, base[:n], buf[:n]) == 0, lib.b200_last_error()
            if it % 50 == 0:
                torch.cuda.synchronize()
                assert torch.equal(_bits(buf[:n]), _bits(want[:n])), f"call {it}, {n} rows"
                assert ring.epoch(0) == it and ring.counter(0) == 0
                assert (ring.regions[0][: 2 * ring.slot].view(torch.int16) == SENT).all(), f"call {it}: not re-armed"
    finally:
        ring.close()


def test_argument_checks_with_device_pointers(b200, lib):
    """Rejected before any launch: dim 8200 (> 8192), a message one chunk larger than the slot, a misaligned
    x; rows == 0 launches nothing.  A valid launch afterwards still works."""
    ring = Ring(lib, 1)
    try:
        x = torch.zeros(1, 8200, dtype=torch.bfloat16, device="cuda")
        count = b200._cabi.launch_count()
        assert ring.launch(0, x, x) != 0 and b"max 8192" in lib.b200_last_error()
        rows = ring.slot // 16 + 1  # rows * 8 * 2 == slot + 16
        x = torch.zeros(rows, 8, dtype=torch.bfloat16, device="cuda")
        assert ring.launch(0, x, x) != 0 and b"exceeds" in lib.b200_last_error()
        assert ring.launch(0, x[: rows - 1], x[: rows - 1]) == 0  # exactly the slot is fine
        torch.cuda.synchronize()
        assert ring.epoch(0) == 1
        buf = torch.zeros(4 * 1024 + 8, dtype=torch.bfloat16, device="cuda")
        mis = buf[4 : 4 + 4 * 1024].view(4, 1024)  # 8 bytes past a 16-byte boundary
        out = torch.empty(4, 1024, dtype=torch.bfloat16, device="cuda")
        assert ring.launch(0, mis, out) != 0 and b"aligned" in lib.b200_last_error()
        assert ring.launch(0, out, out, rows=0) == 0
        torch.cuda.synchronize()
        assert ring.epoch(0) == 1 and b200._cabi.launch_count() == count + 1
        x = torch.randn(4, 1024, device="cuda").to(torch.bfloat16)
        assert ring.launch(0, x, out) == 0, lib.b200_last_error()
        torch.cuda.synchronize()
        assert torch.equal(_bits(out), _bits(_sendable(x))) and ring.epoch(0) == 2
    finally:
        ring.close()


# ------------------------------------------------------------------ the Python layer (distributed.py)
@pytest.fixture
def gloo_world1():
    import torch.distributed as dist

    assert not dist.is_initialized()
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        yield dist.group.WORLD
    finally:
        dist.destroy_process_group()


class _Fallback:
    def __init__(self):
        self.calls = []

    def all_reduce(self, x):
        self.calls.append(x)
        return x

    def all_gather(self, x):
        raise AssertionError("not used")


def test_python_communicator_world1(b200, lib, gloo_world1):
    """B200AllReduce over an in-process gloo group of one rank: b200_ar_alloc, the IPC handle path, all_reduce
    in place / with out= / fused; B200DistributedImpl's hand-off to the fallback; no use after destroy()."""
    D = import_module("mini-sglang_b200.distributed")
    comm = D.B200AllReduce(0, 1, gloo_world1, torch.device("cuda", torch.cuda.current_device()))
    g = torch.Generator(device="cuda").manual_seed(12)
    rows, dim = 130, 1024
    x = _randn(g, rows, dim, torch.bfloat16, 3.0)
    x[:, ::7] = -0.0
    want = _sendable(x)
    try:
        y = x.clone()
        assert comm.all_reduce(y) is y
        _assert_bits(y, want, "in place")
        out = torch.empty_like(x)
        comm.all_reduce(x, out=out)
        _assert_bits(out, want, "out=")
        w = (torch.rand(dim, generator=g, device="cuda") + 0.5).to(torch.bfloat16)
        res0 = _randn(g, rows, dim, torch.bfloat16)
        res, o = res0.clone(), torch.empty_like(x)
        comm.all_reduce(x, out=o, residual=res, weight=w, eps=1e-6)
        y_ref, r_ref = want.clone(), res0.clone()
        b200.ops.fused_add_rmsnorm(y_ref, r_ref, w, 1e-6)
        _assert_bits(res, r_ref, "fused residual")
        _assert_bits(o, y_ref, "fused out")
        o_out, o_res = o_norm.ref_fused_add_rmsnorm(want.cpu(), res0.cpu(), w.cpu(), 1e-6)
        _assert_bits(res, o_res, "fused residual vs oracle")
        _ulp_close(o, o_out, "fused out vs oracle")

        # fits(x) implies the kernel accepts x; what does not fit goes to the fallback, without a launch
        buf = torch.zeros(rows * dim + 16, dtype=torch.bfloat16, device="cuda")
        aligned = buf[8 : 8 + rows * dim].view(rows, dim)
        misaligned = buf[4 : 4 + rows * dim].view(rows, dim)
        big = torch.zeros(comm.max_bytes // (2 * dim) + 1, dim, dtype=torch.bfloat16, device="cuda")
        assert comm.fits(x) and comm.fits(aligned)
        assert not comm.fits(misaligned) and not comm.fits(big)
        fb = _Fallback()
        impl = D.B200DistributedImpl(comm, fb)
        for t in (aligned, misaligned, big, x[:, :512]):
            t.copy_(torch.ones_like(t))
            count, handed = b200._cabi.launch_count(), len(fb.calls)
            impl.all_reduce(t)
            torch.cuda.synchronize()
            kernel = comm.fits(t) and t.is_contiguous()
            assert b200._cabi.launch_count() == count + int(kernel)
            assert len(fb.calls) == handed + int(not kernel)
            assert (t == 1).all()
    finally:
        comm.destroy()
    comm.destroy()  # idempotent
    with pytest.raises(RuntimeError, match="destroyed"):
        comm.all_reduce(x)
