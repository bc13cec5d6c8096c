"""CPU rehearsal of the decode kernel's box-mode K/V loads (attn_decode_tc.cu, producer warps), restated in
tools/decode_tail_ab.tile_loads: for every box size, range end and tile position, the transaction bytes a stage
announces on its mbarrier must equal the bytes its loads deliver (too many announced bytes hang the kernel), and the
exact-tail loads must cover every key of the range exactly once, stay inside one page and read at most 7 rows past
the end of the range."""
import pytest

from tools.decode_tail_ab import TILE, box_rows_for, modelled_read_over_need, range_rows_read, tile_loads

STAGE_BYTES = 2 * TILE * 128


def _cases(rb):
    # tile starts are multiples of 128 (chunks are whole tiles); the range ends anywhere in the tile or past it
    for tile_begin in (0, 128, 384):
        for n_valid in range(1, TILE + 1):
            yield tile_begin, tile_begin + n_valid
    yield 0, 1000  # a full tile of a longer range


@pytest.mark.parametrize("rb", [8, 16, 32, 64])
@pytest.mark.parametrize("exact", [True, False])
def test_announced_bytes_equal_the_bytes_loaded(rb, exact):
    for tile_begin, kv_end in _cases(rb):
        loads, tx = tile_loads(rb, tile_begin, kv_end, exact)
        assert tx == sum(rows for (_, _, rows, _) in loads) * 128, (rb, tile_begin, kv_end)
        assert 0 < tx <= STAGE_BYTES
        if not exact:
            assert tx == STAGE_BYTES  # the whole-box loads: a full stage, as before the exact tail


@pytest.mark.parametrize("rb", [8, 16, 32, 64])
def test_exact_tail_covers_each_key_once(rb):
    for page_size in {8: (8, 24), 16: (16, 48), 32: (32, 96), 64: (64, 128)}[rb]:
        assert box_rows_for(page_size) == rb
        for tile_begin, kv_end in _cases(rb):
            loads, _ = tile_loads(rb, tile_begin, kv_end, True)
            end = min(kv_end, tile_begin + TILE)
            for half in (0, 1):
                seen = [0] * TILE
                for (h, row0, rows, pos0) in loads:
                    if h != half:
                        continue
                    assert rows in (8, rb) and row0 % 8 == 0 and row0 + rows <= TILE
                    assert pos0 == tile_begin + row0  # smem row = key position within the tile
                    assert pos0 // page_size == (pos0 + rows - 1) // page_size, "a box crosses a page"
                    assert pos0 < kv_end, "a box wholly past the end is issued"
                    for i in range(row0, row0 + rows):
                        seen[i] += 1
                assert all(seen[i] == 1 for i in range(end - tile_begin)), (rb, tile_begin, kv_end)
                assert all(s <= 1 for s in seen)
                assert sum(seen) - (end - tile_begin) <= 7  # rows past the end that still come from HBM


@pytest.mark.parametrize("n", [1, 2, 7, 8, 9, 15, 16, 17, 63, 64, 65, 127, 128, 129, 255, 256, 1000])
def test_rows_read_per_range(n):
    for rb in (8, 16, 32, 64):
        exact, whole = range_rows_read(rb, 0, n, True), range_rows_read(rb, 0, n, False)
        assert exact == -(-n // 8) * 8 if n % rb else exact == n
        assert whole == -(-n // rb) * rb
    # a later split-KV chunk starts on a tile boundary
    assert range_rows_read(64, 256, 256 + n, True) == range_rows_read(64, 0, n, True)


def test_bench_schedule_model():
    """The cfg1 bench schedule at page size 64 reads about 3.5 % more K/V rows than it needs with whole boxes,
    under 0.5 % with exact tails; page size 8 boxes are the tail boxes already."""
    m = modelled_read_over_need(64, "cfg1", 40)
    assert m["box_rows"] == 64 and 1.03 < m["exact_tail_0"] < 1.04 and 1.0 < m["exact_tail_1"] < 1.005
    m8 = modelled_read_over_need(8, "cfg1", 40)
    assert m8["exact_tail_0"] == m8["exact_tail_1"]
    assert box_rows_for(1) == 0 and box_rows_for(24) == 8 and box_rows_for(48) == 16 and box_rows_for(256) == 64
