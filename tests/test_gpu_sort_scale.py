"""GPU: Sort and TopK at scale against the vectorised reference of tests/sortscale.py.  Every output is compared bit for bit, the row
column (input position) included, with partref.assert_tables_equal, and checked with sortref.assert_sorted.  Full sorts also assert
cb200_stats.sort_passes against the digits that vary in the packed keys, computed on the host by the encoder's host compile
(sortkey_test.cpp), and every TopK case asserts that the radix select ran (sort_select_rows > 0) exactly when the operator wants only
the first rows of some sort: every TopK (fetch <= chunkRows) over more than one chunk, and a larger fetch without a skip.

Which case fails when a mechanism is wrong:
- a size on, or one row either side of, a 4096-row tile, a 512-row warp slice or a 1024-row select block: test_edge_sizes;
- k_sort_scatter's __match_any_sync ranking with every lane on one digit, a slice or a tile on one digit: test_digit_runs;
- the constant-digit skip (k_sort_keys' AND / OR) when one row differs, at row 0, the last row or mid-tile: test_one_row_differs;
- ordered, reversed and periodic inputs, one digit varying at either end of the key: test_patterns;
- k_scan_totals' carry between its 1024-chunk iterations (more than 16 384 tiles) and the concatenation of chunks past the default
  chunkRows: test_full_sort_past_2_26_rows; four words over 2^24 rows: test_four_word_sort_2_24_rows;
- TopK's candidates carried over 101 or 102 rounds, ties across chunks, rounds that replace every or no candidate, the select deciding in each
  word, NULLs / float specials / extremes on the cut-off, large and growing dictionaries: test_topk."""
import time

import numpy as np
import pyarrow as pa
import pytest

import sortref as R
import sortscale as S

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


@pytest.fixture(scope="module")
def sk(tmp_path_factory):
    return S.sortkey_lib(tmp_path_factory.mktemp("sortkey"))


def run(cb, table, keys, fetch=None, skip=None, inputs=None, chunk=None, batch=1 << 20):
    """(output table or None, stats) of Sort(scan) over `table` in record batches of `batch` rows (or `inputs`)"""
    cfg = {"spark.comet.b200.chunkRows": str(chunk)} if chunk else None
    ins = inputs if inputs is not None else [table.to_batches(max_chunksize=batch)]
    with cb.native.Plan(S.plan(cb.proto, table, keys, fetch, skip), ins, config=cfg, batch_size=1 << 27) as p:
        got = p.collect()
        return got, p.stats()


def full_sort(cb, sk, table, keys, chunk=None, batch=1 << 20):
    """a full sort, checked against the reference, its pass count against the host-derived digits; -> stats"""
    got, st = run(cb, table, keys, chunk=chunk, batch=batch)
    S.check(got, S.sort_table(table, keys), keys)
    assert st["sort_select_rows"] == 0, st
    want = S.digit_passes(S.host_words(sk, table, keys))
    assert st["sort_passes"] == want, (st["sort_passes"], want)
    return st


# ---- full sorts at the tile / slice / block edges --------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [1, 2, 3, 4])
def test_edge_sizes(cb, sk, W):
    """every edge size, random keys of W words (one INT64 key per word, and for W = 4 also 7 INT32 keys with mixed directions)"""
    for n in S.EDGE_SIZES:
        t, keys = S.words_table(S.random_words(n, W, n + W))
        full_sort(cb, sk, t, keys)
    if W == 4:
        for n in S.EDGE_SIZES:
            t, keys = S.words_table(S.random_words(n, 4, n), "i32", desc=[True, False, False, True, True, False, True])
            full_sort(cb, sk, t, keys)


@pytest.mark.parametrize("W", [1, 2, 4])
def test_digit_runs(cb, sk, W):
    """the last word constant over runs of 32 rows (all lanes of a warp step on one digit), 512 rows (a warp's slice) and 4096 rows (a
    tile); and one tile, the last full or the partial one, on one digit while the others are random"""
    n = 5 * S.TILE + 700
    for length in (32, 512, S.TILE):
        t, keys = S.words_table(S.runs(n, W, length, length + W))
        full_sort(cb, sk, t, keys)
    for tile in (0, 2, 5):
        t, keys = S.words_table(S.tile_on_one_digit(n, W, tile, tile + W))
        full_sort(cb, sk, t, keys)


@pytest.mark.parametrize("W", [1, 2, 3, 4])
def test_one_row_differs(cb, sk, W):
    """every row equal but one, which differs in one digit: exactly one pass; at row 0, mid-tile, the last row of a full tile and the
    last row of the partial last tile, in the lowest digit of the last word and the top digit of the first"""
    n = 3 * S.TILE + 100
    for at in (0, S.TILE + 1000, 2 * S.TILE - 1, n - 1):
        for word, digit in ((W - 1, 0), (0, S.top_digit(W)), (W // 2, 3)):
            t, keys = S.words_table(S.one_row_differs(n, W, at, word, digit, at + word))
            st = full_sort(cb, sk, t, keys)
            assert st["sort_passes"] == 1


@pytest.mark.parametrize("W", [1, 2, 3, 4])
def test_patterns(cb, sk, W):
    """sorted, reverse-sorted and sawtooth inputs of periods 32, 512 and 4096; keys that differ only in the lowest digit of the last
    word or only in the top digit of the first (256 values over 100 000 rows: long runs of ties)"""
    n = 100_000
    for kind, period in (("sorted", None), ("reverse", None), ("sawtooth", 32), ("sawtooth", 512), ("sawtooth", S.TILE)):
        t, keys = S.words_table(S.pattern(n, W, kind, period, W))
        full_sort(cb, sk, t, keys, batch=30_000)
    for where in ("low", "top"):
        t, keys = S.words_table(S.one_digit_varies(n, W, where, W))
        st = full_sort(cb, sk, t, keys, batch=30_000)
        assert st["sort_passes"] == 1


# ---- the two large sorts ------------------------------------------------------------------------------------------------------------
def need_device_memory(bytes_needed, what):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < bytes_needed:
        pytest.skip(f"{what}: needs about {bytes_needed / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")


def test_full_sort_past_2_26_rows(cb, sk):
    """2^26 + 4097 rows, one INT64 key of random bits (one word, 8 passes): 16 385 tiles, so the histogram's 1025 scan chunks take
    k_scan_totals through two 1024-wide iterations, and the scan hands the sort two chunks (2^26 rows and 4097) to concatenate.
    Device memory: input and concatenated columns (2 x 16 B / row), keys and indices (2 x 12 B), histogram (1 B), gathered output
    (16 B): about 75 B per row, 5 GiB; 8 GiB asked for."""
    n = (1 << 26) + 4097
    need_device_memory(8 << 30, "2^26 + 4097-row sort")
    t0 = time.time()
    t, keys = S.words_table(S.random_words(n, 1, 26))
    assert S.scan_chunks(n) == 1025
    st = full_sort(cb, sk, t, keys)
    assert st["sort_rows"] == n and st["sort_passes"] == 8
    print(f"2^26 + 4097 rows: {time.time() - t0:.1f} s")


def test_four_word_sort_2_24_rows(cb, sk):
    """about 2^24 rows of a 4-word key whose order is decided in every word: words 0 - 2 of few values, word 3 random.  Device memory
    about 2^24 x (2 x 40 B columns + 2 x 36 B keys / indices + 40 B output): 3 GiB; 6 GiB asked for."""
    n = (1 << 24) + 1
    need_device_memory(6 << 30, "2^24-row 4-word sort")
    t0 = time.time()
    rng = np.random.default_rng(24)
    w = S.random_words(n, 4, 24)
    for j in range(3):
        w[:, j] = rng.integers(0, 2**64, 3 + j, dtype=np.uint64)[rng.integers(0, 3 + j, n)]
    t, keys = S.words_table(w, desc=[False, True, False, True])
    full_sort(cb, sk, t, keys)
    print(f"2^24 rows x 4 words: {time.time() - t0:.1f} s")


# ---- TopK over many chunks ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(S.CASES))
def test_topk(cb, sk, name):
    """chunkRows 2^14 over 101 or 102 chunks: every window of the case, checked against the reference; the radix select runs exactly
    when S.selects says it must, and a single full sort's passes equal the host-derived digits"""
    c = S.CASES[name]
    table, keys, inputs = c.make(c.n)
    order = S.order(table, keys)
    for fetch, skip in c.windows:
        got, st = run(cb, table, keys, fetch, skip, inputs=inputs, chunk=c.chunk, batch=c.batch)
        lo, hi = R.window(len(order), fetch, skip)
        take = pa.array(order[lo:hi], pa.int64())
        want = pa.table([R._array(table.column(i)).take(take) for i in range(table.num_columns)], names=table.column_names)
        S.check(got, want, keys)
        assert (st["sort_select_rows"] > 0) == S.selects(table.num_rows, fetch, skip, c.chunk), (fetch, skip, st["sort_select_rows"])
        if not S.selects(table.num_rows, fetch, skip, c.chunk) and not S.is_topk(fetch, c.chunk):
            assert st["sort_passes"] == S.digit_passes(S.host_words(sk, table, keys)), (fetch, skip, st["sort_passes"])
