"""CPU checks of the sort scale cases (tests/sortscale.py): the vectorised reference equals sortref.order on slices of every input the
GPU file sorts; each generator has the digit shape it claims, read from the host compile of the key encoder (sortkey_test.cpp); the
comparison fails on each kind of wrong answer; and every plan the GPU file builds is accepted and compiles."""
import numpy as np
import pyarrow as pa
import pytest

import sortref as R
import sortscale as S


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


@pytest.fixture(scope="module")
def sk(tmp_path_factory):
    return S.sortkey_lib(tmp_path_factory.mktemp("sortkey"))


def _slices(n, seed):
    """row index sets, in input order: the first 3 000 rows, 3 000 rows from the end, and 3 000 spread over the whole input"""
    rng = np.random.default_rng(seed)
    k = min(3000, n)
    return [np.arange(k), np.arange(n - k, n), np.sort(rng.choice(n, k, replace=False))]


def _same_order(table, keys, seed):
    for rows in _slices(table.num_rows, seed):
        sl = table.take(pa.array(rows))
        got, want = S.order(sl, keys), R.order(sl, keys)
        assert (got == want).all(), (keys, int(np.argmax(got != want)))


# ---- the reference -----------------------------------------------------------------------------------------------------------------------
GENERATED = {
    "random-1w": lambda: S.words_table(S.random_words(20_000, 1, 1)),
    "random-4w-desc": lambda: S.words_table(S.random_words(20_000, 4, 2), desc=[True, False, True, False]),
    "i32x8": lambda: S.words_table(S.random_words(20_000, 4, 3), "i32", desc=[True, False, False, True, True, False, True]),
    "runs-32": lambda: S.words_table(S.runs(20_000, 2, 32, 4)),
    "tile": lambda: S.words_table(S.tile_on_one_digit(20_000, 3, 2, 5)),
    "one-row": lambda: S.words_table(S.one_row_differs(20_000, 2, 19_999, 0, 7, 6)),
    "sawtooth": lambda: S.words_table(S.pattern(20_000, 2, "sawtooth", 512, 7)),
    "reverse": lambda: S.words_table(S.pattern(20_000, 1, "reverse", None, 8)),
    "low-digit": lambda: S.words_table(S.one_digit_varies(20_000, 4, "low", 9)),
    "top-digit": lambda: S.words_table(S.one_digit_varies(20_000, 3, "top", 10)),
}


@pytest.mark.parametrize("name", list(GENERATED))
def test_reference_matches_sortref_on_generated(name):
    t, keys = GENERATED[name]()
    _same_order(t, keys, len(name))


@pytest.mark.parametrize("name", list(S.CASES))
def test_reference_matches_sortref_on_gpu_cases(name):
    """the GPU inputs themselves (at their full size), sliced; also with the direction and null placement of every key flipped"""
    c = S.CASES[name]
    t, keys, _ = c.make(c.n)
    _same_order(t, keys, 1)
    _same_order(t, [(k, not d, not nf) for k, d, nf in keys], 2)


def test_reference_on_dictionaries_that_differ_by_chunk():
    """chunks with different dictionaries (growing, and a reordered one): ranks by the strings' bytes, not by the codes"""
    bs, t = S.string_batches(30_000, 2000, 5000, True, 3, null_rate=0.1)
    d = pa.array(S.dictionary_words(5000, 3)[::-1])
    extra = pa.record_batch([pa.DictionaryArray.from_arrays(pa.array(np.arange(5000, dtype=np.int32) % 7), d),
                             pa.array(np.zeros(5000, np.int32)), pa.array(np.arange(30_000, 35_000))], names=["s", "v", "row"])
    t = pa.Table.from_batches(bs + [extra])
    for keys in ([(0, False, True)], [(0, True, False), (1, False, True)]):
        _same_order(t, keys, 3)
        got, want = S.order(t, keys), R.order(t, keys)
        assert (got == want).all()


# ---- digit shapes, through the host compile of the encoder ----------------------------------------------------------------------------
def _words(sk, gen_table):
    t, keys = gen_table
    return S.host_words(sk, t, keys)


@pytest.mark.parametrize("kind,W,desc", [("i64", 1, None), ("i64", 2, [True, False]), ("i64", 3, None), ("i64", 4, [False, True, True, False]),
                                         ("i32", 4, [True, False] * 3 + [True]), ("i32", 1, [False, True])])
def test_key_columns_encode_to_the_generator_words(sk, kind, W, desc):
    w = S.random_words(5000, W, W)
    assert (_words(sk, S.words_table(w, kind, desc)) == S.fit(w)).all()


@pytest.mark.parametrize("W", [1, 2, 3, 4])
def test_one_row_differs_in_one_digit(sk, W):
    n = 3 * S.TILE + 100
    for at in (0, S.TILE + 1000, n - 1):
        for word, digit in ((W - 1, 0), (0, S.top_digit(W)), (W // 2, 3)):
            w = _words(sk, S.words_table(S.one_row_differs(n, W, at, word, digit, at + word)))
            assert S.varying_digits(w) == [(word, digit)]
            assert np.flatnonzero((w != w[(at + 1) % n]).any(axis=1)).tolist() == [at]


@pytest.mark.parametrize("W", [1, 2, 3, 4])
def test_one_digit_varies(sk, W):
    w = _words(sk, S.words_table(S.one_digit_varies(50_000, W, "low", W)))
    assert S.varying_digits(w) == [(W - 1, 0)] and len(np.unique(w[:, W - 1])) == 256
    w = _words(sk, S.words_table(S.one_digit_varies(50_000, W, "top", W)))
    assert S.varying_digits(w) == [(0, S.top_digit(W))] and len(np.unique(w[:, 0])) == 256


def test_runs_and_tiles_on_one_digit(sk):
    n = 5 * S.TILE + 700
    for length in (32, 512, S.TILE):
        w = _words(sk, S.words_table(S.runs(n, 2, length, length)))
        last = w[:, 1]
        for s in range(0, n, length):
            assert (last[s:s + length] == last[s]).all()
        assert len(np.unique(last)) == -(-n // length)
        assert len(S.varying_digits(w)) == 16
    for tile in (0, 2, 5):
        w = _words(sk, S.words_table(S.tile_on_one_digit(n, 3, tile, tile)))
        rows = w[tile * S.TILE:(tile + 1) * S.TILE, 2]
        assert (rows == rows[0]).all()
        assert len(np.unique(w[:, 2])) > n - S.TILE                           # the other tiles: random


def test_patterns_shapes(sk):
    n = 100_000
    w = _words(sk, S.words_table(S.pattern(n, 2, "sorted", None, 1)))
    assert (np.diff(w[:, 1].astype(np.int64)) == 1).all() and S.varying_digits(w) == [(1, 0), (1, 1), (1, 2)]
    w = _words(sk, S.words_table(S.pattern(n, 2, "reverse", None, 1)))
    assert (np.diff(w[:, 1].astype(np.int64)) == -1).all()
    for period in (32, 512, S.TILE):
        w = _words(sk, S.words_table(S.pattern(n, 1, "sawtooth", period, 1)))
        assert (w[:, 0] == np.arange(n) % period).all()


@pytest.mark.parametrize("j", [0, 1, 2, 3])
def test_decided_in_word(sk, j):
    """the key at each TopK cut-off shares words 0 .. j - 1 with many rows and no other row has its words 0 .. j"""
    w = _words(sk, S.words_table(S.decided_in_word(S.TOPK_ROWS, 4, j, 11 + j)))
    for k in range(j):
        assert len(np.unique(w[:, k])) == 2
    srt = w[np.lexsort(w.T[::-1])]
    for fetch in (1, 1000, 4096, S.TOPK_CHUNK):
        cut = srt[fetch - 1]
        assert (srt[:, :j] == cut[:j]).all(axis=1).sum() > S.TOPK_ROWS >> (j + 1)
        assert (srt[:, :j + 1] == cut[:j + 1]).all(axis=1).sum() == 1


def test_chunk_trends():
    n, c = S.TOPK_ROWS, S.TOPK_CHUNK
    for improving in (True, False):
        w = S.chunk_trend(n, c, improving, 1)[:, 0]
        hi = [w[k:k + c].max() for k in range(0, n, c)]
        lo = [w[k:k + c].min() for k in range(0, n, c)]
        for k in range(1, len(hi)):
            assert (hi[k] < lo[k - 1]) if improving else (lo[k] > hi[k - 1])


@pytest.mark.parametrize("name", list(S.CASES))
def test_topk_cases_run_over_100_rounds(name):
    c = S.CASES[name]
    batch = c.batch or S.TOPK_CHUNK // 4
    assert S.rounds(c.n, c.chunk, batch) >= 100


def test_tie_run_spans_chunks():
    """the cut-off falls inside the run of V, whose rows sit in every chunk"""
    n, fetch, c = S.TOPK_ROWS, 4096, S.CASES["topk-tie-run"]
    w = S.tie_run_across_chunks(n, fetch, 7)[:, 0]
    V = np.uint64(1 << 62)
    assert (w < V).sum() < fetch < (w <= V).sum()
    chunks = np.flatnonzero(w == V) // (c.batch * -(-S.TOPK_CHUNK // c.batch))
    assert len(np.unique(chunks)) == S.rounds(n, S.TOPK_CHUNK, c.batch)


def test_cutoff_specials_sit_on_the_cut_offs():
    """asc, NULLs first: NULL f64 rows are sorted rows [0, 2048), -NaN payloads [2048, 4096), -NaN [4096, 6144), -Inf [6144, 8192)"""
    t, cls = S.cutoff_table(S.TOPK_ROWS, 2048, 41)
    order = S.order(t, [(0, False, True), (1, True, False), (2, False, True)])
    assert (cls[order[:8192]] == np.repeat([0, 1, 2, 3], 2048)).all()
    order = S.order(t, [(0, True, False)])
    assert (cls[order[:4096]] == np.repeat([8, 7], 2048)).all()                # +NaN payload, then +NaN


def test_large_dictionary():
    c = S.CASES["strings-large-dict"]
    t, _, inputs = c.make(c.n)
    d = inputs[0][0].column(0).dictionary
    assert len(d) >= 100_000 and len(set(d.to_pylist())) == len(d)
    c = S.CASES["strings-growing-dict"]
    _, _, inputs = c.make(c.n)
    sizes = [len(b.column(0).dictionary) for b in inputs[0]]
    assert sizes == sorted(sizes) and sizes[-1] >= 100_000 and len(set(sizes)) > 100


def test_digit_passes_and_selects():
    w = np.array([[0x0100, 0xFF], [0x0000, 0xFF]], np.uint64)
    assert S.varying_digits(w) == [(0, 1)] and S.digit_passes(w) == 1
    assert S.digit_passes(S.random_words(1, 4, 0)) == 0
    assert S.scan_chunks(S.TILE * 16 * 1024) == 1024 and S.scan_chunks(S.TILE * 16 * 1024 + 1) == 1025
    n, c = 10 * S.TOPK_CHUNK, S.TOPK_CHUNK
    assert S.selects(n, 1, None, c) and S.selects(n, c, 5, c) and S.selects(n, c + 1, None, c)
    assert not S.selects(n, c + 1, 5, c) and not S.selects(n, None, 5, c) and not S.selects(n, n, None, c)


# ---- the comparison fails on wrong answers ---------------------------------------------------------------------------------------------
def _fails(got, want, keys):
    try:
        S.check(got, want, keys)
    except AssertionError:
        return True
    return False


def _take(t, rows):
    return pa.table([R._array(t.column(i)).take(pa.array(rows, pa.int64())) for i in range(t.num_columns)], names=t.column_names)


def test_comparison_catches_corruptions():
    t, keys = S.words_table(S.one_digit_varies(3 * S.TILE + 5, 2, "low", 1, distinct=50))
    o = S.order(t, keys)
    want = S.sort_table(t, keys)
    assert not _fails(want, want, keys)
    k0 = np.asarray(want.column(1))
    # two tied rows swapped
    i = int(np.flatnonzero(k0[:-1] == k0[1:])[10])
    sw = o.copy()
    sw[[i, i + 1]] = sw[[i + 1, i]]
    assert _fails(_take(t, sw), want, keys)
    # one row out of order across a tile edge (distinct keys)
    rt, rkeys = S.words_table(S.random_words(3 * S.TILE + 5, 1, 2))
    ro = S.order(rt, rkeys)
    sw = ro.copy()
    sw[[S.TILE - 1, S.TILE]] = sw[[S.TILE, S.TILE - 1]]
    assert _fails(_take(rt, sw), S.sort_table(rt, rkeys), rkeys)
    # the last row of a fetch window replaced by the next tied row
    fetch = i + 1
    w = S.sort_table(t, keys, fetch)
    assert not _fails(_take(t, o[:fetch]), w, keys)
    assert _fails(_take(t, np.concatenate([o[:fetch - 1], o[fetch:fetch + 1]])), w, keys)
    # a window off by one, either way, and with a skip
    assert _fails(_take(t, o[1:fetch + 1]), w, keys)
    assert _fails(_take(t, o[:fetch - 1]), w, keys)
    assert _fails(_take(t, o[:fetch + 1]), w, keys)
    w = S.sort_table(t, keys, fetch, 7)
    assert _fails(_take(t, o[6:fetch]), w, keys) and _fails(_take(t, o[8:fetch + 1]), w, keys)
    # a candidate (earlier input) losing a tie to a later row
    assert _fails(_take(t, np.sort(o[:fetch])), w, keys)


# ---- plans ------------------------------------------------------------------------------------------------------------------------------
def _plans(P):
    for W in (1, 2, 3, 4):
        t, keys = S.words_table(S.random_words(3, W, 0))
        yield S.plan(P, t, keys)
    t, keys = S.words_table(S.random_words(3, 4, 0), "i32", desc=[True, False, False, True, True, False, True])
    yield S.plan(P, t, keys)
    t, keys = S.words_table(S.random_words(3, 4, 0), desc=[False, True, False, True])
    yield S.plan(P, t, keys)
    for c in S.CASES.values():
        t, keys, _ = c.make(S.TOPK_CHUNK + 10)
        for fetch, skip in c.windows:
            yield S.plan(P, t, keys, fetch, skip)


def test_plans_supported_and_compile(cb):
    plans = list(_plans(cb.proto))
    assert len(plans) > 60
    for p in plans:
        ok, why = cb.native.supports(p)
        assert ok, why
        assert cb.native.compile_plan(p) is not None
