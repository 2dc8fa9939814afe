"""GPU parity for the Parquet page decoders on hand-built pages (tests/pagecases.py, pinned on CPU by tests/test_parquet_pages_cpu.py):
every RLE / bit-packed run shape and dictionary bit width 0..32 through k_pq_rle_scan / k_pq_rle_decode<4, 8, 16> / k_pq_rle_direct,
definition levels in every layout on both level paths, tiny pages, PLAIN fallback, mixed codecs per row group and Snappy element
forms through the segmented and serial decoders.  Values are compared bit-exact (floats by their bits), validity and strings in full.
Malformed pages must raise, never return a batch."""
import decimal
import struct

import numpy as np
import pytest

import pagecases as PC
import pqwrite as W

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def _dt(P, kind):
    return P.DECIMAL(*PC.TYPES[kind][2]) if PC.TYPES[kind][2] else getattr(P, PC.TYPES[kind][1])


def _run(cb, names, raws, tag, chunk_rows=1 << 20):
    P = cb.proto
    paths = [cb.native.register_memory_file(f"pages_{tag}_{i}", np.frombuffer(r, dtype=np.uint8).copy()) for i, r in enumerate(raws)]
    fields = [(n, _dt(P, n), True) for n in names]
    try:
        with cb.native.Plan(P.native_scan(fields, fields, paths), [], config={"spark.comet.b200.chunkRows": str(chunk_rows)}) as p:
            return p.collect()
    finally:
        for i in range(len(raws)):
            cb.native.register_memory_file(f"pages_{tag}_{i}", None)


def _values(arr, kind):
    """the device's column in the writer's convention: ints, float bit patterns, unscaled decimals, bytes; None at NULLs"""
    import pyarrow as pa
    if pa.types.is_dictionary(arr.type):
        arr = arr.cast(arr.type.value_type)
    if kind == "date":
        arr = arr.cast(pa.int32())
    if kind in ("f32", "f64"):
        bits = np.asarray(arr.fill_null(0)).view(np.uint32 if kind == "f32" else np.uint64)
        return [int(b) if ok else None for b, ok in zip(bits, arr.is_valid().to_pylist())]
    out = arr.to_pylist()
    if PC.TYPES[kind][2]:
        ctx = decimal.Context(prec=60)
        return [None if v is None else int(v.scaleb(PC.TYPES[kind][2][1], context=ctx)) for v in out]
    if kind == "s":
        return [None if v is None else v.encode() for v in out]
    return out


def _check(res, case):
    exp = PC.expected(case)
    for j, name in enumerate(case[1]):
        v, ok = exp[name]
        want = [x if k else None for x, k in zip(v, ok)]
        got = _values(res.column(j).combine_chunks(), name)
        assert len(got) == len(want), name
        bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
        assert not bad, (name, len(bad), bad[:5], [got[i] for i in bad[:5]], [want[i] for i in bad[:5]])


@pytest.mark.parametrize("name", sorted(PC.cases()))
def test_page_matrix(cb, name):
    """Every case of the matrix: dictionary widths 0..32 for 4-, 8- and 16-byte values and strings, run shapes including RLE runs of 1
    (more runs than a page's run table holds: the direct decoder), level layouts and paths, tiny pages, PLAIN fallback, codecs per row
    group, Snappy element forms."""
    case = PC.cases()[name]()
    res = _run(cb, case[1], PC.file_bytes(case), name, case[2])
    _check(res, case)


def test_fast_path_is_taken_when_statistics_promise_no_nulls(cb):
    """null_count = 0 selects the verify-only path: a NULL in such a chunk is reported as corrupt statistics.  The same file without
    Statistics decodes its NULL (NULL-aware path), in every level shape including one RLE run per row."""
    col = PC.column("i64")
    for shape in PC.SHAPES:
        vals, valid = list(range(300)), [i != 150 for i in range(300)]
        raw = W.write_file([col], [[W.chunk(col, vals, valid, 100, level_shape=shape, null_count=0)]])
        with pytest.raises(cb.native.CometB200Error, match="null_count = 0"):
            _run(cb, ["i64"], [raw], "fast")
        raw = W.write_file([col], [[W.chunk(col, vals, valid, 100, level_shape=shape, null_count=None)]])
        assert _values(_run(cb, ["i64"], [raw], "aware").column(0).combine_chunks(), "i64") == [v if ok else None for v, ok in zip(vals, valid)]


def test_many_short_runs_decode_on_both_level_paths(cb):
    """Alternating NULLs as one RLE run per row (about n runs, past the n / 8 + 64 a page's run table holds), and dictionary indices the
    same way: decoded on the NULL-aware path and verified on the fast path.  Before k_pq_rle_direct such pages were refused at execute
    time."""
    col = PC.column("i32")
    n = 5000
    dictionary = list(range(-3, 4))
    vals = [dictionary[i % 7] for i in range(n)]
    for valid, nc in (([i % 2 == 0 for i in range(n)], "exact"), ([True] * n, "exact")):
        for ver in (1, 2):
            ch = W.chunk(col, vals, valid, n, dictionary=dictionary, index_shape="rle1", level_shape="rle1", version=ver, null_count=nc)
            got = _values(_run(cb, ["i32"], [W.write_file([col], [[ch]])], "short").column(0).combine_chunks(), "i32")
            assert got == [v if ok else None for v, ok in zip(vals, valid)]


# ---- malformed pages: each bound below is checked by the kernel before it reads -------------------------------------------------
def _dict_file(idx_stream, num_values=16, dict_size=4, optional=False):
    col = PC.column("i64", optional=optional)
    dictionary = list(range(100, 100 + dict_size))
    pages = [W.dict_page(col, dictionary), W.Page(W.DATA_PAGE, num_values, W.RLE_DICTIONARY, idx_stream)]
    return W.write_file([col], [[W.Chunk(pages, [0] * num_values, [True] * num_values)]])


def test_malformed_pages_raise(cb):
    run = lambda raw: _run(cb, ["i64"], [raw], "bad")
    E = cb.native.CometB200Error
    # store_dict: an index at or above the dictionary size -> ExecError 3
    with pytest.raises(E) as ei:
        run(_dict_file(bytes([3]) + W.hybrid([("packed", 2, [0, 1, 2, 3, 4] + [0] * 11)], 3)))
    assert ei.value.code == 3 and "dictionary index" in ei.value.message
    with pytest.raises(E) as ei:                                                  # the same through k_pq_rle_direct (RLE runs of 1)
        run(_dict_file(bytes([3]) + W.hybrid([("rle", 1, i % 5) for i in range(200)], 3), num_values=200))
    assert ei.value.code == 3
    # walk_hybrid: a bit width above 32 is refused before any run is read
    with pytest.raises(E, match="malformed RLE"):
        run(_dict_file(bytes([33]) + W.hybrid([("rle", 16, 1)], 32)))
    # walk_hybrid: the stream ends before num_values values (seen != want in k_pq_rle_scan)
    with pytest.raises(E, match="malformed RLE"):
        run(_dict_file(bytes([2]) + W.hybrid([("rle", 9, 1)], 2)))
    # walk_hybrid: a packed run whose wanted values lie past the page (HYB_TRUNCATED, checked before the run is handed out)
    with pytest.raises(E, match="truncated page"):
        run(_dict_file(bytes([2]) + W.hybrid([("packed", 2, [1] * 16)], 2)[:-2]))
    # k_pq_resolve: a v1 level length of 0, or one past the page, on a page with values
    col = PC.column("i64")
    for prefix, what in ((0, "malformed RLE"), (10**6, "truncated page")):
        page = W.Page(W.DATA_PAGE, 20, W.PLAIN, struct.pack("<I", prefix) + W.plain(W.INT64, list(range(20))))
        with pytest.raises(E, match=what):
            run(W.write_file([col], [[W.Chunk([page], list(range(20)), [True] * 20, null_count=None)]]))
        with pytest.raises(E, match=what):                                         # the fast path's page goes through the same check
            run(W.write_file([col], [[W.Chunk([page], list(range(20)), [True] * 20, null_count=0)]]))
    # the planner: BIT_PACKED levels, and a v2 page of an optional column without levels
    bp = W.Page(W.DATA_PAGE, 16, W.PLAIN, b"\xff\xff" + W.plain(W.INT64, list(range(16))), def_encoding=W.BIT_PACKED)
    with pytest.raises(cb.native.Unsupported, match="definition level encoding 4"):
        run(W.write_file([col], [[W.Chunk([bp], list(range(16)), [True] * 16)]]))
    v2 = W.data_page(col, list(range(16)), [True] * 16, version=2)
    v2.levels = b""
    with pytest.raises(E, match="no definition levels"):
        run(W.write_file([col], [[W.Chunk([v2], list(range(16)), [True] * 16)]]))


def test_out_of_scope_physical_types_are_refused(cb):
    """BOOLEAN and INT96 pages stay outside the device decoder: refused, not misread"""
    P = cb.proto
    for phys, dt in ((0, P.BOOL), (3, P.TIMESTAMP)):
        col = W.Column("x", phys, optional=False)
        page = W.Page(W.DATA_PAGE, 8, W.PLAIN, b"\x55" if phys == 0 else bytes(96))
        raw = W.write_file([col], [[W.Chunk([page], [0] * 8, [True] * 8)]])
        path = cb.native.register_memory_file("pages_oos", np.frombuffer(raw, dtype=np.uint8).copy())
        try:
            with pytest.raises(cb.native.CometB200Error):
                with cb.native.Plan(P.native_scan([("x", dt, True)], [("x", dt, True)], [path]), []) as p:
                    p.collect()
        finally:
            cb.native.register_memory_file("pages_oos", None)
