"""GPU: the Sort operator (ORDER BY, and TopK through fetch / skip) against the CPU reference (tests/sortref.py).  Every output column is
compared bit-exact -- values, float bits, validity, strings spelled out -- with the reference's stable order, and every output is also
checked with the reference comparator alone.  Inputs cover every key type and physical layout a source hands the operator: Arrow
streams (booleans as bitmaps, dictionaries with int8 / int16 / int32 indices, growing or replaced between batches), device tables
(8-byte decimals), the Parquet scan, a filter / projection pipeline below the sort and a Final hash aggregate (host-resident results)."""
import numpy as np
import pyarrow as pa
import pytest

import partref
import sortref as R
from test_gpu_partition_layouts import WORDS, device_table, expected_table, make_values, parquet_table, scan_of, supports, table_of, write_parquet

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def sort_plan(cb, child, types, keys, fetch=None, skip=None):
    """keys: (column index, descending, nulls_first)"""
    P = cb.proto
    return P.sort(child, [P.sort_order(P.bound(i, types[i]), d, nf) for i, d, nf in keys], fetch=fetch, skip=skip)


def collect(cb, plan, inputs, config=None, batch_size=8192):
    """(table or None, stats): every batch of cb200_execute (batchSize slices) concatenated"""
    with cb.native.Plan(plan, inputs, config=config, batch_size=batch_size) as p:
        got = p.collect()
        return got, p.stats()


def check(got, tbl, keys, fetch=None, skip=None):
    want = R.sort_table(tbl, keys, fetch, skip)
    if want.num_rows == 0:
        assert got is None or got.num_rows == 0
        return
    assert got is not None
    partref.assert_tables_equal(got, want)
    R.assert_sorted(got, keys)


def stream_case(cb, n, keys, names=None, seed=1, chunk=8192, fetch=None, skip=None, config=None):
    cols = make_values(n, seed)
    tbl, types = table_of(cols, names)
    ks = [(tbl.column_names.index(k), d, nf) for k, d, nf in keys]
    plan = sort_plan(cb, cb.proto.scan(types), types, ks, fetch, skip)
    got, stats = collect(cb, plan, [tbl.to_batches(max_chunksize=chunk)] if n else [tbl], config)
    check(got, tbl, ks, fetch, skip)
    return got, stats


ALL = ["b", "i8", "i16", "i32", "date", "i64", "ts", "f32", "f64", "d9", "d18", "d38", "s8", "s16", "s32"]
OPTS = [(False, True), (False, False), (True, True), (True, False)]   # (descending, nulls_first)


# ---- key types, directions, null placement -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("desc,nulls_first", OPTS)
@pytest.mark.parametrize("key", ALL)
def test_each_key_type(cb, key, desc, nulls_first):
    """one key of each type (NULLs, MIN / MAX, +-0.0, +-Inf, NaN payloads, decimal +-(10^p - 1)); the row number rides along"""
    stream_case(cb, 20_000, [(key, desc, nulls_first)], names=[key, "row"], seed=ALL.index(key) + 3)


@pytest.mark.parametrize("keys", ["i8+i16", "b+f32+s8", "d9+d38+date", "s16+i32+date+b+d18",
                                  "b+i8+i16+date+s8+s16+f32+i32", "d38+f64+s32+i16+b"])
def test_key_combinations(cb, keys):
    """up to 8 keys and up to 256 bits of packed key; every column has NULLs in its own rows; mixed directions and null placements"""
    names = keys.split("+")
    rng = np.random.default_rng(len(names))
    ks = [(k, *OPTS[int(rng.integers(4))]) for k in names]
    stream_case(cb, 40_000, ks, names=ALL + ["row"], seed=len(names) * 5)
    stream_case(cb, 40_000, ks, names=ALL + ["row"], seed=len(names) * 5, fetch=700, config={"spark.comet.b200.chunkRows": "16384"})


def test_ties_and_constant_digits(cb):
    """many ties (input order must survive) and keys whose digits are equal in every row: a constant column runs no pass, a small range
    one or two"""
    P = cb.proto
    n = 100_000
    rng = np.random.default_rng(8)
    tbl = pa.table({"k": pa.array(rng.integers(0, 3, n), pa.int64()), "c": pa.array(np.full(n, 7, np.int32)),
                    "d": pa.array(rng.integers(18000, 18200, n).astype(np.int32), pa.date32()), "row": pa.array(np.arange(n))})
    types = [P.INT64, P.INT32, P.DATE, P.INT64]
    for ks, passes in (([(1, False, True)], 0), ([(0, True, True)], 1), ([(1, True, True), (0, False, True)], 1), ([(2, False, True)], 2),
                       ([(2, True, False), (0, False, True)], 3)):
        got, stats = collect(cb, sort_plan(cb, P.scan(types), types, ks), [tbl.to_batches(max_chunksize=30_000)])
        check(got, tbl, ks)
        assert stats["sort_passes"] == passes, (ks, stats["sort_passes"])
    # TopK where the cut-off falls inside a run of equal keys: the first rows of the run in input order are kept
    cfg = {"spark.comet.b200.chunkRows": "30000"}
    for ks, fetch in (([(1, False, True)], 1000), ([(0, True, True)], 25_000), ([(0, False, True), (1, True, False)], 12_345),
                      ([(2, True, True)], 777)):
        got, _ = collect(cb, sort_plan(cb, P.scan(types), types, ks, fetch), [tbl.to_batches(max_chunksize=30_000)], cfg)
        check(got, tbl, ks, fetch)


@pytest.mark.parametrize("n", [0, 1, 1023, 3 * 2**20 + 17])
def test_sizes(cb, n):
    keys = [("f64", True, False), ("s16", False, True), ("i32", False, True)]
    stream_case(cb, n, keys, names=["b", "i32", "f64", "d18", "s16", "row"], seed=n % 97, chunk=1 << 18)


# ---- fetch / skip (TopK) -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fetch,skip", [(0, None), (1, None), (100, None), (5000, None), (25_000, None), (60_000, None), (10**6, None),
                                        (None, 7), (None, 60_000), (100, 30), (25_000, 24_999), (40, 40), (50, 200)])
def test_fetch_skip(cb, fetch, skip):
    """chunkRows 20 000 over 50 000 rows: a fetch within one chunk is a TopK that carries candidates across chunks, a larger one a full
    sort of the concatenated chunks; sorted[skip : fetch] either way"""
    keys = [("i16", False, True), ("s8", True, False), ("d18", False, False)]
    stream_case(cb, 50_000, keys, names=["i16", "s8", "d18", "f32", "b", "row"], seed=13, chunk=7000, fetch=fetch, skip=skip,
                config={"spark.comet.b200.chunkRows": "20000"})


def test_topk_input_with_projection(cb):
    """TakeOrderedAndProject: Scan("TopKInput") -> Sort{fetch, skip} -> Projection (CometExecUtils.getTopKNativePlan)"""
    P = cb.proto
    cols = make_values(30_000, 4)
    tbl, types = table_of(cols, ["f64", "s32", "d38", "row"])
    ks = [(0, True, False), (3, False, True)]
    topk = sort_plan(cb, P.scan(types, source="TopKInput"), types, ks, fetch=777, skip=5)
    plan = P.projection(topk, [P.bound(3, P.INT64), P.bound(1, P.STRING), P.bound(0, P.DOUBLE)])
    got, _ = collect(cb, plan, [tbl.to_batches(max_chunksize=4000)], config={"spark.comet.b200.chunkRows": "10000"})
    want = R.sort_table(tbl, ks, 777, 5)
    partref.assert_tables_equal(got, want.select([3, 1, 0]))


def test_outputs_through_execute_device(cb):
    """the same sort read back through cb200_execute with several batch sizes and through cb200_execute_device"""
    from test_gpu_scan_export import assert_device_matches, device_batches
    P = cb.proto
    cols = make_values(30_000, 6)
    tbl, types = table_of(cols, ["b", "i8", "d9", "d38", "s8", "f32", "row"])
    ks = [(4, False, False), (2, True, True)]
    plan = sort_plan(cb, P.scan(types), types, ks)
    want = R.sort_table(tbl, ks)
    for bs in (8192, 1000, 30_000):
        got, _ = collect(cb, plan, [tbl.to_batches(max_chunksize=5000)], batch_size=bs)
        partref.assert_tables_equal(got, want)
    assert_device_matches(device_batches(cb, plan, [tbl.to_batches(max_chunksize=5000)]), want)


# ---- sources ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("index", [pa.int8(), pa.int16(), pa.int32()])
@pytest.mark.parametrize("mode", ["same", "growing", "shuffled"])
def test_dictionary_streams(cb, index, mode):
    """each record batch carries its own dictionary: the same one, one that grows batch by batch, or a shuffled one; small chunks make
    the full sort concatenate several chunks and TopK rebuild its keys from a grown dictionary"""
    P = cb.proto
    rng = np.random.default_rng(5)
    per, k = 4000, 10
    batches, plain = [], []
    for b in range(k):
        words = WORDS[:30 + 7 * b] if mode == "growing" else WORDS
        order = rng.permutation(len(words)) if mode == "shuffled" else np.arange(len(words))
        d = pa.array([words[i] for i in order])
        s = pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, len(words), per), index, mask=rng.random(per) < 0.1), d)
        v = pa.array(rng.integers(-50, 50, per).astype(np.int32))
        batches.append(pa.record_batch([s, v], names=["s", "v"]))
        plain.append(pa.record_batch([s.dictionary_decode(), v], names=["s", "v"]))
    tbl = pa.Table.from_batches(plain)
    types = [P.STRING, P.INT32]
    cfg = {"spark.comet.b200.chunkRows": "8000"}
    for ks, fetch in (([(0, False, True)], None), ([(1, True, False), (0, True, True)], None), ([(0, True, False), (1, False, True)], 3000)):
        got, _ = collect(cb, sort_plan(cb, P.scan(types), types, ks, fetch), [batches], cfg)
        check(got, tbl, ks, fetch)


@pytest.mark.parametrize("keys", ["b", "i8", "i16", "d9", "d18", "d38", "s8+i32", "f32+s16+date+ts", "d9+d18+s32"])
def test_device_tables(cb, keys):
    """device columns, decimal(9, 2) and decimal(18, 0) 8 bytes wide; chunkRows below the table: the slices are concatenated"""
    cols = make_values(30_000, 21 + len(keys))
    tbl, types = table_of(cols)
    t = device_table(cb, tbl, types, dec8=("d9", "d18"))
    ks = [(tbl.column_names.index(k), i % 2 == 1, i % 3 == 0) for i, k in enumerate(keys.split("+"))]
    got, _ = collect(cb, sort_plan(cb, cb.proto.scan(types), types, ks), [t], config={"spark.comet.b200.chunkRows": "10240"})
    check(got, tbl, ks)


@pytest.mark.parametrize("as_int", [True, False])
@pytest.mark.parametrize("keys", ["i8", "i16", "d7", "d12", "d28", "i32w+date", "ts+f32", "f64+i64", "sd", "sp+d7+i8"])
def test_native_scan(cb, tmp_path, as_int, keys):
    """Sort over NativeScan: INT32-backed int8 / int16 / decimal(7, 2), INT64 or FLBA decimals, dictionary and PLAIN string pages"""
    n = 90_000
    cols = parquet_table(n, 31)
    path = str(tmp_path / "p.parquet")
    write_parquet(path, cols, as_int)
    names = ["i8", "i16", "i32", "i32w", "date", "d7", "i64", "ts", "d12", "d28", "f32", "f64", "sd", "sp", "row"]
    scan, types = scan_of(cb, cols, names, path)
    ks = [(names.index(k), i == 0, i != 1) for i, k in enumerate(keys.split("+"))]
    fetch = 1000 if "+" in keys else None
    got, _ = collect(cb, sort_plan(cb, scan, types, ks, fetch), [], config={"spark.comet.b200.chunkRows": "50000"})
    check(got, expected_table(cols, names), ks, fetch)


def test_pipeline_below_and_above(cb):
    """Filter + Projection below the sort (their kernel feeds it), and a Filter + Projection above it (fed by the sort, order kept)"""
    P = cb.proto
    cols = make_values(60_000, 9)
    tbl, types = table_of(cols, ["i32", "f64", "s16", "d18", "row"])
    below = P.projection(P.filter_(P.scan(types), P.gt(P.bound(0, P.INT32), P.literal(0, P.INT32))),
                         [P.bound(4, P.INT64), P.bound(2, P.STRING), P.bound(1, P.DOUBLE), P.bound(3, P.DECIMAL(18, 0))])
    btypes = [P.INT64, P.STRING, P.DOUBLE, P.DECIMAL(18, 0)]
    ks = [(1, True, True), (2, False, False)]
    plan = P.projection(P.filter_(sort_plan(cb, below, btypes, ks), P.is_not_null(P.bound(2, P.DOUBLE))),
                        [P.bound(0, P.INT64), P.bound(1, P.STRING)])
    got, _ = collect(cb, plan, [tbl.to_batches(max_chunksize=8192)], config={"spark.comet.b200.chunkRows": "16384"})
    i32 = tbl.column("i32").combine_chunks()
    kept = tbl.filter(np.asarray(i32.fill_null(0)) > 0).select(["row", "s16", "f64", "d18"])
    srt = R.sort_table(kept, ks)
    want = srt.filter(np.asarray(srt.column(2).is_valid())).select([0, 1])
    partref.assert_tables_equal(got, want)


def test_q1_order_by(cb):
    """TPC-H Q1 ends in ORDER BY l_returnflag, l_linestatus: Sort over the Final aggregate, whose results are host-resident"""
    from comet_b200 import tpch
    P = cb.proto
    cols = tpch.gen_lineitem(200_000, seed=42)
    tbl = tpch.lineitem_table(cols, "dec", dictionary=True)
    with cb.native.Plan(tpch.q1_partial_plan("dec"), [tbl.to_batches(max_chunksize=8192)]) as p:
        state = p.collect()
    final = tpch.q1_final_plan("dec")
    unsorted, _ = collect(cb, final, [state])
    out_types = [P.STRING, P.STRING] + [None] * 7 + [P.INT64]   # group keys ... count(*)
    ks = [(0, False, True), (1, False, True)]
    got, _ = collect(cb, sort_plan(cb, final, out_types, ks), [state])
    assert got.num_rows == 4
    check(got, unsorted, ks)
    got, _ = collect(cb, sort_plan(cb, final, out_types, [(1, True, True), (9, True, False)]), [state])   # by linestatus DESC, count DESC
    check(got, unsorted, [(1, True, True), (9, True, False)])


def test_plain_utf8_refused(cb):
    P = cb.proto
    tbl = pa.table({"s": pa.array(["b", "a", None]), "v": pa.array([1, 2, 3])})
    plan = sort_plan(cb, P.scan([P.STRING, P.INT64]), [P.STRING, P.INT64], [(0, False, True)])
    assert supports(cb, plan)[0]   # a plan-time answer: the column's encoding is known only when a batch arrives
    with pytest.raises(cb.native.Unsupported, match="plain string columns"):
        collect(cb, plan, [tbl])


def test_partial_aggregate_state(cb):
    """Sort over HashAggregate(Partial), whose state keeps booleans one byte per row: keys on the BOOLEAN group key and the SUM state's
    is_empty flag ((b, k) is unique per state row, so the order has no ties)"""
    P = cb.proto
    rng = np.random.default_rng(17)
    n = 60_000
    from test_gpu_partition_layouts import _dec
    tbl = pa.table({"b": pa.array(rng.random(n) < 0.5, mask=rng.random(n) < 0.1), "k": pa.array(rng.integers(0, 5000, n), pa.int64()),
                    "v": _dec(rng.integers(-10**9, 10**9, n), 12, 2, mask=rng.random(n) < 0.3)})
    agg = P.hash_agg(P.scan([P.BOOL, P.INT64, P.DECIMAL(12, 2)]), [P.bound(0, P.BOOL), P.bound(1, P.INT64)],
                     [P.agg_sum(P.bound(2, P.DECIMAL(12, 2)), P.DECIMAL(22, 2))], P.PARTIAL)
    state, stats = collect(cb, agg, [tbl.to_batches(max_chunksize=8192)])
    assert stats["agg_strategies"] & cb.native.AGG_TABLE
    types = [P.BOOL, P.INT64, P.DECIMAL(22, 2), P.BOOL]
    ks = [(3, True, False), (0, False, False), (1, True, True)]
    got, _ = collect(cb, sort_plan(cb, agg, types, ks), [tbl.to_batches(max_chunksize=8192)])
    check(got, state, ks)
