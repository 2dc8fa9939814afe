"""GPU: the SortMergeJoin operator (inner, left / right / full outer, left semi and left anti equi-joins) against the CPU reference
(tests/smjref.py).  Every output column is compared bit-exact and in order.  Inputs are sorted by the keys, as
Spark hands them to the operator, except where a Sort below the join does it; NULL-extended columns are checked in every stored layout
and exported as valid Arrow."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import smjref as R
import partref
from test_gpu_join import KEYS, check, collect, side
from test_gpu_partition_layouts import WORDS, _dec, _words, device_table, expected_table, parquet_table, scan_of, write_parquet

pytestmark = pytest.mark.gpu

JTS = [R.INNER, R.LEFT_OUTER, R.RIGHT_OUTER, R.FULL_OUTER, R.LEFT_SEMI, R.LEFT_ANTI]
JT = {R.INNER: 0, R.LEFT_OUTER: 1, R.RIGHT_OUTER: 2, R.FULL_OUTER: 3, R.LEFT_SEMI: 4, R.LEFT_ANTI: 5}
OUTER = [R.LEFT_OUTER, R.RIGHT_OUTER, R.FULL_OUTER]


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def _plain(a):
    a = a.combine_chunks() if isinstance(a, pa.ChunkedArray) else a
    return a.dictionary_decode() if pa.types.is_dictionary(a.type) else a


def sorted_by(tbl, keys):
    """tbl's rows in ascending key order, NULLs first, equal keys in input order (Spark's default SortOrder)"""
    if tbl.num_rows == 0:
        return tbl
    plain = pa.table({f"k{i}": _plain(tbl.column(k)) for i, k in enumerate(keys)})
    idx = pc.sort_indices(plain, sort_keys=[(f"k{i}", "ascending") for i in range(len(keys))], null_placement="at_start")
    return tbl.take(idx)


def smj_plan(cb, lchild, ltypes, rchild, rtypes, lk, rk, jt):
    P = cb.proto
    return P.sort_merge_join(lchild, rchild, [P.bound(i, ltypes[i]) for i in lk], [P.bound(i, rtypes[i]) for i in rk], JT[jt],
                             [P.sort_order(P.bound(i, ltypes[i])) for i in lk])


def inputs_of(tbl, chunk):
    return [tbl.to_batches(max_chunksize=chunk)] if tbl.num_rows else [tbl]


def case(cb, left, ltypes, right, rtypes, lk, rk, jt, lchunk=5000, rchunk=3000, config=None, linputs=None, rinputs=None):
    P = cb.proto
    plan = smj_plan(cb, P.scan(ltypes), ltypes, P.scan(rtypes), rtypes, lk, rk, jt)
    li = linputs if linputs is not None else inputs_of(left, lchunk)
    ri = rinputs if rinputs is not None else inputs_of(right, rchunk)
    got, stats = collect(cb, plan, li + ri, config)
    want = R.sort_merge_join_table(left, right, lk, rk, jt)
    check(got, want)
    if got is not None:
        got.validate(full=True)
    return got, want, stats


def sorted_sides(n_l, n_r, keys, seed, domain, **kw):
    ks = [f"k{i}" for i in range(len(keys))]
    left, lt = side(n_l, keys, seed, domain, **kw)
    right, rt = side(n_r, keys, seed + 100, domain, **kw)
    return sorted_by(left, ks), lt, sorted_by(right, ks), rt


# ---- join types and key types --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("jt", JTS)
@pytest.mark.parametrize("key", KEYS)
def test_each_key_type(cb, key, jt):
    """one key of each type, NULLs on both sides, N:M duplicates, keys on one side only"""
    n_l, n_r, dom = (300, 200, 2) if key == "b" else (3000, 2000, 1500) if key in ("i8", "s8", "s16", "s32") else (8000, 5000, 3000)
    left, lt, right, rt = sorted_sides(n_l, n_r, [key], KEYS.index(key) + 1, dom)
    case(cb, left, lt, right, rt, [0], [0], jt)


@pytest.mark.parametrize("shape", ["1:1", "1:N", "N:M", "none", "all", "skew", "null_left", "null_right"])
@pytest.mark.parametrize("jt", JTS)
def test_multiplicities(cb, shape, jt):
    """unique keys, duplicates on one side or both, no key in common, every key in common, one key owning most build rows, and a side
    whose keys are all NULL"""
    P = cb.proto
    rng = np.random.default_rng(len(shape) + JT[jt])
    def keys(n, kind):
        if kind == "unique":
            return rng.permutation(int(n * 1.3))[:n]
        if kind == "dup":
            return rng.integers(0, n // 20, n)
        if kind == "high":
            return rng.integers(10**6, 2 * 10**6, n)
        if kind == "skew":
            return np.where(rng.random(n) < 0.9, 7, rng.integers(0, 500, n))
        if kind == "few7":
            return np.concatenate([[7], rng.integers(0, 500, n - 1)])
        return rng.integers(0, 50, n)
    lkind, rkind = {"1:1": ("unique", "unique"), "1:N": ("unique", "dup"), "N:M": ("dup", "dup"), "none": ("dup", "high"),
                    "all": ("small", "small"), "skew": ("few7", "skew"), "null_left": ("dup", "dup"), "null_right": ("dup", "dup")}[shape]
    def tbl(n, kind, all_null):
        mask = np.ones(n, bool) if all_null else rng.random(n) < 0.05
        t = pa.table({"k": pa.array(keys(n, kind), pa.int64(), mask=mask), "row": pa.array(np.arange(n, dtype=np.int64))})
        return sorted_by(t, ["k"])
    n_l, n_r = (200, 20_000) if shape == "skew" else (3_000, 2_000)
    if jt == R.RIGHT_OUTER and shape == "skew":   # the skewed side is the build side
        n_l, n_r, lkind, rkind = n_r, n_l, rkind, lkind
    left, right = tbl(n_l, lkind, shape == "null_left"), tbl(n_r, rkind, shape == "null_right")
    types = [P.INT64, P.INT64]
    case(cb, left, types, right, types, [0], [0], jt)


# ---- sizes ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_l,n_r", [(0, 500), (500, 0), (0, 0), (1, 500), (500, 1), (1, 1), (1, 0), (0, 1)])
@pytest.mark.parametrize("jt", JTS)
def test_empty_and_one_row(cb, n_l, n_r, jt):
    """an empty or one-row side; the empty-side rules give every row of the other side NULL-extended, or nothing"""
    left, lt, right, rt = sorted_sides(n_l, n_r, ["i32", "s8"], n_l + 5, 3, spread=0.0)
    got, want, stats = case(cb, left, lt, right, rt, [0, 1], [0, 1], jt)
    assert stats["join_out_rows"] == want.num_rows


@pytest.mark.parametrize("jt", JTS)
def test_batches_and_chunks(cb, jt):
    """several input batches per side and a small chunkRows: probe-side outer output and FullOuter's unmatched build rows each leave in
    several batches of at most chunkRows rows"""
    P = cb.proto
    ks = ["k0", "k1"]
    left, lt = side(20_000, ["i64", "s32"], 1, 3000, spread=0.0)
    right, rt = side(16_000, ["i64", "s32"], 2, 6000, spread=0.0)     # about half the right keys match no left row
    left, right = sorted_by(left, ks), sorted_by(right, ks)
    cfg = {"spark.comet.b200.chunkRows": "2048"}
    plan = smj_plan(cb, P.scan(lt), lt, P.scan(rt), rt, [0, 1], [0, 1], jt)
    sizes = []
    with cb.native.Plan(plan, [left.to_batches(max_chunksize=7000), right.to_batches(max_chunksize=3000)], config=cfg, batch_size=1 << 22) as p:
        batches = []
        while True:
            b = p.execute()
            if b is None:
                break
            batches.append(b)
            sizes.append(b.num_rows)
        stats = p.stats()
    got = pa.Table.from_batches(batches)
    want = R.sort_merge_join_table(left, right, [0, 1], [0, 1], jt)
    partref.assert_tables_equal(got, want)
    got.validate(full=True)
    assert max(sizes) <= 2048
    build_n, probe_n = (20_000, 16_000) if jt == R.RIGHT_OUTER else (16_000, 20_000)
    assert stats["join_build_rows"] == build_n and stats["join_probe_rows"] == probe_n and stats["join_out_rows"] == want.num_rows
    if jt in OUTER:
        assert len(sizes) > 10
    if jt == R.FULL_OUTER:   # the unmatched right rows leave after the left-outer part, in batches of their own
        lo = R.sort_merge_join_table(left, right, [0, 1], [0, 1], R.LEFT_OUTER).num_rows
        cum = np.cumsum(sizes)
        assert lo in cum and (cum > lo).sum() >= 3


@pytest.mark.parametrize("jt", OUTER)
def test_aggregate_over_null_extended_columns(cb, jt):
    """a Partial HashAggregate fed by many join batches sums and counts a NULL-extended column of each side; the Final aggregate gives
    the numpy answer (the accumulator sees one layout in every batch)"""
    P = cb.proto
    left, lt, right, rt = sorted_sides(9_000, 7_000, ["i32"], 3, 4000, spread=0.0)
    j = smj_plan(cb, P.scan(lt), lt, P.scan(rt), rt, [0], [0], jt)
    n_l = len(lt)
    aggs = [P.agg_sum(P.bound(1, P.INT64), P.INT64), P.agg_count([P.bound(1, P.INT64)]),
            P.agg_sum(P.bound(n_l + 1, P.INT64), P.INT64), P.agg_count([P.bound(n_l + 1, P.INT64)])]
    partial = P.hash_agg(j, [], aggs, P.PARTIAL)
    with cb.native.Plan(partial, [left.to_batches(max_chunksize=2500), right.to_batches(max_chunksize=2000)],
                        config={"spark.comet.b200.chunkRows": "1024"}) as p:
        state = p.collect()
    st = [P.INT64, P.INT64, P.INT64, P.INT64]
    final = P.hash_agg(P.scan(st, source="shuffle"), [], [P.agg_sum(P.unbound("a", P.INT64), P.INT64), P.agg_count([P.unbound("b", P.INT64)]),
                                                          P.agg_sum(P.unbound("c", P.INT64), P.INT64), P.agg_count([P.unbound("d", P.INT64)])], P.FINAL)
    res, _ = collect(cb, final, [state])
    want = R.sort_merge_join_table(left, right, [0], [0], jt)
    lrow, rrow = want.column(1), want.column(n_l + 1)
    assert list(res.to_pylist()[0].values()) == [pc.sum(lrow).as_py(), lrow.length() - lrow.null_count,
                                                 pc.sum(rrow).as_py(), rrow.length() - rrow.null_count]
    assert lrow.null_count > 0 or rrow.null_count > 0


# ---- NULL-extended columns in every stored layout ---------------------------------------------------------------------------------------
def layout_table(n, seed, key_dom):
    """a key k (int32) and one payload column per stored layout: bitmap booleans, decimal(9, 2) / decimal(18, 0) (8 bytes wide on a
    device table), decimal(38, 4), dictionary strings with 1 / 2 / 4-byte codes"""
    import comet_b200.proto as P
    rng = np.random.default_rng(seed)
    m = lambda: rng.random(n) < 0.1
    ids = rng.integers(0, len(WORDS), n)
    cols = {"k": pa.array(np.sort(rng.integers(0, key_dom, n)).astype(np.int32)),
            "b": pa.array(rng.random(n) < 0.5, mask=m()),
            "d9": _dec(rng.integers(-10**8, 10**8, n), 9, 2, m()),
            "d18": _dec(rng.integers(-10**17, 10**17, n), 18, 0, m()),
            "d38": _dec(_words([int(v) * 10**20 + 7 for v in rng.integers(-10**17, 10**17, n)]), 38, 4, m()),
            "s8": pa.DictionaryArray.from_arrays(pa.array(ids, pa.int8(), mask=m()), pa.array(WORDS)),
            "s16": pa.DictionaryArray.from_arrays(pa.array(ids, pa.int16(), mask=m()), pa.array(WORDS)),
            "s32": pa.DictionaryArray.from_arrays(pa.array(ids, pa.int32(), mask=m()), pa.array(WORDS))}
    types = [P.INT32, P.BOOL, P.DECIMAL(9, 2), P.DECIMAL(18, 0), P.DECIMAL(38, 4), P.STRING, P.STRING, P.STRING]
    return pa.table(cols), types


@pytest.mark.parametrize("source", ["stream", "device"])
@pytest.mark.parametrize("sizes", [(6000, 5000), (0, 5000), (6000, 0)])
@pytest.mark.parametrize("jt", OUTER)
def test_null_extended_layouts(cb, jt, sizes, source):
    """bitmap booleans, 8- and 16-byte decimals and 1 / 2 / 4-byte dictionary codes NULL-extended; with an empty side a column has
    no source batch (the type's Arrow layout, an empty dictionary).  Exported and validated as Arrow."""
    left, lt = layout_table(sizes[0], 1, 3000)
    right, rt = layout_table(sizes[1], 2, 3000)
    li = ri = None
    if source == "device":
        if not (sizes[0] and sizes[1]):
            pytest.skip("a device table has rows")
        li = [device_table(cb, left, lt, dec8=["d9", "d18"])]
        ri = [device_table(cb, right, rt, dec8=["d9", "d18"])]
    case(cb, left, lt, right, rt, [0], [0], jt, config={"spark.comet.b200.chunkRows": "3000"}, linputs=li, rinputs=ri)


@pytest.mark.parametrize("jt", OUTER)
def test_null_extended_byte_booleans_and_int32_backed_int8(cb, tmp_path, jt):
    """booleans a Projection writes one byte per row, and int8 / decimal(7, 2) a NativeScan reads from Parquet INT32, NULL-extended"""
    P = cb.proto
    n = 6000
    a, b = parquet_table(n, 41), parquet_table(n, 42)
    names = ["i32", "i8", "d7", "sd", "row"]
    a = {k: a[k] for k in names}
    b = {k: b[k] for k in names}
    for cols, seed in ((a, 1), (b, 2)):   # a sorted key column shared by both files
        cols["i32"] = (pa.array(np.sort(np.random.default_rng(seed).integers(0, 4000, n)).astype(np.int32)), P.INT32)
    pa_path, pb_path = str(tmp_path / "a.parquet"), str(tmp_path / "b.parquet")
    write_parquet(pa_path, a, True)
    write_parquet(pb_path, b, True)
    scan_l, types = scan_of(cb, a, names, pa_path)
    scan_r, _ = scan_of(cb, b, names, pb_path)
    # right: (i32, i8, d7, sd, row, row > 3000 as a byte-per-row boolean)
    proj_r = P.projection(scan_r, [P.bound(i, t) for i, t in enumerate(types)] + [P.gt(P.bound(4, types[4]), P.literal(3000, types[4]))])
    rtypes = types + [P.BOOL]
    plan = smj_plan(cb, scan_l, types, proj_r, rtypes, [0], [0], jt)
    got, _ = collect(cb, plan, [], config={"spark.comet.b200.chunkRows": "2500"})
    ltbl, rtbl = expected_table(a, names), expected_table(b, names)
    rtbl = rtbl.append_column("gt", pc.greater(rtbl.column("row"), pa.scalar(3000, rtbl.column("row").type)))
    want = R.sort_merge_join_table(ltbl, rtbl, [0], [0], jt)
    check(got, want)
    got.validate(full=True)


# ---- strings -------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("jt", JTS)
def test_string_dictionaries_differ_between_sides(cb, jt):
    """each side's batches carry their own dictionary, with strings the other side lacks"""
    P = cb.proto
    def batches(k, per, words, seed):
        r = np.random.default_rng(seed)
        out = []
        for b in range(k):
            codes = np.sort(r.integers(0, len(words), per))
            s = pa.DictionaryArray.from_arrays(pa.array(codes, pa.int16(), mask=r.random(per) < 0.1), pa.array(words))
            out.append(pa.record_batch([s, pa.array(np.arange(b * per, (b + 1) * per, dtype=np.int64))], names=["s", "v"]))
        return out
    lb = batches(5, 2000, sorted(WORDS[:70] + [f"only-left-{i}" for i in range(10)]), 1)
    rb = batches(4, 1500, sorted(WORDS[30:] + [f"only-right-{i}" for i in range(10)]), 2)
    plainify = lambda bs: pa.Table.from_batches([pa.record_batch([b.column(0).dictionary_decode(), b.column(1)], names=["s", "v"]) for b in bs])
    types = [P.STRING, P.INT64]
    case(cb, plainify(lb), types, plainify(rb), types, [0], [0], jt, linputs=[lb], rinputs=[rb], config={"spark.comet.b200.chunkRows": "4000"})


@pytest.mark.parametrize("jt", JTS)
def test_repeated_dictionary_values(cb, jt):
    """device-table dictionaries that hold a value more than once: equal strings match whichever code they have"""
    P = cb.proto
    dict_l, dict_r = ["x", "y", "x", "z", "y", "", ""], ["y", "y", "q", "x", "", "z", "x"]
    def table(n, d, seed):
        r = np.random.default_rng(seed)
        codes = r.integers(0, len(d), n).astype(np.int32)
        tbl = pa.table({"s": pa.DictionaryArray.from_arrays(pa.array(codes, mask=r.random(n) < 0.1), pa.array(d)),
                        "v": pa.array(np.arange(n, dtype=np.int64))})
        return sorted_by(tbl, ["s"])
    types = [P.STRING, P.INT64]
    left, right = table(3000, dict_l, 1), table(2500, dict_r, 2)
    case(cb, left, types, right, types, [0], [0], jt, linputs=[device_table(cb, left, types)], rinputs=[device_table(cb, right, types)],
         config={"spark.comet.b200.chunkRows": "2048"})


# ---- the Comet shape -----------------------------------------------------------------------------------------------------------------------
def sorted_scan(cb, types, keys):
    P = cb.proto
    return P.sort(P.scan(types), [P.sort_order(P.bound(k, types[k])) for k in keys])


@pytest.mark.parametrize("jt", JTS)
def test_scan_sort_smj_sort_scan(cb, jt):
    """Scan -> Sort -> SortMergeJoin <- Sort <- Scan over unsorted inputs: the reference's answer over the sorted sides"""
    left, lt = side(15_000, ["i64", "s16"], 11, 2000, spread=0.0)
    right, rt = side(10_000, ["i64", "s16"], 12, 2000, spread=0.0)
    plan = smj_plan(cb, sorted_scan(cb, lt, [0, 1]), lt, sorted_scan(cb, rt, [0, 1]), rt, [0, 1], [0, 1], jt)
    got, _ = collect(cb, plan, [left.to_batches(max_chunksize=4000), right.to_batches(max_chunksize=4000)],
                     config={"spark.comet.b200.chunkRows": "8192"})
    want = R.sort_merge_join_table(sorted_by(left, ["k0", "k1"]), sorted_by(right, ["k0", "k1"]), [0, 1], [0, 1], jt)
    check(got, want)


@pytest.mark.parametrize("outer_jt", [R.INNER, R.LEFT_OUTER, R.FULL_OUTER])
@pytest.mark.parametrize("inner_jt", [R.INNER, R.LEFT_OUTER, R.RIGHT_OUTER])
def test_smj_over_smj(cb, inner_jt, outer_jt):
    """an SMJ over an SMJ on the same key with no Sort between, as Spark plans it from the first join's output ordering"""
    P = cb.proto
    a, at = side(6000, ["i32"], 21, 1500, spread=0.0)
    b, bt = side(5000, ["i32"], 22, 1500, spread=0.0)
    c, ct = side(4000, ["i32"], 23, 1500, spread=0.0)
    a, b, c = sorted_by(a, ["k0"]), sorted_by(b, ["k0"]), sorted_by(c, ["k0"])
    j1 = smj_plan(cb, P.scan(at), at, P.scan(bt), bt, [0], [0], inner_jt)
    key = 0 if inner_jt != R.RIGHT_OUTER else len(at)      # the key column whose order the first join keeps
    jtypes = at + bt
    j2 = smj_plan(cb, j1, jtypes, P.scan(ct), ct, [key], [0], outer_jt)
    got, _ = collect(cb, j2, [a.to_batches(max_chunksize=2000), b.to_batches(max_chunksize=2000), c.to_batches(max_chunksize=2000)],
                     config={"spark.comet.b200.chunkRows": "4096"})
    ab = R.sort_merge_join_table(a, b, [0], [0], inner_jt)
    check(got, R.sort_merge_join_table(ab, c, [key], [0], outer_jt))


@pytest.mark.parametrize("jt", [R.INNER, R.LEFT_OUTER, R.FULL_OUTER])
def test_partial_final_aggregate_above(cb, jt):
    """Sort -> SMJ -> Projection -> Partial -> Final, grouped by a string of the left side, summing a right-side payload"""
    P = cb.proto
    left, lt = side(20_000, ["i32"], 31, 5000, spread=0.0)
    right, rt = side(15_000, ["i32"], 32, 5000, spread=0.0)
    j = smj_plan(cb, sorted_scan(cb, lt, [0]), lt, sorted_scan(cb, rt, [0]), rt, [0], [0], jt)
    n_l = len(lt)
    proj = P.projection(j, [P.bound(3, P.STRING), P.bound(n_l + 1, P.INT64)])
    partial = P.hash_agg(proj, [P.bound(0, P.STRING)], [P.agg_sum(P.bound(1, P.INT64), P.INT64), P.agg_count([P.bound(1, P.INT64)])], P.PARTIAL)
    with cb.native.Plan(partial, [left.to_batches(max_chunksize=6000), right.to_batches(max_chunksize=6000)],
                        config={"spark.comet.b200.chunkRows": "8192"}) as p:
        state = p.collect()
    final = P.hash_agg(P.scan([P.STRING, P.INT64, P.INT64], source="shuffle"), [P.bound(0, P.STRING)],
                       [P.agg_sum(P.unbound("s", P.INT64), P.INT64), P.agg_count([P.unbound("c", P.INT64)])], P.FINAL)
    res, _ = collect(cb, final, [state])
    want = R.sort_merge_join_table(sorted_by(left, ["k0"]), sorted_by(right, ["k0"]), [0], [0], jt)
    exp = {}
    for g, v in zip(want.column(3).to_pylist(), want.column(n_l + 1).to_pylist()):
        s, c = exp.get(g, (None, 0))
        exp[g] = (s if v is None else (s or 0) + v, c + (v is not None))
    got = {r["col_0"]: (r["col_1"], r["col_2"]) for r in res.to_pylist()}
    assert got == exp


@pytest.mark.parametrize("jt", JTS)
def test_device_tables(cb, jt):
    """device columns on both sides, 8-byte decimals on the right, chunkRows below the tables"""
    names = ["d18", "s8", "i32"]
    left, lt, right, rt = sorted_sides(12_000, 9_000, names, 5, 2000)
    dl = device_table(cb, left, lt)
    dr = device_table(cb, right, rt, dec8=["k0"])
    case(cb, left, lt, right, rt, [0, 1, 2], [0, 1, 2], jt, linputs=[dl], rinputs=[dr], config={"spark.comet.b200.chunkRows": "5120"})


@pytest.mark.parametrize("jt", JTS)
def test_native_scan(cb, tmp_path, jt):
    """both sides NativeScans of Parquet files, sorted by a Sort above each scan"""
    P = cb.proto
    n = 6000
    a, b = parquet_table(n, 51), parquet_table(n, 52)
    names = ["i16", "d12", "sd", "row"]
    pa_path, pb_path = str(tmp_path / "a.parquet"), str(tmp_path / "b.parquet")
    write_parquet(pa_path, {k: a[k] for k in names}, False)
    write_parquet(pb_path, {k: b[k] for k in names}, False)
    scan_l, types = scan_of(cb, a, names, pa_path)
    scan_r, _ = scan_of(cb, b, names, pb_path)
    order = lambda s: P.sort(s, [P.sort_order(P.bound(0, types[0])), P.sort_order(P.bound(3, types[3]))])
    plan = smj_plan(cb, order(scan_l), types, order(scan_r), types, [0], [0], jt)
    got, _ = collect(cb, plan, [], config={"spark.comet.b200.chunkRows": "2500"})
    ltbl, rtbl = sorted_by(expected_table(a, names), ["i16", "row"]), sorted_by(expected_table(b, names), ["i16", "row"])
    check(got, R.sort_merge_join_table(ltbl, rtbl, [0], [0], jt))


# ---- cross-operator equality ---------------------------------------------------------------------------------------------------------------
def test_inner_smj_is_the_inner_hash_join(cb):
    P = cb.proto
    left, lt, right, rt = sorted_sides(15_000, 10_000, ["i64", "s32", "d38"], 61, 800)
    ks = [0, 1, 2]
    inputs = lambda: [left.to_batches(max_chunksize=5000), right.to_batches(max_chunksize=4000)]
    smj, _ = collect(cb, smj_plan(cb, P.scan(lt), lt, P.scan(rt), rt, ks, ks, R.INNER), inputs())
    hj, _ = collect(cb, P.hash_join(P.scan(lt), P.scan(rt), [P.bound(i, lt[i]) for i in ks], [P.bound(i, rt[i]) for i in ks], P.INNER,
                                    P.BUILD_RIGHT), inputs())
    assert smj.num_rows > 0
    partref.assert_tables_equal(smj, hj)
