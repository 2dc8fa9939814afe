"""GPU: the row operators fed by each other's output -- Sort over HashJoin, HashJoin over Sort / TopK, HashJoin over HashJoin,
ShuffleWriter(HashPartitioning) over HashJoin and Sort, HashAggregate over Sort and HashJoin, and Sort / TopK / join build /
ShuffleWriter over a Partial aggregate that migrates from dense to hash.  The expected output of a stack is the single-operator
references composed (tests/joinref.py, sortref.py, partref.py, aggref.py).  Where the operators fix the order (join output order,
Sort ties in input order, the TopK candidate rule) every column is compared bit-exact and in order; where it is open (aggregate
output, a join built on aggregate state) the rows are compared as a multiset.  Every test also checks the counters that prove the
intended path ran, and that the lower operator emitted more than one batch, so the upper one had to concatenate or remap."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import aggref as A
import exprs as E
import joinref as J
import partref
import sortref as S
from test_gpu_join import side
from test_gpu_partition_layouts import WORDS, _dec, device_table, expected_table, make_values, parquet_table, scan_of, write_parquet

pytestmark = pytest.mark.gpu

JT = {"inner": 0, "left_semi": 4, "left_anti": 5}
MODES = [("inner", False), ("inner", True), ("left_semi", False), ("left_anti", False)]
CHUNK = 2048


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def config(chunk_rows=CHUNK, **extra):
    return {"spark.comet.b200.chunkRows": str(chunk_rows), **{k: str(v) for k, v in extra.items()}}


def run(cb, plan, inputs, cfg=None, batch_size=1 << 22):
    """(batches, the partition starts that came with each, counters): every batch of cb200_execute"""
    batches, starts = [], []
    with cb.native.Plan(plan, inputs, config=cfg, batch_size=batch_size) as p:
        while True:
            b = p.execute()
            if b is None:
                break
            batches.append(b)
            starts.append(p.partition_starts())
        return batches, starts, p.stats()


def plain_table(batches):
    """the batches as one table, dictionaries spelled out (each batch may carry its own dictionary)"""
    if not batches:
        return None
    return pa.concat_tables([pa.table([partref.plain(c) for c in b.columns], names=b.schema.names) for b in batches])


def check(batches, want):
    """the batches, concatenated, equal `want` bit-exact and in order"""
    if want.num_rows == 0:
        assert sum(b.num_rows for b in batches) == 0
        return
    partref.assert_tables_equal(plain_table(batches), want)


def canonical(t):
    """t's rows in the order of all its columns: equal multisets of rows give equal tables"""
    return S.sort_table(t, [(i, False, True) for i in range(t.num_columns)])


def sort_plan(P, child, types, keys, fetch=None, skip=None):
    return P.sort(child, [P.sort_order(P.bound(i, types[i]), d, nf) for i, d, nf in keys], fetch=fetch, skip=skip)


def join_plan(P, lchild, ltypes, rchild, rtypes, lk, rk, jt, build_left=False):
    return P.hash_join(lchild, rchild, [P.bound(i, ltypes[i]) for i in lk], [P.bound(i, rtypes[i]) for i in rk], JT[jt],
                       P.BUILD_LEFT if build_left else P.BUILD_RIGHT)


def out_types(lt, rt, jt):
    return lt + rt if jt == "inner" else lt


def replaced_dicts(tbl, cols, chunk, seed):
    """tbl as record batches of `chunk` rows in which each dictionary column named in `cols` carries its own shuffled dictionary: the
    dictionary is replaced between batches, the values stay"""
    rng = np.random.default_rng(seed)
    out = []
    for b in tbl.to_batches(max_chunksize=chunk):
        arrays = []
        for name, a in zip(b.schema.names, b.columns):
            if name in cols:
                d = a.dictionary.to_pylist()
                perm = rng.permutation(len(d))
                inv = np.argsort(perm)                                     # old code -> new code
                idx = a.indices
                codes = inv[np.asarray(idx.fill_null(0))].astype(idx.type.to_pandas_dtype())
                a = pa.DictionaryArray.from_arrays(pa.array(codes, idx.type, mask=np.asarray(idx.is_null())), pa.array([d[i] for i in perm]))
            arrays.append(a)
        out.append(pa.record_batch(arrays, names=b.schema.names))
    return out


def cut_inside_run(table, keys, fetch):
    """rows fetch - 1 and fetch of the sorted table tie on every key"""
    srt = S.sort_table(table, keys)
    if srt.num_rows <= fetch:
        return False
    ranks = [S.key_ranks(srt.column(c), d, nf) for c, d, nf in keys]
    return all(r[fetch - 1] == r[fetch] for r in ranks)


# ---- Sort over HashJoin -------------------------------------------------------------------------------------------------------------------
def sort_join_case(n_l, n_r, jt, build_left, seed=1):
    """both sides keyed on k0 (int32) with a boolean k1 (bitmaps with NULLs), payloads row, pf, ps; the probe side's ps dictionary is
    replaced between its batches.  Sort keys: a boolean of each half, then the probe half's string."""
    left, lt = side(n_l, ["i32", "b"], seed, max(n_r // 2, 1))
    right, rt = side(n_r, ["i32", "b"], seed + 50, max(n_r // 2, 1))
    li = replaced_dicts(left, {"ps"}, 1500, seed) if not build_left else left.to_batches(max_chunksize=1000)
    ri = replaced_dicts(right, {"ps"}, 1000, seed) if build_left else right.to_batches(max_chunksize=1000)
    if jt == "inner":
        keys = [(1, False, True), (6, True, False), (9 if build_left else 4, True, True)]
    else:
        keys = [(1, True, False), (4, False, True)]
    return left, lt, right, rt, [li or left, ri or right], keys


@pytest.mark.parametrize("fetch,skip", [(None, None), (700, None), (900, 150)])
@pytest.mark.parametrize("jt,build_left", MODES)
def test_sort_over_join(cb, jt, build_left, fetch, skip):
    """a full sort and a TopK (fetch < chunkRows: candidates merged across join output batches, cut inside a run of equal keys) over
    the join's output; ties keep join output order"""
    P = cb.proto
    left, lt, right, rt, inputs, keys = sort_join_case(6000, 3000, jt, build_left)
    j = join_plan(P, P.scan(lt), lt, P.scan(rt), rt, [0], [0], jt, build_left)
    joined, _, _ = run(cb, j, inputs, config())
    want_join = J.join_table(left, right, [0], [0], jt, build_left)
    check(joined, want_join)
    assert len(joined) >= 2 and max(b.num_rows for b in joined) <= CHUNK
    if fetch is not None:
        assert cut_inside_run(want_join, keys, fetch)
    got, _, stats = run(cb, sort_plan(P, j, out_types(lt, rt, jt), keys, fetch, skip), inputs, config())
    want = S.sort_table(want_join, keys, fetch, skip)
    check(got, want)
    S.assert_sorted(plain_table(got), keys)
    assert len(got) == 1
    assert stats["join_out_rows"] == want_join.num_rows and stats["join_probe_rows"] == (right if build_left else left).num_rows
    assert stats["sort_passes"] > 0 and stats["sort_rows"] >= want_join.num_rows


@pytest.mark.parametrize("n_l,n_r", [(0, 50), (50, 0), (1, 50), (50, 1), (1, 1), (0, 0)])
def test_sort_over_join_sizes(cb, n_l, n_r):
    """0 and 1 row on each side: inner and semi joins of an empty side give nothing to sort, an anti join every probe row"""
    P = cb.proto
    for jt, build_left in MODES:
        left, lt, right, rt, inputs, keys = sort_join_case(n_l, n_r, jt, build_left, seed=n_l + 7 * n_r + 3)
        j = join_plan(P, P.scan(lt), lt, P.scan(rt), rt, [0], [0], jt, build_left)
        for fetch in (None, 1):
            got, _, stats = run(cb, sort_plan(P, j, out_types(lt, rt, jt), keys, fetch), inputs, config())
            want_join = J.join_table(left, right, [0], [0], jt, build_left)
            check(got, S.sort_table(want_join, keys, fetch))
            assert stats["join_out_rows"] == want_join.num_rows


def test_sort_over_join_hand_off(cb):
    """the top of Sort over an inner join read through cb200_execute in spark.comet.batchSize slices and through
    cb200_execute_device with the reported value_width"""
    from test_gpu_scan_export import assert_device_matches, device_batches
    P = cb.proto
    left, lt, right, rt, inputs, keys = sort_join_case(5000, 2500, "inner", False, seed=9)
    plan = sort_plan(P, join_plan(P, P.scan(lt), lt, P.scan(rt), rt, [0], [0], "inner"), lt + rt, keys)
    want = S.sort_table(J.join_table(left, right, [0], [0], "inner"), keys)
    for bs in (1000, 4096):
        got, _, _ = run(cb, plan, inputs, config(), batch_size=bs)
        assert len(got) == (want.num_rows + bs - 1) // bs
        check(got, want)
    assert_device_matches(device_batches(cb, plan, inputs, config()), want)


# ---- HashJoin over Sort / TopK ----------------------------------------------------------------------------------------------------------
def sorted_sides(seed):
    """left: a TopK input (stream, one key s16 + i32); right: a full sort input whose s16 key dictionary is replaced between batches"""
    left, lt = side(4000, ["s16", "i32"], seed, 300)
    right, rt = side(5000, ["s16", "i32"], seed + 1, 300)
    return left, lt, left.to_batches(max_chunksize=1000), right, rt, replaced_dicts(right, {"k0"}, 1000, seed)


@pytest.mark.parametrize("jt,build_left", MODES)
def test_join_over_sort(cb, jt, build_left):
    """one side a full Sort (one batch above chunkRows whose string key carries the dictionary the concatenation made), the other a
    TopK; joined on the string key"""
    P = cb.proto
    left, lt, li, right, rt, ri = sorted_sides(21)
    lkeys, rkeys = [(1, True, False), (2, False, True)], [(0, False, True), (2, True, True)]
    ls, rs = sort_plan(P, P.scan(lt), lt, lkeys, fetch=1500), sort_plan(P, P.scan(rt), rt, rkeys)
    sorted_r, _, _ = run(cb, rs, [ri], config())
    assert len(sorted_r) == 1 and sorted_r[0].num_rows == right.num_rows > CHUNK
    got, _, stats = run(cb, join_plan(P, ls, lt, rs, rt, [0], [0], jt, build_left), [li, ri], config())
    want = J.join_table(S.sort_table(left, lkeys, 1500), S.sort_table(right, rkeys), [0], [0], jt, build_left)
    check(got, want)
    assert want.num_rows > 0 and stats["join_out_rows"] == want.num_rows
    assert stats["join_build_rows"] == (1500 if build_left else right.num_rows)


@pytest.mark.parametrize("empty", ["left", "right"])
@pytest.mark.parametrize("fetch,skip", [(0, None), (None, 5000), (300, 400)])
def test_join_over_empty_sort(cb, empty, fetch, skip):
    """a Sort that emits nothing (fetch = 0, skip at or past its rows) on either side: inner and semi joins give nothing, an anti join
    every probe row"""
    P = cb.proto
    left, lt, li, right, rt, ri = sorted_sides(31)
    right = right.slice(0, 4000)
    ri = replaced_dicts(right, {"k0"}, 1000, 31)
    keys = [(0, False, True), (2, False, True)]
    lf, lsk = (fetch, skip) if empty == "left" else (None, None)
    rf, rsk = (fetch, skip) if empty == "right" else (None, None)
    ls, rs = sort_plan(P, P.scan(lt), lt, keys, lf, lsk), sort_plan(P, P.scan(rt), rt, keys, rf, rsk)
    for jt, build_left in MODES:
        got, _, stats = run(cb, join_plan(P, ls, lt, rs, rt, [0], [0], jt, build_left), [li, ri], config())
        want = J.join_table(S.sort_table(left, keys, lf, lsk), S.sort_table(right, keys, rf, rsk), [0], [0], jt, build_left)
        check(got, want)
        if jt == "left_anti" and empty == "right":
            assert want.num_rows == left.num_rows
        assert stats["join_out_rows"] == want.num_rows


# ---- HashJoin over HashJoin ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("outer", ["build_half", "probe_half", "anti_empty"])
@pytest.mark.parametrize("jt", ["inner", "left_semi", "left_anti"])
def test_join_over_join(cb, jt, outer):
    """the outer join's probe side is an inner join's output, with no Projection between them: keyed on a string of the inner build
    half (gathered, carrying the inner build dictionary) or on a column of its probe half (no NULLs, against a build key with NULLs);
    or the inner join is an anti join with an empty build side, whose raw probe batches (dictionaries replaced) reach the outer join"""
    P = cb.proto
    a, at = side(5000, ["i32", "s8"], 41, 1200)
    b, bt = side(0 if outer == "anti_empty" else 2400, ["i32", "s16"], 42, 1200)
    rng = np.random.default_rng(43)
    n_c = 1500
    c = pa.table({"s": pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, len(WORDS), n_c), pa.int32(), mask=rng.random(n_c) < 0.1),
                                                       pa.array(WORDS)),
                  "k": pa.array(rng.integers(0, 5000, n_c), pa.int64(), mask=rng.random(n_c) < 0.1),
                  "row": pa.array(np.arange(n_c, dtype=np.int64))})
    ct = [P.STRING, P.INT64, P.INT64]
    inner_jt = "left_anti" if outer == "anti_empty" else "inner"
    j1 = join_plan(P, P.scan(at), at, P.scan(bt), bt, [0], [0], inner_jt)
    j1t = out_types(at, bt, inner_jt)
    inputs = [replaced_dicts(a, {"ps"}, 1000, 44), b.to_batches(max_chunksize=1000) or b, c.to_batches(max_chunksize=500)]
    lk, rk = {"build_half": ([9], [0]), "probe_half": ([2], [1]), "anti_empty": ([4], [0])}[outer]
    inner_out, _, _ = run(cb, j1, inputs[:2], config())
    want1 = J.join_table(a, b, [0], [0], inner_jt)
    check(inner_out, want1)
    assert len(inner_out) >= 2
    got, _, stats = run(cb, join_plan(P, j1, j1t, P.scan(ct), ct, lk, rk, jt), inputs, config())
    want = J.join_table(want1, c, lk, rk, jt)
    check(got, want)
    assert 0 < want.num_rows < want1.num_rows or jt == "inner"
    assert stats["join_build_rows"] == b.num_rows + n_c and stats["join_out_rows"] == want1.num_rows + want.num_rows


# ---- ShuffleWriter over HashJoin and over Sort ------------------------------------------------------------------------------------------
def check_partitioned(oracle, got, starts, want, keys, n_parts):
    """each batch the partitioning of the reference's rows at the same place"""
    row0 = 0
    for b, st in zip(got, starts):
        want_starts, _, part = partref.partition(oracle, want.slice(row0, b.num_rows), keys, n_parts)
        assert st == want_starts, row0
        partref.assert_tables_equal(plain_table([b]), part)
        row0 += b.num_rows
    assert row0 == want.num_rows


@pytest.mark.parametrize("as_int,n_l,n_r,chunk", [(True, 20_000, 600, 8192), (False, 200_000, 300, 65_536)])
def test_partition_over_join_and_sort(cb, oracle, tmp_path, as_int, n_l, n_r, chunk):
    """NativeScan (int8 stored as INT32, decimal(7, 2) as INT32 or FLBA, decimal(28, 2), dictionary string pages) joined on int8 with
    a device table (bitmap booleans, 8-byte decimal(18, 0), int16-index dictionary); keys: a gathered boolean, the INT32-backed
    int8, the 8-byte decimal and the dictionary strings.  The large case sorts far more than one 4096-row tile and partitions many
    1024-row blocks."""
    P = cb.proto
    names = ["i8", "d7", "d28", "sd", "row"]
    cols = parquet_table(n_l, 51)
    path = str(tmp_path / "l.parquet")
    write_parquet(path, {k: cols[k] for k in names}, as_int)
    scan, lt = scan_of(cb, cols, names, path)
    rcols = make_values(n_r, 52)
    right = pa.table({k: rcols[k][0] for k in ["i8", "b", "d18", "s16", "row"]})
    rt = [rcols[k][1] for k in right.column_names]
    j = join_plan(P, scan, lt, P.scan(rt), rt, [0], [0], "inner")
    want_join = J.join_table(expected_table(cols, names), right, [0], [0], "inner")
    types = lt + rt
    sort_keys = [(7, False, True), (4, True, False), (9, False, False)]
    want_sort = S.sort_table(want_join, sort_keys)
    for keys, n_parts in (([6, 0, 7, 3], 200), ([8, 1, 2], 7)):
        hp = P.hash_partitioning([P.bound(k, types[k]) for k in keys], n_parts)
        got, starts, stats = run(cb, P.shuffle_writer(j, hp), [device_table(cb, right, rt, dec8=("d18",))], config(chunk))
        assert len(got) >= 2 and max(b.num_rows for b in got) <= chunk
        check_partitioned(oracle, got, starts, want_join, keys, n_parts)
        assert stats["join_out_rows"] == want_join.num_rows
        got, starts, stats = run(cb, P.shuffle_writer(sort_plan(P, j, types, sort_keys), hp), [device_table(cb, right, rt, dec8=("d18",))],
                                 config(chunk))
        assert len(got) == 1 and stats["sort_passes"] > 0
        check_partitioned(oracle, got, starts, want_sort, keys, n_parts)


# ---- HashAggregate over Sort and over HashJoin ------------------------------------------------------------------------------------------
def final_rows(table, key_types, aggs):
    cols = [A.pyvalues(table.column(i), t) for i, t in enumerate(key_types + [a.result_type() for a in aggs])]
    nk = len(key_types)
    out = {}
    for r in range(table.num_rows):
        key = tuple(c[r] for c in cols[:nk])
        assert key not in out, key
        out[key] = [c[r] for c in cols[nk:]]
    return out


def partial_then_final(cb, partial, inputs, cfg, key_types, aggs):
    """(Final result {key: [values]}, the Partial's counters)"""
    state, _, stats = run(cb, partial, inputs, cfg)
    assert state
    res, _, _ = run(cb, A.merge_plan(key_types, aggs), [state])
    return final_rows(plain_table(res), key_types, aggs), stats


def test_aggregate_over_sort(cb):
    """a Partial grouped by the Sort's key runs on the stream strategy (runs of equal keys); a string predicate over the Sort's
    concatenated dictionary filters its input; SUM / AVG(decimal), MIN / MAX, COUNT and a FILTER clause, then Final"""
    P = cb.proto
    rng = np.random.default_rng(61)
    n = 40_000
    tbl = pa.table({"g": pa.array(rng.integers(0, 600, n), pa.int64()),
                    "v": _dec(rng.integers(-10**9, 10**9, n), 12, 2, rng.random(n) < 0.1),
                    "s": pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, len(WORDS), n), pa.int16(), mask=rng.random(n) < 0.1),
                                                        pa.array(WORDS)),
                    "x": pa.array(rng.integers(-1000, 1000, n).astype(np.int32), mask=rng.random(n) < 0.1)})
    types = [P.INT64, P.DECIMAL(12, 2), P.STRING, P.INT32]
    batches = replaced_dicts(tbl, {"s"}, 5000, 62)
    srt = sort_plan(P, P.scan(types), types, [(0, False, True)])
    words = [w for w in WORDS if w.startswith("ab")]
    pred = P.in_(P.bound(2, P.STRING), [P.literal(w, P.STRING) for w in words])
    v, x = E.Col(1, P.DECIMAL(12, 2)), E.Col(3, P.INT32)
    aggs = [A.Agg("sum", v, P.DECIMAL(22, 2)), A.Agg("avg", v, P.DECIMAL(16, 6), sum_dt=P.DECIMAL(22, 2)), A.Agg("min", x, P.INT32),
            A.Agg("max", x, P.INT32), A.Agg("count", v), A.Agg("sum", v, P.DECIMAL(22, 2), filt=E.Cmp("gt", x, E.Lit(0, P.INT32)))]
    partial = P.hash_agg(P.filter_(srt, pred), [P.bound(0, P.INT64)], [a.proto() for a in aggs], P.PARTIAL)
    got, stats = partial_then_final(cb, partial, [batches], config(8192, **{"spark.comet.b200.streamAgg.minRows": 0}), [P.INT64], aggs)
    assert stats["agg_strategies"] & cb.native.AGG_STREAM and stats["sort_passes"] > 0
    kept = tbl.filter(pc.is_in(partref.plain(tbl.column("s")), value_set=pa.array(words)).fill_null(False))
    want = A.aggregate(kept, types, [0], aggs)
    assert got == want and len(want) > 100


@pytest.mark.parametrize("shape", ["dense_bool", "table"])
def test_aggregate_over_join(cb, shape):
    """an aggregate pipeline fed by an inner join: dense, grouped by a gathered boolean, or the key table over keys of both halves"""
    P = cb.proto
    left, lt = side(8000, ["i32", "b", "d9"], 71, 1500)
    right, rt = side(3000, ["i32", "s16"], 72, 1500)
    types = lt + rt                                       # 0 k0, 1 b, 2 d9, 3 row, 4 pf, 5 ps | 6 k0, 7 s16, 8 row, 9 pf, 10 ps
    d = E.Col(2, P.DECIMAL(9, 2))
    aggs = [A.Agg("sum", d, P.DECIMAL(19, 2)), A.Agg("avg", d, P.DECIMAL(13, 6), sum_dt=P.DECIMAL(19, 2)), A.Agg("min", d, P.DECIMAL(9, 2)),
            A.Agg("max", E.Col(8, P.INT64), P.INT64), A.Agg("count", E.Col(9, P.DOUBLE)),
            A.Agg("count", d, filt=E.Cmp("gt", E.Col(3, P.INT64), E.Lit(4000, P.INT64)))]
    key_cols = [1] if shape == "dense_bool" else [1, 7, 5]
    j = join_plan(P, P.scan(lt), lt, P.scan(rt), rt, [0], [0], "inner")
    partial = P.hash_agg(j, [P.bound(k, types[k]) for k in key_cols], [a.proto() for a in aggs], P.PARTIAL)
    inputs = [replaced_dicts(left, {"ps"}, 2000, 73), right.to_batches(max_chunksize=1000)]
    got, stats = partial_then_final(cb, partial, inputs, config(**{"spark.comet.b200.streamAgg.minRows": -1}), [types[k] for k in key_cols], aggs)
    assert stats["agg_strategies"] & (cb.native.AGG_DENSE if shape == "dense_bool" else cb.native.AGG_TABLE)
    want_join = J.join_table(left, right, [0], [0], "inner")
    assert stats["join_out_rows"] == want_join.num_rows > 4 * CHUNK
    assert got == A.aggregate(want_join, types, key_cols, aggs)


# ---- row operators over a Partial aggregate that migrates from dense to hash ------------------------------------------------------------
def migrating(cb):
    """A Partial grouped by (k, b): k's dictionary has 6 values in the first batches (dense) and 300 later (hash), b is a nullable
    boolean; SUM(v decimal(12, 2)) and COUNT(v).  The dense state leaves as a host-resident flush (booleans become a bitmap on the
    device), the hash state as kernel output (booleans one byte per row).  -> (plan, input batches, state types, standalone state
    batches)"""
    P = cb.proto
    rng = np.random.default_rng(81)
    small = [f"s{i}" for i in range(6)]
    big = [f"b{i:03d}" for i in range(294)] + small
    batches = []
    for bi in range(10):
        names, n = (small if bi < 4 else big), 3000
        k = pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, len(names), n).astype(np.int32)), pa.array(names))
        b = pa.array(rng.random(n) < 0.5, mask=rng.random(n) < 0.1)
        v = _dec(rng.integers(-10**9, 10**9, n), 12, 2, rng.random(n) < 0.3)
        batches.append(pa.record_batch([k, b, v], names=["k", "b", "v"]))
    dt = P.DECIMAL(12, 2)
    plan = P.hash_agg(P.scan([P.STRING, P.BOOL, dt]), [P.bound(0, P.STRING), P.bound(1, P.BOOL)],
                      [P.agg_sum(P.bound(2, dt), P.DECIMAL(22, 2)), P.agg_count([P.bound(2, dt)])], P.PARTIAL)
    state_types = [P.STRING, P.BOOL, P.DECIMAL(22, 2), P.BOOL, P.INT64]
    state, _, stats = run(cb, plan, [batches], config(3000))
    assert stats["agg_strategies"] & cb.native.AGG_MIGRATED and len(state) >= 2
    return plan, batches, state_types, [plain_table([s]) for s in state]


STATE_KEYS = [(1, False, True), (3, True, False), (0, False, True), (2, True, True), (4, False, False)]   # b, is_empty, then the rest


@pytest.mark.parametrize("fetch,skip", [(None, None), (40, None), (60, 7)])
def test_sort_over_migrated_aggregate(cb, fetch, skip):
    """a full Sort (concatenates the flush and the hash output) and a TopK (merges candidates of both) keyed on the boolean group key
    and the SUM state's is_empty flag; every state column is a key, so rows that tie are equal"""
    P = cb.proto
    plan, batches, types, state = migrating(cb)
    want = S.sort_table(pa.concat_tables(state), STATE_KEYS, fetch, skip)
    got, _, stats = run(cb, sort_plan(P, plan, types, STATE_KEYS, fetch, skip), [batches], config(3000))
    check(got, want)
    assert stats["agg_strategies"] & cb.native.AGG_MIGRATED and stats["sort_passes"] > 0


@pytest.mark.parametrize("jt", ["inner", "left_semi", "left_anti"])
def test_join_built_on_migrated_aggregate(cb, jt):
    """the join's build side is the migrated state, keyed on (k, b); its match order follows the build input order, which the hash
    strategy does not fix, so inner output is compared as a multiset (semi / anti keep probe order)"""
    P = cb.proto
    plan, batches, types, state = migrating(cb)
    rng = np.random.default_rng(82)
    n = 5000
    names = [f"b{i:03d}" for i in range(0, 294, 3)] + [f"s{i}" for i in range(6)] + ["zz"]
    probe = pa.table({"k": pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, len(names), n).astype(np.int8)), pa.array(names)),
                      "b": pa.array(rng.random(n) < 0.5, mask=rng.random(n) < 0.05), "row": pa.array(np.arange(n, dtype=np.int64))})
    pt = [P.STRING, P.BOOL, P.INT64]
    got, _, stats = run(cb, join_plan(P, P.scan(pt), pt, plan, types, [0, 1], [0, 1], jt), [probe.to_batches(max_chunksize=2000), batches],
                        config(3000))
    want = J.join_table(probe, pa.concat_tables(state), [0, 1], [0, 1], jt)
    assert want.num_rows > 0
    if jt == "inner":
        partref.assert_tables_equal(canonical(plain_table(got)), canonical(want))
    else:
        check(got, want)
    assert stats["join_build_rows"] == sum(s.num_rows for s in state)


def test_partition_over_migrated_aggregate(cb, oracle):
    """ShuffleWriter over the migrated state, batch by batch (the flush, then the hash output): each batch holds its standalone
    counterpart's rows, with the reference's partition starts and each row in its own partition"""
    P = cb.proto
    plan, batches, types, state = migrating(cb)
    for keys in ([1, 3], [0], [3, 0, 1]):
        hp = P.hash_partitioning([P.bound(k, types[k]) for k in keys], 7)
        got, starts, _ = run(cb, P.shuffle_writer(plan, hp), [batches], config(3000))
        assert len(got) == len(state)
        for b, st, want in zip(got, starts, state):
            out = plain_table([b])
            partref.assert_tables_equal(canonical(out), canonical(want))
            assert st == partref.partition(oracle, want, keys, 7)[0]
            pids = np.array([oracle.pmod(int(h), 7) for h in partref.key_hashes(oracle, out, keys)])
            assert (pids == np.searchsorted(np.array(st), np.arange(out.num_rows), side="right") - 1).all()
