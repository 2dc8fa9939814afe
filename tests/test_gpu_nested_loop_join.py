"""GPU: BroadcastNestedLoopJoin against the CPU reference (tests/nljref.py), bit-exact and in order, and the pairs its condition was
evaluated on (cb200_stats.join_cond_pairs).  Covers every accepted shape x the join-condition suite's conditions, no condition (cross
products, semi / anti / outer by build emptiness), sides of 0 / 1 / 500 rows, chunkRows at its minimum with one probe row's pairs across
slices and groups, a probe batch of more than 2^32 pairs under an aggregate, ANSI errors, stored layouts (device tables, NativeScan,
dictionary strings, 16-byte decimals, bitmap booleans) and compositions (the TPC-DS Q90 / Q28 cross join of single-row aggregates, the
multi-column NOT IN shape, a band join under an aggregate)."""
import numpy as np
import pyarrow as pa
import pytest

import exprs as E
import nljref as R
import strpred_ref as S
from joinref import INNER, LEFT_ANTI, LEFT_SEMI
from smjref import LEFT_OUTER, RIGHT_OUTER
from test_gpu_join import check, collect
from test_gpu_join_condition import NCOL, conditions, side
from test_gpu_partition_layouts import _dec, device_table, expected_table, parquet_table, scan_of, write_parquet

pytestmark = pytest.mark.gpu

JT = {INNER: 0, LEFT_OUTER: 1, RIGHT_OUTER: 2, LEFT_SEMI: 4, LEFT_ANTI: 5}
SHAPES = R.ACCEPTED
IDS = [f"{jt}-{'build_left' if bl else 'build_right'}" for jt, bl in SHAPES]


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def nlj_plan(cb, lchild, rchild, jt, cond, build_left=False):
    P = cb.proto
    return P.broadcast_nested_loop_join(lchild, rchild, JT[jt], P.BUILD_LEFT if build_left else P.BUILD_RIGHT,
                                        condition=cond.proto() if cond is not None else None)


def batches(t, chunk):
    return t.to_batches(max_chunksize=chunk) if t.num_rows else t


def run(cb, left, lt, right, rt, jt, cond, build_left=False, config=None, linputs=None, rinputs=None, chunk=4000):
    P = cb.proto
    plan = nlj_plan(cb, P.scan(lt), P.scan(rt), jt, cond, build_left)
    li = linputs if linputs is not None else [batches(left, chunk)]
    ri = rinputs if rinputs is not None else [batches(right, chunk)]
    got, stats = collect(cb, plan, li + ri, config)
    want = R.nlj_table(left, right, jt, cond, build_left)
    check(got, want)
    if got is not None:
        got.validate(full=True)
    assert stats["join_cond_pairs"] == R.candidate_count(left, right, cond), (stats["join_cond_pairs"], R.candidate_count(left, right, cond))
    assert stats["join_build_rows"] == (left if build_left else right).num_rows
    return got, want, stats


# ---- every accepted shape, every condition ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cond", list(conditions()))
@pytest.mark.parametrize("jt,build_left", SHAPES, ids=IDS)
def test_conditions(cb, jt, build_left, cond):
    left, lt = side(200, 1, 800)
    right, rt = side(120, 2, 800)
    run(cb, left, lt, right, rt, jt, conditions()[cond], build_left, chunk=64)


# ---- no condition, and the side sizes -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cond", [None, "lt_int"])
@pytest.mark.parametrize("n_l,n_r", [(a, b) for a in (0, 1, 500) for b in (0, 1, 500)])
@pytest.mark.parametrize("jt,build_left", SHAPES, ids=IDS)
def test_side_sizes(cb, jt, build_left, n_l, n_r, cond):
    """without a condition: the cross product for inner / outer joins; semi / anti by whether the build side is empty"""
    left, lt = side(n_l, 5, 3)
    right, rt = side(n_r, 6, 3)
    got, _, stats = run(cb, left, lt, right, rt, jt, conditions()[cond] if cond else None, build_left, chunk=200)
    if cond is None and jt in (INNER, LEFT_OUTER, RIGHT_OUTER) and n_l and n_r:
        assert got.num_rows == n_l * n_r
    build, probe = (left, right) if build_left else (right, left)
    no_output = build.num_rows == 0 and jt in (INNER, LEFT_SEMI)   # the probe side is never read
    assert stats["join_probe_rows"] == (0 if no_output else probe.num_rows)


def narrow(n, seed, lo=0, hi=40):
    import comet_b200.proto as P
    rng = np.random.default_rng(seed)
    return (pa.table({"a": pa.array(rng.integers(lo, hi, n).astype(np.int32), mask=rng.random(n) < 0.05), "row": pa.array(np.arange(n, dtype=np.int64))}),
            [P.INT32, P.INT64])


def uneven(t, sizes):
    """t cut into batches of the given sizes, cycling (a size of 0 gives an empty batch)"""
    whole = t.combine_chunks().to_batches()[0]
    out, at, i = [], 0, 0
    while at < t.num_rows:
        k = min(sizes[i % len(sizes)], t.num_rows - at)
        out.append(whole.slice(at, k))
        at += k
        i += 1
    return out


@pytest.mark.parametrize("n_probe,n_build", [(700, 1500), (2100, 300), (9, 1030)])
@pytest.mark.parametrize("cond", [None, "lt", "none_pass"])
@pytest.mark.parametrize("jt,build_left", SHAPES, ids=IDS)
def test_min_chunk_rows(cb, jt, build_left, n_probe, n_build, cond):
    """chunkRows 1024: with m above it one probe row's pairs span two slices and each group is one row; below it a group holds
    1024 / m rows and a probe batch several groups.  Probe batches of uneven sizes; output batches stay at most chunkRows rows."""
    import comet_b200.proto as P
    probe, pt = narrow(n_probe, 1)
    build, bt = narrow(n_build, 2)
    left, lt, right, rt = (build, bt, probe, pt) if build_left else (probe, pt, build, bt)
    c = {None: None, "lt": E.Cmp("lt", E.Col(0, P.INT32), E.Col(2, P.INT32)),
         "none_pass": E.Cmp("gt", E.Col(0, P.INT32), E.Lit(100, P.INT32))}[cond]
    sizes = [1, 333, 0, 77, 1024, 5]
    pin = [uneven(probe, sizes)]
    bin_ = [uneven(build, sizes[::-1])]
    got, _, _ = run(cb, left, lt, right, rt, jt, c, build_left, config={"spark.comet.b200.chunkRows": "1024"},
                    linputs=bin_ if build_left else pin, rinputs=pin if build_left else bin_)


# ---- above 2^32 pairs in one probe batch -----------------------------------------------------------------------------------------------
def band_sides(n_events, n_ranges, seed):
    rng = np.random.default_rng(seed)
    t = rng.integers(0, 10**9, n_events).astype(np.int64)
    lo = rng.integers(0, 10**9, n_ranges).astype(np.int64)
    hi = lo + rng.integers(1, 40_000, n_ranges)
    return t, lo, hi


def band_counts(t, lo, hi):
    """ranges [lo, hi) holding each t: #(lo <= t) - #(hi <= t), since lo < hi"""
    return np.searchsorted(np.sort(lo), t, side="right") - np.searchsorted(np.sort(hi), t, side="right")


def test_above_2_32_pairs_in_one_probe_batch(cb):
    """70 000 event times x 70 000 ranges: 4.9e9 pairs in one probe batch, inner band join under COUNT / SUM, then the same as LeftSemi"""
    P = cb.proto
    n = 70_000
    t, lo, hi = band_sides(n, n, 3)
    ev, rg = pa.table({"t": t}), pa.table({"lo": lo, "hi": hi})
    band = P.and_(P.gt_eq(P.bound(0, P.INT64), P.bound(1, P.INT64)), P.lt(P.bound(0, P.INT64), P.bound(2, P.INT64)))
    cnt = band_counts(t, lo, hi)
    j = P.broadcast_nested_loop_join(P.scan([P.INT64]), P.scan([P.INT64, P.INT64]), 0, P.BUILD_RIGHT, condition=band)
    agg = P.hash_agg(j, [], [P.agg_count([P.bound(0, P.INT64)]), P.agg_sum(P.bound(0, P.INT64), P.INT64)], P.PARTIAL)
    got, stats = collect(cb, agg, [ev.to_batches(), rg.to_batches()])
    row = list(got.to_pylist()[0].values())
    assert row[0] == int(cnt.sum()) and row[1] == int((t * cnt).sum()), (row, int(cnt.sum()))
    assert stats["join_cond_pairs"] == n * n and n * n > 2**32
    assert stats["join_probe_rows"] == n and stats["join_out_rows"] == int(cnt.sum())
    semi = P.broadcast_nested_loop_join(P.scan([P.INT64]), P.scan([P.INT64, P.INT64]), 4, P.BUILD_RIGHT, condition=band)
    got, stats = collect(cb, P.hash_agg(semi, [], [P.agg_count([P.bound(0, P.INT64)])], P.PARTIAL), [ev.to_batches(), rg.to_batches()])
    assert got.to_pylist()[0][got.column_names[0]] == int((cnt > 0).sum())
    assert stats["join_cond_pairs"] == n * n


# ---- ANSI errors --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("jt,build_left", SHAPES, ids=IDS)
def test_ansi_overflow_only_from_a_pair(cb, jt, build_left):
    """l.a + 1 overflows at INT32_MAX: ARITHMETIC_OVERFLOW once that row is in a pair, none when the other side is empty"""
    P = cb.proto
    cond = E.Cmp("gt", E.Arith("add", E.Col(0, P.INT32), E.Lit(1, P.INT32), P.INT32, E.ANSI), E.Col(1, P.INT32))
    t = [P.INT32]
    left = pa.table({"a": pa.array(np.r_[np.zeros(999), [2**31 - 1]].astype(np.int32))})
    right = pa.table({"b": pa.array(np.zeros(50, np.int32))})
    run(cb, left, t, right.slice(0, 0), t, jt, cond, build_left)     # no pair: no error (the empty-side rules)
    with pytest.raises(E.AnsiError):
        R.nlj_table(left, right, jt, cond, build_left)
    with pytest.raises(cb.native.CometB200Error) as ei:
        collect(cb, nlj_plan(cb, P.scan(t), P.scan(t), jt, cond, build_left), [left.to_batches(max_chunksize=4000), right.to_batches(max_chunksize=4000)])
    assert ei.value.error_class == "ARITHMETIC_OVERFLOW", str(ei.value)
    run(cb, left.slice(0, 999), t, right, t, jt, cond, build_left)   # without the row: every pair is fine


# ---- stored layouts -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("jt,build_left", SHAPES, ids=IDS)
def test_device_tables(cb, jt, build_left):
    """bitmap booleans and 8-byte decimals in the condition and the output"""
    P = cb.proto
    def tbl(n, seed):
        rng = np.random.default_rng(seed)
        m = lambda: rng.random(n) < 0.1
        return pa.table({"b": pa.array(rng.random(n) < 0.5, mask=m()), "m": _dec(rng.integers(-10**6, 10**6, n), 12, 2, m()),
                         "w": _dec(rng.integers(-10**6, 10**6, n), 18, 0, m())})
    types = [P.BOOL, P.DECIMAL(12, 2), P.DECIMAL(18, 0)]
    left, right = tbl(600, 1), tbl(400, 2)
    cond = E.Logic("or", E.Logic("and", E.Col(0, P.BOOL), E.Not(E.Col(3, P.BOOL))),
                   E.Logic("and", E.Cmp("lt", E.Col(1, P.DECIMAL(12, 2)), E.Col(4, P.DECIMAL(12, 2))),
                           E.Cmp("gt_eq", E.Col(2, P.DECIMAL(18, 0)), E.Col(5, P.DECIMAL(18, 0)))))
    for c in (cond, None):
        run(cb, left, types, right, types, jt, c, build_left, config={"spark.comet.b200.chunkRows": "3072"},
            linputs=[device_table(cb, left, types, dec8=["m", "w"])], rinputs=[device_table(cb, right, types, dec8=["m", "w"])])


@pytest.mark.parametrize("jt,build_left", SHAPES, ids=IDS)
def test_native_scan(cb, tmp_path, jt, build_left):
    """INT32-backed int8 and INT32 / FLBA decimals and dictionary-page strings read by NativeScan, compared in the condition"""
    P = cb.proto
    n_l, n_r = 400, 300
    a, b = parquet_table(n_l, 51), parquet_table(n_r, 52)
    names = ["i32", "i8", "d7", "d28", "sd", "row"]
    a = {k: a[k] for k in names}
    b = {k: b[k] for k in names}
    pa_path, pb_path = str(tmp_path / "a.parquet"), str(tmp_path / "b.parquet")
    write_parquet(pa_path, a, True)
    write_parquet(pb_path, b, True)
    scan_l, types = scan_of(cb, a, names, pa_path)
    scan_r, _ = scan_of(cb, b, names, pb_path)
    k = len(names)
    cond = E.Logic("or", E.Cmp("lt", E.Col(1, types[1]), E.Col(k + 1, types[1])),
                   E.Logic("and", E.Cmp("lt", E.Col(2, types[2]), E.Col(k + 2, types[2])), E.Cmp("gt_eq", E.Col(3, types[3]), E.Col(k + 3, types[3]))))
    got, stats = collect(cb, nlj_plan(cb, scan_l, scan_r, jt, cond, build_left), [], config={"spark.comet.b200.chunkRows": "2048"})
    ltbl, rtbl = expected_table(a, names), expected_table(b, names)
    check(got, R.nlj_table(ltbl, rtbl, jt, cond, build_left))
    assert stats["join_cond_pairs"] == n_l * n_r


@pytest.mark.parametrize("jt,build_left", SHAPES, ids=IDS)
def test_dictionary_strings_and_wide_decimals(cb, jt, build_left):
    """dictionary strings on both sides (each side its own batches), read by the condition and gathered into the output, and 16-byte
    decimals compared"""
    P = cb.proto
    left, lt = side(450, 31, 50)
    right, rt = side(350, 32, 50)
    cond = E.Logic("and", E.Cmp("gt_eq", E.Col(4, P.DECIMAL(30, 2)), E.Col(NCOL + 4, P.DECIMAL(30, 2))),
                   E.Logic("or", S.StrCmp("neq", S.StrCol(6), "ab"), S.StrCmp("eq", S.StrCol(NCOL + 6), "abc")))
    run(cb, left, lt, right, rt, jt, cond, build_left, chunk=100, config={"spark.comet.b200.chunkRows": "4096"})


# ---- compositions -------------------------------------------------------------------------------------------------------------------------
def test_q90_q28_cross_join_of_single_row_aggregates(cb):
    """three single-row aggregates over Scans, cross-joined with no condition (TPC-DS Q28 puts six in FROM, Q90 two)"""
    P = cb.proto
    rng = np.random.default_rng(90)
    tabs = [pa.table({"v": pa.array(rng.integers(-1000, 1000, n).astype(np.int64)), "q": pa.array(rng.integers(0, 100, n).astype(np.int32))})
            for n in (5000, 12000, 700)]
    t = [P.INT64, P.INT32]
    def agg(i):   # SUM(v), COUNT(v) WHERE q between i * 10 and i * 10 + 40
        f = P.filter_(P.scan(t), P.and_(P.gt_eq(P.bound(1, P.INT32), P.literal(i * 10, P.INT32)), P.lt(P.bound(1, P.INT32), P.literal(i * 10 + 40, P.INT32))))
        return P.hash_agg(f, [], [P.agg_sum(P.bound(0, P.INT64), P.INT64), P.agg_count([P.bound(0, P.INT64)])], P.PARTIAL)
    singles = [collect(cb, agg(i), [tabs[i].to_batches(max_chunksize=4096)])[0] for i in range(3)]
    want = [v for s in singles for v in s.to_pylist()[0].values()]
    for bl in (False, True):
        side_ = P.BUILD_LEFT if bl else P.BUILD_RIGHT
        plan = P.broadcast_nested_loop_join(P.broadcast_nested_loop_join(agg(0), agg(1), 0, side_), agg(2), 0, side_)
        got, stats = collect(cb, plan, [tabs[i].to_batches(max_chunksize=4096) for i in range(3)])
        assert got.num_rows == 1 and list(got.to_pylist()[0].values()) == want, (got.to_pylist(), want)
        assert stats["join_cond_pairs"] == 0


def not_in_cond(cb):
    """(l.a, l.b) NOT IN (SELECT x, y): per column (l = r OR isnull(l = r)), ANDed"""
    P = cb.proto
    eq_or_null = lambda l, r: E.Logic("or", E.Cmp("eq", l, r), E.IsNull(E.Cmp("eq", l, r)))
    return E.Logic("and", eq_or_null(E.Col(0, P.INT32), E.Col(3, P.INT32)), eq_or_null(E.Col(1, P.INT64), E.Col(4, P.INT64)))


@pytest.mark.parametrize("n_build", [0, 1, 40, 3000])
def test_multi_column_not_in(cb, n_build):
    """LeftAnti with the null-aware rewrite's condition, NULLs on both sides, an empty build side keeping every row"""
    P = cb.proto
    rng = np.random.default_rng(n_build)
    def tbl(n, seed):
        r = np.random.default_rng(seed)
        return pa.table({"a": pa.array(r.integers(0, 6, n).astype(np.int32), mask=r.random(n) < 0.1),
                         "b": pa.array(r.integers(0, 8, n).astype(np.int64), mask=r.random(n) < 0.1), "row": pa.array(np.arange(n, dtype=np.int64))})
    left, right = tbl(5000, 1), tbl(n_build, 2 + int(rng.integers(0, 5)))
    t = [P.INT32, P.INT64, P.INT64]
    got, _, _ = run(cb, left, t, right.select(["a", "b"]), t[:2], LEFT_ANTI, not_in_cond(cb), chunk=1500)
    if n_build == 0:
        assert got.num_rows == left.num_rows


def test_band_join_under_an_aggregate(cb):
    """events x ranges with t >= lo AND t < hi, grouped by the range id: COUNT(*) and SUM(t) per range"""
    P = cb.proto
    t, lo, hi = band_sides(20_000, 1000, 8)
    t, lo, hi = t // 1000, lo // 1000, lo // 1000 + (hi - lo) // 10
    ev = pa.table({"t": t})
    rg = pa.table({"id": np.arange(1000, dtype=np.int32), "lo": lo, "hi": hi})
    band = P.and_(P.gt_eq(P.bound(0, P.INT64), P.bound(2, P.INT64)), P.lt(P.bound(0, P.INT64), P.bound(3, P.INT64)))
    j = P.broadcast_nested_loop_join(P.scan([P.INT64]), P.scan([P.INT32, P.INT64, P.INT64]), 0, P.BUILD_RIGHT, condition=band)
    agg = P.hash_agg(j, [P.bound(1, P.INT32)], [P.agg_count([P.bound(0, P.INT64)]), P.agg_sum(P.bound(0, P.INT64), P.INT64)], P.PARTIAL)
    got, stats = collect(cb, agg, [ev.to_batches(max_chunksize=6000), rg.to_batches()], config={"spark.comet.b200.chunkRows": "65536"})
    rows = {r[0]: r[1:] for r in (tuple(d.values()) for d in got.to_pylist())}
    st = np.sort(t)
    for i in range(1000):
        a, b = np.searchsorted(st, lo[i], "left"), np.searchsorted(st, hi[i], "left")
        if b > a:
            assert rows[i][0] == b - a and rows[i][1] == int(st[a:b].sum()), i
        else:
            assert i not in rows
    assert stats["join_cond_pairs"] == 20_000 * 1000
