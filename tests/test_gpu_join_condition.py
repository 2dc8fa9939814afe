"""GPU: HashJoin and SortMergeJoin with a join condition against the CPU reference (tests/condjoinref.py), bit-exact and in order, and
the candidates the condition was evaluated on (cb200_stats.join_cond_pairs).  Covers every operator x join type x build side, conditions
between the sides on every comparable type and over one side only, OR / CASE / IS NULL, a string predicate on a dictionary column,
literal TRUE / FALSE, ANSI errors, candidate shapes (all / none / alternating pass, a key with thousands of matches across small slices,
skew, NULL keys, empty and one-row sides), stored layouts (device tables, NativeScan) and compositions (an aggregate above, Sorts below,
the TPC-H Q21 and TPC-DS Q16 shapes)."""
import numpy as np
import pyarrow as pa
import pytest

import condjoinref as R
import exprs as E
import strpred_ref as S
from joinref import INNER, LEFT_ANTI, LEFT_SEMI
from smjref import FULL_OUTER, LEFT_OUTER, RIGHT_OUTER
from test_gpu_join import check, collect
from test_gpu_partition_layouts import WORDS, _dec, _words, device_table, expected_table, parquet_table, scan_of, write_parquet
from test_gpu_sort_merge_join import sorted_by

pytestmark = pytest.mark.gpu

JT = {INNER: 0, LEFT_OUTER: 1, RIGHT_OUTER: 2, FULL_OUTER: 3, LEFT_SEMI: 4, LEFT_ANTI: 5}
MODES = ([("smj", jt, False) for jt in (INNER, LEFT_OUTER, RIGHT_OUTER, FULL_OUTER, LEFT_SEMI, LEFT_ANTI)] +
         [("hash", INNER, False), ("hash", INNER, True), ("hash", LEFT_SEMI, False), ("hash", LEFT_ANTI, False)])


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def join_plan(cb, op, lchild, ltypes, rchild, rtypes, lk, rk, jt, cond, build_left=False):
    P = cb.proto
    lkeys, rkeys = [P.bound(i, ltypes[i]) for i in lk], [P.bound(i, rtypes[i]) for i in rk]
    c = cond.proto() if cond is not None else None
    if op == "hash":
        return P.hash_join(lchild, rchild, lkeys, rkeys, JT[jt], P.BUILD_LEFT if build_left else P.BUILD_RIGHT, condition=c)
    return P.sort_merge_join(lchild, rchild, lkeys, rkeys, JT[jt], [P.sort_order(k) for k in lkeys], condition=c)


def run(cb, op, left, lt, right, rt, lk, rk, jt, cond, build_left=False, config=None, linputs=None, rinputs=None, chunk=4000):
    P = cb.proto
    plan = join_plan(cb, op, P.scan(lt), lt, P.scan(rt), rt, lk, rk, jt, cond, build_left)
    li = linputs if linputs is not None else ([left.to_batches(max_chunksize=chunk)] if left.num_rows else [left])
    ri = rinputs if rinputs is not None else ([right.to_batches(max_chunksize=chunk)] if right.num_rows else [right])
    got, stats = collect(cb, plan, li + ri, config)
    want = R.cond_join_table(left, right, lk, rk, jt, cond, build_left)
    check(got, want)
    if got is not None:
        got.validate(full=True)
    n_cand = R.candidate_count(left, right, lk, rk, jt, build_left) if cond is not None else 0
    assert stats["join_cond_pairs"] == n_cand, (stats["join_cond_pairs"], n_cand)
    return got, want, stats


# a side: k (int64 key), a (int32), d (date), m (decimal(12, 2)), w (decimal(30, 2)), f (float64), s (dictionary string)
NCOL = 7


def side(n, seed, dom, null_frac=0.1, key_nulls=0.05):
    import comet_b200.proto as P
    rng = np.random.default_rng(seed)
    m = lambda f=null_frac: rng.random(n) < f
    k = np.sort(rng.integers(0, dom, n))
    cols = {"k": pa.array(k, mask=m(key_nulls)),
            "a": pa.array(rng.integers(-20, 20, n).astype(np.int32), mask=m()),
            "d": pa.array(rng.integers(0, 40, n).astype(np.int32), pa.date32(), mask=m()),
            "m": _dec(rng.integers(-3000, 3000, n), 12, 2, m()),
            "w": _dec(_words([int(v) * 10**20 + 3 for v in rng.integers(-50, 50, n)]), 30, 2, m()),
            "f": pa.array(rng.standard_normal(n), mask=m()),
            "s": pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, 12, n), pa.int16(), mask=m()), pa.array(WORDS))}
    return pa.table(cols), [P.INT64, P.INT32, P.DATE, P.DECIMAL(12, 2), P.DECIMAL(30, 2), P.DOUBLE, P.STRING]


def L(i, dt):
    return E.Col(i, dt)


def Rc(i, dt):
    return E.Col(NCOL + i, dt)


def conditions():
    import comet_b200.proto as P
    return {
        "neq_int": E.Cmp("neq", L(1, P.INT32), Rc(1, P.INT32)),
        "lt_int": E.Cmp("lt", L(1, P.INT32), Rc(1, P.INT32)),
        "ge_date": E.Cmp("gt_eq", L(2, P.DATE), Rc(2, P.DATE)),
        "lt_dec8": E.Cmp("lt", L(3, P.DECIMAL(12, 2)), Rc(3, P.DECIMAL(12, 2))),
        "ge_dec16": E.Cmp("gt_eq", L(4, P.DECIMAL(30, 2)), Rc(4, P.DECIMAL(30, 2))),
        "lt_float": E.Cmp("lt", L(5, P.DOUBLE), Rc(5, P.DOUBLE)),
        "left_only": E.Cmp("gt_eq", L(1, P.INT32), E.Lit(0, P.INT32)),
        "right_only": E.Cmp("lt", Rc(1, P.INT32), E.Lit(5, P.INT32)),
        "or_isnull": E.Logic("or", E.IsNull(Rc(5, P.DOUBLE)), E.Cmp("gt", L(5, P.DOUBLE), Rc(5, P.DOUBLE))),
        "case": E.If(E.Cmp("gt", L(1, P.INT32), E.Lit(0, P.INT32)), E.Cmp("lt", L(2, P.DATE), Rc(2, P.DATE)), E.IsNull(Rc(1, P.INT32))),
        "strpred": E.Logic("and", S.StrCmp("neq", S.StrCol(NCOL + 6), "abc"), E.Cmp("neq", L(1, P.INT32), Rc(1, P.INT32))),
        "true": E.Lit(True, P.BOOL),
        "false": E.Lit(False, P.BOOL),
    }


# ---- every operator x join type x build side, every condition ----------------------------------------------------------------------------
@pytest.mark.parametrize("cond", list(conditions()))
@pytest.mark.parametrize("op,jt,build_left", MODES)
def test_conditions(cb, op, jt, build_left, cond):
    left, lt = side(5000, 1, 800)
    right, rt = side(3000, 2, 800)
    run(cb, op, left, lt, right, rt, [0], [0], jt, conditions()[cond], build_left)


@pytest.mark.parametrize("op,jt,build_left", MODES)
def test_literal_true_equals_no_condition(cb, op, jt, build_left):
    P = cb.proto
    left, lt = side(4000, 3, 500)
    right, rt = side(2500, 4, 500)
    plain, _ = collect(cb, join_plan(cb, op, P.scan(lt), lt, P.scan(rt), rt, [0], [0], jt, None, build_left),
                       [left.to_batches(max_chunksize=4000), right.to_batches(max_chunksize=4000)])
    got, _, _ = run(cb, op, left, lt, right, rt, [0], [0], jt, E.Lit(True, P.BOOL), build_left)
    assert got.equals(plain)


# ---- candidate shapes ---------------------------------------------------------------------------------------------------------------------
def shaped(cb, shape):
    """(left, right, condition): all pass, none pass, alternating pass, one key with thousands of matches, N:M skew, NULL keys"""
    import comet_b200.proto as P
    rng = np.random.default_rng(7)
    def tbl(k, a, kmask=None):
        return pa.table({"k": pa.array(np.asarray(k, np.int64), mask=kmask), "a": pa.array(np.asarray(a, np.int32))}), [P.INT64, P.INT32]
    ne = E.Cmp("neq", E.Col(1, P.INT32), E.Col(3, P.INT32))
    if shape in ("all", "none", "alternating"):
        k = np.repeat(np.arange(300), 3)
        left, lt = tbl(k, np.zeros(len(k)))
        rv = {"all": np.ones(len(k)), "none": np.zeros(len(k)), "alternating": np.arange(len(k)) % 2}[shape]
        right, rt = tbl(k, rv)
        return left, lt, right, rt, ne
    if shape == "big_key":   # 3 left rows x 5000 right rows of one key: their candidates span many slices
        left, lt = tbl([1, 2, 2, 2, 3], [0, 1, 2, 3, 4])
        right, rt = tbl(np.sort(np.r_[np.full(5000, 2), [1, 3, 4]]), rng.integers(0, 4, 5003))
        return left, lt, right, rt, ne
    if shape == "skew":
        k = np.sort(np.r_[np.zeros(2000), rng.integers(1, 400, 3000)])
        left, lt = tbl(k, rng.integers(0, 3, len(k)))
        kr = np.sort(np.r_[np.zeros(40), rng.integers(1, 400, 2000)])
        right, rt = tbl(kr, rng.integers(0, 3, len(kr)))
        return left, lt, right, rt, E.Cmp("lt", E.Col(1, P.INT32), E.Col(3, P.INT32))
    if shape == "null_keys":
        k = np.sort(rng.integers(0, 50, 1000))
        left, lt = tbl(k, rng.integers(0, 3, 1000), rng.random(1000) < 0.3)
        right, rt = tbl(k, rng.integers(0, 3, 1000), rng.random(1000) < 0.3)
        return left, lt, right, rt, ne
    raise ValueError(shape)


@pytest.mark.parametrize("chunk", ["64", "1000", "65536"])
@pytest.mark.parametrize("shape", ["all", "none", "alternating", "big_key", "skew", "null_keys"])
@pytest.mark.parametrize("op,jt,build_left", MODES)
def test_candidate_shapes(cb, op, jt, build_left, shape, chunk):
    """small chunkRows: one probe row's candidates straddle condition slices, and output batches stay at most chunkRows rows"""
    left, lt, right, rt, cond = shaped(cb, shape)
    run(cb, op, left, lt, right, rt, [0], [0], jt, cond, build_left, config={"spark.comet.b200.chunkRows": chunk}, chunk=700)


@pytest.mark.parametrize("n_l,n_r", [(0, 500), (500, 0), (0, 0), (1, 500), (500, 1), (1, 1)])
@pytest.mark.parametrize("op,jt,build_left", MODES)
def test_empty_and_one_row_sides(cb, op, jt, build_left, n_l, n_r):
    left, lt = side(n_l, 5, 3, key_nulls=0)
    right, rt = side(n_r, 6, 3, key_nulls=0)
    run(cb, op, left, lt, right, rt, [0], [0], jt, conditions()["lt_int"], build_left)


# ---- ANSI errors --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op,jt,build_left", MODES)
def test_ansi_overflow_only_from_a_candidate(cb, op, jt, build_left):
    """l.a + 1 overflows at INT32_MAX: no error while that row has no candidate, ARITHMETIC_OVERFLOW once it has one"""
    P = cb.proto
    cond = E.Cmp("gt", E.Arith("add", E.Col(1, P.INT32), E.Lit(1, P.INT32), P.INT32, E.ANSI), E.Col(3, P.INT32))
    types = [P.INT64, P.INT32]
    left = pa.table({"k": pa.array(np.arange(2000, dtype=np.int64)), "a": pa.array(np.r_[np.zeros(1999), [2**31 - 1]].astype(np.int32))})
    right = pa.table({"k": pa.array(np.arange(0, 1998, 2, dtype=np.int64)), "a": pa.array(np.zeros(999, np.int32))})
    run(cb, op, left, types, right, types, [0], [0], jt, cond, build_left)
    right2 = pa.table({"k": pa.array(np.r_[np.arange(0, 1998, 2), [1999]].astype(np.int64)), "a": pa.array(np.zeros(1000, np.int32))})
    with pytest.raises(E.AnsiError):
        R.cond_join_table(left, right2, [0], [0], jt, cond, build_left)
    with pytest.raises(cb.native.CometB200Error) as ei:
        collect(cb, join_plan(cb, op, P.scan(types), types, P.scan(types), types, [0], [0], jt, cond, build_left),
                [left.to_batches(max_chunksize=4000), right2.to_batches(max_chunksize=4000)])
    assert ei.value.error_class == "ARITHMETIC_OVERFLOW", str(ei.value)


# ---- stored layouts -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op,jt,build_left", MODES)
def test_device_tables(cb, op, jt, build_left):
    """bitmap booleans and 8-byte decimals in the condition"""
    P = cb.proto
    def tbl(n, seed):
        rng = np.random.default_rng(seed)
        m = lambda: rng.random(n) < 0.1
        return pa.table({"k": pa.array(np.sort(rng.integers(0, 700, n)).astype(np.int32)), "b": pa.array(rng.random(n) < 0.5, mask=m()),
                         "m": _dec(rng.integers(-10**6, 10**6, n), 12, 2, m()), "w": _dec(rng.integers(-10**6, 10**6, n), 18, 0, m())})
    types = [P.INT32, P.BOOL, P.DECIMAL(12, 2), P.DECIMAL(18, 0)]
    left, right = tbl(6000, 1), tbl(4000, 2)
    cond = E.Logic("or", E.Logic("and", E.Col(1, P.BOOL), E.Not(E.Col(5, P.BOOL))),
                   E.Logic("and", E.Cmp("lt", E.Col(2, P.DECIMAL(12, 2)), E.Col(6, P.DECIMAL(12, 2))),
                           E.Cmp("gt_eq", E.Col(3, P.DECIMAL(18, 0)), E.Col(7, P.DECIMAL(18, 0)))))
    run(cb, op, left, types, right, types, [0], [0], jt, cond, build_left, config={"spark.comet.b200.chunkRows": "3072"},
        linputs=[device_table(cb, left, types, dec8=["m", "w"])], rinputs=[device_table(cb, right, types, dec8=["m", "w"])])


@pytest.mark.parametrize("op,jt,build_left", MODES)
def test_native_scan(cb, tmp_path, op, jt, build_left):
    """INT32-backed int8 and INT32 / FLBA decimals read by NativeScan, compared in the condition"""
    P = cb.proto
    n = 5000
    a, b = parquet_table(n, 51), parquet_table(n, 52)
    names = ["i32", "i8", "d7", "d28", "row"]
    a = {k: a[k] for k in names}
    b = {k: b[k] for k in names}
    for cols, seed in ((a, 1), (b, 2)):
        cols["i32"] = (pa.array(np.sort(np.random.default_rng(seed).integers(0, 3000, n)).astype(np.int32)), P.INT32)
    pa_path, pb_path = str(tmp_path / "a.parquet"), str(tmp_path / "b.parquet")
    write_parquet(pa_path, a, True)
    write_parquet(pb_path, b, True)
    scan_l, types = scan_of(cb, a, names, pa_path)
    scan_r, _ = scan_of(cb, b, names, pb_path)
    k = len(names)
    cond = E.Logic("or", E.Cmp("neq", E.Col(1, types[1]), E.Col(k + 1, types[1])),
                   E.Logic("and", E.Cmp("lt", E.Col(2, types[2]), E.Col(k + 2, types[2])), E.Cmp("gt_eq", E.Col(3, types[3]), E.Col(k + 3, types[3]))))
    plan = join_plan(cb, op, scan_l, types, scan_r, types, [0], [0], jt, cond, build_left)
    got, stats = collect(cb, plan, [], config={"spark.comet.b200.chunkRows": "2048"})
    ltbl, rtbl = expected_table(a, names), expected_table(b, names)
    check(got, R.cond_join_table(ltbl, rtbl, [0], [0], jt, cond, build_left))
    assert stats["join_cond_pairs"] == R.candidate_count(ltbl, rtbl, [0], [0], jt, build_left)


# ---- composition --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("jt", [INNER, LEFT_OUTER, FULL_OUTER])
def test_aggregate_above(cb, jt):
    import pyarrow.compute as pc
    P = cb.proto
    left, lt = side(6000, 11, 900)
    right, rt = side(4000, 12, 900)
    cond = conditions()["lt_int"]
    j = join_plan(cb, "smj", P.scan(lt), lt, P.scan(rt), rt, [0], [0], jt, cond)
    agg = P.hash_agg(j, [], [P.agg_sum(P.bound(0, P.INT64), P.INT64), P.agg_count([P.bound(NCOL + 1, P.INT32)])], P.PARTIAL)
    got, _ = collect(cb, agg, [left.to_batches(max_chunksize=4000), right.to_batches(max_chunksize=4000)], config={"spark.comet.b200.chunkRows": "5000"})
    want = R.cond_join_table(left, right, [0], [0], jt, cond)
    row = got.to_pylist()[0]
    assert list(row.values())[0] == pc.sum(want.column(0)).as_py()
    assert list(row.values())[-1] == want.column(NCOL + 1).length() - want.column(NCOL + 1).null_count


@pytest.mark.parametrize("jt", [INNER, LEFT_OUTER, RIGHT_OUTER, FULL_OUTER, LEFT_SEMI, LEFT_ANTI])
def test_scan_sort_smj_sort_scan(cb, jt):
    """Scan -> Sort -> SortMergeJoin(cond) <- Sort <- Scan over unsorted inputs"""
    P = cb.proto
    left, lt = side(8000, 21, 1500)
    right, rt = side(6000, 22, 1500)
    rng = np.random.default_rng(0)
    left, right = left.take(rng.permutation(left.num_rows)), right.take(rng.permutation(right.num_rows))
    srt = lambda t: P.sort(P.scan(t), [P.sort_order(P.bound(0, t[0]))])
    cond = conditions()["neq_int"]
    got, stats = collect(cb, join_plan(cb, "smj", srt(lt), lt, srt(rt), rt, [0], [0], jt, cond),
                         [left.to_batches(max_chunksize=3000), right.to_batches(max_chunksize=3000)], config={"spark.comet.b200.chunkRows": "4096"})
    ls, rs = sorted_by(left, ["k"]), sorted_by(right, ["k"])
    check(got, R.cond_join_table(ls, rs, [0], [0], jt, cond))
    assert stats["join_cond_pairs"] == R.candidate_count(ls, rs, [0], [0], jt)


def lineitem(n, seed):
    """l_orderkey (sorted), l_suppkey, l_receiptdate > l_commitdate as a flag, l_row"""
    rng = np.random.default_rng(seed)
    ok = np.sort(rng.integers(0, n // 4, n)).astype(np.int64)
    return pa.table({"l_orderkey": pa.array(ok), "l_suppkey": pa.array(rng.integers(0, 50, n).astype(np.int64)),
                     "late": pa.array(rng.random(n) < 0.5), "l_row": pa.array(np.arange(n, dtype=np.int64))})


def test_q21_shape(cb):
    """l1 semi-joined to l2 on l_orderkey with l_suppkey <> l_suppkey, then anti-joined to late l3 rows the same way, counted"""
    P = cb.proto
    t = [P.INT64, P.INT64, P.BOOL, P.INT64]
    l1 = lineitem(20_000, 1)
    l3 = l1.filter(l1.column("late"))
    cond = E.Cmp("neq", E.Col(1, P.INT64), E.Col(5, P.INT64))
    semi = join_plan(cb, "smj", P.filter_(P.scan(t), P.bound(2, P.BOOL)), t, P.scan(t), t, [0], [0], LEFT_SEMI, cond)
    anti = join_plan(cb, "smj", semi, t, P.filter_(P.scan(t), P.bound(2, P.BOOL)), t, [0], [0], LEFT_ANTI, cond)
    got, _ = collect(cb, anti, [l1.to_batches(max_chunksize=8192), l1.to_batches(max_chunksize=8192), l1.to_batches(max_chunksize=8192)],
                     config={"spark.comet.b200.chunkRows": "8192"})
    want = R.cond_join_table(R.cond_join_table(l3, l1, [0], [0], LEFT_SEMI, cond).rename_columns(l1.column_names), l3, [0], [0], LEFT_ANTI, cond)
    check(got, want)


def test_q16_shape(cb):
    """catalog_sales semi-joined to itself on the order number with a different warehouse, anti-joined to returns, over Sorts"""
    P = cb.proto
    rng = np.random.default_rng(16)
    n = 15_000
    cs = pa.table({"order": pa.array(rng.integers(0, 4000, n).astype(np.int64)), "wh": pa.array(rng.integers(0, 5, n).astype(np.int32), mask=rng.random(n) < 0.05),
                   "row": pa.array(np.arange(n, dtype=np.int64))})
    cr = pa.table({"order": pa.array(rng.integers(0, 4000, 3000).astype(np.int64))})
    t, tr = [P.INT64, P.INT32, P.INT64], [P.INT64]
    srt = lambda child, ty: P.sort(child, [P.sort_order(P.bound(0, ty[0]))])
    cond = E.Cmp("neq", E.Col(1, P.INT32), E.Col(4, P.INT32))
    semi = join_plan(cb, "smj", srt(P.scan(t), t), t, srt(P.scan(t), t), t, [0], [0], LEFT_SEMI, cond)
    anti = join_plan(cb, "smj", semi, t, srt(P.scan(tr), tr), tr, [0], [0], LEFT_ANTI, None)
    got, _ = collect(cb, anti, [cs.to_batches(max_chunksize=5000), cs.to_batches(max_chunksize=5000), cr.to_batches(max_chunksize=5000)])
    css = sorted_by(cs, ["order"])
    s = R.cond_join_table(css, css, [0], [0], LEFT_SEMI, cond).rename_columns(cs.column_names)
    want = R.cond_join_table(s, sorted_by(cr, ["order"]), [0], [0], LEFT_ANTI, None)
    check(got, want)
