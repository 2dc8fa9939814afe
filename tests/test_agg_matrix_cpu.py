"""CPU checks of the aggregate test matrix: the CPU reference (tests/aggref.py) agrees with pyarrow and with the oracle's
accumulators, and every plan of the matrix is accepted by the planner and NVRTC-compiles for sm_90a."""
import math

import numpy as np
import pyarrow as pa
import pytest

import aggcases
import aggref as R
import exprs as E
from comet_b200 import proto as P


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def _ordinary_table(seed):
    rng = np.random.default_rng(seed)
    n = 5000
    k1 = rng.integers(-5, 5, n)
    k2 = rng.integers(0, 3, n)
    iv = rng.integers(-10 ** 12, 10 ** 12, n)
    fv = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 6, n)
    im, fm, km = rng.random(n) < 0.1, rng.random(n) < 0.1, rng.random(n) < 0.05
    return pa.table({"k1": pa.array(k1, mask=km), "k2": pa.array(k2.astype(np.int32)), "i": pa.array(iv, mask=im), "f": pa.array(fv, mask=fm)})


def test_reference_matches_pyarrow_group_by():
    """COUNT / SUM / MIN / MAX / MEAN over int and float columns (no NaN: pyarrow's float min / max does not follow totalOrder)."""
    t = _ordinary_table(1)
    dts = [P.INT64, P.INT32, P.INT64, P.DOUBLE]
    i, f = E.Col(2, P.INT64), E.Col(3, P.DOUBLE)
    aggs = [R.Agg("count", i), R.Agg("sum", i, P.INT64), R.Agg("min", i, P.INT64), R.Agg("max", i, P.INT64), R.Agg("avg", i, P.DOUBLE),
            R.Agg("count", f), R.Agg("sum", f, P.DOUBLE), R.Agg("min", f, P.DOUBLE), R.Agg("max", f, P.DOUBLE), R.Agg("avg", f, P.DOUBLE)]
    got = R.aggregate(t, dts, [0, 1], aggs)
    exp = t.group_by(["k1", "k2"]).aggregate([("i", "count"), ("i", "sum"), ("i", "min"), ("i", "max"), ("i", "mean"),
                                              ("f", "count"), ("f", "sum"), ("f", "min"), ("f", "max"), ("f", "mean")])
    rows = exp.to_pylist()
    assert len(rows) == len(got)
    for r in rows:
        g = got[(r["k1"], r["k2"])]
        assert g[:4] == [r["i_count"], r["i_sum"], r["i_min"], r["i_max"]]
        assert g[5] == r["f_count"] and g[7] == r["f_min"] and g[8] == r["f_max"]
        for mine, theirs in ((g[4], r["i_mean"]), (g[6], r["f_sum"]), (g[9], r["f_mean"])):
            assert (mine is None) == (theirs is None)
            if mine is not None:
                assert math.isclose(mine, theirs, rel_tol=1e-12, abs_tol=1e-9)


def test_reference_ungrouped_matches_pyarrow():
    t = _ordinary_table(2)
    dts = [P.INT64, P.INT32, P.INT64, P.DOUBLE]
    got = R.aggregate(t, dts, [], [R.Agg("sum", E.Col(2, P.INT64), P.INT64), R.Agg("min", E.Col(3, P.DOUBLE), P.DOUBLE),
                                   R.Agg("count", E.Col(3, P.DOUBLE))])
    assert got == {(): [pa.compute.sum(t["i"]).as_py(), pa.compute.min(t["f"]).as_py(), pa.compute.count(t["f"]).as_py()]}


def test_reference_float_rules():
    """IEEE special values, totalOrder MIN / MAX with exact bits, and one rounding of the exact sum."""
    nan_p, neg_nan = aggcases.NAN_PAYLOAD, aggcases.NEG_NAN
    vals = [[1.0, math.nan], [math.inf, -math.inf], [math.inf, 1.0], [1e308, 1e308, -1e308], [0.1] * 10, [-0.0, 0.0], [nan_p, 1.0, neg_nan, -math.inf]]
    keys = [i for i, v in enumerate(vals) for _ in v]
    t = pa.table({"k": pa.array(keys, type=pa.int64()), "v": pa.array([x for v in vals for x in v], type=pa.float64())})
    v = E.Col(1, P.DOUBLE)
    got = R.aggregate(t, [P.INT64, P.DOUBLE], [0], [R.Agg("sum", v, P.DOUBLE), R.Agg("min", v, P.DOUBLE), R.Agg("max", v, P.DOUBLE)])
    assert math.isnan(got[(0,)][0]) and math.isnan(got[(1,)][0]) and got[(2,)][0] == math.inf
    assert got[(3,)][0] == 1e308                          # exact: the row-ordered prefix 2e308 does not overflow here
    assert got[(4,)][0] == 1.0                            # math.fsum([0.1] * 10) rounds to 1.0
    assert R.f64_bits(got[(5,)][1]) == R.f64_bits(-0.0) and R.f64_bits(got[(5,)][2]) == 0
    assert R.f64_bits(got[(6,)][1]) == R.f64_bits(neg_nan) and R.f64_bits(got[(6,)][2]) == R.f64_bits(nan_p)
    assert got[(4,)][0] == math.fsum([0.1] * 10)


def test_reference_sum_int_matches_oracle(oracle):
    """SUM(int) in Legacy / TRY / ANSI vs the oracle's SumIntGroups (sum_int.rs), values near the i64 edges."""
    rng = np.random.default_rng(5)
    n = 400
    g = rng.integers(0, 8, n)
    v = rng.integers(-2 ** 62, 2 ** 62, n) * rng.integers(0, 3, n)
    valid = rng.random(n) > 0.1
    valid[g == 7] = False                                  # one group all NULL
    t = pa.table({"g": pa.array(g), "v": pa.array(v, mask=~valid)})
    for mode in (R.LEGACY, R.TRY):
        got = R.aggregate(t, [P.INT64, P.INT64], [0], [R.Agg("sum", E.Col(1, P.INT64), P.INT64, mode=mode)])
        acc = oracle.SumIntGroups(8, mode)
        acc.update(v, valid.astype(np.uint8), g)
        for k in range(8):
            exp = int(acc.sums[k]) if acc.sums_valid[k] else None
            assert got[(k,)][0] == exp, (mode, k)
    small = pa.table({"g": pa.array(g), "v": pa.array(v // 2 ** 40, mask=~valid)})
    got = R.aggregate(small, [P.INT64, P.INT64], [0], [R.Agg("sum", E.Col(1, P.INT64), P.INT64, mode=R.ANSI)])
    acc = oracle.SumIntGroups(8, R.ANSI)
    acc.update(v // 2 ** 40, valid.astype(np.uint8), g)
    assert all(got[(k,)][0] == (int(acc.sums[k]) if acc.sums_valid[k] else None) for k in range(8))
    with pytest.raises(E.AnsiError):
        R.aggregate(t, [P.INT64, P.INT64], [0], [R.Agg("sum", E.Col(1, P.INT64), P.INT64, mode=R.ANSI)])


def test_reference_sum_decimal_matches_oracle(oracle):
    """SUM(decimal) state and result vs the oracle's SumDecimalGroups (sum_decimal.rs), incl. merge of two partial states."""
    rng = np.random.default_rng(6)
    n = 600
    g = rng.integers(0, 6, n)
    m = 10 ** 12 - 1
    v = [int(x) for x in rng.choice([m, -m, -1, 0, 12345], n)]
    valid = rng.random(n) > 0.1
    valid[g == 5] = False
    col = R.arrow_column([x if ok else None for x, ok in zip(v, valid)], P.DECIMAL(12, 2))
    t = pa.table({"g": pa.array(g), "v": col})
    a = R.Agg("sum", E.Col(1, P.DECIMAL(12, 2)), P.DECIMAL(22, 2))
    st = R.partial(t, [P.INT64, P.DECIMAL(12, 2)], [0], [a])
    acc = oracle.SumDecimalGroups(6, 22)
    acc.update(oracle.dec_from_ints(v), valid.astype(np.uint8), g)
    s, sv, empty = acc.state()
    for k in range(6):
        exp = (oracle.dec_to_ints(s[k:k + 1])[0] if sv[k] else None, bool(empty[k]))
        assert tuple(st[(k,)][0]) == exp
    halves = [R.partial(t.slice(0, n // 2), [P.INT64, P.DECIMAL(12, 2)], [0], [a]), R.partial(t.slice(n // 2), [P.INT64, P.DECIMAL(12, 2)], [0], [a])]
    res = R.final([(k, v) for h in halves for k, v in h.items()], [a])
    out, ok = acc.evaluate()
    for k in range(6):
        assert res[(k,)][0] == (oracle.dec_to_ints(out[k:k + 1])[0] if ok[k] else None)


def test_reference_avg_f64_merge_skips_null_partial_sums():
    """avg.rs:148-175: a partition that saw no batch contributes (NULL, 0); the merge skips the NULL sum."""
    a = R.Agg("avg", E.Col(0, P.DOUBLE), P.DOUBLE)
    res = R.final([((), [(None, 0)]), ((), [(6.0, 3)]), ((), [(None, 0)])], [a], ungrouped=True)
    assert res == {(): [2.0]}
    assert R.final([((), [(None, 0)])], [a], ungrouped=True) == {(): [None]}


def test_matrix_reaches_every_strategy():
    n = {s: sum(1 for c in aggcases.CASES if c.strategy == s) for s in aggcases.EXPECTED_BITS}
    assert n["dense"] >= 5 and n["table"] >= 10 and n["stream"] >= 5 and n["migrate"] >= 1 and n["ungrouped"] >= 3 and n["empty"] >= 1
    names = [c.name for c in aggcases.CASES]
    assert len(names) == len(set(names))
    kinds = {a.kind for c in aggcases.CASES for a in c.aggs}
    assert kinds == {"count", "sum", "avg", "min", "max"}


@pytest.mark.parametrize("case", aggcases.CASES, ids=lambda c: c.name)
def test_matrix_plan_supported_and_compiles(cb, case):
    plans = [case.partial_plan(), case.merge_plan(R.FINAL), case.merge_plan(R.PARTIAL_MERGE)]
    for plan in plans:
        ok, why = cb.native.supports(plan)
        assert ok, why
        assert cb.native.compile_plan(plan)


@pytest.mark.parametrize("case", aggcases.CASES, ids=lambda c: c.name)
def test_matrix_reference_runs(case):
    """The reference evaluates every case and its state batch round-trips through Arrow (garbage under the NULL slots included)."""
    st = R.partial(case.table(), case.dts, case.key_cols, case.aggs)
    rows = [(k, v) for k, v in st.items()]
    b = R.state_batch(rows, case.key_types, case.aggs, garbage_seed=1)
    back = R.state_rows_of(pa.Table.from_batches([b]), len(case.key_cols), case.aggs, R.state_schema(case.key_types, case.aggs))
    assert len(back) == len(rows)
    for (k1, s1), (k2, s2) in zip(rows, back):
        assert k1 == k2
        assert [[R.f64_bits(x) if isinstance(x, float) else x for x in s] for s in s1] == \
               [[R.f64_bits(x) if isinstance(x, float) else x for x in s] for s in s2]
