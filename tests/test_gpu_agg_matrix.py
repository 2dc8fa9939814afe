"""GPU parity of the aggregate operator against the CPU reference (tests/aggref.py) over the matrix of tests/aggcases.py: key types,
aggregate functions, special values, batch layouts and the dense / key-table / stream / dense -> hash strategies.

Each case runs Partial -> Final, Partial -> PartialMerge -> Final, and a Final fed with a state batch the reference built (with bytes
under its NULL slots).  Comparison rules:
  integers, decimals, counts, dates, timestamps, keys, MIN / MAX (floats included, by their bits)   exact
  SUM(f64)   within 1 ULP of the exact sum of its inputs; NaN / +Inf / -Inf by class
  AVG(f64)   within 2 ULP of the correctly rounded exact mean; the same class rule
A Partial may emit a key more than once (stream runs, a dense -> hash migration), so Partial output is compared after a reference
merge, each of its float sums allowed its own 1 ULP."""
import collections
import math
import types

import numpy as np
import pyarrow as pa
import pytest

import aggcases
import aggref as R
import exprs as E

pytestmark = pytest.mark.gpu

STRATEGY_RUNS = collections.Counter()


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def run(cb, plan, inputs, cfg=None):
    """-> (result table or None, cb200_stats.agg_strategies)"""
    with cb.native.Plan(plan, inputs, config=cfg) as p:
        out = p.collect()
        return out, p.stats()["agg_strategies"]


def rows_of(table, case, state=True):
    if table is None:
        return []
    if state:
        return R.state_rows_of(table, len(case.key_cols), case.aggs, R.state_schema(case.key_types, case.aggs))
    cols = [R.pyvalues(table.column(i), t) for i, t in enumerate(case.key_types + [a.result_type() for a in case.aggs])]
    nk = len(case.key_cols)
    return [(tuple(c[r] for c in cols[:nk]), [c[r] for c in cols[nk:]]) for r in range(table.num_rows)]


def fclass(x):
    return "nan" if math.isnan(x) else "+inf" if x == math.inf else "-inf" if x == -math.inf else "finite"


def f64_within(got, exact, ulps, slack=0.0, what=""):
    """`got` within `ulps` ULP (+ slack) of `exact` (a float already rounded from the exact value); non-finite by class."""
    assert (got is None) == (exact is None), what
    if got is None:
        return
    assert fclass(got) == fclass(exact), f"{what}: got {got!r}, want {exact!r}"
    if fclass(exact) == "finite":
        tol = ulps * math.ulp(exact) + slack
        assert abs(got - exact) <= tol, f"{what}: got {got!r}, want {exact!r} (tolerance {tol!r})"


def same(got, exp, what):
    g = R.f64_bits(got) if isinstance(got, float) else got
    e = R.f64_bits(exp) if isinstance(exp, float) else exp
    assert g == e, f"{what}: got {got!r}, want {exp!r}"


def check_states(got_rows, exp, case, stage, f64_exp=None):
    """Library state rows (keys may repeat) vs the reference's states, merged by the reference.  f64_exp: states whose float sums are
    exact over the states the library merged (each of those already carries its own rounding)."""
    merged = R.merge(got_rows, case.aggs)
    assert set(merged) == set(exp), f"{stage}: group keys differ: extra {list(set(merged) - set(exp))[:3]}, missing {list(set(exp) - set(merged))[:3]}"
    n_rows = collections.Counter(k for k, _ in got_rows)
    for ai, a in enumerate(case.aggs):
        for key in exp:
            g, e = merged[key][ai], exp[key][ai]
            what = f"{stage} agg {ai} ({a.kind}) key {key}"
            if a.f64_sum and f64_exp is not None:
                e = f64_exp[key][ai]
            if a.f64_sum:
                sums = [s[ai][0] for k, s in got_rows if k == key and s[ai][0] is not None] if n_rows[key] > 1 else []
                slack = sum(math.ulp(x) for x in sums if math.isfinite(x))
                f64_within(g[0], e[0], 1, slack, what)
                if a.kind == "avg":
                    same(g[1], e[1], what + " count")
            else:
                for x, y in zip(g, e):
                    same(x, y, what)


def check_results(got_rows, exp, case, stage, f64_exp=None):
    """Final results vs the reference's.  f64_exp: results whose float sums / means are exact over the states the library merged."""
    got = dict(got_rows)
    assert len(got) == len(got_rows), f"{stage}: a key appears twice in Final output"
    assert set(got) == set(exp), f"{stage}: group keys differ: extra {list(set(got) - set(exp))[:3]}, missing {list(set(exp) - set(got))[:3]}"
    for ai, a in enumerate(case.aggs):
        for key in exp:
            what = f"{stage} agg {ai} ({a.kind}) key {key}"
            g, e = got[key][ai], (f64_exp or exp)[key][ai]
            if a.f64_sum:
                f64_within(g, e, 1 if a.kind == "sum" else 2, 0.0, what)
            else:
                same(g, exp[key][ai], what)


def bitwise(rows):
    b = lambda x: ("f", R.f64_bits(x)) if isinstance(x, float) else tuple(b(y) for y in x) if isinstance(x, (tuple, list)) else x
    return [b(r) for r in rows]


def f64_final_over(state_rows, case):
    return R.final(state_rows, case.aggs, ungrouped=not case.key_cols)


@pytest.mark.parametrize("case", aggcases.CASES, ids=lambda c: c.name)
def test_agg_matrix(cb, case):
    table = case.table()
    exp_state = R.partial(table, case.dts, case.key_cols, case.aggs)
    exp = R.aggregate(table, case.dts, case.key_cols, case.aggs)
    grouped = bool(case.key_cols)
    # Partial: the strategy the case targets must be the one that ran
    state, bits = run(cb, case.partial_plan(), [case.batches()], case.config())
    assert bits == aggcases.EXPECTED_BITS[case.strategy], f"strategy bits {bits:#x}, case targets {case.strategy}"
    STRATEGY_RUNS[case.strategy] += 1
    got_state = rows_of(state, case)
    if grouped and table.num_rows == 0:
        assert got_state == [] and exp == {}
        return
    check_states(got_state, exp_state, case, "partial")

    # Partial -> Final
    res, _ = run(cb, case.merge_plan(R.FINAL), [state])
    check_results(rows_of(res, case, state=False), exp, case, "partial->final", f64_final_over(got_state, case))

    # Partial -> PartialMerge -> Final
    merged, _ = run(cb, case.merge_plan(R.PARTIAL_MERGE), [state])
    got_merged = rows_of(merged, case)
    check_states(got_merged, exp_state, case, "partial->merge", R.merge(got_state, case.aggs))
    res2, _ = run(cb, case.merge_plan(R.FINAL), [merged])
    check_results(rows_of(res2, case, state=False), exp, case, "partial->merge->final", f64_final_over(got_merged, case))

    # Final over reference-built state: two partial states per group (odd and even rows), garbage under every NULL slot, and for
    # an ungrouped AVG(f64) the (NULL sum, 0) state of a partition that saw no batch (avg.rs:148-153)
    n = table.num_rows
    halves = [R.partial(table.take(pa.array(range(h, n, 2), type=pa.int64())), case.dts, case.key_cols, case.aggs) for h in (0, 1)]
    ref_rows = [(k, v) for h in halves for k, v in h.items()]
    if not grouped and any(a.f64_sum and a.kind == "avg" for a in case.aggs):
        empty = R.partial(table.slice(0, 0), case.dts, case.key_cols, case.aggs)[()]
        ref_rows.append(((), [(None, 0) if a.f64_sum and a.kind == "avg" else s for a, s in zip(case.aggs, empty)]))
    batch = R.state_batch(ref_rows, case.key_types, case.aggs, garbage_seed=case.seed)
    res3, _ = run(cb, case.merge_plan(R.FINAL), [[batch]])
    ref_final = R.final(ref_rows, case.aggs, ungrouped=not grouped)
    check_results(rows_of(res3, case, state=False), ref_final, case, "reference state->final")

    # the dense fold has a fixed order: float results repeat bit for bit
    if case.strategy in ("dense", "ungrouped") and any(a.f64_sum for a in case.aggs):
        state_b, _ = run(cb, case.partial_plan(), [case.batches()], case.config())
        assert bitwise(rows_of(state_b, case)) == bitwise(got_state)
        res_b, _ = run(cb, case.merge_plan(R.FINAL), [state_b])
        assert bitwise(rows_of(res_b, case, state=False)) == bitwise(rows_of(res, case, state=False))


def test_agg_matrix_ran_every_strategy():
    """Every strategy was reached by at least one case of this session (the matrix cannot quietly collapse onto one path)."""
    if sum(STRATEGY_RUNS.values()) < len(aggcases.CASES):
        pytest.skip("only part of the matrix ran in this session")
    for s in ("dense", "table", "stream", "migrate", "ungrouped"):
        assert STRATEGY_RUNS[s] > 0, s


def test_ungrouped_avg_f64_final_skips_null_partial_sums(cb):
    """avg.rs:148-175: the Partial of a partition that saw no batch emits (NULL, 0); the ungrouped merge skips the NULL sum.  The
    NULL slot here holds a NaN: reading it would make the average NaN."""
    P = cb.proto
    a = R.Agg("avg", E.Col(0, P.DOUBLE), P.DOUBLE)
    ref_rows = [((), [(None, 0)]), ((), [(6.0, 3)]), ((), [(None, 0)]), ((), [(1.5, 1)])]
    batch = R.state_batch(ref_rows, [], [a], garbage_seed=1)
    assert batch.column(0).null_count == 2
    res, _ = run(cb, R.merge_plan([], [a]), [[batch]])
    assert res.column(0).to_pylist() == [7.5 / 4]


def test_f64_sum_overflowing_prefix_is_never_a_wrong_finite_value(cb):
    """[1e308, 1e308, -1e308]: the exact sum (1e308) is finite, the row-ordered reference gives +Inf.  The library's double-double
    result depends on the merge order (DESIGN.md section 6): it is the exact sum within 1 ULP or a non-finite value, never another
    finite number."""
    P = cb.proto
    vals = [1e308, 1e308, -1e308]
    exact = 1e308
    for keys, cfg in ((None, None), ([7] * len(vals), aggcases.TABLE_CFG), ([7] * len(vals), aggcases.STREAM_CFG)):
        cols = {"v": pa.array(vals, type=pa.float64())}
        dts = [P.DOUBLE]
        if keys:
            cols = {"k": pa.array(keys, type=pa.int64()), **cols}
            dts = [P.INT64, P.DOUBLE]
        v = E.Col(len(dts) - 1, P.DOUBLE)
        aggs = [R.Agg("sum", v, P.DOUBLE), R.Agg("avg", v, P.DOUBLE)]
        kc = [0] if keys else []
        partial, _ = run(cb, R.partial_plan(dts, kc, aggs), [pa.table(cols).to_batches()], cfg)
        res, _ = run(cb, R.merge_plan(dts[:len(kc)], aggs), [partial])
        s, avg = res.column(len(kc)).to_pylist()[0], res.column(len(kc) + 1).to_pylist()[0]
        assert not math.isfinite(s) or abs(s - exact) <= math.ulp(exact), s
        exact_avg = 1e308 / 3
        assert not math.isfinite(avg) or abs(avg - exact_avg) <= 2 * math.ulp(exact_avg), avg


@pytest.mark.parametrize("strategy", ["ungrouped", "dense", "table", "stream"])
def test_f64_sum_keeps_the_low_word_over_many_rows(cb, strategy):
    """2^53 every 61st row, 1.0 elsewhere: a plain double sum drops every 1.0 added to a large partial, the double-double keeps them
    in its low word.  Each thread folds many rows here, which the matrix's small groups do not reach."""
    P = cb.proto
    n = 1 << 22
    v = np.ones(n)
    v[::61] = 2.0 ** 53
    k = {"ungrouped": None, "dense": np.arange(n) % 2 == 0, "table": np.arange(n) % 3, "stream": np.arange(n) // 4096}[strategy]
    dts = [P.DOUBLE] if k is None else [P.BOOL if strategy == "dense" else P.INT64, P.DOUBLE]
    cols = [pa.array(v)] if k is None else [pa.array(k), pa.array(v)]
    kc = [] if k is None else [0]
    x = E.Col(len(dts) - 1, P.DOUBLE)
    aggs = [R.Agg("sum", x, P.DOUBLE), R.Agg("avg", x, P.DOUBLE)]
    cfg = aggcases.STREAM_CFG if strategy == "stream" else aggcases.TABLE_CFG
    state, bits = run(cb, R.partial_plan(dts, kc, aggs), [pa.table(cols, names=[f"c{i}" for i in range(len(cols))]).to_batches(max_chunksize=1 << 17)], cfg)
    assert bits == aggcases.EXPECTED_BITS[strategy]
    res, _ = run(cb, R.merge_plan(dts[:len(kc)], aggs), [state])
    groups = {(): np.ones(n, dtype=bool)} if k is None else {(int(g) if strategy != "dense" else bool(g),): k == g for g in np.unique(k)}
    got = dict(rows_of(res, types.SimpleNamespace(key_cols=kc, key_types=dts[:len(kc)], aggs=aggs), state=False))
    assert set(got) == set(groups)
    for key, m in groups.items():
        exact = int(m.sum()) + int(m[::61].sum()) * (2 ** 53 - 1)     # the exact sum
        f64_within(got[key][0], float(exact), 1, 0.0, f"sum {key}")
        f64_within(got[key][1], R.round_fraction(R.Fraction(exact, int(m.sum()))), 2, 0.0, f"avg {key}")
