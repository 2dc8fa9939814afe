"""CPU checks of distinct-aggregate plans: the four-stage reference (tests/distinctref.py) against the direct SQL answer computed with
pyarrow, the planner's acceptance and refusals for per-expression aggregate modes, the output schema of a mixed operator, and NVRTC
compilation of every mixed and keys-only kernel of tests/distinctcases.py."""
from decimal import Decimal

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import aggref as R
import distinctcases
import distinctref as D
import exprs as E
from comet_b200 import proto as P


@pytest.fixture(scope="module")
def native():
    from comet_b200 import native
    return native


# ---- the reference against the direct answer ----------------------------------------------------------------------------------------
def _table(seed, n=4000, key_card=12, x_card=25):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, key_card, n)
    x = rng.integers(-x_card, x_card, n)
    y = rng.integers(-10 ** 9, 10 ** 9, n)
    yd = rng.integers(-10 ** 11, 10 ** 11, n)
    km, xm, ym = rng.random(n) < 0.03, rng.random(n) < 0.05, rng.random(n) < 0.05
    km[:] = km & (k != 3)
    xm[k == 3] = True                     # group 3: every x is NULL
    ym[k == 3] = True                     # and every y
    ctx = __import__("decimal").Context(prec=40)
    return pa.table({"k": pa.array(k, mask=km), "x": pa.array(x, mask=xm), "y": pa.array(y, mask=ym),
                     "yd": pa.array([Decimal(int(v)).scaleb(-2, context=ctx) for v in yd], type=pa.decimal128(12, 2))})


DTS = [P.INT64, P.INT64, P.INT64, P.DECIMAL(12, 2)]


def _chain(key_cols):
    """over the columns k, x, y, yd of _table: group by key_cols (k or nothing), distinct x"""
    y, yd = E.Col(2, P.INT64), E.Col(3, P.DECIMAL(12, 2))
    ordinary = [R.Agg("sum", y, P.INT64), R.Agg("count", y), R.Agg("min", yd, P.DECIMAL(12, 2)), R.Agg("sum", yd, P.DECIMAL(22, 2))]
    dist = [("count", None, None, R.LEGACY), ("sum", P.INT64, None, R.LEGACY), ("avg", P.DOUBLE, None, R.LEGACY)]
    return D.Chain(DTS, key_cols, [1], ordinary, dist)


def _unscaled(v):
    return None if v is None else int(v.scaleb(2))


def test_reference_chain_matches_direct_answer_grouped():
    """SELECT k, COUNT(DISTINCT x), SUM(DISTINCT x), AVG(DISTINCT x), SUM(y), COUNT(y), MIN(yd), SUM(yd) GROUP BY k: NULL x, NULL keys
    and a group whose x and y are all NULL."""
    t = _table(1)
    got = _chain([0]).answer(t)
    dedup = t.group_by(["k", "x"]).aggregate([]).group_by("k").aggregate([("x", "count"), ("x", "sum"), ("x", "mean")])
    plain = t.group_by("k").aggregate([("y", "sum"), ("y", "count"), ("yd", "min"), ("yd", "sum")])
    exp = {r["k"]: r for r in dedup.to_pylist()}
    for r in plain.to_pylist():
        exp[r["k"]].update(r)
    assert set(got) == {(k,) for k in exp}
    assert None in exp and exp[3]["x_count"] == 0 and exp[3]["x_sum"] is None
    for k, r in exp.items():
        g = got[(k,)]
        assert g[:4] == [r["y_sum"], r["y_count"], _unscaled(r["yd_min"]), _unscaled(r["yd_sum"])], k
        assert g[4:6] == [r["x_count"], r["x_sum"]], k
        assert (g[6] is None) == (r["x_mean"] is None) and (g[6] is None or abs(g[6] - r["x_mean"]) <= 1e-12 * abs(r["x_mean"]) + 1e-12), k


def test_reference_chain_matches_direct_answer_global():
    """SELECT COUNT(DISTINCT x), SUM(DISTINCT x), AVG(DISTINCT x), SUM(y), ... FROM t: no outer key; and over no rows."""
    t = _table(2)
    got = _chain([]).answer(t)
    ux = pc.unique(t["x"]).drop_null()
    assert got[()][:2] == [pc.sum(t["y"]).as_py(), pc.count(t["y"]).as_py()]
    assert got[()][2:4] == [_unscaled(pc.min(t["yd"]).as_py()), _unscaled(pc.sum(t["yd"]).as_py())]
    assert got[()][4:6] == [len(ux), pc.sum(ux).as_py()]
    assert abs(got[()][6] - pc.mean(ux).as_py()) <= 1e-12 * abs(pc.mean(ux).as_py())
    empty = _chain([]).answer(t.slice(0, 0))
    assert empty == {(): [None, 0, None, None, 0, None, None]}


def test_reference_stage3_offsets_advance_over_merging_aggregates_only():
    """Interleaved agg_exprs give the same answers as Spark's order (merging aggregates first), reordered."""
    t = _table(3)
    c = _chain([0])
    inter = D.Chain(DTS, [0], [1], c.ordinary, c.distinct_specs, [("d", 0), ("o", 0), ("o", 1), ("d", 1), ("o", 2), ("d", 2), ("o", 3)])
    a, b = c.answer(t), inter.answer(t)
    pos = {e: i for i, e in enumerate(c.order)}
    for k in a:
        assert b[k] == [a[k][pos[e]] for e in inter.order]


# ---- planning -----------------------------------------------------------------------------------------------------------------------
K, X = P.INT64, P.INT32


def supported(native, plan):
    ok, why = native.supports(plan)
    assert ok or why
    return ok


SUM_STATE = [P.DECIMAL(22, 2), P.BOOL]


def _stage3(expr_modes, mode=P.PARTIAL, offset=2, child=None, aggs=None):
    """group by k over (k, x, sum state...): SUM(y) merging, COUNT(x) Partial, in expr_modes' order"""
    child = child or P.scan([K, X] + SUM_STATE, source="shuffle")
    merge = P.agg_sum(P.unbound("y", P.DECIMAL(12, 2)), P.DECIMAL(22, 2))
    count = P.agg_count([P.bound(1, X)])
    if aggs is None:
        aggs = [merge if m != P.PARTIAL else count for m in expr_modes]
    return P.hash_agg(child, [P.bound(0, K)], aggs, mode, expr_modes=expr_modes, initial_input_buffer_offset=offset)


def test_mixed_modes_are_accepted(native):
    assert supported(native, _stage3([P.PARTIAL_MERGE, P.PARTIAL]))
    assert supported(native, _stage3([P.PARTIAL, P.PARTIAL_MERGE]))
    assert supported(native, _stage3([P.PARTIAL_MERGE, P.PARTIAL], mode=P.PARTIAL_MERGE))
    # uniform lists, and a PartialMerge operator with or without its offset
    assert supported(native, _stage3([P.PARTIAL_MERGE], mode=P.PARTIAL_MERGE))
    assert supported(native, P.hash_agg(P.scan([K, X] + SUM_STATE), [P.bound(0, K), P.bound(1, X)],
                                      [P.agg_sum(P.unbound("y", P.DECIMAL(12, 2)), P.DECIMAL(22, 2))], P.PARTIAL_MERGE, initial_input_buffer_offset=2))
    # a global distinct: no grouping keys, state from column 1
    g = P.hash_agg(P.scan([X] + SUM_STATE), [], [P.agg_sum(P.unbound("y", P.DECIMAL(12, 2)), P.DECIMAL(22, 2)), P.agg_count([P.bound(0, X)])],
                   P.PARTIAL, expr_modes=[P.PARTIAL_MERGE, P.PARTIAL], initial_input_buffer_offset=1)
    assert supported(native, g)


@pytest.mark.parametrize("modes,mode", [([P.PARTIAL_MERGE, P.FINAL], P.PARTIAL), ([P.FINAL, P.PARTIAL], P.PARTIAL),
                                        ([P.PARTIAL_MERGE, P.PARTIAL], P.FINAL), ([P.FINAL, P.FINAL], P.PARTIAL)])
def test_final_in_a_mixed_list_is_refused(native, modes, mode):
    assert not supported(native, _stage3(modes, mode=mode))
    with pytest.raises(native.Unsupported):
        native.compile_plan(_stage3(modes, mode=mode))


@pytest.mark.parametrize("what", ["length", "past_child", "state_type", "negative_offset"])
def test_malformed_mixed_plans_are_plan_errors(native, what):
    if what == "length":
        plan = _stage3([P.PARTIAL_MERGE, P.PARTIAL, P.PARTIAL], aggs=[P.agg_count([P.bound(1, X)])] * 2)
    elif what == "past_child":
        plan = _stage3([P.PARTIAL_MERGE, P.PARTIAL], offset=3)
    elif what == "state_type":
        plan = _stage3([P.PARTIAL_MERGE, P.PARTIAL], offset=1)   # the state would start at x (INT32), not the DECIMAL sum
    else:
        plan = _stage3([P.PARTIAL_MERGE, P.PARTIAL], offset=-1)
    with pytest.raises(native.CometB200Error) as e:
        native.compile_plan(plan)
    assert not isinstance(e.value, native.Unsupported)


def test_partial_expressions_read_any_child_column(native):
    """The Partial aggregate of a mixed operator is resolved against the whole child schema, state columns included."""
    child = P.scan([K, X] + SUM_STATE, source="shuffle")
    plan = _stage3([P.PARTIAL_MERGE, P.PARTIAL], aggs=[P.agg_sum(P.unbound("y", P.DECIMAL(12, 2)), P.DECIMAL(22, 2)),
                                                        P.agg_max(P.bound(2, P.DECIMAL(22, 2)), P.DECIMAL(22, 2))], child=child)
    with pytest.raises(native.Unsupported):  # MIN / MAX over decimal(p > 18) is outside the hot path: the argument was resolved
        native.compile_plan(plan)
    plan = _stage3([P.PARTIAL_MERGE, P.PARTIAL], aggs=[P.agg_sum(P.unbound("y", P.DECIMAL(12, 2)), P.DECIMAL(22, 2)),
                                                        P.agg_count([P.bound(3, P.BOOL)])], child=child)
    assert supported(native, plan)


def test_mixed_output_schema(native):
    """Group columns, then every aggregate's state columns in agg_exprs order -- the layout of a Partial operator."""
    t = _table(4).slice(0, 500)
    for modes in ([P.PARTIAL_MERGE, P.PARTIAL], [P.PARTIAL, P.PARTIAL_MERGE]):
        c = D.Chain(DTS, [0], [1], [R.Agg("sum", E.Col(3, P.DECIMAL(12, 2)), P.DECIMAL(22, 2))], [("count", None, None, R.LEGACY)],
                    [("o", 0), ("d", 0)] if modes[0] == P.PARTIAL_MERGE else [("d", 0), ("o", 0)])
        assert c.expr_modes() == modes
        want = [P.INT64] + ([P.DECIMAL(22, 2), P.BOOL, P.INT64] if modes[0] == P.PARTIAL_MERGE else [P.INT64, P.DECIMAL(22, 2), P.BOOL])
        assert [repr(x) for x in c.stage3_schema()] == [repr(x) for x in want]
        assert supported(native, c.stage3_plan())
        assert c.stage3(list(c.stage2(list(c.stage1(t).items())).items()))


# ---- every kernel of the GPU cases compiles --------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", distinctcases.CASES, ids=lambda c: c.name)
def test_distinct_chain_compiles(native, case):
    c = case.chain()
    for plan in (c.stage1_plan(), c.stage2_plan(case.offset2), c.stage3_plan(), c.stage4_plan()):
        assert native.compile_plan(plan)


@pytest.mark.parametrize("case", distinctcases.CASES, ids=lambda c: c.name)
def test_distinct_case_reference_runs(case):
    """Each case's stages chain on the CPU: stage 4 over stage 3 over ... is the whole answer, and it has every outer key."""
    c = case.chain()
    t = case.table()
    s3 = c.stage3(list(c.stage2(list(c.stage1(t).items())).items()))
    ans = c.answer(t)
    assert c.stage4(list(s3.items())) == ans
    keys = {tuple(r) for r in zip(*[R.pyvalues(t.column(i), d) for i, d in enumerate(c.key_types)])} if c.key_cols else {()}
    assert set(ans) == keys


def test_keys_only_final_compiles(native):
    for keys in ([P.INT64], [P.STRING], [P.BOOL, P.INT32]):
        plan = P.hash_agg(P.scan(keys, source="shuffle"), [P.bound(i, t) for i, t in enumerate(keys)], [], P.FINAL)
        assert native.compile_plan(plan)


def test_wide_decimal_distinct_column_is_refused(native):
    """A distinct column is a group key of stages 1 and 2; decimal(p > 18) keys do not pack into the hash key words."""
    c = D.Chain([P.INT64, P.DECIMAL(20, 2)], [0], [1], [], [("count", None, None, R.LEGACY)])
    assert not supported(native, c.stage1_plan())
