"""CPU: join conditions.  The reference (tests/condjoinref.py) against a brute-force nested-loop statement of the semantics and
hand-worked cases, and which HashJoin / SortMergeJoin plans with a condition the planner accepts, refuses (code 1) or rejects as
malformed (code 4), with the condition kernel's place in the compiled plan (NVRTC, no device)."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

import condjoinref as R
import exprs as E
from comet_b200 import proto as P
from joinref import INNER, LEFT_ANTI, LEFT_SEMI
from smjref import FULL_OUTER, LEFT_OUTER, RIGHT_OUTER, sort_merge_join_table
import joinref

JTS = [INNER, LEFT_OUTER, RIGHT_OUTER, FULL_OUTER, LEFT_SEMI, LEFT_ANTI]
JT = {INNER: 0, LEFT_OUTER: 1, RIGHT_OUTER: 2, FULL_OUTER: 3, LEFT_SEMI: 4, LEFT_ANTI: 5}


def _t(**cols):
    return pa.table({k: pa.array(v) for k, v in cols.items()})


def _rows(t):
    return [tuple(r.values()) for r in t.to_pylist()]


# ---- the reference against the nested loop ----------------------------------------------------------------------------------------------
def brute_force(left, right, lk, rk, jt, cond, build_left=False):
    """every (left row, right row) pair in probe-major order, a match when the keys are equal and non-NULL and the condition, evaluated on
    that one pair, is TRUE"""
    lkeys, rkeys = joinref.key_tuples(left, lk), joinref.key_tuples(right, rk)
    probe_right = jt == RIGHT_OUTER or (jt == INNER and build_left)
    order = ([(i, j) for j in range(right.num_rows) for i in range(left.num_rows)] if probe_right else
             [(i, j) for i in range(left.num_rows) for j in range(right.num_rows)])
    def ok(i, j):
        if lkeys[i] is None or lkeys[i] != rkeys[j]:
            return False
        return R.passes(left, right, [(i, j)], cond)[0]
    match = [(i, j) for i, j in order if ok(i, j)]
    if jt == INNER:
        return match
    lhit, rhit = {i for i, _ in match}, {j for _, j in match}
    if jt in (LEFT_SEMI, LEFT_ANTI):
        return [i for i in range(left.num_rows) if (i in lhit) == (jt == LEFT_SEMI)]
    if jt == RIGHT_OUTER:
        out = []
        for j in range(right.num_rows):
            out += [(i, jj) for i, jj in match if jj == j] or [(None, j)]
        return out
    out = []
    for i in range(left.num_rows):
        out += [(ii, j) for ii, j in match if ii == i] or [(i, None)]
    if jt == FULL_OUTER:
        out += [(None, j) for j in range(right.num_rows) if j not in rhit]
    return out


def _random_sides(seed, n_l, n_r, dom):
    rng = np.random.default_rng(seed)
    def side(n):
        return pa.table({"k": pa.array(rng.integers(0, dom, n), mask=rng.random(n) < 0.15),
                         "x": pa.array(rng.integers(-5, 5, n).astype(np.int32), mask=rng.random(n) < 0.15),
                         "f": pa.array(rng.standard_normal(n), mask=rng.random(n) < 0.1)})
    return side(n_l), side(n_r)


def _conds():
    lx, rx, lf, rf = E.Col(1, P.INT32), E.Col(4, P.INT32), E.Col(2, P.DOUBLE), E.Col(5, P.DOUBLE)
    return {"neq": E.Cmp("neq", lx, rx), "lt": E.Cmp("lt", lx, rx), "left_only": E.Cmp("gt_eq", lx, E.Lit(0, P.INT32)),
            "right_only": E.IsNull(rx), "or": E.Logic("or", E.Cmp("lt", lf, rf), E.IsNull(lx)),
            "case": E.If(E.Cmp("gt", lx, E.Lit(0, P.INT32)), E.Cmp("lt", lf, rf), E.Cmp("eq", lx, rx))}


@pytest.mark.parametrize("cond", list(_conds()))
@pytest.mark.parametrize("jt,build_left", [(jt, False) for jt in JTS] + [(INNER, True)])
@pytest.mark.parametrize("seed", [1, 2])
def test_reference_matches_the_nested_loop(seed, jt, build_left, cond):
    left, right = _random_sides(seed, 40, 30, 6)
    c = _conds()[cond]
    rows, n_cand = R.output_rows(left, right, [0], [0], jt, c, build_left)
    assert rows == brute_force(left, right, [0], [0], jt, c, build_left)
    assert n_cand == sum(1 for i in joinref.key_tuples(left, [0]) for j in joinref.key_tuples(right, [0]) if i is not None and i == j)


@pytest.mark.parametrize("jt,build_left", [(jt, False) for jt in JTS] + [(INNER, True)])
def test_literal_true_is_no_condition(jt, build_left):
    left, right = _random_sides(3, 60, 50, 8)
    got = R.cond_join_table(left, right, [0], [0], jt, E.Lit(True, P.BOOL), build_left)
    want = joinref.join_table(left, right, [0], [0], jt, build_left) if build_left else sort_merge_join_table(left, right, [0], [0], jt)
    assert _rows(got) == _rows(want)


# ---- hand-worked cases --------------------------------------------------------------------------------------------------------------------
LEFT = _t(k=[1, 1, 2, None, 3], a=[10, 20, 30, 40, 50])
RIGHT = _t(k=[1, 1, 2, 4, None], b=[15, 25, 5, 0, 99])
LT = E.Cmp("lt", E.Col(1, P.INT64), E.Col(3, P.INT64))   # l.a < r.b


def test_left_outer_row_whose_candidates_all_fail():
    """left row 1 (a=20) has candidates b=15 and b=25: 25 passes.  Row 2 (a=30) has b=5 only: it fails, so the row is NULL-extended"""
    got = _rows(R.cond_join_table(LEFT, RIGHT, [0], [0], LEFT_OUTER, LT))
    assert got == [(1, 10, 1, 15), (1, 10, 1, 25), (1, 20, 1, 25), (2, 30, None, None), (None, 40, None, None), (3, 50, None, None)]


def test_is_null_does_not_revive_an_unmatched_row():
    """r.b IS NULL is TRUE on a NULL-extended row, but the condition never sees one"""
    cond = E.IsNull(E.Col(3, P.INT64))
    got = _rows(R.cond_join_table(LEFT, RIGHT, [0], [0], LEFT_OUTER, cond))
    assert got == [(1, 10, None, None), (1, 20, None, None), (2, 30, None, None), (None, 40, None, None), (3, 50, None, None)]
    assert R.cond_join_table(LEFT, RIGHT, [0], [0], LEFT_SEMI, cond).num_rows == 0


def test_null_condition_is_no_match():
    left = _t(k=[1, 1], a=[None, 5])
    right = _t(k=[1], b=[3])
    cond = E.Cmp("gt", E.Col(1, P.INT64), E.Col(3, P.INT64))
    assert _rows(R.cond_join_table(left, right, [0], [0], INNER, cond)) == [(1, 5, 1, 3)]
    assert _rows(R.cond_join_table(left, right, [0], [0], LEFT_ANTI, cond)) == [(1, None)]
    assert _rows(R.cond_join_table(left, right, [0], [0], LEFT_OUTER, cond)) == [(1, None, None, None), (1, 5, 1, 3)]


def test_anti_keeps_null_keys_and_failed_rows():
    got = _rows(R.cond_join_table(LEFT, RIGHT, [0], [0], LEFT_ANTI, LT))
    assert got == [(2, 30), (None, 40), (3, 50)]
    assert _rows(R.cond_join_table(LEFT, RIGHT, [0], [0], LEFT_SEMI, LT)) == [(1, 10), (1, 20)]


def test_full_outer_build_row_whose_candidates_fail():
    """right row 2 (b=5) has one candidate (a=30), which fails: it leaves as unmatched, after the left rows, with the NULL-key row"""
    got = _rows(R.cond_join_table(LEFT, RIGHT, [0], [0], FULL_OUTER, LT))
    assert got == [(1, 10, 1, 15), (1, 10, 1, 25), (1, 20, 1, 25), (2, 30, None, None), (None, 40, None, None), (3, 50, None, None),
                   (None, None, 2, 5), (None, None, 4, 0), (None, None, None, 99)]
    assert _rows(R.cond_join_table(LEFT, RIGHT, [0], [0], RIGHT_OUTER, LT)) == [
        (1, 10, 1, 15), (1, 10, 1, 25), (1, 20, 1, 25), (None, None, 2, 5), (None, None, 4, 0), (None, None, None, 99)]


def test_ansi_error_only_from_candidates():
    """a + 1 overflows on left row 1 only; it raises when that row is a candidate"""
    big = 2**31 - 1
    left = pa.table({"k": pa.array([1, 2]), "a": pa.array([0, big], pa.int32())})
    cond = E.Cmp("gt", E.Arith("add", E.Col(1, P.INT32), E.Lit(1, P.INT32), P.INT32, E.ANSI), E.Lit(0, P.INT32))
    right = pa.table({"k": pa.array([1, 3]), "b": pa.array([0, 0], pa.int32())})
    assert _rows(R.cond_join_table(left, right, [0], [0], LEFT_OUTER, cond)) == [(1, 0, 1, 0), (2, big, None, None)]
    with pytest.raises(E.AnsiError):
        R.cond_join_table(left, pa.table({"k": pa.array([2]), "b": pa.array([0], pa.int32())}), [0], [0], LEFT_OUTER, cond)


# ---- the planner --------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def native():
    import comet_b200
    from comet_b200 import native
    return native


def _why(native, plan):
    err = native._Error()
    ok = native.lib().cb200_supports(plan, len(plan), C.byref(err))
    return ok, err.code, err.message.decode(errors="replace")


TYPES = [P.INT32, P.INT64, P.DOUBLE, P.DECIMAL(12, 2), P.STRING, P.DT("BYTES")]


def _hj(jt, build_left, cond, types=TYPES):
    return P.hash_join(P.scan(types), P.scan(types), [P.bound(0, P.INT32)], [P.bound(0, P.INT32)], jt, P.BUILD_LEFT if build_left else P.BUILD_RIGHT,
                       condition=cond)


def _smj(jt, cond, types=TYPES):
    return P.sort_merge_join(P.scan(types), P.scan(types), [P.bound(0, P.INT32)], [P.bound(0, P.INT32)], jt, [P.sort_order(P.bound(0, P.INT32))],
                             condition=cond)


def _accepted():
    out = [("hash", JT[INNER], False), ("hash", JT[INNER], True), ("hash", JT[LEFT_SEMI], False), ("hash", JT[LEFT_ANTI], False)]
    return out + [("smj", JT[jt], False) for jt in JTS]


def _plan(op, jt, build_left, cond):
    return _hj(jt, build_left, cond) if op == "hash" else _smj(jt, cond)


CONDS = [P.neq(P.bound(1, P.INT64), P.bound(7, P.INT64)),                                   # left vs right
         P.lt(P.bound(3, P.DECIMAL(12, 2)), P.bound(9, P.DECIMAL(12, 2))),
         P.is_null(P.bound(8, P.DOUBLE)),                                                    # right side only
         P.and_(P.gt(P.bound(2, P.DOUBLE), P.literal(0.5, P.DOUBLE)), P.is_not_null(P.bound(4, P.STRING))),
         P.eq(P.bound(10, P.STRING), P.literal("abc", P.STRING)),                            # a string predicate on a right column
         P.literal(True, P.BOOL)]


@pytest.mark.parametrize("op,jt,build_left", _accepted())
def test_every_accepted_join_accepts_a_condition(native, op, jt, build_left):
    for cond in CONDS:
        ok, code, why = _why(native, _plan(op, jt, build_left, cond))
        assert ok, (op, jt, build_left, code, why)


@pytest.mark.parametrize("op,jt,build_left", _accepted())
def test_plan_errors(native, op, jt, build_left):
    """a condition that is not boolean, or reads a column past left ++ right (12 columns): code 4"""
    for cond in (P.bound(1, P.INT64), P.add(P.bound(0, P.INT32), P.bound(6, P.INT32), P.INT32), P.is_null(P.bound(12, P.INT32))):
        ok, code, why = _why(native, _plan(op, jt, build_left, cond))
        assert not ok and code == 4 and "condition" in why, (cond, code, why)


@pytest.mark.parametrize("op,jt,build_left", _accepted())
def test_unsupported_expressions_are_refused_naming_the_condition(native, op, jt, build_left):
    for cond in (P.gt(P.bound(1, P.INT32), P.bound(11, P.INT32)),       # int32 vs binary
                 P.lt(P.bound(4, P.STRING), P.bound(10, P.STRING)),     # string column vs string column
                 P.gt(P.bound(0, P.INT32), P.bound(1, P.INT64))):       # int32 vs int64
        ok, code, why = _why(native, _plan(op, jt, build_left, cond))
        assert not ok and code == 1 and "condition" in why, (cond, code, why)


def test_scope_refusals_stay_with_a_condition(native):
    cond = CONDS[0]
    for jt in (JT[LEFT_OUTER], JT[RIGHT_OUTER], JT[FULL_OUTER]):
        ok, code, why = _why(native, _hj(jt, False, cond))
        assert not ok and code == 1 and "outer" in why, why
    for jt in (JT[LEFT_SEMI], JT[LEFT_ANTI]):
        ok, code, why = _why(native, _hj(jt, True, cond))
        assert not ok and code == 1 and "BuildLeft" in why, why
    plan = P.hash_join(P.scan(TYPES), P.scan(TYPES), [P.bound(0, P.INT32)], [P.bound(0, P.INT32)], JT[LEFT_ANTI], P.BUILD_RIGHT, condition=cond,
                       null_aware=True)
    ok, code, why = _why(native, plan)
    assert not ok and code == 1 and "null-aware" in why, why


def test_compile_plan_lists_the_condition_kernel_in_node_order(native):
    """cb200_compile_plan: the pipeline above the join, the join's condition, then the left child's and the right child's"""
    lt, rt = [P.INT64, P.DOUBLE, P.STRING], [P.STRING, P.INT32, P.DECIMAL(12, 2)]
    left = P.filter_(P.scan(lt), P.gt(P.bound(1, P.DOUBLE), P.literal(0.5, P.DOUBLE)))
    right = P.filter_(P.scan(rt), P.is_not_null(P.bound(2, P.DECIMAL(12, 2))))
    below = native.compile_plan(left) + native.compile_plan(right)
    cond = P.neq(P.bound(0, P.INT64), P.cast(P.bound(4, P.INT32), P.INT64))
    for op in ("hash", "smj"):
        for jt in ([0, 4, 5] if op == "hash" else range(6)):
            if op == "hash":
                j = P.hash_join(left, right, [P.bound(2, P.STRING)], [P.bound(0, P.STRING)], jt, P.BUILD_RIGHT, condition=cond)
                plain = P.hash_join(left, right, [P.bound(2, P.STRING)], [P.bound(0, P.STRING)], jt, P.BUILD_RIGHT)
            else:
                j = P.sort_merge_join(left, right, [P.bound(2, P.STRING)], [P.bound(0, P.STRING)], jt, [P.sort_order(P.bound(2, P.STRING))], condition=cond)
                plain = P.sort_merge_join(left, right, [P.bound(2, P.STRING)], [P.bound(0, P.STRING)], jt, [P.sort_order(P.bound(2, P.STRING))])
            keys = native.compile_plan(j)
            assert native.compile_plan(plain) == below
            assert len(keys) == len(below) + 1 and keys[1:] == below, (op, jt)
            assert keys[0] not in below
            above = native.compile_plan(P.projection(j, [P.add(P.bound(0, P.INT64), P.literal(1, P.INT64), P.INT64)]))
            assert len(above) == len(keys) + 1 and above[1:] == keys, (op, jt)
