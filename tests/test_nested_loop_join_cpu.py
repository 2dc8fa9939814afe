"""CPU: the BroadcastNestedLoopJoin reference (tests/nljref.py) against a brute-force nested loop and hand-worked cases, and which plans
the planner accepts (with their output schemas), refuses (code 1) or rejects as malformed (code 4), with the condition kernel's place in
the compiled plan (NVRTC, no device)."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

import condjoinref
import exprs as E
import nljref as R
from comet_b200 import proto as P
from joinref import INNER, LEFT_ANTI, LEFT_SEMI
from smjref import FULL_OUTER, LEFT_OUTER, RIGHT_OUTER

JT = {INNER: 0, LEFT_OUTER: 1, RIGHT_OUTER: 2, FULL_OUTER: 3, LEFT_SEMI: 4, LEFT_ANTI: 5}


def _t(**cols):
    return pa.table({k: pa.array(v) for k, v in cols.items()})


def _rows(t):
    return [tuple(r.values()) for r in t.to_pylist()]


# ---- the reference against the nested loop ----------------------------------------------------------------------------------------------
def brute_force(left, right, jt, cond, build_left):
    """two loops, the streamed side outside, the condition evaluated on one pair at a time"""
    def ok(i, j):
        return cond is None or condjoinref.passes(left, right, [(i, j)], cond)[0]
    n_l, n_r = left.num_rows, right.num_rows
    if jt in (LEFT_SEMI, LEFT_ANTI):
        return [i for i in range(n_l) if any(ok(i, j) for j in range(n_r)) == (jt == LEFT_SEMI)]
    out = []
    if build_left:   # the right side is streamed: Inner / BuildLeft and RightOuter
        for j in range(n_r):
            hits = [(i, j) for i in range(n_l) if ok(i, j)]
            out += hits or ([(None, j)] if jt == RIGHT_OUTER else [])
        return out
    for i in range(n_l):
        hits = [(i, j) for j in range(n_r) if ok(i, j)]
        out += hits or ([(i, None)] if jt == LEFT_OUTER else [])
    return out


def _random_sides(seed, n_l, n_r):
    rng = np.random.default_rng(seed)
    def side(n):
        return pa.table({"t": pa.array(rng.integers(0, 30, n), mask=rng.random(n) < 0.15),
                         "x": pa.array(rng.integers(-5, 5, n).astype(np.int32), mask=rng.random(n) < 0.15),
                         "f": pa.array(rng.standard_normal(n), mask=rng.random(n) < 0.1)})
    return side(n_l), side(n_r)


def _conds():
    lt, rt, lx, rx, lf, rf = E.Col(0, P.INT64), E.Col(3, P.INT64), E.Col(1, P.INT32), E.Col(4, P.INT32), E.Col(2, P.DOUBLE), E.Col(5, P.DOUBLE)
    return {"none": None, "lt": E.Cmp("lt", lx, rx), "band": E.Logic("and", E.Cmp("gt_eq", lt, rt), E.Cmp("lt", lt, E.Arith("add", rt, E.Lit(5, P.INT64), P.INT64))),
            "left_only": E.Cmp("gt_eq", lx, E.Lit(0, P.INT32)), "right_only": E.IsNull(rx), "or": E.Logic("or", E.Cmp("lt", lf, rf), E.IsNull(lx)),
            "case": E.If(E.Cmp("gt", lx, E.Lit(0, P.INT32)), E.Cmp("lt", lf, rf), E.Cmp("eq", lx, rx)),
            "not_in": E.Logic("and", E.Logic("or", E.Cmp("eq", lx, rx), E.IsNull(E.Cmp("eq", lx, rx))),
                              E.Logic("or", E.Cmp("eq", lt, rt), E.IsNull(E.Cmp("eq", lt, rt))))}


@pytest.mark.parametrize("cond", list(_conds()))
@pytest.mark.parametrize("jt,build_left", R.ACCEPTED)
@pytest.mark.parametrize("seed", [1, 2])
def test_reference_matches_the_nested_loop(seed, jt, build_left, cond):
    left, right = _random_sides(seed, 23, 17)
    c = _conds()[cond]
    rows, n_cand = R.output_rows(left, right, jt, c, build_left)
    assert rows == brute_force(left, right, jt, c, build_left)
    assert n_cand == (23 * 17 if c is not None else 0)
    got = R.nlj_table(left, right, jt, c, build_left)
    assert got.num_rows == len(rows)


@pytest.mark.parametrize("jt,build_left", R.ACCEPTED)
def test_conditions_give_true_false_and_null(jt, build_left):
    """x < r.x is NULL on a NULL x: such pairs fail, as FALSE ones do"""
    left, right = _random_sides(5, 30, 20)
    c = _conds()["lt"]
    ok = condjoinref.passes(left, right, R.candidates(30, 20, build_left), c)
    v, valid = c.eval(condjoinref.node_columns(condjoinref.pair_table(left, right, R.candidates(30, 20, build_left))))
    assert (~np.asarray(valid)).any() and (np.asarray(valid) & ~np.asarray(v, bool)).any() and any(ok)
    assert R.output_rows(left, right, jt, c, build_left)[0] == brute_force(left, right, jt, c, build_left)


def test_refused_shapes_have_no_reference():
    left, right = _random_sides(1, 3, 3)
    for jt, build_left in ((LEFT_OUTER, True), (RIGHT_OUTER, False), (FULL_OUTER, False), (FULL_OUTER, True), (LEFT_SEMI, True), (LEFT_ANTI, True)):
        with pytest.raises(ValueError):
            R.output_rows(left, right, jt, None, build_left)


# ---- hand-worked cases --------------------------------------------------------------------------------------------------------------------
EV = _t(t=[5, 12, None, 30])                       # event times
RG = _t(lo=[0, 10, 10], hi=[10, 20, 11])           # ranges [lo, hi)
BAND = E.Logic("and", E.Cmp("gt_eq", E.Col(0, P.INT64), E.Col(1, P.INT64)), E.Cmp("lt", E.Col(0, P.INT64), E.Col(2, P.INT64)))


def test_band_join():
    assert _rows(R.nlj_table(EV, RG, INNER, BAND)) == [(5, 0, 10), (12, 10, 20)]
    assert _rows(R.nlj_table(EV, RG, LEFT_OUTER, BAND)) == [(5, 0, 10), (12, 10, 20), (None, None, None), (30, None, None)]
    assert _rows(R.nlj_table(EV, RG, LEFT_SEMI, BAND)) == [(5,), (12,)]
    assert _rows(R.nlj_table(EV, RG, LEFT_ANTI, BAND)) == [(None,), (30,)]
    # BuildLeft streams the right side: its rows in order, each one's passing left rows in left order
    assert _rows(R.nlj_table(EV, RG, INNER, BAND, build_left=True)) == [(5, 0, 10), (12, 10, 20)]
    assert _rows(R.nlj_table(EV, RG, RIGHT_OUTER, BAND, build_left=True)) == [(5, 0, 10), (12, 10, 20), (None, 10, 11)]


def test_cross_product_order():
    l, r = _t(a=[1, 2]), _t(b=[10, 20, 30])
    assert _rows(R.nlj_table(l, r, INNER, None)) == [(1, 10), (1, 20), (1, 30), (2, 10), (2, 20), (2, 30)]
    assert _rows(R.nlj_table(l, r, INNER, None, build_left=True)) == [(1, 10), (2, 10), (1, 20), (2, 20), (1, 30), (2, 30)]


def test_empty_sides():
    empty = EV.slice(0, 0)
    none_r = RG.slice(0, 0)
    for cond in (None, BAND):
        assert R.nlj_table(EV, none_r, INNER, cond).num_rows == 0
        assert R.nlj_table(EV, none_r, LEFT_SEMI, cond).num_rows == 0
        assert _rows(R.nlj_table(EV, none_r, LEFT_ANTI, cond)) == [(5,), (12,), (None,), (30,)]
        assert _rows(R.nlj_table(EV, none_r, LEFT_OUTER, cond)) == [(5, None, None), (12, None, None), (None, None, None), (30, None, None)]
        assert _rows(R.nlj_table(none_r.select(["lo"]), RG, RIGHT_OUTER, None if cond is None else E.Cmp("lt", E.Col(0, P.INT64), E.Col(1, P.INT64)),
                                 build_left=True)) == [(None, 0, 10), (None, 10, 20), (None, 10, 11)]
        for jt, bl in R.ACCEPTED:   # an empty streamed side, or (Inner / BuildLeft) an empty build side with an inner join
            if jt != RIGHT_OUTER:
                assert R.nlj_table(empty, RG, jt, cond, bl).num_rows == 0
        assert R.output_rows(empty, RG, INNER, cond)[1] == 0


def test_literal_false_and_an_all_null_condition():
    false = E.Lit(False, P.BOOL)
    all_null = E.Cmp("lt", E.Col(0, P.INT64), E.Lit(None, P.INT64))
    for cond in (false, all_null):
        assert R.nlj_table(EV, RG, INNER, cond).num_rows == 0
        assert R.nlj_table(EV, RG, LEFT_SEMI, cond).num_rows == 0
        assert _rows(R.nlj_table(EV, RG, LEFT_ANTI, cond)) == [(5,), (12,), (None,), (30,)]
        assert _rows(R.nlj_table(EV, RG, LEFT_OUTER, cond)) == [(5, None, None), (12, None, None), (None, None, None), (30, None, None)]
        assert R.output_rows(EV, RG, INNER, cond)[1] == 12


def test_is_null_does_not_revive_an_extended_row():
    """r.lo IS NULL is TRUE on a NULL-extended row, but the condition never sees one"""
    cond = E.IsNull(E.Col(1, P.INT64))
    assert _rows(R.nlj_table(EV, RG, LEFT_OUTER, cond)) == [(5, None, None), (12, None, None), (None, None, None), (30, None, None)]


def test_multi_column_not_in():
    """(a, b) NOT IN (SELECT x, y): a left row is kept unless some right row makes every column's comparison TRUE or NULL"""
    left = _t(a=[1, 1, 2, None, 3], b=[1, 2, 2, 9, None])
    right = _t(x=[1, 2], y=[1, None])
    eq_or_null = lambda l, r: E.Logic("or", E.Cmp("eq", l, r), E.IsNull(E.Cmp("eq", l, r)))
    cond = E.Logic("and", eq_or_null(E.Col(0, P.INT64), E.Col(2, P.INT64)), eq_or_null(E.Col(1, P.INT64), E.Col(3, P.INT64)))
    # (1, 1) = (1, 1); (2, 2) vs (2, NULL) is NULL; (NULL, 9) vs (1, 1): NULL AND FALSE = FALSE, vs (2, NULL): NULL AND NULL -> dropped;
    # (3, NULL) vs (1, 1) FALSE, vs (2, NULL) FALSE -> kept; (1, 2) vs (1, 1) FALSE, vs (2, NULL) FALSE -> kept
    assert _rows(R.nlj_table(left, right, LEFT_ANTI, cond)) == [(1, 2), (3, None)]
    assert _rows(R.nlj_table(left, right.slice(0, 0), LEFT_ANTI, cond)) == _rows(left)


def test_ansi_error_only_from_a_pair():
    big = 2**31 - 1
    left = pa.table({"a": pa.array([0, big], pa.int32())})
    cond = E.Cmp("gt", E.Arith("add", E.Col(0, P.INT32), E.Lit(1, P.INT32), P.INT32, E.ANSI), E.Col(1, P.INT32))
    right = pa.table({"b": pa.array([0], pa.int32())})
    with pytest.raises(E.AnsiError):
        R.nlj_table(left, right, LEFT_OUTER, cond)
    assert _rows(R.nlj_table(left, right.slice(0, 0), LEFT_OUTER, cond)) == [(0, None), (big, None)]


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
SHAPES = [(JT[jt], bl) for jt, bl in R.ACCEPTED]
REFUSED = [(JT[LEFT_OUTER], True), (JT[RIGHT_OUTER], False), (JT[FULL_OUTER], False), (JT[FULL_OUTER], True), (JT[LEFT_SEMI], True),
           (JT[LEFT_ANTI], True)]
NAMES = {0: "inner", 1: "left outer", 2: "right outer", 3: "full outer", 4: "left semi", 5: "left anti"}


def _nlj(jt, build_left, cond, lt=TYPES, rt=TYPES):
    return P.broadcast_nested_loop_join(P.scan(lt), P.scan(rt), jt, P.BUILD_LEFT if build_left else P.BUILD_RIGHT, condition=cond)


CONDS = [None,
         P.neq(P.bound(1, P.INT64), P.bound(7, P.INT64)),                                   # left vs right
         P.lt(P.bound(3, P.DECIMAL(12, 2)), P.bound(9, P.DECIMAL(12, 2))),
         P.and_(P.gt_eq(P.bound(0, P.INT32), P.bound(6, P.INT32)), P.lt(P.bound(2, P.DOUBLE), P.bound(8, P.DOUBLE))),   # a band
         P.is_null(P.bound(8, P.DOUBLE)),                                                    # right side only
         P.eq(P.bound(10, P.STRING), P.literal("abc", P.STRING)),                            # a string predicate on a right column
         P.literal(True, P.BOOL), P.literal(False, P.BOOL)]


@pytest.mark.parametrize("jt,build_left", SHAPES)
def test_every_accepted_shape_with_and_without_a_condition(native, jt, build_left):
    for cond in CONDS:
        ok, code, why = _why(native, _nlj(jt, build_left, cond))
        assert ok, (jt, build_left, code, why)


COMPARABLE = [P.INT8, P.INT16, P.INT32, P.INT64, P.FLOAT, P.DOUBLE, P.DATE, P.TIMESTAMP, P.DECIMAL(12, 2), P.DECIMAL(30, 2), P.BOOL]


@pytest.mark.parametrize("t", COMPARABLE, ids=repr)
@pytest.mark.parametrize("jt,build_left", SHAPES)
def test_comparisons_over_every_type(native, jt, build_left, t):
    for cmp in (P.lt, P.gt_eq, P.neq):
        ok, code, why = _why(native, _nlj(jt, build_left, cmp(P.bound(0, t), P.bound(2, t)), [t, P.INT32], [t, P.INT32]))
        assert ok, (t, code, why)


@pytest.mark.parametrize("jt,build_left", SHAPES)
def test_output_schema(native, jt, build_left):
    """inner and outer: the left columns, then the right ones; semi / anti: the left columns.  A Filter above compares each output column
    with a literal of the type it must have (a comparison of different types is refused)."""
    lt, rt = [P.INT32, P.STRING, P.DECIMAL(12, 2)], [P.INT64, P.INT32, P.DATE, P.BOOL]
    lit = {"INT32": 1, "INT64": 1, "DATE": 1, "BOOL": True, "DECIMAL": 1}
    schema = lt if jt in (JT[LEFT_SEMI], JT[LEFT_ANTI]) else lt + rt
    for cond in (None, P.lt(P.bound(0, P.INT32), P.bound(4, P.INT32))):
        j = _nlj(jt, build_left, cond, lt, rt)
        with native.Plan(j, []) as p:
            assert p.n_cols == len(schema)
        for i, t in enumerate(schema):
            if t.name == "STRING":
                continue
            assert _why(native, P.filter_(j, P.eq(P.bound(i, t), P.literal(lit[t.name], t))))[0], (jt, i, t)
            other = P.INT16 if t.name != "INT16" else P.INT32
            assert not _why(native, P.filter_(j, P.eq(P.bound(i, t), P.literal(1, other))))[0], (jt, i, t)
        assert _why(native, P.filter_(j, P.eq(P.bound(len(schema), P.INT32), P.literal(1, P.INT32))))[1] == 4   # past the last column


@pytest.mark.parametrize("jt,build_left", REFUSED)
def test_refused_shapes_name_the_join_type_and_build_side(native, jt, build_left):
    for cond in (None, CONDS[1]):
        ok, code, why = _why(native, _nlj(jt, build_left, cond))
        assert not ok and code == 1, (code, why)
        assert NAMES[jt] + " nested-loop join" in why and ("BuildLeft" if build_left else "BuildRight") in why, why


def test_a_side_without_columns_is_refused(native):
    """a COUNT(*) over a cross join may prune a side to no columns"""
    for lt, rt in (([], TYPES), (TYPES, []), ([], [])):
        for jt, bl in SHAPES:
            ok, code, why = _why(native, _nlj(jt, bl, None, lt, rt))
            assert not ok and code == 1 and "without columns" in why, (lt, rt, code, why)


def test_plan_errors(native):
    one_child = P._op("broadcast_nested_loop_join", P.f_varint(1, 0) + P.f_varint(2, 1), (P.scan(TYPES),))
    three = P._op("broadcast_nested_loop_join", P.f_varint(1, 0) + P.f_varint(2, 1), (P.scan(TYPES),) * 3)
    cases = [(one_child, "two children"), (three, "two children"), (_nlj(6, False, None), "join type"), (_nlj(-1, False, None), "join type"),
             (P.broadcast_nested_loop_join(P.scan(TYPES), P.scan(TYPES), 0, 2), "build side")]
    for plan, what in cases:
        ok, code, why = _why(native, plan)
        assert not ok and code == 4 and what in why, (what, code, why)


@pytest.mark.parametrize("jt,build_left", SHAPES)
def test_condition_plan_errors(native, jt, build_left):
    """a condition that is not boolean, or reads a column past left ++ right (12 columns): code 4"""
    for cond in (P.bound(1, P.INT64), P.add(P.bound(0, P.INT32), P.bound(6, P.INT32), P.INT32), P.is_null(P.bound(12, P.INT32))):
        ok, code, why = _why(native, _nlj(jt, build_left, cond))
        assert not ok and code == 4 and "condition" in why, (cond, code, why)


@pytest.mark.parametrize("jt,build_left", SHAPES)
def test_unsupported_expressions_are_refused_naming_the_condition(native, jt, build_left):
    for cond in (P.gt(P.bound(1, P.INT32), P.bound(11, P.INT32)),       # int32 vs binary
                 P.lt(P.bound(4, P.STRING), P.bound(10, P.STRING)),     # string column vs string column
                 P.gt(P.bound(0, P.INT32), P.bound(1, P.INT64))):       # int32 vs int64
        ok, code, why = _why(native, _nlj(jt, build_left, cond))
        assert not ok and code == 1 and why.startswith("join condition: "), (cond, code, why)


def test_compile_plan_lists_the_condition_kernel_in_node_order(native):
    """cb200_compile_plan: the pipeline above the join, the join's condition, then the left child's and the right child's; a join
    without a condition compiles no kernel of its own"""
    lt, rt = [P.INT64, P.DOUBLE, P.STRING], [P.STRING, P.INT32, P.DECIMAL(12, 2)]
    left = P.filter_(P.scan(lt), P.gt(P.bound(1, P.DOUBLE), P.literal(0.5, P.DOUBLE)))
    right = P.filter_(P.scan(rt), P.is_not_null(P.bound(2, P.DECIMAL(12, 2))))
    below = native.compile_plan(left) + native.compile_plan(right)
    cond = P.neq(P.bound(0, P.INT64), P.cast(P.bound(4, P.INT32), P.INT64))
    for jt, bl in SHAPES:
        side = P.BUILD_LEFT if bl else P.BUILD_RIGHT
        j = P.broadcast_nested_loop_join(left, right, jt, side, condition=cond)
        plain = P.broadcast_nested_loop_join(left, right, jt, side)
        keys = native.compile_plan(j)
        assert native.compile_plan(plain) == below
        assert len(keys) == len(below) + 1 and keys[1:] == below, (jt, bl)
        assert keys[0] not in below
        above = native.compile_plan(P.projection(j, [P.add(P.bound(0, P.INT64), P.literal(1, P.INT64), P.INT64)]))
        assert len(above) == len(keys) + 1 and above[1:] == keys, (jt, bl)
        lit = native.compile_plan(P.broadcast_nested_loop_join(left, right, jt, side, condition=P.literal(False, P.BOOL)))
        assert len(lit) == len(below) + 1 and lit[1:] == below, (jt, bl)
