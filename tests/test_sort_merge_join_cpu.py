"""CPU: the SortMergeJoin reference (tests/smjref.py) against pyarrow's joins and hand-worked order cases, and which
SortMergeJoin plans the planner accepts, refuses (cb200_supports says no, code 1) or rejects as malformed (code 4), with their output
schemas and the pipeline kernels below and above a join (NVRTC, no device)."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

import joinref
import smjref as R


# ---- the reference ------------------------------------------------------------------------------------------------------------------------
def _sides(n_l, n_r, seed, dom):
    rng = np.random.default_rng(seed)
    def side(n, prefix):
        return pa.table({f"{prefix}a": pa.array(rng.integers(0, dom, n), mask=rng.random(n) < 0.1),
                         f"{prefix}b": pa.array([f"s{i}" for i in rng.integers(0, 3, n)], mask=rng.random(n) < 0.1),
                         f"{prefix}row": pa.array(np.arange(n))})
    return side(n_l, "l"), side(n_r, "r")


def _multiset(pairs):
    return sorted(pairs, key=lambda p: tuple((v is None, v or 0) for v in p))


@pytest.mark.parametrize("keys", [[0], [1], [0, 1]])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_reference_matches_pyarrow(keys, seed):
    """as multisets of (left row, right row): pyarrow matches no NULL key either and NULL-extends the same rows"""
    left, right = _sides(700, 500, seed, 40)
    lk, rk = [left.column_names[k] for k in keys], [right.column_names[k] for k in keys]
    for jt, pj in ((R.INNER, "inner"), (R.LEFT_OUTER, "left outer"), (R.RIGHT_OUTER, "right outer"), (R.FULL_OUTER, "full outer")):
        want = left.join(right, keys=lk, right_keys=rk, join_type=pj, coalesce_keys=False)
        got = R.sort_merge_join_table(left, right, keys, keys, jt)
        assert _multiset(zip(got.column(2).to_pylist(), got.column(5).to_pylist())) == \
            _multiset(zip(want.column("lrow").to_pylist(), want.column("rrow").to_pylist())), jt
    for jt, pj in ((R.LEFT_SEMI, "left semi"), (R.LEFT_ANTI, "left anti")):
        want = sorted(left.join(right, keys=lk, right_keys=rk, join_type=pj).column("lrow").to_pylist())
        assert sorted(R.sort_merge_join_table(left, right, keys, keys, jt).column(2).to_pylist()) == want


def _t(**cols):
    return pa.table({k: pa.array(v, pa.int64()) for k, v in cols.items()})


def _rows(t):
    return [tuple(r.values()) for r in t.to_pylist()]


def test_inner_semi_anti_are_the_hash_joins():
    """the types HashJoin also runs give its BuildRight output"""
    left, right = _sides(300, 200, 7, 30)
    for jt in (R.INNER, R.LEFT_SEMI, R.LEFT_ANTI):
        assert R.sort_merge_join_table(left, right, [0, 1], [0, 1], jt).equals(joinref.join_table(left, right, [0, 1], [0, 1], jt))


def test_left_outer_unmatched_row_in_its_place():
    left = _t(k=[1, 2, 3, 3], v=[10, 11, 12, 13])
    right = _t(k=[3, 1, 3], w=[20, 21, 22])
    assert _rows(R.sort_merge_join_table(left, right, [0], [0], R.LEFT_OUTER)) == [
        (1, 10, 1, 21), (2, 11, None, None), (3, 12, 3, 20), (3, 12, 3, 22), (3, 13, 3, 20), (3, 13, 3, 22)]


def test_right_outer_follows_right_order():
    """right rows in input order, each one's matches in left input order -- not the left order of the other types"""
    left = _t(k=[2, 1, 2], v=[10, 11, 12])
    right = _t(k=[1, 3, 2, None], w=[20, 21, 22, 23])
    assert _rows(R.sort_merge_join_table(left, right, [0], [0], R.RIGHT_OUTER)) == [
        (1, 11, 1, 20), (None, None, 3, 21), (2, 10, 2, 22), (2, 12, 2, 22), (None, None, None, 23)]
    assert _rows(R.sort_merge_join_table(left, right, [0], [0], R.INNER)) == [(2, 10, 2, 22), (1, 11, 1, 20), (2, 12, 2, 22)]


def test_full_outer_trailing_unmatched_right_rows():
    """everything LeftOuter gives, then the right rows no left row matched in right input order, NULL keys among them"""
    left = _t(k=[1, None, 4, 1], v=[10, 11, 12, 13])
    right = _t(k=[None, 5, 1, 7, None], w=[20, 21, 22, 23, 24])
    assert _rows(R.sort_merge_join_table(left, right, [0], [0], R.FULL_OUTER)) == [
        (1, 10, 1, 22), (None, 11, None, None), (4, 12, None, None), (1, 13, 1, 22),
        (None, None, None, 20), (None, None, 5, 21), (None, None, 7, 23), (None, None, None, 24)]


def _empty():
    return pa.table({"k": pa.array([], pa.int64()), "w": pa.array([], pa.int64())})


@pytest.mark.parametrize("jt,want", [(R.INNER, []), (R.LEFT_OUTER, [(1, 0, None, None), (None, 1, None, None)]), (R.RIGHT_OUTER, []),
                                     (R.FULL_OUTER, [(1, 0, None, None), (None, 1, None, None)]), (R.LEFT_SEMI, []),
                                     (R.LEFT_ANTI, [(1, 0), (None, 1)])])
def test_right_side_empty(jt, want):
    left = _t(k=[1, None], v=[0, 1])
    assert _rows(R.sort_merge_join_table(left, _empty(), [0], [0], jt)) == want


@pytest.mark.parametrize("jt,want", [(R.INNER, []), (R.LEFT_OUTER, []), (R.RIGHT_OUTER, [(None, None, 1, 0), (None, None, None, 1)]),
                                     (R.FULL_OUTER, [(None, None, 1, 0), (None, None, None, 1)]), (R.LEFT_SEMI, []), (R.LEFT_ANTI, [])])
def test_left_side_empty(jt, want):
    right = _t(k=[1, None], w=[0, 1])
    assert _rows(R.sort_merge_join_table(_empty(), right, [0], [0], jt)) == want


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


def _smj(P, ltypes, rtypes, lk, rk, jt=0, n_options=None, **kw):
    opts = [P.sort_order(P.bound(i, ltypes[i])) for i in lk]
    if n_options is not None:
        opts = [P.sort_order(P.bound(0, ltypes[0]))] * n_options
    return P.sort_merge_join(P.scan(ltypes), P.scan(rtypes), [P.bound(i, ltypes[i]) for i in lk], [P.bound(i, rtypes[i]) for i in rk], jt,
                             opts, **kw)


def _types(P):
    return [P.BOOL, P.INT8, P.INT16, P.INT32, P.INT64, P.DATE, P.TIMESTAMP, P.DT("TIMESTAMP_NTZ"), P.DECIMAL(9, 2), P.DECIMAL(18, 0),
            P.DECIMAL(38, 4), P.STRING]


def _jts(P):
    return [P.INNER, P.LEFT_OUTER, P.RIGHT_OUTER, P.FULL_OUTER, P.LEFT_SEMI, P.LEFT_ANTI]


def test_accepted_plans(native):
    from comet_b200 import proto as P
    types = _types(P)
    for i, t in enumerate(types):
        for jt in _jts(P):
            ok, _, why = _why(native, _smj(P, types, types[::-1], [i], [len(types) - 1 - i], jt))
            assert ok, (t, jt, why)
    seven_plus_bool = [0, 1, 2, 3, 5, 11, 4, 0]                            # 2 + 9 + 17 + 33 + 33 + 33 + 65 + 2 = 194
    for jt in _jts(P):
        assert _why(native, _smj(P, types, types, seven_plus_bool, seven_plus_bool, jt))[0], jt
    assert _why(native, _smj(P, types, types, [10, 9, 3], [10, 9, 3], P.FULL_OUTER))[0]   # 129 + 65 + 33


def test_refused_plans(native):
    """outside the operator's scope: cb200_supports says no with code 1 (Unsupported)"""
    from comet_b200 import proto as P
    types = [P.INT32] * 9 + [P.DOUBLE, P.FLOAT, P.DT("BYTES")]
    cases = [
        (_smj(P, types, types, [0], [0], condition=P.gt(P.bound(1, P.INT32), P.bound(11, P.INT32))), "condition"),
        (_smj(P, types, types, [0], [0], P.FULL_OUTER, condition=P.gt(P.bound(1, P.INT32), P.bound(11, P.INT32))), "condition"),
        (_smj(P, types, types, [9], [9]), "float64"),
        (_smj(P, types, types, [10], [10], P.LEFT_OUTER), "float32"),
        (_smj(P, types, types, [11], [11]), "binary"),
        (_smj(P, types, types, list(range(9)), list(range(9))), "more than 8 sort-merge join keys"),
        (_smj(P, types, types, list(range(8)), list(range(8))), "256 bits"),             # 8 x 33 bits
        (P.sort_merge_join(P.scan(types), P.scan(types), [P.add(P.bound(0, P.INT32), P.bound(1, P.INT32), P.INT32)], [P.bound(0, P.INT32)],
                           P.INNER, [P.sort_order(P.bound(0, P.INT32))]), "Projection below the join"),
    ]
    for plan, what in cases:
        ok, code, why = _why(native, plan)
        assert not ok and code == 1 and what in why, (what, code, why)
    assert _why(native, _smj(P, [P.INT16] * 8, [P.INT16] * 8, list(range(8)), list(range(8))))[0]   # 8 x 17 bits


def test_malformed_plans(native):
    """plan errors: cb200_supports says no with code 4"""
    from comet_b200 import proto as P
    types = [P.INT32, P.INT64, P.DECIMAL(12, 2), P.DECIMAL(12, 3)]
    cases = [
        (_smj(P, types, types, [], []), "without keys"),
        (_smj(P, types, types, [0, 1], [0]), "2 left keys and 1 right keys"),
        (P.sort_merge_join(P.scan(types), P.scan(types), [P.bound(4, P.INT32)], [P.bound(0, P.INT32)], P.INNER,
                           [P.sort_order(P.bound(0, P.INT32))]), "out of range"),
        (P.sort_merge_join(P.scan(types), P.scan(types[:2]), [P.bound(2, P.INT32)], [P.bound(2, P.INT32)], P.INNER,
                           [P.sort_order(P.bound(0, P.INT32))]), "out of range"),
        (_smj(P, types, types, [0], [1]), "int32 on the left and int64 on the right"),
        (_smj(P, types, types, [2], [3], P.FULL_OUTER), "decimal128(12,2) on the left and decimal128(12,3)"),
        (_smj(P, types, types, [0, 1], [0, 1], n_options=1), "1 sort options for 2 keys"),
        (_smj(P, types, types, [0], [0], n_options=0), "0 sort options for 1 keys"),
        (_smj(P, types, types, [0], [0], n_options=2), "2 sort options for 1 keys"),
        (_smj(P, types, types, [0], [0], 6), "unknown join type 6"),
    ]
    for plan, what in cases:
        ok, code, why = _why(native, plan)
        assert not ok and code == 4 and what in why, (what, code, why)


def test_output_schema(native):
    """inner and outer: the left columns, then the right ones; semi / anti: the left columns.  A Filter above the join compares each
    output column with a literal of the type it must have (a comparison of different types is refused)."""
    from comet_b200 import proto as P
    lt, rt = [P.INT32, P.STRING, P.DECIMAL(12, 2)], [P.INT64, P.INT32, P.DATE, P.BOOL]
    lit = {"INT32": 1, "INT64": 1, "DATE": 1, "BOOL": True, "DECIMAL": 1}
    for jt in _jts(P):
        schema = lt if jt in (P.LEFT_SEMI, P.LEFT_ANTI) else lt + rt
        j = _smj(P, lt, rt, [0], [1], jt)
        with native.Plan(j, []) as p:
            assert p.n_cols == len(schema)
        for i, t in enumerate(schema):
            if t.name == "STRING":
                continue
            assert _why(native, P.filter_(j, P.eq(P.bound(i, t), P.literal(lit[t.name], t))))[0], (jt, i, t)
            other = P.INT16 if t.name != "INT16" else P.INT32
            assert not _why(native, P.filter_(j, P.eq(P.bound(i, t), P.literal(1, other))))[0], (jt, i, t)
        assert _why(native, P.filter_(j, P.eq(P.bound(len(schema), P.INT32), P.literal(1, P.INT32))))[1] == 4   # past the last column


def test_pipelines_below_and_above_compile(native):
    """cb200_compile_plan walks both sides of a sort-merge join as it walks a hash join's: the pipeline above it, then the left child's,
    then the right child's, whichever side builds"""
    from comet_b200 import proto as P
    lt, rt = [P.INT64, P.DOUBLE, P.STRING], [P.STRING, P.INT32, P.DECIMAL(12, 2)]
    left = P.projection(P.filter_(P.scan(lt), P.gt(P.bound(1, P.DOUBLE), P.literal(0.5, P.DOUBLE))), [P.bound(0, P.INT64), P.bound(2, P.STRING)])
    right = P.filter_(P.scan(rt), P.is_not_null(P.bound(2, P.DECIMAL(12, 2))))
    below = native.compile_plan(left) + native.compile_plan(right)
    hj = P.hash_join(left, right, [P.bound(1, P.STRING)], [P.bound(0, P.STRING)], P.INNER, P.BUILD_RIGHT)
    assert native.compile_plan(hj) == below
    for jt in _jts(P):
        j = P.sort_merge_join(P.sort(left, [P.sort_order(P.bound(1, P.STRING))]), P.sort(right, [P.sort_order(P.bound(0, P.STRING))]),
                              [P.bound(1, P.STRING)], [P.bound(0, P.STRING)], jt, [P.sort_order(P.bound(1, P.STRING))])
        assert native.compile_plan(j) == below, jt
        above = P.hash_agg(P.projection(j, [P.bound(0, P.INT64), P.bound(1, P.STRING)]), [P.bound(1, P.STRING)],
                           [P.agg_sum(P.bound(0, P.INT64), P.INT64)], P.PARTIAL)
        keys = native.compile_plan(above)
        assert len(keys) > len(below) and keys[len(keys) - len(below):] == below, jt
