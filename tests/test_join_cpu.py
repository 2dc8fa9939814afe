"""CPU: the HashJoin reference (tests/joinref.py) against pyarrow's hash join and hand-worked cases, and which HashJoin plans the planner
accepts, refuses (cb200_supports says no, code 1) or rejects as malformed (code 4), with their output schemas and the pipeline kernels
below and above a join (NVRTC, no device)."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

import joinref as R


# ---- the reference ------------------------------------------------------------------------------------------------------------------------
def _pairs(t, lcol, rcol):
    return sorted(zip(t.column(lcol).to_pylist(), t.column(rcol).to_pylist()))


def _sides(n_l, n_r, seed, dom):
    rng = np.random.default_rng(seed)
    def side(n, prefix):
        return pa.table({f"{prefix}a": pa.array(rng.integers(0, dom, n), mask=rng.random(n) < 0.1),
                         f"{prefix}b": pa.array([f"s{i}" for i in rng.integers(0, 3, n)], mask=rng.random(n) < 0.1),
                         f"{prefix}row": pa.array(np.arange(n))})
    return side(n_l, "l"), side(n_r, "r")


@pytest.mark.parametrize("keys", [[0], [1], [0, 1]])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_reference_matches_pyarrow(keys, seed):
    """as multisets: pyarrow's hash join does not match NULL keys either, and its row order is its own"""
    left, right = _sides(700, 500, seed, 40)
    lk, rk = [left.column_names[k] for k in keys], [right.column_names[k] for k in keys]
    inner = left.join(right, keys=lk, right_keys=rk, join_type="inner", coalesce_keys=False)
    for build_left in (False, True):
        got = R.join_table(left, right, keys, keys, R.INNER, build_left)
        assert _pairs(got, 2, 5) == _pairs(inner, "lrow", "rrow")
    for jt, pj in ((R.LEFT_SEMI, "left semi"), (R.LEFT_ANTI, "left anti")):
        want = sorted(left.join(right, keys=lk, right_keys=rk, join_type=pj).column("lrow").to_pylist())
        assert sorted(R.join_table(left, right, keys, keys, jt).column(2).to_pylist()) == want


def _t(**cols):
    return pa.table({k: pa.array(v) for k, v in cols.items()})


def _rows(t):
    return [tuple(r.values()) for r in t.to_pylist()]


def test_null_keys_on_each_side():
    left = _t(k=[1, None, 2, None], v=[10, 11, 12, 13])
    right = _t(k=[None, 1, 2, None], w=[20, 21, 22, 23])
    assert _rows(R.join_table(left, right, [0], [0], R.INNER)) == [(1, 10, 1, 21), (2, 12, 2, 22)]
    assert _rows(R.join_table(left, right, [0], [0], R.LEFT_SEMI)) == [(1, 10), (2, 12)]
    assert _rows(R.join_table(left, right, [0], [0], R.LEFT_ANTI)) == [(None, 11), (None, 13)]   # a NULL key matches nothing: kept


def test_n_to_m_duplicates_and_order():
    """probe rows in input order, each one's matches in build input order; BuildLeft probes the right side"""
    left = _t(k=[5, 7, 5, 9], v=[0, 1, 2, 3])
    right = _t(k=[5, 5, 7, 8, 5], w=[0, 1, 2, 3, 4])
    assert _rows(R.join_table(left, right, [0], [0], R.INNER)) == [
        (5, 0, 5, 0), (5, 0, 5, 1), (5, 0, 5, 4), (7, 1, 7, 2), (5, 2, 5, 0), (5, 2, 5, 1), (5, 2, 5, 4)]
    assert _rows(R.join_table(left, right, [0], [0], R.INNER, build_left=True)) == [
        (5, 0, 5, 0), (5, 2, 5, 0), (5, 0, 5, 1), (5, 2, 5, 1), (7, 1, 7, 2), (5, 0, 5, 4), (5, 2, 5, 4)]
    assert _rows(R.join_table(left, right, [0], [0], R.LEFT_SEMI)) == [(5, 0), (7, 1), (5, 2)]
    assert _rows(R.join_table(left, right, [0], [0], R.LEFT_ANTI)) == [(9, 3)]


def test_empty_build_side():
    left = _t(k=[1, None, 2], v=[0, 1, 2])
    right = pa.table({"k": pa.array([], pa.int64()), "w": pa.array([], pa.int64())})
    assert R.join_table(left, right, [0], [0], R.INNER).num_rows == 0
    assert R.join_table(left, right, [0], [0], R.LEFT_SEMI).num_rows == 0
    assert _rows(R.join_table(left, right, [0], [0], R.LEFT_ANTI)) == [(1, 0), (None, 1), (2, 2)]
    assert R.join_table(right, left, [0], [0], R.INNER, build_left=True).num_rows == 0


def test_multi_key_equal_in_one_key_only():
    left = _t(a=[1, 1, 2, 2], b=["x", "y", "x", None])
    right = _t(a=[1, 2, 2], b=["y", "y", None])
    assert _rows(R.join_table(left, right, [0, 1], [0, 1], R.INNER)) == [(1, "y", 1, "y")]
    assert _rows(R.join_table(left, right, [0, 1], [0, 1], R.LEFT_ANTI)) == [(1, "x"), (2, "x"), (2, None)]


def test_strings_compare_by_value_not_code():
    """dictionaries that differ between the sides, and one that repeats a value"""
    left = pa.table({"s": pa.DictionaryArray.from_arrays(pa.array([0, 1, 2, 3]), pa.array(["a", "b", "a", "c"]))})
    right = pa.table({"s": pa.DictionaryArray.from_arrays(pa.array([1, 0]), pa.array(["c", "a"]))})
    assert _rows(R.join_table(left, right, [0], [0], R.INNER)) == [("a", "a"), ("a", "a"), ("c", "c")]


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


def _join(P, ltypes, rtypes, lk, rk, jt=0, build=1, **kw):
    return P.hash_join(P.scan(ltypes), P.scan(rtypes), [P.bound(i, ltypes[i]) for i in lk], [P.bound(i, rtypes[i]) for i in rk], jt, build, **kw)


def _types(P):
    return [P.BOOL, P.INT8, P.INT16, P.INT32, P.INT64, P.DATE, P.TIMESTAMP, P.DT("TIMESTAMP_NTZ"), P.DECIMAL(9, 2), P.DECIMAL(18, 0),
            P.DECIMAL(38, 4), P.STRING]


def test_accepted_plans(native):
    from comet_b200 import proto as P
    types = _types(P)
    for i, t in enumerate(types):
        for jt, build in ((P.INNER, P.BUILD_RIGHT), (P.INNER, P.BUILD_LEFT), (P.LEFT_SEMI, P.BUILD_RIGHT), (P.LEFT_ANTI, P.BUILD_RIGHT)):
            ok, _, why = _why(native, _join(P, types, types[::-1], [i], [len(types) - 1 - i], jt, build))
            assert ok, (t, jt, build, why)
    eight = [0, 1, 2, 3, 5, 11, 4, 8]                                      # 2 + 9 + 17 + 33 + 33 + 33 + 65 + 65 = 257 > 256
    assert not _why(native, _join(P, types, types, eight, eight))[0]
    seven_plus_bool = [0, 1, 2, 3, 5, 11, 4, 0]                            # 2 + 9 + 17 + 33 + 33 + 33 + 65 + 2 = 194
    assert _why(native, _join(P, types, types, seven_plus_bool, seven_plus_bool))[0]
    assert _why(native, _join(P, types, types, [10, 9, 3], [10, 9, 3]))[0]   # 129 + 65 + 33
    ok, code, why = _why(native, _join(P, types, types, [10, 9, 4], [10, 9, 4]))   # 129 + 65 + 65
    assert not ok and code == 1 and "256 bits" in why


def test_refused_plans(native):
    """outside the operator's scope: cb200_supports says no with code 1 (Unsupported)"""
    from comet_b200 import proto as P
    types = [P.INT32] * 9 + [P.DOUBLE, P.FLOAT, P.DT("BYTES")]
    cases = [
        (_join(P, types, types, [0], [0], P.LEFT_OUTER), "outer"),
        (_join(P, types, types, [0], [0], P.RIGHT_OUTER), "outer"),
        (_join(P, types, types, [0], [0], P.FULL_OUTER), "outer"),
        (_join(P, types, types, [0], [0], P.LEFT_SEMI, P.BUILD_LEFT), "BuildLeft"),
        (_join(P, types, types, [0], [0], P.LEFT_ANTI, P.BUILD_LEFT), "BuildLeft"),
        (_join(P, types, types, [0], [0], condition=P.gt(P.bound(1, P.INT32), P.bound(11, P.INT32))), "condition"),
        (_join(P, types, types, [0], [0], P.LEFT_ANTI, null_aware=True), "null-aware"),
        (_join(P, types, types, [9], [9]), "float64"),
        (_join(P, types, types, [10], [10]), "float32"),
        (_join(P, types, types, [11], [11]), "binary"),
        (_join(P, types, types, list(range(9)), list(range(9))), "8 hash join keys"),
        (_join(P, types, types, list(range(8)), list(range(8))), "256 bits"),             # 8 x 33 bits
        (P.hash_join(P.scan(types), P.scan(types), [P.add(P.bound(0, P.INT32), P.bound(1, P.INT32), P.INT32)], [P.bound(0, P.INT32)],
                     P.INNER, P.BUILD_RIGHT), "Projection below the join"),
    ]
    for plan, what in cases:
        ok, code, why = _why(native, plan)
        assert not ok and code == 1 and what in why, (what, code, why)
    assert _why(native, _join(P, [P.INT16] * 8, [P.INT16] * 8, list(range(8)), list(range(8))))[0]   # 8 x 17 bits


def test_malformed_plans(native):
    """plan errors: cb200_supports says no with code 4"""
    from comet_b200 import proto as P
    types = [P.INT32, P.INT64, P.DECIMAL(12, 2), P.DECIMAL(12, 3)]
    cases = [
        (_join(P, types, types, [], []), "without keys"),
        (_join(P, types, types, [0, 1], [0]), "2 left keys and 1 right keys"),
        (P.hash_join(P.scan(types), P.scan(types), [P.bound(4, P.INT32)], [P.bound(0, P.INT32)], P.INNER, P.BUILD_RIGHT), "out of range"),
        (P.hash_join(P.scan(types), P.scan(types[:2]), [P.bound(2, P.INT32)], [P.bound(2, P.INT32)], P.INNER, P.BUILD_RIGHT), "out of range"),
        (_join(P, types, types, [0], [1]), "int32 on the left and int64 on the right"),
        (_join(P, types, types, [2], [3]), "decimal128(12,2) on the left and decimal128(12,3)"),
    ]
    for plan, what in cases:
        ok, code, why = _why(native, plan)
        assert not ok and code == 4 and what in why, (what, code, why)


def test_output_schema(native):
    """inner: the left columns, then the right ones, whatever the build side; semi / anti: the left columns.  A Filter above the join
    compares each output column with a literal of the type it must have (a comparison of different types is refused)."""
    from comet_b200 import proto as P
    lt, rt = [P.INT32, P.STRING, P.DECIMAL(12, 2)], [P.INT64, P.INT32, P.DATE, P.BOOL]
    lit = {"INT32": 1, "INT64": 1, "DATE": 1, "BOOL": True, "DECIMAL": 1}
    for jt, build, schema in ((P.INNER, P.BUILD_RIGHT, lt + rt), (P.INNER, P.BUILD_LEFT, lt + rt), (P.LEFT_SEMI, P.BUILD_RIGHT, lt),
                              (P.LEFT_ANTI, P.BUILD_RIGHT, lt)):
        j = _join(P, lt, rt, [0], [1], jt, build)
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
    """cb200_compile_plan walks both sides of a join: the pipeline above it, then the left child's, then the right child's"""
    from comet_b200 import proto as P
    lt, rt = [P.INT64, P.DOUBLE, P.STRING], [P.STRING, P.INT32, P.DECIMAL(12, 2)]
    left = P.projection(P.filter_(P.scan(lt), P.gt(P.bound(1, P.DOUBLE), P.literal(0.5, P.DOUBLE))), [P.bound(0, P.INT64), P.bound(2, P.STRING)])
    right = P.filter_(P.scan(rt), P.is_not_null(P.bound(2, P.DECIMAL(12, 2))))
    for jt, build in ((P.INNER, P.BUILD_LEFT), (P.INNER, P.BUILD_RIGHT), (P.LEFT_SEMI, P.BUILD_RIGHT)):
        j = P.hash_join(left, right, [P.bound(1, P.STRING)], [P.bound(0, P.STRING)], jt, build)
        below = native.compile_plan(left) + native.compile_plan(right)
        assert native.compile_plan(j) == below
        above = P.hash_agg(P.projection(j, [P.bound(0, P.INT64), P.bound(1, P.STRING)]), [P.bound(1, P.STRING)],
                           [P.agg_sum(P.bound(0, P.INT64), P.INT64)], P.PARTIAL)
        keys = native.compile_plan(above)
        assert len(keys) > len(below) and keys[len(keys) - len(below):] == below
