"""CPU: the stacked row-operator plans of tests/test_gpu_operator_stacks.py -- accepted by the planner, their pipeline kernels compiled
in the documented walk order (NVRTC, no device) -- and the composition of the CPU references those tests rely on, pinned on small
hand-worked cases."""
import numpy as np
import pyarrow as pa
import pytest

import joinref as J
import partref
import sortref as S


@pytest.fixture(scope="module")
def native():
    import comet_b200
    from comet_b200 import native
    return native


def _join(P, l, lt, r, rt, lk, rk, jt=0, build=1):
    return P.hash_join(l, r, [P.bound(i, lt[i]) for i in lk], [P.bound(i, rt[i]) for i in rk], jt, build)


def _sort(P, child, types, keys, fetch=None, skip=None):
    return P.sort(child, [P.sort_order(P.bound(i, types[i]), d, nf) for i, d, nf in keys], fetch=fetch, skip=skip)


def stacked_plans(P):
    """name -> plan: one of each stack the GPU suite runs"""
    side = [P.INT32, P.BOOL, P.INT64, P.DOUBLE, P.STRING]                 # k0, k1, row, pf, ps
    scan = lambda: P.scan(side)
    inner = _join(P, scan(), side, scan(), side, [0], [0], P.INNER, P.BUILD_RIGHT)
    dec = P.DECIMAL(12, 2)
    state = [P.STRING, P.BOOL, P.DECIMAL(22, 2), P.BOOL, P.INT64]
    partial = P.hash_agg(P.scan([P.STRING, P.BOOL, dec]), [P.bound(0, P.STRING), P.bound(1, P.BOOL)],
                         [P.agg_sum(P.bound(2, dec), P.DECIMAL(22, 2)), P.agg_count([P.bound(2, dec)])], P.PARTIAL)
    plans = {}
    for jt, build in ((P.INNER, P.BUILD_RIGHT), (P.INNER, P.BUILD_LEFT), (P.LEFT_SEMI, P.BUILD_RIGHT), (P.LEFT_ANTI, P.BUILD_RIGHT)):
        j = _join(P, scan(), side, scan(), side, [0], [0], jt, build)
        types = side + side if jt == P.INNER else side
        for fetch, skip in ((None, None), (700, None), (900, 150), (0, None)):
            plans[f"sort_over_join_{jt}_{build}_{fetch}_{skip}"] = _sort(P, j, types, [(1, False, True), (4, True, True)], fetch, skip)
        plans[f"join_over_sort_{jt}_{build}"] = _join(P, _sort(P, scan(), side, [(4, False, True)], 1500), side,
                                                      _sort(P, scan(), side, [(4, True, False)]), side, [4], [4], jt, build)
        plans[f"join_over_join_{jt}"] = _join(P, inner, side + side, P.scan([P.STRING, P.INT64]), [P.STRING, P.INT64], [9], [0], jt)
        plans[f"join_over_anti_{jt}"] = _join(P, _join(P, scan(), side, scan(), side, [0], [0], P.LEFT_ANTI), side,
                                              P.scan([P.STRING, P.INT64]), [P.STRING, P.INT64], [4], [0], jt)
        plans[f"join_built_on_partial_{jt}"] = _join(P, P.scan([P.STRING, P.BOOL, P.INT64]), [P.STRING, P.BOOL, P.INT64], partial, state,
                                                     [0, 1], [0, 1], jt)
    hp = P.hash_partitioning([P.bound(1, P.BOOL), P.bound(0, P.INT32), P.bound(4, P.STRING)], 200)
    plans["partition_over_join"] = P.shuffle_writer(inner, hp)
    plans["partition_over_sort"] = P.shuffle_writer(_sort(P, inner, side + side, [(2, False, True)]), hp)
    plans["partition_over_partial"] = P.shuffle_writer(partial, P.hash_partitioning([P.bound(1, P.BOOL), P.bound(3, P.BOOL)], 7))
    plans["agg_over_sort"] = P.hash_agg(P.filter_(_sort(P, scan(), side, [(2, False, True)]), P.eq(P.bound(4, P.STRING), P.literal("ab", P.STRING))),
                                        [P.bound(2, P.INT64)], [P.agg_sum(P.bound(0, P.INT32), P.INT64), P.agg_count([P.bound(3, P.DOUBLE)])], P.PARTIAL)
    plans["agg_over_join"] = P.hash_agg(inner, [P.bound(1, P.BOOL), P.bound(9, P.STRING)],
                                        [P.agg_min(P.bound(3, P.DOUBLE), P.DOUBLE), P.agg_max(P.bound(7, P.INT64), P.INT64)], P.PARTIAL)
    for fetch in (None, 40):
        plans[f"sort_over_partial_{fetch}"] = _sort(P, partial, state, [(1, False, True), (3, True, False), (0, False, True)], fetch)
    return plans


def test_stacked_plans_accepted(native):
    from comet_b200 import proto as P
    for name, plan in stacked_plans(P).items():
        ok, why = native.supports(plan)
        assert ok, (name, why)


def test_stacked_plans_compile_in_walk_order(native):
    """cb200_compile_plan lists a node's own pipeline kernels, then its left child's, then its right child's"""
    from comet_b200 import proto as P
    side = [P.INT32, P.BOOL, P.INT64, P.DOUBLE, P.STRING]
    pos = lambda child: P.filter_(child, P.gt(P.bound(3, P.DOUBLE), P.literal(0.0, P.DOUBLE)))
    below_l, below_r = pos(P.scan(side)), P.filter_(P.scan(side), P.is_not_null(P.bound(1, P.BOOL)))
    kl, kr = native.compile_plan(below_l), native.compile_plan(below_r)
    assert kl and kr and kl != kr
    # an aggregate over a Sort: the aggregate's kernels, then those below the Sort
    srt = _sort(P, below_l, side, [(2, False, True)])
    agg = lambda child: P.hash_agg(P.filter_(child, P.eq(P.bound(4, P.STRING), P.literal("ab", P.STRING))), [P.bound(2, P.INT64)],
                                   [P.agg_sum(P.bound(0, P.INT32), P.INT64)], P.PARTIAL)
    own = native.compile_plan(agg(P.scan(side)))
    assert own and native.compile_plan(agg(srt)) == own + kl
    # an aggregate over a join: the aggregate's kernels, then the left child's, then the right child's, whichever side builds
    for build in (P.BUILD_RIGHT, P.BUILD_LEFT):
        j = _join(P, below_l, side, below_r, side, [0], [0], P.INNER, build)
        agg_j = lambda child: P.hash_agg(child, [P.bound(1, P.BOOL), P.bound(9, P.STRING)], [P.agg_max(P.bound(7, P.INT64), P.INT64)], P.PARTIAL)
        own = native.compile_plan(agg_j(P.scan(side + side)))
        assert own and native.compile_plan(agg_j(j)) == own + kl + kr
    # a join over a join over a Sort: the inner join's left (the Sort's child), its right, then the outer right
    inner = _join(P, srt, side, below_r, side, [0], [0])
    outer = _join(P, inner, side + side, pos(P.scan(side)), side, [2], [2], P.LEFT_SEMI)
    assert native.compile_plan(outer) == kl + kr + kl
    # a ShuffleWriter over a Sort over a join
    assert native.compile_plan(P.shuffle_writer(_sort(P, inner, side + side, [(2, False, True)]), P.hash_partitioning([P.bound(1, P.BOOL)], 8))) == kl + kr


# ---- the references composed ----------------------------------------------------------------------------------------------------------
def _sides():
    probe = pa.table({"k": pa.array([2, 1, 2, None, 3, 1], pa.int64()), "p": pa.array(["a", "b", "c", "d", "e", "f"])})
    build = pa.table({"k": pa.array([1, 2, 1, 2, 4], pa.int64()), "b": pa.array([10, 20, 30, 40, 50], pa.int64())})
    return probe, build


def test_sort_ties_over_join_follow_join_order():
    """join output: probe rows in order, each one's matches in build order; a sort on a key with ties keeps that order"""
    probe, build = _sides()
    j = J.join_table(probe, build, [0], [0], J.INNER)
    assert list(zip(j.column("l1").to_pylist(), j.column("r1").to_pylist())) == \
        [("a", 20), ("a", 40), ("b", 10), ("b", 30), ("c", 20), ("c", 40), ("f", 10), ("f", 30)]
    s = S.sort_table(j, [(0, False, True)])                                # by k: 1 before 2, ties in join order
    assert list(zip(s.column("l1").to_pylist(), s.column("r1").to_pylist())) == \
        [("b", 10), ("b", 30), ("f", 10), ("f", 30), ("a", 20), ("a", 40), ("c", 20), ("c", 40)]
    s = S.sort_table(j, [(0, True, True)])
    assert s.column("r1").to_pylist() == [20, 40, 20, 40, 10, 30, 10, 30]


def test_topk_cut_inside_a_run_keeps_earliest_join_rows():
    probe, build = _sides()
    j = J.join_table(probe, build, [0], [0], J.INNER)
    top = S.sort_table(j, [(0, False, True)], fetch=3)                     # the run of k = 1 has 4 rows: the first 3 in join order
    assert list(zip(top.column("l1").to_pylist(), top.column("r1").to_pylist())) == [("b", 10), ("b", 30), ("f", 10)]
    mid = S.sort_table(j, [(0, False, True)], fetch=6, skip=3)
    assert list(zip(mid.column("l1").to_pylist(), mid.column("r1").to_pylist())) == [("f", 30), ("a", 20), ("a", 40)]
    assert S.sort_table(j, [(0, False, True)], fetch=0).num_rows == 0 and S.sort_table(j, [(0, False, True)], skip=8).num_rows == 0


def test_anti_join_with_empty_build_returns_probe_rows():
    probe, build = _sides()
    out = J.join_table(probe, build.slice(0, 0), [0], [0], J.LEFT_ANTI)
    partref.assert_tables_equal(out, probe)
    assert J.join_table(probe, build.slice(0, 0), [0], [0], J.LEFT_SEMI).num_rows == 0
    assert J.join_table(probe, build.slice(0, 0), [0], [0], J.INNER).num_rows == 0
    # and an outer join over it sees those rows unchanged
    c = pa.table({"p": pa.array(["d", "e", "x"])})
    assert J.join_table(out, c, [1], [0], J.INNER).column("l1").to_pylist() == ["d", "e"]


def test_partitioning_join_batches_equals_partitioning_reference_slices(oracle):
    """a join emits each probe batch's output in slices of at most chunkRows rows; partitioning those batches one by one equals
    partitioning the same slices of the reference join over the whole probe side"""
    rng = np.random.default_rng(5)
    probe = pa.table({"k": pa.array(rng.integers(0, 20, 300), pa.int32()), "v": pa.array(rng.random(300) < 0.5)})
    build = pa.table({"k": pa.array(rng.integers(0, 20, 60), pa.int32()), "s": pa.array([f"s{i % 7}" for i in range(60)]).dictionary_encode()})
    chunk_rows = 64
    whole = J.join_table(probe, build, [0], [0], J.INNER)
    row0, n_batches = 0, 0
    for pb in probe.to_batches(max_chunksize=100):
        out = J.join_table(pa.Table.from_batches([pb]), build, [0], [0], J.INNER)
        for at in range(0, out.num_rows, chunk_rows):
            piece = out.slice(at, chunk_rows)
            ref = whole.slice(row0, piece.num_rows)
            a, b = partref.partition(oracle, piece, [1, 3], 7), partref.partition(oracle, ref, [1, 3], 7)
            assert a[0] == b[0]
            partref.assert_tables_equal(a[2], b[2])
            row0 += piece.num_rows
            n_batches += 1
    assert row0 == whole.num_rows and n_batches > 3
