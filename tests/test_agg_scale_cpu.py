"""CPU checks of the high-cardinality aggregate cases (tests/aggscale.py): the vectorised reference and its comparison agree with
tests/aggref.py on slices of every input, the comparison fails on a wrong group, and every plan NVRTC-compiles for sm_90a."""
import numpy as np
import pyarrow as pa
import pytest

import aggref as R
import aggscale as A


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def aggref_outputs(d, aggset):
    """aggref's Partial state batch and Final result table for the input d"""
    tbl, kc, ag = d.table(), list(range(len(d.keys))), A.aggs(len(d.keys), aggset)
    st = R.partial(tbl, d.dts, kc, ag)
    state = pa.Table.from_batches([R.state_batch(list(st.items()), d.key_types, ag)])
    res = R.aggregate(tbl, d.dts, kc, ag)
    types = d.key_types + [a.result_type() for a in ag]
    cols = [[k[i] for k in res] for i in range(len(kc))] + [[v[ai] for v in res.values()] for ai in range(len(ag))]
    result = pa.table([R.arrow_column(c, t) for c, t in zip(cols, types)], names=[f"r{i}" for i in range(len(types))])
    return state, result


@pytest.mark.parametrize("name,gen", A.all_data(), ids=[n for n, _ in A.all_data()])
def test_reference_matches_aggref_on_a_slice(name, gen):
    """20 000 rows of every input: every function, NULL keys, all-NULL groups, NaN / +-Inf, the type's decimal edges."""
    d = gen().slice(0, 20_000)
    ref = d.ref()
    for aggset in A.MERGE_SETS:
        state, result = aggref_outputs(d, aggset)
        assert A.check(state, ref, "aggref partial", "state", aggset) == ref.ng
        assert A.check(result, ref, "aggref final", "result", aggset, fed=state) == ref.ng
    if name in ("growth", "all-new", "hot-cold"):      # small groups: the slice reaches what the reference must get right
        assert (ref.result[1][0] == 0).any(), "no group whose i64 values are all NULL"
        assert (ref.f64[8].cls != 0).any(), "no group whose f64 sum is NaN or infinite"


def test_comparison_fails_on_a_wrong_group():
    d = A.growth(n=20_000, pool=12_000)
    ref = d.ref()
    state, result = aggref_outputs(d, "int-dec")
    fstate, fresult = aggref_outputs(d, "dec-f64")

    def mutated(tbl, col, fn):
        cols = list(tbl.columns)
        cols[col] = fn(cols[col].combine_chunks())
        return pa.table(cols, names=tbl.column_names)
    g = ref.sample[3]
    # the totals of two groups swapped (what a relocation to the wrong range would do), one group lost, one f64 sum 2 ULP off
    swap = lambda a: pa.array(np.concatenate([a.to_numpy(zero_copy_only=False)[1::-1], a.to_numpy(zero_copy_only=False)[2:]]), mask=~np.asarray(a.is_valid()))
    for bad, kind in ((mutated(state, 1, swap), "state"), (state.slice(1), "state"), (mutated(result, 1, swap), "result")):
        with pytest.raises(AssertionError):
            A.check(bad, ref, "mutated", kind, "int-dec")
    keys = A.from_arrow(fresult.column(0), A.I64)
    row = int(np.flatnonzero(ref.locate([keys]) == g)[0])
    f = fresult.column(3).to_numpy(zero_copy_only=False).copy()
    assert np.isfinite(f[row])
    f[row] = np.nextafter(np.nextafter(f[row], np.inf), np.inf)
    with pytest.raises(AssertionError, match="group"):
        A.check(mutated(fresult, 3, lambda a: pa.array(f, mask=~np.asarray(a.is_valid()))), ref, "mutated", "result", "dec-f64", fed=fstate)


def test_inputs_reach_their_edges():
    """the named rows are where the GPU cases need them"""
    early, late = A.reserved(True), A.reserved(False)
    for d, first_null, first_neg in ((early, 3, 1), (late, 400_001, 420_000)):
        k = d.keys[0]
        assert int(np.flatnonzero(~k.valid)[0]) == first_null and int(np.flatnonzero(k.values == -1)[0]) == first_neg
    assert not (A.growth().keys[0].values == -1).any()
    h = A.hot_cold()
    _, counts = np.unique(h.keys[0].values, return_counts=True)
    assert (counts > 10_000).sum() == 8 and len(counts) > 1_000_000
    assert len(np.unique(A.all_new().keys[0].values)) == A.all_new().n


@pytest.mark.parametrize("keys", A.KEY_SETS, ids=lambda ks: "-".join(k.name.lower() for k in ks))
@pytest.mark.parametrize("aggset", A.MERGE_SETS)
def test_plans_supported_and_compile(cb, keys, aggset):
    for plan in (A.partial_plan(keys, aggset), A.merge_plan(keys, aggset, R.FINAL), A.merge_plan(keys, aggset, R.PARTIAL_MERGE)):
        ok, why = cb.native.supports(plan)
        assert ok, why
        assert cb.native.compile_plan(plan)


def test_merge_plan_of_all_twelve_is_refused_as_a_hash_staging_limit(cb):
    """a Partial takes all twelve aggregates; a merging hash aggregate refuses them (its state columns do not fit the staging ring),
    naming the hash kernel rather than the dense accumulators"""
    ok, why = cb.native.supports(A.partial_plan([A.I64], "all"))
    assert ok, why
    assert cb.native.compile_plan(A.partial_plan([A.I64], "all"))
    ok, why = cb.native.supports(A.merge_plan([A.I64], "all", R.FINAL))
    assert not ok and "hash aggregate" in why and "dense" not in why, why
