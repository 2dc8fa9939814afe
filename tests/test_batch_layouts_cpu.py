"""CPU side of tests/test_gpu_batch_layouts.py: the layout builder (tests/layoutcases.py) pinned against pyarrow and the C data
interface, the plans of the GPU file compiled, and the aggregate accumulator layout over every subset of nullable inputs, generated
by codegen.cpp through a host-only driver (csrc/layout_test.cpp): each layout refines those with fewer nullable inputs, the word map
the aggregate moves its totals by is that refinement, and the benchmark plans compile to the kernels they did before."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pyarrow as pa
import pytest

import aggref as R
import exprs as E
import layoutcases as L

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "datafusion-comet_b200", "csrc")


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


@pytest.fixture(scope="module")
def lt(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("layout") / "libcb200_layout.so")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-fPIC", "-shared", f"-I{cuda}/include", "-o", so,
                           os.path.join(CSRC, "layout_test.cpp"), os.path.join(CSRC, "codegen.cpp"), os.path.join(CSRC, "plan.cpp"),
                           "-Wl,--no-undefined"])
    lib = C.CDLL(so)
    for f in (lib.lt_layout, lib.lt_widen):
        f.argtypes = [C.c_char_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_char_p, C.c_size_t]
    return lib


# ---- the builder --------------------------------------------------------------------------------------------------------------------------
def small_table(n=24):
    return pa.table({"i": pa.array(range(n), pa.int64()), "b": pa.array([i % 3 == 0 for i in range(n)]),
                     "s": pa.DictionaryArray.from_arrays(pa.array([i % 4 for i in range(n)], pa.int16()), pa.array(["w", "x", "y", "z"])),
                     "u": pa.array([f"u{i}" for i in range(n)])})


@pytest.mark.parametrize("offset", [0, 3, 13])
@pytest.mark.parametrize("how", ["none", "zero", "unknown"])
def test_validity_layouts_without_nulls(how, offset):
    t = small_table()
    rec = [{c: how for c in t.column_names} | {"_offset": offset}, {}, {}]
    bs = L.chunked(t, 8, rec)
    assert pa.Table.from_batches(bs).to_pylist() == t.to_pylist()
    for length, nc, off, has in L.exported(bs[0]):
        # pyarrow's exporter counts the NULLs of "unknown" and drops the buffer of "zero": `source` puts them back
        assert (length, off, has, nc) == (8, offset, how == "unknown", 0)
    assert bs.unknown[0] == (frozenset(range(4)) if how == "unknown" else frozenset())
    assert bs.zero[0] == (frozenset(range(4)) if how == "zero" else frozenset())
    assert L.device_validity(bs[0]) == [False] * 4


def test_null_layouts_and_splits():
    t = small_table(30)
    t = t.set_column(0, "i", pa.array([None if i % 5 == 0 else i for i in range(8)] + [None] * 8 + list(range(14)), pa.int64()))
    rec = [{"i": "nulls", "_split": [3, 5], "_empty": True}, {"i": "allnull", "b": "unknown", "_offset": 9}, {"i": "none"}, {}]
    bs = L.chunked(t, 8, rec)
    assert [b.num_rows for b in bs] == [0, 3, 0, 5, 8, 8, 6]
    assert L.chunk_of(bs, 8) == [0, 0, 0, 0, 1, 2, 3]
    assert pa.Table.from_batches(bs).to_pylist() == t.to_pylist()
    assert L.device_validity(bs[1])[0] and L.device_validity(bs[4])[0] and not L.device_validity(bs[5])[0]
    assert L.exported(bs[4])[0][1] == 8 and L.exported(bs[4])[1][2] == 9
    assert bs.unknown[4] == frozenset([1])
    with pytest.raises(AssertionError):
        L.chunked(t, 8, [{"i": "none"}])                                  # the first chunk holds NULLs
    with pytest.raises(AssertionError):
        L.chunked(t, 8, [{"i": "nulls", "_split": [3, 4]}])               # the batches must fill the chunk exactly


def test_dictionary_identity_and_remap():
    t = small_table()
    bs = L.chunked(t, 8, [{}, {"_dict": {"s": "remap"}, "s": "unknown"}, {"_dict": {"s": "identity"}}])
    assert bs[0].column(2).dictionary.to_pylist() == ["w", "x", "y", "z"] and bs[1].column(2).dictionary.to_pylist() == ["z", "y", "x", "w"]
    assert bs[1].column(2).indices.type == pa.int16()
    assert pa.Table.from_batches(bs).column("s").to_pylist() == t.column("s").to_pylist()


def test_source_exports_unknown_null_count():
    """the stream `source` hands null_count -1 for every column marked "unknown" (and leaves the others as pyarrow exports them)"""
    t = small_table()
    bs = L.chunked(t, 8, [{"i": "zero"}, {"i": "unknown", "u": "unknown", "_empty": True}, {"i": "none"}])
    st = L._Stream()
    L.source(bs)._export_to_c(C.addressof(st))
    seen = []
    while True:
        arr = L._Array()
        assert st.get_next(C.byref(st), C.byref(arr)) == 0
        if not arr.release:
            break
        seen.append([(arr.children[c].contents.null_count, bool(arr.children[c].contents.buffers[0])) for c in (0, 3)])
        C.CFUNCTYPE(None, C.POINTER(L._Array))(arr.release)(C.byref(arr))
    st.release(C.byref(st))
    assert seen == [[(0, True), (0, False)], [(0, True), (0, True)], [(-1, True), (-1, True)], [(0, False), (0, False)]]


def test_row_groups_with_and_without_statistics(tmp_path):
    import pyarrow.parquet as pq
    x = [None] * 1024 + list(range(1024)) + [None if i % 7 == 0 else i for i in range(1024)]
    s = [f"v{i % 3}" for i in range(2048)] + [f"distinct-value-{i:06d}" * 3 for i in range(1024)]
    t = pa.table({"x": pa.array(x, pa.int64()), "s": pa.array(s)})
    for stats in (True, False):
        md = L.write_row_groups(str(tmp_path / f"{stats}.parquet"), t, 1024, statistics=stats, dictionary_limit=4096)
        assert md.num_row_groups == 3 and all(md.row_group(g).num_rows == 1024 for g in range(3))
        nulls = [md.row_group(g).column(0).statistics.null_count if md.row_group(g).column(0).is_stats_set else None for g in range(3)]
        assert nulls == ([1024, 0, 147] if stats else [None] * 3)
    assert pq.read_table(str(tmp_path / "True.parquet")).equals(t)


# ---- the plans of the GPU file compile ----------------------------------------------------------------------------------------------
def test_gpu_plans_compile(cb):
    import test_gpu_batch_layouts as T
    T.P = cb.proto
    P = cb.proto
    n = 0
    for which in ("counts", "modes", "dec", "f64"):
        aggs = T.agg_list(which)
        for key in ("kd", "ki", "kc"):
            case = T.agg_case(key, aggs)
            n += len(cb.native.compile_plan(R.partial_plan(T.dts(), case.key_cols, aggs)))
            n += len(cb.native.compile_plan(R.merge_plan(case.key_types, aggs, R.FINAL)))
        n += len(cb.native.compile_plan(R.partial_plan(T.dts(), [], aggs)))
    keys = [(T.NAMES.index("x"), False, True), (T.NAMES.index("kd"), True, False)]
    n += len(cb.native.compile_plan(P.sort(P.scan(T.dts()), [P.sort_order(P.bound(i, T.dts()[i]), d, f) for i, d, f in keys], fetch=700)))
    x, flag, a, b = T.col("x"), T.col("flag"), T.col("a"), T.col("b")
    pred = E.Logic("or", E.IsNull(x), E.Logic("and", flag, E.Cmp("gt", a, b)))
    n += len(cb.native.compile_plan(P.projection(P.filter_(P.scan(T.dts()), pred.proto()), [E.IsNull(x).proto(), x.proto()])))
    assert n > 20


# ---- the accumulator layout over every subset of nullable inputs -------------------------------------------------------------------------
def layout(lt, plan, validity, nullable_before, hash_):
    out = (C.c_int * 512)()
    err = C.create_string_buffer(512)
    assert lt.lt_layout(plan, len(plan), validity, nullable_before, hash_, out, 512, err, 512) == 0, err.value
    nw, nr = out[0], out[1]
    return list(out[2:2 + nw]), list(out[2 + nw:2 + nw + nr])


def widen(lt, plan, before, batch, hash_):
    out = (C.c_int * 512)()
    err = C.create_string_buffer(512)
    n = lt.lt_widen(plan, len(plan), before, batch, hash_, out, 512, err, 512)
    assert n != -1, err.value
    return None if n == -2 else list(out[:n])


def partition(roles):
    """words as the sets of roles that share them"""
    by = {}
    for r, w in enumerate(roles):
        if w >= 0:
            by.setdefault(w, set()).add(r)
    return sorted(frozenset(s) for s in by.values())


def refines(fine, coarse):
    return all(any(f <= c for c in coarse) for f in fine)


def layout_plans(cb):
    P = cb.proto
    t = [P.STRING, P.INT64, P.INT32, P.DECIMAL(12, 2), P.DOUBLE, P.BOOL, P.INT32]
    x, y, d, f, flag, a = (E.Col(i, t[i]) for i in range(1, 7))
    A = R.Agg
    sets = [
        [A("count", x), A("count", E.Lit(1, P.INT32)), A("sum", x, P.INT64), A("avg", x, P.DOUBLE), A("min", x, P.INT64)],
        [A("count", x, filt=flag), A("sum", y, P.INT64, mode=R.TRY), A("count", E.Arith("add", y, a, P.INT32)), A("count", y),
         A("sum", d, P.DECIMAL(22, 2)), A("avg", d, P.DECIMAL(16, 6), sum_dt=P.DECIMAL(22, 2), filt=flag)],
        [A("sum", f, P.DOUBLE), A("avg", f, P.DOUBLE, filt=flag), A("count", f), A("count", E.Lit(1, P.INT32)), A("max", f, P.DOUBLE),
         A("sum", y, P.INT64, mode=R.ANSI), A("count", x)],
    ]
    return t, sets


@pytest.mark.parametrize("hash_", [0, 1], ids=["dense", "hash"])
@pytest.mark.parametrize("which", [0, 1, 2])
def test_layouts_refine_and_widen_by_the_generated_map(lt, cb, which, hash_):
    P = cb.proto
    t, sets = layout_plans(cb)
    aggs = sets[which]
    plan = R.partial_plan(t, [1 if hash_ else 0], aggs)
    cols = range(1, len(t))
    masks = [sum(1 << c for c in s) for k in range(len(cols) + 1) for s in itertools.combinations(cols, k)]
    lay = {m: layout(lt, plan, m, 0, hash_) for m in masks}
    for m in masks:
        kinds, roles = lay[m]
        # the layout depends on the columns that ever had validity, not on this batch's alone
        for sub in (s for s in masks if s & m == s):
            assert layout(lt, plan, sub, m, hash_) == (kinds, roles)
        for sub in (s for s in masks if s & m == s):
            sk, sr = lay[sub]
            assert refines(partition(roles), partition(sr)), (sub, m)
            wmap = widen(lt, plan, sub, m, hash_)
            assert wmap is not None and len(wmap) == len(kinds)
            for r, (w, o) in enumerate(zip(roles, sr)):       # role by role: each new word starts as the word its role had
                assert (w < 0) == (o < 0)
                if w >= 0:
                    assert wmap[w] == o and kinds[w] == sk[o]
    assert len(lay[0][0]) < len(lay[masks[-1]][0])                   # the flips matter: every plan here has words to split
    # a layout never narrows: going back to fewer nullable inputs is not a widening
    assert widen(lt, plan, masks[-1], 0, hash_) == list(range(len(lay[masks[-1]][0])))


def test_compiled_benchmark_kernels_unchanged(cb):
    """the plans of bench.py (Q1, Q6 and Config 1, both money types) compile to the same kernels as before the layout change"""
    from comet_b200 import tpch
    want = {("q1_partial_plan", "dec"): ["b84783df8963af71_176e"], ("q1_final_plan", "dec"): ["4d6a4bcf93fc6d50_1f69"],
            ("q6_partial_plan", "dec"): ["964dae03c38c5d0c_990"], ("q6_final_plan", "dec"): ["33ad549a87420bd2_75c"],
            ("config1_plan", "dec"): ["e8696220ef4a6f20_516", "55067cfcaab25154_310"],
            ("q1_partial_plan", "f64"): ["c88fee897c096730_df2"], ("q1_final_plan", "f64"): ["ef0170dd73ab48ed_1139"],
            ("q6_partial_plan", "f64"): ["d8807d19e6ddba44_906"], ("q6_final_plan", "f64"): ["ac236d05d1f2b2de_53e"],
            ("config1_plan", "f64"): ["e83d955de78ef34b_468", "55067cfcaab25154_310"]}
    for (name, v), keys in want.items():
        assert cb.native.compile_plan(getattr(tpch, name)(v)) == keys, (name, v)
