"""GPU: every stateful operator fed device chunks whose physical layouts differ, against the CPU references.  Consecutive chunks of
real inputs differ in whether a column has a validity buffer (NativeScan gives one only to row groups whose statistics allow NULLs;
the Arrow stream source only when a batch has null_count != 0 and a buffer), in its stored width (narrow dictionary codes, or
int32 when a batch dictionary is remapped) and in bit offsets.  Each test runs at least two chunks (chunkRows = 1024), in both
orders, compares every output column with the reference for the logical table (tests/layoutcases.py builds the layouts), and
checks through cb200_stats that the chunks and the strategy it targets ran."""
import types

import numpy as np
import pyarrow as pa
import pytest

import aggcases
import aggref as R
import condjoinref
import exprs as E
import joinref
import layoutcases as L
import partref
import smjref
import sortref
from test_gpu_agg_matrix import check_results, check_states, rows_of
from test_gpu_sort_merge_join import JT as SMJ_JT, JTS as SMJ_JTS

pytestmark = pytest.mark.gpu

C = 1024                       # chunkRows at its minimum: every recipe entry is one device chunk
CFG = {"spark.comet.b200.chunkRows": str(C)}
P = None


@pytest.fixture(scope="module")
def cb():
    global P
    import comet_b200
    P = comet_b200.proto
    return comet_b200


def run(cb, plan, inputs, cfg=None, batch_size=8192):
    """-> (table or None, stats)"""
    with cb.native.Plan(plan, inputs, config={**CFG, **(cfg or {})}, batch_size=batch_size) as p:
        out = p.collect()
        return out, p.stats()


# ---- the logical table: NULLs exactly where a chunk's recipe asks for them -------------------------------------------------------------
I32, I64, DBL, BOOL, STR = "INT32", "INT64", "DOUBLE", "BOOL", "STRING"
NAMES = ["kd", "ki", "kc", "x", "y", "d", "w", "f", "flag", "a", "b"]
VALUE_COLS = ["x", "y", "d", "w", "f", "flag", "a", "b"]
ROTATION = ["none", "nulls", "zero", "unknown"]
KEY_NAMES = ["apple", "kiwi", "fig", "plum", "lime"]


def dts():
    return [P.STRING, P.INT64, P.INT64, P.INT64, P.INT32, P.DECIMAL(12, 2), P.DECIMAL(20, 2), P.DOUBLE, P.BOOL, P.INT32, P.INT32]


def recipe_of(n_chunks, reverse=False, extra=None):
    """each value column walks ROTATION from its own start, so the columns flip independently; `reverse` runs the chunks backwards"""
    rec = []
    for c in range(n_chunks):
        spec = {col: ROTATION[(c + i) % len(ROTATION)] for i, col in enumerate(VALUE_COLS)}
        spec.update((extra or {}).get(c, {}))
        rec.append(spec)
    return rec[::-1] if reverse else rec


def table_for(recipe, seed, key_dict_modes=None):
    """the logical table of `recipe` (C rows per chunk)"""
    rng = np.random.default_rng(seed)
    n = C * len(recipe)
    t = dts()
    cols = {}
    masks = {}
    for col in VALUE_COLS:
        m = np.zeros(n, dtype=bool)
        for c, spec in enumerate(recipe):
            how = spec.get(col)
            if how == "nulls":
                m[c * C:(c + 1) * C] = rng.random(C) < 0.25
                m[c * C] = True
            elif how == "allnull":
                m[c * C:(c + 1) * C] = True
        masks[col] = m
    val = lambda col, xs: [None if z else v for v, z in zip(xs, masks[col].tolist())]
    cols["kd"] = pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, len(KEY_NAMES), n), pa.int8()), pa.array(KEY_NAMES))
    cols["ki"] = pa.array(rng.integers(-200, 200, n) * 7919, pa.int64())
    cols["kc"] = pa.array(np.repeat(np.arange(n // 4 + 1, dtype=np.int64), 4)[:n] * 3 - 50, pa.int64())
    cols["x"] = R.arrow_column(val("x", [int(v) for v in rng.integers(-10**12, 10**12, n)]), t[3])
    cols["y"] = R.arrow_column(val("y", [int(v) for v in rng.integers(-2**31, 2**31 - 1, n)]), t[4])
    cols["d"] = R.arrow_column(val("d", [int(v) for v in rng.integers(-10**12 + 1, 10**12, n)]), t[5])
    cols["w"] = R.arrow_column(val("w", [int(v) * 10**3 + 7 for v in rng.integers(-10**16, 10**16, n)]), t[6])
    cols["f"] = R.arrow_column(val("f", [float(v) for v in rng.standard_normal(n) * 1e6]), t[7])
    cols["flag"] = pa.array(val("flag", [bool(v) for v in rng.integers(0, 2, n)]), pa.bool_())
    cols["a"] = R.arrow_column(val("a", [int(v) for v in rng.integers(-10**6, 10**6, n)]), t[9])
    cols["b"] = R.arrow_column(val("b", [int(v) for v in rng.integers(-10**6, 10**6, n)]), t[10])
    return pa.table(cols)


def col(name):
    return E.Col(NAMES.index(name), dts()[NAMES.index(name)])


def agg_list(which):
    A = R.Agg
    x, y, d, w, f, flag, a, b = (col(c) for c in VALUE_COLS)
    ab = E.Arith("add", a, b, P.INT32)
    if which == "counts":   # COUNT(x) beside COUNT(*), SUM and AVG: the row-count words the layout used to share
        return [A("count", x), A("count", E.Lit(1, P.INT32)), A("sum", x, P.INT64), A("avg", x, P.DOUBLE), A("count", x, filt=flag),
                A("count", ab), A("sum", ab, P.INT64), A("count", y, filt=E.IsNull(x, negate=True))]
    if which == "modes":    # Legacy / TRY / ANSI integer sums and MIN / MAX beside the counts
        return [A("sum", y, P.INT64, mode=R.TRY), A("sum", y, P.INT64, mode=R.ANSI), A("sum", y, P.INT64), A("min", x, P.INT64),
                A("max", y, P.INT32), A("count", y), A("count", E.Lit(1, P.INT32)), A("max", d, P.DECIMAL(12, 2))]
    if which == "dec":
        return [A("sum", d, P.DECIMAL(22, 2)), A("avg", d, P.DECIMAL(16, 6), sum_dt=P.DECIMAL(22, 2)), A("count", d),
                A("sum", w, P.DECIMAL(30, 2), filt=flag), A("count", E.Lit(1, P.INT32))]
    if which == "f64":
        return [A("sum", f, P.DOUBLE), A("avg", f, P.DOUBLE), A("min", f, P.DOUBLE), A("max", f, P.DOUBLE), A("count", f),
                A("avg", f, P.DOUBLE, filt=flag), A("count", E.Lit(1, P.INT32)), A("sum", E.Cast(a, P.DOUBLE), P.DOUBLE, filt=flag)]
    raise KeyError(which)


STRATEGY = {"dense": ("kd", {}), "table": ("ki", aggcases.TABLE_CFG), "stream": ("kc", aggcases.STREAM_CFG)}


def agg_case(key, aggs):
    k = NAMES.index(key)
    return types.SimpleNamespace(aggs=aggs, key_cols=[k], key_types=[dts()[k]])


def same_table(got, want):
    """an operator that produced no batch returns None"""
    if got is None:
        assert want.num_rows == 0
    else:
        partref.assert_tables_equal(got, want)


def check_agg(cb, inputs, table, key, aggs, strategy_cfg, expected_bits, n_chunks):
    """Partial over `inputs` -> state vs the reference's; Final over it -> results vs the reference's"""
    case = agg_case(key, aggs)
    plan = R.partial_plan(dts(), case.key_cols, aggs)
    state, st = run(cb, plan, inputs, strategy_cfg)
    assert st["pipeline_rows"] == table.num_rows and st["pipeline_launches"] >= n_chunks
    assert st["agg_strategies"] == expected_bits
    got_state = rows_of(state, case)
    check_states(got_state, R.partial(table, dts(), case.key_cols, aggs), case, "partial")
    res, _ = run(cb, R.merge_plan(case.key_types, aggs, R.FINAL), [state])
    check_results(rows_of(res, case, state=False), R.aggregate(table, dts(), case.key_cols, aggs), case, "final",
                  R.final(got_state, aggs))


# ---- HashAggregate: arguments, FILTER columns and a + b whose validity flips between chunks --------------------------------------------
@pytest.mark.parametrize("reverse", [False, True], ids=["fwd", "rev"])
@pytest.mark.parametrize("which", ["counts", "modes", "dec", "f64"])
@pytest.mark.parametrize("strategy", ["dense", "table", "stream"])
def test_aggregate_over_flipping_validity(cb, strategy, which, reverse):
    rec = recipe_of(5, reverse, extra={2: {"x": "allnull", "d": "allnull", "f": "allnull"}, 4: {"_split": [300, 724], "_offset": 3}})
    rec[1]["_empty"] = True
    tbl = table_for(rec, seed=len(which) * 7 + reverse)
    key, cfg = STRATEGY[strategy]
    batches = L.chunked(tbl, C, rec)
    check_agg(cb, [L.source(batches)], tbl, key, agg_list(which), cfg, aggcases.EXPECTED_BITS[strategy], len(rec))


@pytest.mark.parametrize("first", ["none", "zero", "unknown", "nulls"])
def test_count_beside_count_star_one_flip(cb, first):
    """the smallest shape of the layout change: COUNT(x), COUNT(*), SUM(x), AVG(x) ungrouped and grouped, x without validity in
    one chunk and with it in the next (and the other way round)"""
    other = "nulls" if first != "nulls" else "none"
    rec = [{"x": first}, {"x": other}, {"x": first}]
    tbl = table_for(rec, seed=3)
    x = col("x")
    aggs = [R.Agg("count", x), R.Agg("count", E.Lit(1, P.INT32)), R.Agg("sum", x, P.INT64), R.Agg("avg", x, P.DOUBLE)]
    for key, cfg, bits in (("kd", {}, 1), ("ki", aggcases.TABLE_CFG, 2)):
        check_agg(cb, [L.source(L.chunked(tbl, C, rec))], tbl, key, aggs, cfg, bits, 3)
    plan = R.partial_plan(dts(), [], aggs)
    state, st = run(cb, plan, [L.source(L.chunked(tbl, C, rec))])
    assert st["pipeline_launches"] >= 3
    res, _ = run(cb, R.merge_plan([], aggs, R.FINAL), [state])
    want = R.aggregate(tbl, dts(), [], aggs)[()]
    got = res.to_pylist()[0]
    assert [got[f"col_{i}"] for i in range(3)] == want[:3]
    assert abs(got["col_3"] - want[3]) <= 2 * abs(np.spacing(want[3]))


def test_dense_to_hash_migration_after_a_flip(cb):
    """a dictionary key grows past the dense path after the argument's validity flipped: the dense state flushed, then hashed"""
    rec = [{"x": "none"}, {"x": "nulls"}, {"x": "none"}, {"x": "unknown"}]
    tbl = table_for(rec, seed=11)
    names = [f"g{i:03d}" for i in range(200)]
    rng = np.random.default_rng(5)
    codes = np.concatenate([rng.integers(0, 3, 2 * C), rng.integers(0, 200, 2 * C)]).astype(np.int16)
    tbl = tbl.set_column(0, "kd", pa.DictionaryArray.from_arrays(pa.array(codes), pa.array(names)))
    batches, row = L.chunked(tbl, C, rec), 0
    for i, bt in enumerate(batches):   # the batch dictionaries hold 3 names, then all 200: the plan-wide one grows
        d = names[:3] if row < 2 * C else names
        batches[i] = bt.set_column(0, "kd", pa.DictionaryArray.from_arrays(pa.array(codes[row:row + bt.num_rows]), pa.array(d)))
        row += bt.num_rows
    x = col("x")
    aggs = [R.Agg("count", x), R.Agg("count", E.Lit(1, P.INT32)), R.Agg("sum", x, P.INT64), R.Agg("avg", x, P.DOUBLE)]
    check_agg(cb, [L.source(batches)], tbl, "kd", aggs, aggcases.TABLE_CFG, aggcases.EXPECTED_BITS["migrate"], 4)


# ---- NativeScan: row groups with and without NULLs, all NULL, with and without statistics ------------------------------------------------
@pytest.mark.parametrize("statistics", [True, False])
@pytest.mark.parametrize("reverse", [False, True], ids=["fwd", "rev"])
def test_aggregate_over_native_scan_row_groups(cb, tmp_path, statistics, reverse):
    rec = [{"x": "none", "d": "nulls"}, {"x": "nulls", "d": "none"}, {"x": "allnull", "d": "none"}, {"x": "none", "d": "nulls"}]
    rec = rec[::-1] if reverse else rec
    tbl = table_for(rec, seed=21 + reverse)
    names = ["kd", "ki", "x", "d"]
    sub = tbl.select(names).set_column(0, "kd", tbl.column("kd").cast(pa.string()))
    path = str(tmp_path / "rg.parquet")
    md = L.write_row_groups(path, sub, C, statistics=statistics)
    assert md.num_row_groups == 4
    t = [P.STRING, P.INT64, P.INT64, P.DECIMAL(12, 2)]
    fields = [(k, dt, True) for k, dt in zip(names, t)]
    x, d = E.Col(2, t[2]), E.Col(3, t[3])
    flag = E.Cmp("gt", x, E.Lit(0, P.INT64))
    aggs = [R.Agg("count", x), R.Agg("count", E.Lit(1, P.INT32)), R.Agg("sum", x, P.INT64), R.Agg("avg", x, P.DOUBLE),
            R.Agg("sum", d, P.DECIMAL(22, 2)), R.Agg("count", d, filt=flag), R.Agg("min", d, P.DECIMAL(12, 2))]
    for key in (0, 1):
        case = types.SimpleNamespace(aggs=aggs, key_cols=[key], key_types=[t[key]])
        plan = P.hash_agg(P.native_scan(fields, fields, [path]), [P.bound(key, t[key])], [a.proto() for a in aggs], P.PARTIAL)
        state, st = run(cb, plan, [], aggcases.TABLE_CFG)
        assert st["pipeline_launches"] >= 4 and st["pipeline_rows"] == sub.num_rows          # one row group per chunk
        got = rows_of(state, case)
        check_states(got, R.partial(sub, t, [key], aggs), case, "partial")
        res, _ = run(cb, R.merge_plan(case.key_types, aggs, R.FINAL), [state])
        check_results(rows_of(res, case, state=False), R.aggregate(sub, t, [key], aggs), case, "final", R.final(got, aggs))


# ---- Final / PartialMerge over state batches with and without validity on a state column ---------------------------------------------
@pytest.mark.parametrize("mode", [R.FINAL, R.PARTIAL_MERGE])
def test_merge_over_mixed_state_batches(cb, mode):
    rec = recipe_of(4)
    tbl = table_for(rec, seed=31)
    aggs = agg_list("counts")[:6]
    case = agg_case("ki", aggs)
    states, rows = [], []
    for c in range(len(rec)):   # the Partial state of each chunk: SUM(x) is NULL in some groups (a validity buffer), or in none
        st = list(R.partial(tbl.slice(c * C, C), dts(), case.key_cols, aggs).items())
        rows += st
        states.append(R.state_batch(st, case.key_types, aggs))
    assert any(b.column(3).null_count for b in states) and any(b.column(3).buffers()[0] is None for b in states)
    for order in (states, states[::-1]):
        batches = list(order)
        out, st = run(cb, R.merge_plan(case.key_types, aggs, mode), [batches], aggcases.TABLE_CFG)
        assert st["pipeline_launches"] >= 2
        if mode == R.FINAL:
            check_results(rows_of(out, case, state=False), R.aggregate(tbl, dts(), case.key_cols, aggs), case, "final", R.final(rows, aggs))
        else:
            check_states(rows_of(out, case), R.partial(tbl, dts(), case.key_cols, aggs), case, "merge", R.merge(rows, aggs))


# ---- Sort and TopK ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fetch", [None, 700])
@pytest.mark.parametrize("reverse", [False, True], ids=["fwd", "rev"])
def test_sort_and_topk_over_flipping_chunks(cb, fetch, reverse):
    """keys and payloads flip validity, the dictionary key is narrow in one chunk and remapped to int32 in the next; TopK carries
    candidates from a chunk of another layout"""
    rec = recipe_of(4, reverse, extra={1: {"_dict": {"kd": "remap"}, "_offset": 5}, 3: {"_dict": {"kd": "remap"}}})
    tbl = table_for(rec, seed=41 + reverse)
    keys = [(NAMES.index("x"), False, True), (NAMES.index("kd"), True, False), (NAMES.index("flag"), False, False), (NAMES.index("kc"), False, True)]
    plan = P.sort(P.scan(dts()), [P.sort_order(P.bound(i, dts()[i]), dsc, nf) for i, dsc, nf in keys], fetch=fetch)
    got, st = run(cb, plan, [L.source(L.chunked(tbl, C, rec))])
    partref.assert_tables_equal(got, sortref.sort_table(tbl, keys, fetch))
    assert st["sort_rows"] >= tbl.num_rows and st["sort_passes"] > 0


# ---- HashJoin and SortMergeJoin --------------------------------------------------------------------------------------------------------
def join_sides(seed, reverse):
    rec_l = recipe_of(3, reverse, extra={1: {"_dict": {"kd": "remap"}}})
    rec_r = recipe_of(2, not reverse, extra={0: {"_split": [500, 524], "_offset": 1}})
    left, right = table_for(rec_l, seed), table_for(rec_r, seed + 1)
    # sorted join keys (SortMergeJoin reads sorted sides), so the rows, and with them the NULLs of each chunk, stay in place
    small = lambda t: t.set_column(1, "ki", pa.array(np.sort(np.asarray(t.column("ki").to_numpy()) % 211), pa.int64()))
    return small(left), rec_l, small(right), rec_r


@pytest.mark.parametrize("reverse", [False, True], ids=["fwd", "rev"])
@pytest.mark.parametrize("jt,build_left", [("inner", False), ("inner", True), ("left_semi", False), ("left_anti", False)])
def test_hash_join_over_flipping_chunks(cb, jt, build_left, reverse):
    left, rec_l, right, rec_r = join_sides(51 + reverse, reverse)
    lk = [NAMES.index("ki")]
    for cond in (None, E.Cmp("lt", col("x"), E.Col(len(NAMES) + NAMES.index("x"), P.INT64))):   # the condition reads flipping columns
        plan = P.hash_join(P.scan(dts()), P.scan(dts()), [P.bound(lk[0], P.INT64)], [P.bound(lk[0], P.INT64)], {"inner": 0, "left_semi": 4, "left_anti": 5}[jt],
                           P.BUILD_LEFT if build_left else P.BUILD_RIGHT, condition=None if cond is None else cond.proto())
        got, st = run(cb, plan, [L.source(L.chunked(left, C, rec_l)), L.source(L.chunked(right, C, rec_r))])
        want = joinref.join_table(left, right, lk, lk, jt, build_left) if cond is None else condjoinref.cond_join_table(left, right, lk, lk, jt, cond, build_left)
        same_table(got, want)
        assert st["join_out_rows"] == want.num_rows and st["join_build_rows"] == (left if build_left else right).num_rows
        assert cond is None or st["join_cond_pairs"] > 0


@pytest.mark.parametrize("reverse", [False, True], ids=["fwd", "rev"])
@pytest.mark.parametrize("jt", SMJ_JTS)
def test_sort_merge_join_over_flipping_chunks(cb, jt, reverse):
    left, rec_l, right, rec_r = join_sides(61 + reverse, reverse)
    lk = [NAMES.index("ki")]
    for cond in (None, E.Cmp("gt", col("f"), E.Col(len(NAMES) + NAMES.index("f"), P.DOUBLE))):
        plan = P.sort_merge_join(P.scan(dts()), P.scan(dts()), [P.bound(lk[0], P.INT64)], [P.bound(lk[0], P.INT64)], SMJ_JT[jt],
                                 [P.sort_order(P.bound(lk[0], P.INT64))], condition=None if cond is None else cond.proto())
        got, st = run(cb, plan, [L.source(L.chunked(left, C, rec_l)), L.source(L.chunked(right, C, rec_r))])
        want = smjref.sort_merge_join_table(left, right, lk, lk, jt) if cond is None else condjoinref.cond_join_table(left, right, lk, lk, jt, cond)
        same_table(got, want)
        assert st["join_out_rows"] == want.num_rows


# ---- ShuffleWriter -------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("native_scan", [False, True])
def test_shuffle_writer_over_flipping_chunks(cb, oracle, tmp_path, native_scan):
    rec = recipe_of(4, extra={2: {"_offset": 3, "_split": [1000, 24]}})
    tbl = table_for(rec, seed=71).drop_columns(["kd", "flag"])   # NativeScan reads no BOOLEAN Parquet column
    rec = [{k: v for k, v in s.items() if k != "flag"} for s in rec]
    t = [dt for dt, nm in zip(dts(), NAMES) if nm not in ("kd", "flag")]
    names = tbl.column_names
    if native_scan:
        path = str(tmp_path / "sw.parquet")
        L.write_row_groups(path, tbl, C)
        fields = [(k, dt, True) for k, dt in zip(names, t)]
        child, inputs = P.native_scan(fields, fields, [path]), []
    else:
        child, inputs = P.scan(t), [L.source(L.chunked(tbl, C, rec))]
    keys = ["x", "d", "b"]
    plan = P.shuffle_writer(child, P.hash_partitioning([P.bound(names.index(k), t[names.index(k)]) for k in keys], 7))
    row0 = 0
    with cb.native.Plan(plan, inputs, config=CFG) as p:
        while True:
            b = p.execute()
            if b is None:
                break
            want_starts, _, want = partref.partition(oracle, tbl.slice(row0, b.num_rows), keys, 7)
            assert p.partition_starts() == want_starts
            partref.assert_tables_equal(b, want)
            row0 += b.num_rows
    assert row0 == tbl.num_rows


# ---- Filter + Projection ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("reverse", [False, True], ids=["fwd", "rev"])
def test_filter_projection_over_flipping_chunks(cb, reverse):
    rec = recipe_of(4, reverse, extra={1: {"_offset": 7}, 2: {"_split": [9, 1015], "_empty": True}})
    tbl = table_for(rec, seed=81 + reverse)
    x, y, flag, a, b = col("x"), col("y"), col("flag"), col("a"), col("b")
    pred = E.Logic("or", E.IsNull(x), E.Logic("and", flag, E.Cmp("gt", a, b)))
    outs = [E.IsNull(y), E.IsNull(flag, negate=True), E.Logic("and", flag, E.Cmp("lt", a, E.Lit(0, P.INT32))),
            E.Logic("or", E.Not(flag), E.Cmp("gt", x, E.Lit(0, P.INT64))),
            E.CaseWhen([E.IsNull(a), E.Cmp("gt", b, a)], [E.Lit(-1, P.INT64), x], E.Lit(7, P.INT64)),
            E.In(a, [E.Lit(v, P.INT32) for v in tbl.column("a").to_pylist()[:40:3] if v is not None] + [E.Lit(None, P.INT32)]), x, flag]
    plan = P.projection(P.filter_(P.scan(dts()), pred.proto()), [o.proto() for o in outs])
    got, st = run(cb, plan, [L.source(L.chunked(tbl, C, rec))])
    cols = R.exprs_columns(tbl, dts())
    keep = [v is True for v in R.node_values(pred, cols)]
    want = [[v for v, k in zip(R.node_values(o, cols), keep) if k] for o in outs]
    assert st["pipeline_rows"] >= tbl.num_rows
    for i, o in enumerate(outs):
        assert R.pyvalues(got.column(i), o.dt) == want[i], i


# ---- plain (non-dictionary) Utf8 group keys: the device dictionary builder ------------------------------------------------------------
def utf8_plan(aggs):
    return P.hash_agg(P.scan([P.STRING, P.INT64]), [P.bound(0, P.STRING)], [a.proto() for a in aggs], P.PARTIAL)


@pytest.mark.parametrize("reverse", [False, True], ids=["fwd", "rev"])
def test_plain_utf8_keys_across_chunks(cb, reverse):
    """codes stay stable across chunks, NULL key chunks alternate with chunks without NULLs, "" is a group apart from NULL"""
    rng = np.random.default_rng(91 + reverse)
    pool = ["", "a", "bb", "ccc", "a" * 40, "été", "x y"] + [f"k{i}" for i in range(50)]
    rec = [{"s": "nulls", "v": "none"}, {"s": "none", "v": "nulls"}, {"s": "allnull", "v": "zero"}, {"s": "zero", "v": "unknown"}]
    rec = rec[::-1] if reverse else rec
    keys, vals = [], []
    for spec in rec:
        ks = [pool[int(i)] for i in rng.integers(0, len(pool), C)]
        if spec["s"] == "nulls":
            ks = [None if rng.random() < 0.3 else k for k in ks]
        if spec["s"] == "allnull":
            ks = [None] * C
        vs = [int(v) for v in rng.integers(-1000, 1000, C)]
        if spec["v"] == "nulls":
            vs = [None if rng.random() < 0.3 else v for v in vs]
        keys += ks
        vals += vs
    tbl = pa.table({"s": pa.array(keys, pa.string()), "v": pa.array(vals, pa.int64())})
    t = [P.STRING, P.INT64]
    v = E.Col(1, P.INT64)
    aggs = [R.Agg("count", v), R.Agg("count", E.Lit(1, P.INT32)), R.Agg("sum", v, P.INT64), R.Agg("min", v, P.INT64)]
    case = types.SimpleNamespace(aggs=aggs, key_cols=[0], key_types=[P.STRING])
    state, st = run(cb, utf8_plan(aggs), [L.source(L.chunked(tbl, C, rec))])
    assert st["pipeline_launches"] >= 4 and st["agg_strategies"] == cb.native.AGG_DENSE
    got = rows_of(state, case)
    assert len(got) == len({k for k, _ in got})                       # one state row per key: stable codes
    check_states(got, R.partial(tbl, t, [0], aggs), case, "partial")
    assert ("",) in dict(got) and (None,) in dict(got)


@pytest.mark.parametrize("n,bytes_each,ok", [(4096, 8, True), (4097, 8, False), (3000, 400, False)])
def test_plain_utf8_key_dictionary_limits(cb, n, bytes_each, ok):
    """4096 distinct values are accepted; 4097, or more than 1 MiB of distinct bytes, are refused as Unsupported, not answered"""
    vals = [f"{i:0{bytes_each}d}" for i in range(n)]
    rows = vals + vals[: C]                                             # the second chunk repeats keys of the first
    tbl = pa.table({"s": pa.array(rows, pa.string()), "v": pa.array(np.arange(len(rows), dtype=np.int64))})
    aggs = [R.Agg("count", E.Lit(1, P.INT32)), R.Agg("sum", E.Col(1, P.INT64), P.INT64)]
    inputs = [tbl.to_batches(max_chunksize=C)]
    if not ok:
        with pytest.raises(cb.native.Unsupported):
            run(cb, utf8_plan(aggs), inputs, aggcases.TABLE_CFG)
        return
    state, st = run(cb, utf8_plan(aggs), inputs, aggcases.TABLE_CFG)
    case = types.SimpleNamespace(aggs=aggs, key_cols=[0], key_types=[P.STRING])
    check_states(rows_of(state, case), R.partial(tbl, [P.STRING, P.INT64], [0], aggs), case, "partial")
    assert st["pipeline_launches"] >= 2
