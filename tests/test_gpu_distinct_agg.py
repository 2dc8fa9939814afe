"""GPU parity of distinct-aggregate plans (Spark's one-distinct rewrite, tests/distinctref.py): every stage is its own plan fed with the
previous stage's output, and its state or result is compared with the reference under the rules of tests/test_gpu_agg_matrix.py
(integers and decimals exact, SUM(f64) within 1 ULP and AVG(f64) within 2 ULP of the exact value over the states the stage merged)."""
import types

import numpy as np
import pyarrow as pa
import pytest

import aggcases
import aggref as R
import distinctcases
import distinctref as D
import exprs as E
import test_gpu_agg_matrix as M
from comet_b200 import proto as P

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def run(cb, plan, batches, cfg=None):
    return M.run(cb, plan, [batches], cfg)


def as_batches(table, schema, aggs, n_keys):
    """A stage's output as the next stage's input; no output -> one empty batch of the state layout."""
    if table is None or table.num_rows == 0:
        return [R.state_batch([], schema[:n_keys], aggs)]
    return table.to_batches()


def shape(key_types, aggs):
    return types.SimpleNamespace(key_cols=list(range(len(key_types))), key_types=key_types, aggs=aggs)


def state_rows(table, key_types, aggs):
    return M.rows_of(table, shape(key_types, aggs))


def check_stage(got_rows, exp, key_types, aggs, stage, f64_exp):
    if not aggs:  # keys only: a key may repeat (stream runs), the set of keys is the answer
        assert {k for k, _ in got_rows} == set(exp), stage
        return
    M.check_states(got_rows, exp, shape(key_types, aggs), stage, f64_exp)


def run_chain(cb, case, chain, stage3_input=None):
    """Runs the four stages, checks each against the reference, returns the strategy bits of each stage."""
    table = case.table()
    bits = []
    # stage 1: Partial over the scan rows, grouped by (k, x)
    s1, b = run(cb, chain.stage1_plan(), case.batches(), case.config(1))
    bits.append(b)
    got1 = state_rows(s1, chain.inner_types, chain.ordinary)
    exp1 = chain.stage1(table)
    check_stage(got1, exp1, chain.inner_types, chain.ordinary, "stage 1", None)
    # stage 2: PartialMerge (keys only: Partial) over stage 1's state
    s2, b = run(cb, chain.stage2_plan(case.offset2), as_batches(s1, chain.stage2_schema, chain.ordinary, len(chain.inner_types)), case.config(2))
    bits.append(b)
    got2 = state_rows(s2, chain.inner_types, chain.ordinary)
    exp2 = chain.stage2(list(exp1.items()))
    check_stage(got2, exp2, chain.inner_types, chain.ordinary, "stage 2", D.merged_or_keys(got1, chain.ordinary))
    # stage 3: the mixed operator over stage 2's state
    a3 = chain.stage3_aggs()
    in3 = stage3_input if stage3_input is not None else as_batches(s2, chain.stage2_schema, chain.ordinary, len(chain.inner_types))
    s3, b = run(cb, chain.stage3_plan(), in3, case.config(3))
    bits.append(b)
    got3 = state_rows(s3, chain.key_types, a3)
    exp3 = chain.stage3(list(exp2.items()))
    check_stage(got3, exp3, chain.key_types, a3, "stage 3", chain.stage3(got2))
    # stage 4: Final
    s4, b = run(cb, chain.stage4_plan(), as_batches(s3, chain.stage3_schema(), a3, len(chain.key_types)), case.config(4))
    bits.append(b)
    got4 = M.rows_of(s4, shape(chain.key_types, a3), state=False)
    exp4 = chain.stage4(list(exp3.items()))
    M.check_results(got4, exp4, shape(chain.key_types, a3), "stage 4", chain.stage4(got3))
    assert exp4 == chain.answer(table)
    return bits


@pytest.mark.parametrize("case", distinctcases.CASES, ids=lambda c: c.name)
def test_distinct_chain(cb, case):
    bits = run_chain(cb, case, case.chain())
    assert tuple(bits) == case.bits, f"strategy bits {bits}, case targets {case.bits}"


def test_stage3_migrates_dense_to_hash(cb):
    """A mixed stage 3 whose dictionary key starts with 12 values and grows to 300: dense first, then the key table (its partial state
    is flushed, and the Final stage merges it)."""
    case = distinctcases.Case("migrate", [distinctcases.DICT], distinctcases.I64, "dec", "all", None, seed=30, key_card=300, x_card=5000,
                              n=60000)
    chain = case.chain()
    exp2 = chain.stage2(list(chain.stage1(case.table()).items()))
    rows = list(exp2.items())
    small = sorted({k[0] for k, _ in rows if k[0] is not None})[:12]
    # a NULL x every 256 rows: every chunk's x column has a validity buffer (an aggregate argument with a validity buffer in some
    # chunks and not in others changes the accumulator layout between launches, DESIGN.md section 6)
    with_nulls = lambda part: [r for i, (k, st) in enumerate(part) for r in ([(k, st)] + ([((k[0], None), st)] if i % 256 == 0 else []))]
    first = with_nulls([r for r in rows if r[0][0] in small])
    rest = with_nulls([r for r in rows if r[0][0] not in small])
    rows = first + rest
    batches = []
    half = len(first) // 2   # two small-dictionary batches of at least one chunk each: a chunk never mixes in the big dictionary
    assert half >= 1024
    for part, names in ((first[:half], small), (first[half:], small), (rest, sorted({k[0] for k, _ in rows if k[0] is not None}))):
        bt = R.state_batch(part, chain.inner_types, chain.ordinary)
        pos = {s: i for i, s in enumerate(names)}
        keys = pa.DictionaryArray.from_arrays(pa.array([None if k[0] is None else pos[k[0]] for k, _ in part], type=pa.int32()), pa.array(names))
        batches.append(pa.RecordBatch.from_arrays([keys] + bt.columns[1:], names=bt.schema.names))
    cfg = dict(aggcases.TABLE_CFG, **{"spark.comet.b200.chunkRows": "1024"})
    s3, bits = run(cb, chain.stage3_plan(), batches, cfg)
    assert bits == 1 | 8 | 2
    a3 = chain.stage3_aggs()
    got3 = state_rows(s3, chain.key_types, a3)
    check_stage(got3, chain.stage3(rows), chain.key_types, a3, "stage 3", None)
    s4, _ = run(cb, chain.stage4_plan(), s3.to_batches())
    got4 = dict(M.rows_of(s4, shape(chain.key_types, a3), state=False))
    assert got4 == chain.stage4(list(chain.stage3(rows).items()))


@pytest.mark.parametrize("ansi", [False, True])
def test_decimal_sum_overflow_matches_non_distinct(cb, ansi):
    """SUM(y) as decimal(13,2) next to COUNT(DISTINCT x): group 0 has 20 rows of 9e9 (overflows 10^11 only when merged at stage 3),
    the others a few small rows.  Legacy: NULL for group 0, as Partial -> Final gives; ANSI: the query fails, as Partial -> Final does."""
    n_big, dt = 20, P.DECIMAL(13, 2)
    k = [0] * n_big + [1, 1, 2, 3, 3]
    x = list(range(n_big)) + [1, 2, 1, 7, 7]
    y = [9 * 10 ** 11] * n_big + [150, -3, 99, 1, 2]
    t = pa.table({"k": pa.array(k, type=pa.int64()), "x": pa.array(x, type=pa.int64()), "y": R.arrow_column(y, P.DECIMAL(12, 2))})
    dts = [P.INT64, P.INT64, P.DECIMAL(12, 2)]
    mode = R.ANSI if ansi else R.LEGACY
    s = R.Agg("sum", E.Col(2, P.DECIMAL(12, 2)), dt, mode=mode)
    chain = D.Chain(dts, [0], [1], [s], [("count", None, None, R.LEGACY)])
    plain_ok = True
    try:
        st, _ = run(cb, R.partial_plan(dts, [0], [s]), t.to_batches(), aggcases.TABLE_CFG)
        plain, _ = run(cb, R.merge_plan([P.INT64], [s]), st.to_batches())
        plain = dict(M.rows_of(plain, shape([P.INT64], [s]), state=False))
    except cb.native.CometB200Error:
        plain_ok = False
    assert plain_ok == (not ansi)
    batches = t.to_batches()
    try:
        s1, _ = run(cb, chain.stage1_plan(), batches, aggcases.TABLE_CFG)
        s2, _ = run(cb, chain.stage2_plan(), s1.to_batches(), aggcases.TABLE_CFG)
        s3, _ = run(cb, chain.stage3_plan(), s2.to_batches(), aggcases.TABLE_CFG)
        s4, _ = run(cb, chain.stage4_plan(), s3.to_batches())
    except cb.native.CometB200Error:
        assert ansi
        return
    assert not ansi
    got = dict(M.rows_of(s4, shape([P.INT64], chain.stage3_aggs()), state=False))
    assert {key: v[0] for key, v in got.items()} == {key: v[0] for key, v in plain.items()}
    assert got[(0,)] == [None, n_big] and got == chain.answer(t)


def _keys_only_table(strategy, n=5000, seed=40):
    rng = np.random.default_rng(seed)
    if strategy == "dense":
        names = [f"k{i}" for i in range(9)]
        codes = rng.integers(0, len(names), n)
        return pa.table({"k": pa.DictionaryArray.from_arrays(pa.array(codes.astype(np.int32), mask=rng.random(n) < 0.05), pa.array(names))}), [P.STRING]
    v = rng.integers(-500, 500, n)
    if strategy == "stream":
        v = np.sort(v)
    return pa.table({"k": pa.array(v, mask=rng.random(n) < 0.02), "j": pa.array((v % 3).astype(np.int32))}), [P.INT64, P.INT32]


@pytest.mark.parametrize("strategy,bits", [("dense", 1), ("table", 2), ("stream", 4)])
def test_keys_only_partial_and_final(cb, strategy, bits):
    """A HashAggregate with grouping keys and no aggregate expressions (the distinct rewrite's stages 1 and 2): Partial on every
    strategy, then a keys-only Final over its output."""
    t, dts = _keys_only_table(strategy)
    keys = [P.bound(i, d) for i, d in enumerate(dts)]
    cfg = aggcases.STREAM_CFG if strategy == "stream" else aggcases.TABLE_CFG
    st, got_bits = run(cb, P.hash_agg(P.scan(dts), keys, [], P.PARTIAL), t.to_batches(max_chunksize=1000), cfg)
    assert got_bits == bits
    exp = {tuple(r) for r in zip(*[R.pyvalues(t.column(i), d) for i, d in enumerate(dts)])}
    got = [tuple(r) for r in zip(*[R.pyvalues(st.column(i), d) for i, d in enumerate(dts)])]
    assert set(got) == exp
    if strategy != "stream":
        assert len(got) == len(exp)
    fin, _ = run(cb, P.hash_agg(P.scan(dts, source="shuffle"), keys, [], P.FINAL), st.to_batches())
    got_f = [tuple(r) for r in zip(*[R.pyvalues(fin.column(i), d) for i, d in enumerate(dts)])]
    assert sorted(got_f, key=repr) == sorted(exp, key=repr)
