"""GPU parity: high-cardinality hash aggregation (BASELINE config 4 shape: GROUP BY l_orderkey SUM(l_extendedprice))."""
import math

import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def run(cb, plan, inputs, chunk_rows=None):
    cfg = {"spark.comet.b200.chunkRows": str(chunk_rows)} if chunk_rows else None
    with cb.native.Plan(plan, inputs, config=cfg) as p:
        return p.collect()


def unscaled(x):
    return None if x is None else int(x.scaleb(-x.as_tuple().exponent))


def plans(cb, variant):
    P = cb.proto
    m = P.DECIMAL(12, 2) if variant == "dec" else P.DOUBLE
    sdt = P.DECIMAL(22, 2) if variant == "dec" else P.DOUBLE
    partial = P.hash_agg(P.scan([P.INT64, m]), [P.bound(0, P.INT64)], [P.agg_sum(P.bound(1, m), sdt)], P.PARTIAL)
    state = [P.INT64, sdt, P.BOOL] if variant == "dec" else [P.INT64, sdt]
    final = P.hash_agg(P.scan(state, source="shuffle"), [P.bound(0, P.INT64)], [P.agg_sum(P.unbound("c", m), sdt)], P.FINAL)
    return partial, final


@pytest.mark.parametrize("n,chunk", [(10, None), (100_000, None), (700_000, 200_000)])
def test_group_by_orderkey_sum_dec(cb, n, chunk):
    t = cb.tpch
    cols = t.gen_lineitem(n, seed=3)
    tbl = pa.table({"k": pa.array(cols["l_orderkey"]), "v": t._dec_array(cols["l_extendedprice"])})
    partial, final = plans(cb, "dec")
    state = run(cb, partial, [tbl.to_batches(max_chunksize=8192)], chunk)
    res = run(cb, final, [state])
    exp = {}
    for k, v in zip(cols["l_orderkey"].tolist(), cols["l_extendedprice"].tolist()):
        exp[k] = exp.get(k, 0) + v
    got = {k: unscaled(v) for k, v in zip(res.column(0).to_pylist(), res.column(1).to_pylist())}
    assert got == exp
    # partial state: (key, sum d(22,2), is_empty bool); one row per group, unordered
    assert state.num_rows == len(exp) and str(state.schema.field(2).type) == "bool"


def test_group_by_orderkey_sum_f64(cb):
    t = cb.tpch
    n = 300_000
    cols = t.gen_lineitem(n, seed=5)
    price = cols["l_extendedprice"].astype(np.float64) / 100.0
    tbl = pa.table({"k": pa.array(cols["l_orderkey"]), "v": pa.array(price)})
    partial, final = plans(cb, "f64")
    state = run(cb, partial, [tbl.to_batches(max_chunksize=8192)], 120_000)
    res = run(cb, final, [state])
    keys = np.array(res.column(0).to_pylist())
    vals = np.array(res.column(1).to_pylist())
    order = np.argsort(keys)
    uk, inv = np.unique(cols["l_orderkey"], return_inverse=True)
    assert (keys[order] == uk).all()
    for i in range(0, len(uk), 997):
        exact = math.fsum(price[inv == i])
        assert abs(vals[order][i] - exact) <= math.ulp(exact)


def test_null_and_negative_and_sentinel_keys(cb):
    P = cb.proto
    keys = pa.array([None, -1, 5, -1, None, 2**63 - 1, -(2**63), 5, -1], type=pa.int64())   # -1 == the table's EMPTY sentinel pattern
    vals = pa.array([1, 2, 3, 4, 5, 6, 7, 8, None], type=pa.int64())
    plan = P.hash_agg(P.scan([P.INT64, P.INT64]), [P.bound(0, P.INT64)],
                      [P.agg_sum(P.bound(1, P.INT64), P.INT64), P.agg_count([P.bound(1, P.INT64)]), P.agg_min(P.bound(1, P.INT64), P.INT64),
                       P.agg_max(P.bound(1, P.INT64), P.INT64)], P.PARTIAL)
    out = run(cb, plan, [pa.table({"k": keys, "v": vals})])
    got = {r["col_0"]: (r["col_1"], r["col_2"], r["col_3"], r["col_4"]) for r in out.to_pylist()}
    assert got == {None: (6, 2, 1, 5), -1: (6, 2, 2, 4), 5: (11, 2, 3, 8), 2**63 - 1: (6, 1, 6, 6), -(2**63): (7, 1, 7, 7)}


def test_two_keys_date_and_dict_string(cb):
    P = cb.proto
    n = 50_000
    rng = np.random.default_rng(9)
    d = rng.integers(9000, 9400, n).astype(np.int32)
    s = rng.integers(0, 300, n)
    names = [f"name-{i:03d}" for i in range(300)]
    v = rng.integers(-1000, 1000, n)
    tbl = pa.table({"d": pa.array(d, type=pa.date32()), "s": pa.DictionaryArray.from_arrays(pa.array(s.astype(np.int32)), pa.array(names)),
                    "v": pa.array(v)})
    plan = P.hash_agg(P.scan([P.DATE, P.STRING, P.INT64]), [P.bound(0, P.DATE), P.bound(1, P.STRING)],
                      [P.agg_sum(P.bound(2, P.INT64), P.INT64), P.agg_count([P.literal(1, P.INT32)])], P.PARTIAL)
    out = run(cb, plan, [tbl.to_batches(max_chunksize=8192)], 20_000)
    exp = {}
    for a, b, c in zip(d.tolist(), s.tolist(), v.tolist()):
        e = exp.setdefault((a, names[b]), [0, 0])
        e[0] += c
        e[1] += 1
    import datetime
    epoch = datetime.date(1970, 1, 1)
    got = {((r["col_0"] - epoch).days, r["col_1"]): [r["col_2"], r["col_3"]] for r in out.to_pylist()}
    assert got == exp


def test_table_growth_and_rehash(cb):
    """Many small chunks force the table to grow several times."""
    P = cb.proto
    n = 400_000
    k = np.arange(n, dtype=np.int64) * 7919 % 1_000_003
    v = np.ones(n, dtype=np.int64)
    plan = P.hash_agg(P.scan([P.INT64, P.INT64]), [P.bound(0, P.INT64)], [P.agg_sum(P.bound(1, P.INT64), P.INT64)], P.PARTIAL)
    out = run(cb, plan, [pa.table({"k": k, "v": v}).to_batches(max_chunksize=8192)], 16_384)
    assert out.num_rows == len(np.unique(k))
    assert sum(out.column(1).to_pylist()) == n


def test_multi_word_keys_with_nulls(cb):
    """(int64, int64, date32) needs 3 key words + a null-flag word: tag + stored-key probing, collisions resolved by the full key."""
    P = cb.proto
    import datetime
    n = 80_000
    rng = np.random.default_rng(21)
    a = rng.integers(-3, 3, n) * (2**40)
    b = rng.integers(0, 40, n) - 20
    d = rng.integers(9000, 9010, n).astype(np.int32)
    v = rng.integers(-1000, 1000, n)
    ma, mb, md = rng.random(n) < 0.1, rng.random(n) < 0.1, rng.random(n) < 0.1
    tbl = pa.table({"a": pa.array(a, mask=ma), "b": pa.array(b, mask=mb), "d": pa.array(d, type=pa.date32(), mask=md), "v": pa.array(v)})
    plan = P.hash_agg(P.scan([P.INT64, P.INT64, P.DATE, P.INT64]), [P.bound(0, P.INT64), P.bound(1, P.INT64), P.bound(2, P.DATE)],
                      [P.agg_sum(P.bound(3, P.INT64), P.INT64), P.agg_count([P.literal(1, P.INT32)])], P.PARTIAL)
    out = run(cb, plan, [tbl.to_batches(max_chunksize=8192)], 30_000)
    exp = {}
    for i in range(n):
        k = (None if ma[i] else int(a[i]), None if mb[i] else int(b[i]), None if md[i] else int(d[i]))
        e = exp.setdefault(k, [0, 0])
        e[0] += int(v[i])
        e[1] += 1
    epoch = datetime.date(1970, 1, 1)
    got = {(r["col_0"], r["col_1"], None if r["col_2"] is None else (r["col_2"] - epoch).days): [r["col_3"], r["col_4"]] for r in out.to_pylist()}
    assert got == exp


def test_key_nullability_may_change_between_batches(cb):
    """The first chunk has no validity buffers, later chunks do: the key packing must not depend on that."""
    P = cb.proto
    n = 40_000
    rng = np.random.default_rng(22)
    k1 = rng.integers(0, 50, n).astype(np.int32)
    k2 = rng.integers(0, 7, n).astype(np.int32)
    v = rng.integers(0, 100, n)
    m1 = np.zeros(n, dtype=bool)
    m1[n // 2:] = rng.random(n - n // 2) < 0.2           # NULLs only in the second half
    tbl = pa.table({"k1": pa.array(k1, mask=m1), "k2": pa.array(k2), "v": pa.array(v)})
    plan = P.hash_agg(P.scan([P.INT32, P.INT32, P.INT64]), [P.bound(0, P.INT32), P.bound(1, P.INT32)],
                      [P.agg_sum(P.bound(2, P.INT64), P.INT64)], P.PARTIAL)
    for batches in (tbl.to_batches(max_chunksize=4096), [tbl.slice(0, n // 2).to_batches()[0]] + tbl.slice(n // 2).to_batches(max_chunksize=4096)):
        out = run(cb, plan, [batches], 10_000)
        exp = {}
        for i in range(n):
            k = (None if m1[i] else int(k1[i]), int(k2[i]))
            exp[k] = exp.get(k, 0) + int(v[i])
        assert {(r["col_0"], r["col_1"]): r["col_2"] for r in out.to_pylist()} == exp


def test_dense_to_hash_migration_mid_stream(cb):
    """A dictionary key starts with 6 values (dense, thread-private accumulators) and grows to 300 in later batches: the dense
    state is flushed as one partial-state batch, the rest goes through the hash table, and Final merges the duplicates."""
    P = cb.proto
    rng = np.random.default_rng(31)
    names_small = [f"s{i}" for i in range(6)]
    names_big = [f"b{i:03d}" for i in range(294)] + names_small          # overlaps the early groups
    batches, exp = [], {}
    for bi in range(12):
        names = names_small if bi < 4 else names_big
        n = 5000
        codes = rng.integers(0, len(names), n).astype(np.int32)
        vals = rng.integers(-10**6, 10**6, n)
        for c, v in zip(codes.tolist(), vals.tolist()):
            e = exp.setdefault(names[c], [0, 0])
            e[0] += v
            e[1] += 1
        batches.append(pa.RecordBatch.from_arrays([pa.DictionaryArray.from_arrays(pa.array(codes), pa.array(names)), pa.array(vals)], names=["k", "v"]))
    partial = P.hash_agg(P.scan([P.STRING, P.INT64]), [P.bound(0, P.STRING)], [P.agg_sum(P.bound(1, P.INT64), P.INT64), P.agg_count([P.literal(1, P.INT32)])], P.PARTIAL)
    final = P.hash_agg(P.scan([P.STRING, P.INT64, P.INT64], source="shuffle"), [P.bound(0, P.STRING)],
                       [P.agg_sum(P.unbound("s", P.INT64), P.INT64), P.agg_count([P.unbound("c", P.INT32)])], P.FINAL)
    state = run(cb, partial, [batches], 5000)                              # one device chunk per batch
    assert state.num_rows > len(exp)                                       # the early groups appear twice: once per path
    res = run(cb, final, [state])
    assert {r["col_0"]: [r["col_1"], r["col_2"]] for r in res.to_pylist()} == exp


def test_dense_regroup_when_dictionary_grows_and_gains_nulls(cb):
    """A dictionary key stays on the dense path while its plan-global dictionary grows from 3 to 10 values and NULL keys appear
    in a later batch: the accumulated totals move to each wider group layout, the NULL slot staying the last one of its key."""
    P = cb.proto
    rng = np.random.default_rng(47)
    names = [f"k{i}" for i in range(10)]
    batches, exp = [], {}
    for n_values, null_frac in ((3, 0.0), (6, 0.0), (9, 0.15), (10, 0.1)):
        n = 5000
        codes = rng.integers(0, n_values, n).astype(np.int32)
        vals = rng.integers(-10**9, 10**9, n)
        nulls = rng.random(n) < null_frac
        for c, v, isnull in zip(codes.tolist(), vals.tolist(), nulls.tolist()):
            e = exp.setdefault(None if isnull else names[c], [0, 0])
            e[0] += v
            e[1] += 1
        keys = pa.DictionaryArray.from_arrays(pa.array(codes, mask=nulls if null_frac else None), pa.array(names[:n_values]))
        batches.append(pa.RecordBatch.from_arrays([keys, pa.array(vals)], names=["k", "v"]))
    plan = P.hash_agg(P.scan([P.STRING, P.INT64]), [P.bound(0, P.STRING)], [P.agg_sum(P.bound(1, P.INT64), P.INT64), P.agg_count([P.literal(1, P.INT32)])], P.PARTIAL)
    out = run(cb, plan, [batches], 5000)                                   # one device chunk per batch
    assert out.num_rows == len(exp) == 11                                  # dense: every group exactly once, NULL included
    assert {r["col_0"]: [r["col_1"], r["col_2"]] for r in out.to_pylist()} == exp


# ---- stream mode (CB_STREAM): Partial aggregates over clustered keys emit one state row per run, no key table --------------------
def run_cfg(cb, plan, inputs, cfg):
    with cb.native.Plan(plan, inputs, config={k: str(v) for k, v in cfg.items()}) as p:
        return p.collect()


STREAM = {"spark.comet.b200.streamAgg.minRows": 0}


def merge_states(rows, ncols):
    """Final-stage semantics for (sum, count, min, max) state rows keyed by col_0: what merging the partial rows must give."""
    out = {}
    for r in rows:
        e = out.get(r["col_0"])
        if e is None:
            out[r["col_0"]] = [r[f"col_{j}"] for j in range(1, ncols)]
        else:
            for j, f in enumerate(("sum", "sum", "min", "max")[: ncols - 1]):
                a, b = e[j], r[f"col_{j + 1}"]
                if a is None or b is None:
                    e[j] = a if b is None else b
                else:
                    e[j] = a + b if f == "sum" else (min(a, b) if f == "min" else max(a, b))
    return out


@pytest.mark.parametrize("chunk", [None, 150_000])
def test_stream_partial_over_clustered_keys(cb, chunk):
    """Clustered keys (every key ~5 times in a row, some NULL keys and NULL values): runs of equal adjacent keys become state rows.
    A key may appear in more than one state row (runs split at warp / chunk borders); merged by key they are the exact groups."""
    P = cb.proto
    rng = np.random.default_rng(12)
    n = 600_000
    k = np.repeat(np.arange(n // 3, dtype=np.int64) * 3 - 1000, rng.integers(1, 10, n // 3))[:n]      # ~5 adjacent rows per key
    v = rng.integers(-10**6, 10**6, n)
    km, vm = np.zeros(n, dtype=bool), rng.random(n) < 0.1
    km[1000:1040] = True
    km[300_000:300_003] = True
    tbl = pa.table({"k": pa.array(k, mask=km), "v": pa.array(v, mask=vm)})
    plan = P.hash_agg(P.scan([P.INT64, P.INT64]), [P.bound(0, P.INT64)],
                      [P.agg_sum(P.bound(1, P.INT64), P.INT64), P.agg_count([P.bound(1, P.INT64)]), P.agg_min(P.bound(1, P.INT64), P.INT64),
                       P.agg_max(P.bound(1, P.INT64), P.INT64)], P.PARTIAL)
    cfg = dict(STREAM)
    if chunk:
        cfg["spark.comet.b200.chunkRows"] = chunk
    out = run_cfg(cb, plan, [tbl.to_batches(max_chunksize=8192)], cfg)
    exp = {}
    for kk, vv, a, b in zip(k.tolist(), v.tolist(), km.tolist(), vm.tolist()):
        key = None if a else kk
        e = exp.setdefault(key, [None, 0, None, None])
        if not b:
            e[0] = vv if e[0] is None else e[0] + vv
            e[1] += 1
            e[2] = vv if e[2] is None else min(e[2], vv)
            e[3] = vv if e[3] is None else max(e[3], vv)
    assert len(exp) <= out.num_rows < 0.5 * n                       # streamed (no table): at most a few split runs more than groups
    assert merge_states(out.to_pylist(), 5) == exp


def test_stream_partial_feeds_final_decimal_and_f64(cb):
    """The Config 4 shape end to end: streamed Partial state -> Final, decimal sums bit-exact, f64 sums within 1 ULP of the exact sum."""
    t = cb.tpch
    n = 500_000
    cols = t.gen_lineitem(n, seed=11)
    for variant in ("dec", "f64"):
        partial, final = plans(cb, variant)
        price = cols["l_extendedprice"]
        vcol = t._dec_array(price) if variant == "dec" else pa.array(price.astype(np.float64) / 100.0)
        tbl = pa.table({"k": pa.array(cols["l_orderkey"]), "v": vcol})
        state = run_cfg(cb, partial, [tbl.to_batches(max_chunksize=8192)], STREAM)
        uk, inv = np.unique(cols["l_orderkey"], return_inverse=True)
        assert len(uk) <= state.num_rows <= len(uk) + n // 32 + 1024
        res = run(cb, final, [state])
        keys = np.array(res.column(0).to_pylist())
        order = np.argsort(keys)
        assert (keys[order] == uk).all()
        if variant == "dec":
            exp = np.zeros(len(uk), dtype=np.int64)
            np.add.at(exp, inv, price)
            got = np.array([unscaled(x) for x in res.column(1).to_pylist()], dtype=np.int64)[order]
            assert (got == exp).all()
        else:
            vals = np.array(res.column(1).to_pylist())[order]
            pf = price.astype(np.float64) / 100.0
            for i in range(0, len(uk), 4999):
                exact = math.fsum(pf[inv == i])
                assert abs(vals[i] - exact) <= math.ulp(exact)


def test_stream_sample_sees_scattered_keys_and_keeps_the_table(cb):
    """Keys in random order: the sample finds (almost) one run per row, so the key table is used and every group is one state row."""
    P = cb.proto
    n = 300_000
    rng = np.random.default_rng(5)
    k = rng.integers(0, 5000, n)
    v = np.ones(n, dtype=np.int64)
    plan = P.hash_agg(P.scan([P.INT64, P.INT64]), [P.bound(0, P.INT64)], [P.agg_sum(P.bound(1, P.INT64), P.INT64)], P.PARTIAL)
    out = run_cfg(cb, plan, [pa.table({"k": k, "v": v}).to_batches(max_chunksize=8192)], STREAM)
    assert out.num_rows == len(np.unique(k)) and sum(out.column(1).to_pylist()) == n


def test_stream_runs_outgrow_the_estimate(cb):
    """The sampled prefix is clustered (8 rows per key), the tail is not (every row its own key): the launch runs out of state rows,
    is discarded, the arrays grow and it is repeated -- nothing may be lost or counted twice (incl. the shared NULL-key group)."""
    P = cb.proto
    n_head, n_tail = 1_200_000, 900_000
    k = np.concatenate([np.repeat(np.arange(n_head // 8, dtype=np.int64), 8), 10**9 + np.arange(n_tail, dtype=np.int64)])
    km = np.zeros(len(k), dtype=bool)
    km[5:9] = True
    km[n_head + 10:n_head + 12] = True
    v = np.arange(len(k), dtype=np.int64) % 1000
    plan = P.hash_agg(P.scan([P.INT64, P.INT64]), [P.bound(0, P.INT64)], [P.agg_sum(P.bound(1, P.INT64), P.INT64), P.agg_count([P.bound(1, P.INT64)])], P.PARTIAL)
    out = run_cfg(cb, plan, [pa.table({"k": pa.array(k, mask=km), "v": v}).to_batches(max_chunksize=65536)], STREAM)
    got = merge_states(out.to_pylist(), 3)
    assert got[None] == [int(v[km].sum()), int(km.sum())]
    assert len(got) == n_head // 8 + n_tail + 1 - 2          # keys 0 and 1 lose rows to NULL but survive; two tail keys are NULL
    assert sum(e[1] for e in got.values()) == len(k) and sum(e[0] for e in got.values()) == int(v.sum())
