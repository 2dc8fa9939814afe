"""GPU parity: TPC-H Q1 / Q6 / Config 1 through the C ABI vs the CPU oracle (bit-exact for decimals,
1 ULP of the exact sum for float aggregates).  `pytest -m gpu` on an H100."""
import math

import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu

RF = ["A", "N", "R"]
LS = ["F", "O"]


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def dec(o, a):
    return o.dec_from_i64(a)


def run(cb, plan, inputs, chunk_rows=None):
    cfg = {"spark.comet.b200.chunkRows": str(chunk_rows)} if chunk_rows else None
    with cb.native.Plan(plan, inputs, config=cfg) as p:
        t = p.collect()
        assert p.kernel_launches > 0
    return t


def q1_groups(table):
    """{(rf, ls): row dict} from a Q1 result table"""
    d = table.to_pydict()
    out = {}
    for i in range(table.num_rows):
        out[(d["col_0"][i], d["col_1"][i])] = {k: d[k][i] for k in d}
    return out


def unscaled(x):
    """python Decimal -> unscaled integer"""
    return None if x is None else int(x.scaleb(-x.as_tuple().exponent))


@pytest.mark.parametrize("n,chunk", [(1000, None), (200_000, 65536), (1_000_003, 300_000)])
@pytest.mark.parametrize("dictionary", [True, False])
def test_q1_dec_partial_and_final(cb, oracle, n, chunk, dictionary):
    t = cb.tpch
    cols = t.gen_lineitem(n, seed=42)
    tbl = t.lineitem_table(cols, "dec", dictionary=dictionary)
    state = run(cb, t.q1_partial_plan("dec"), [tbl.to_batches(max_chunksize=8192)], chunk)
    assert state.num_columns == 17
    res = run(cb, t.q1_final_plan("dec"), [state])
    exp = oracle.q1_dec(dec(oracle, cols["l_quantity"]), dec(oracle, cols["l_extendedprice"]), dec(oracle, cols["l_discount"]),
                        dec(oracle, cols["l_tax"]), cols["l_shipdate"], cols["l_returnflag"], cols["l_linestatus"], 3, 2,
                        t.Q1_CUTOFF, 1)
    got = q1_groups(res)
    n_exp = 0
    for k, e in enumerate(exp):
        if e is None:
            continue
        n_exp += 1
        g = got[(RF[k // 2], LS[k % 2])]
        names = ["sum_qty", "sum_base", "sum_disc_price", "sum_charge", "avg_qty", "avg_price", "avg_disc"]
        for j, name in enumerate(names):
            assert unscaled(g[f"col_{2 + j}"]) == e[name], (k, name)
        assert g["col_9"] == e["count"]
    assert len(got) == n_exp
    # schema of the final result == golden q1.sql.out:4 types
    assert [str(f.type) for f in res.schema][2:] == ["decimal128(22, 2)", "decimal128(22, 2)", "decimal128(36, 4)",
                                                     "decimal128(38, 6)", "decimal128(16, 6)", "decimal128(16, 6)",
                                                     "decimal128(16, 6)", "int64"]


def test_q1_dec_partial_state_matches_accumulators(cb, oracle):
    t = cb.tpch
    n = 50_000
    cols = t.gen_lineitem(n, seed=7)
    tbl = t.lineitem_table(cols, "dec", dictionary=True)
    state = run(cb, t.q1_partial_plan("dec"), [tbl.to_batches(max_chunksize=8192)])
    keep = cols["l_shipdate"] <= t.Q1_CUTOFF
    gid = (cols["l_returnflag"].astype(np.int64) * 2 + cols["l_linestatus"])[keep]
    acc = oracle.SumDecimalGroups(6, 22)
    acc.update(dec(oracle, cols["l_quantity"][keep]), None, gid)
    s, sv, e = acc.state()
    d = state.to_pydict()
    for i in range(state.num_rows):
        k = RF.index(d["col_0"][i]) * 2 + LS.index(d["col_1"][i])
        assert unscaled(d["col_2"][i]) == oracle.dec_to_ints(s[k:k + 1])[0]
        assert d["col_3"][i] == bool(e[k])  # is_empty
    assert str(state.schema.field(3).type) == "bool" and str(state.schema.field(11).type) == "int64"


@pytest.mark.parametrize("n", [1000, 300_000])
def test_q1_f64(cb, oracle, n):
    t = cb.tpch
    cols = t.gen_lineitem(n, seed=11)
    tbl = t.lineitem_table(cols, "f64", dictionary=True)
    state = run(cb, t.q1_partial_plan("f64"), [tbl.to_batches(max_chunksize=8192)], 100_000)
    res = run(cb, t.q1_final_plan("f64"), [state])
    got = q1_groups(res)
    f = {k: (cols[k].astype(np.float64) / 100.0) for k in ("l_quantity", "l_extendedprice", "l_discount", "l_tax")}
    keep = cols["l_shipdate"] <= t.Q1_CUTOFF
    gid = (cols["l_returnflag"].astype(np.int64) * 2 + cols["l_linestatus"])
    dp = f["l_extendedprice"] * (1.0 - f["l_discount"])
    ch = dp * (1.0 + f["l_tax"])
    for k in range(6):
        m = keep & (gid == k)
        cnt = int(m.sum())
        if cnt == 0:
            assert (RF[k // 2], LS[k % 2]) not in got
            continue
        g = got[(RF[k // 2], LS[k % 2])]
        for j, v in enumerate([f["l_quantity"], f["l_extendedprice"], dp, ch]):
            exact = math.fsum(v[m])
            assert abs(g[f"col_{2 + j}"] - exact) <= math.ulp(exact), (k, j)  # north_star: within 1 ULP
            seq = oracle.sum_f64_groups(v[m], None, None, 1)[0][0]          # reference row-order sum
            assert abs(g[f"col_{2 + j}"] - seq) <= 1e-9 * abs(seq)
        for j, v in enumerate([f["l_quantity"], f["l_extendedprice"], f["l_discount"]]):
            exact_avg = math.fsum(v[m]) / cnt
            assert abs(g[f"col_{6 + j}"] - exact_avg) <= 2 * math.ulp(exact_avg)
        assert g["col_9"] == cnt


@pytest.mark.parametrize("n,chunk", [(5000, None), (500_000, 131072)])
def test_q6_dec(cb, oracle, n, chunk):
    t = cb.tpch
    cols = t.gen_lineitem(n, seed=13)
    tbl = t.lineitem_table(cols, "dec", columns=["l_quantity", "l_extendedprice", "l_discount", "l_shipdate"])
    state = run(cb, t.q6_partial_plan("dec"), [tbl.to_batches(max_chunksize=8192)], chunk)
    assert state.num_rows == 1 and state.num_columns == 2
    res = run(cb, t.q6_final_plan("dec"), [state])
    exp = oracle.q6_dec(dec(oracle, cols["l_quantity"]), dec(oracle, cols["l_extendedprice"]), dec(oracle, cols["l_discount"]),
                        cols["l_shipdate"], t.DATE_1994_01_01, t.DATE_1995_01_01, 5, 7, 2400, 1)
    assert unscaled(res.column(0)[0].as_py()) == exp
    assert str(res.schema.field(0).type) == "decimal128(35, 4)"


def test_q6_f64(cb, oracle):
    t = cb.tpch
    n = 400_000
    cols = t.gen_lineitem(n, seed=17)
    tbl = t.lineitem_table(cols, "f64", columns=["l_quantity", "l_extendedprice", "l_discount", "l_shipdate"])
    state = run(cb, t.q6_partial_plan("f64"), [tbl.to_batches(max_chunksize=8192)], 100_000)
    res = run(cb, t.q6_final_plan("f64"), [state])
    q, p, d = (cols[k].astype(np.float64) / 100.0 for k in ("l_quantity", "l_extendedprice", "l_discount"))
    m = (cols["l_shipdate"] >= t.DATE_1994_01_01) & (cols["l_shipdate"] < t.DATE_1995_01_01) & (d >= 0.05) & (d <= 0.07) & (q < 24.0)
    exact = math.fsum((p * d)[m])
    assert abs(res.column(0)[0].as_py() - exact) <= math.ulp(exact)


def test_q6_empty_input_emits_one_null_row(cb):
    t = cb.tpch
    cols = t.gen_lineitem(100, seed=1)
    cols["l_shipdate"][:] = 0  # nothing passes the filter
    tbl = t.lineitem_table(cols, "dec", columns=["l_quantity", "l_extendedprice", "l_discount", "l_shipdate"])
    state = run(cb, t.q6_partial_plan("dec"), [tbl])
    assert state.num_rows == 1
    assert state.column(1)[0].as_py() is True  # is_empty
    res = run(cb, t.q6_final_plan("dec"), [state])
    assert res.column(0)[0].as_py() is None


@pytest.mark.parametrize("n,chunk", [(1, None), (1023, None), (1024, None), (1025, None), (100_000, 40_000), (1_200_000, None)])
def test_config1_dec(cb, oracle, n, chunk):
    t = cb.tpch
    cols = t.gen_lineitem(n, seed=19)
    tbl = t.lineitem_table(cols, "dec", columns=["l_quantity", "l_extendedprice", "l_shipdate"])
    res = run(cb, t.config1_plan("dec"), [tbl.to_batches(max_chunksize=8192)], chunk)
    eo, ev = oracle.filter_project_dec(dec(oracle, cols["l_quantity"]), dec(oracle, cols["l_extendedprice"]), cols["l_shipdate"],
                                       t.DATE_1998_09_02, 1)
    assert res.num_rows == eo.shape[0]
    got = np.frombuffer(res.column(0).combine_chunks().buffers()[1], dtype=np.uint64)[: 2 * eo.shape[0]].reshape(-1, 2)
    assert (got == eo).all()                      # bit-exact, stable row order
    assert res.column(0).null_count == 0
    assert str(res.schema.field(0).type) == "decimal128(25, 4)"


@pytest.mark.parametrize("n", [777, 600_000])
def test_config1_f64(cb, oracle, n):
    t = cb.tpch
    cols = t.gen_lineitem(n, seed=23)
    tbl = t.lineitem_table(cols, "f64", columns=["l_quantity", "l_extendedprice", "l_shipdate"])
    res = run(cb, t.config1_plan("f64"), [tbl.to_batches(max_chunksize=8192)], 250_000)
    q, p = cols["l_quantity"].astype(np.float64) / 100.0, cols["l_extendedprice"].astype(np.float64) / 100.0
    exp = oracle.filter_project_f64(q, p, cols["l_shipdate"], t.DATE_1998_09_02, 1)
    got = res.column(0).to_numpy()
    assert got.shape == exp.shape and (got.view(np.uint64) == exp.view(np.uint64)).all()  # IEEE mul: bit-exact


def test_config1_all_filtered(cb):
    t = cb.tpch
    cols = t.gen_lineitem(5000, seed=3)
    cols["l_shipdate"][:] = 20000
    tbl = t.lineitem_table(cols, "f64", columns=["l_quantity", "l_extendedprice", "l_shipdate"])
    res = run(cb, t.config1_plan("f64"), [tbl])
    assert res.num_rows == 0


def test_nullable_inputs_q1(cb, oracle):
    """NULL shipdate rows are dropped by the filter, NULL money values are skipped by the accumulators."""
    t = cb.tpch
    n = 60_000
    cols = t.gen_lineitem(n, seed=29)
    rng = np.random.default_rng(5)
    vq = rng.random(n) > 0.1
    vs = rng.random(n) > 0.05
    tbl = t.lineitem_table(cols, "dec", dictionary=True)
    tbl = tbl.set_column(0, "l_quantity", t._dec_array(cols["l_quantity"], valid=vq))
    tbl = tbl.set_column(6, "l_shipdate", pa.array(cols["l_shipdate"], type=pa.date32(), mask=~vs))
    state = run(cb, t.q1_partial_plan("dec"), [tbl.to_batches(max_chunksize=8192)], 20_000)
    res = run(cb, t.q1_final_plan("dec"), [state])
    got = q1_groups(res)
    keep = vs & (cols["l_shipdate"] <= t.Q1_CUTOFF)
    gid = cols["l_returnflag"].astype(np.int64) * 2 + cols["l_linestatus"]
    for k in range(6):
        m = keep & (gid == k)
        if not m.any():
            continue
        g = got[(RF[k // 2], LS[k % 2])]
        assert unscaled(g["col_2"]) == int(cols["l_quantity"][m & vq].sum())
        assert unscaled(g["col_3"]) == int(cols["l_extendedprice"][m].sum())
        assert g["col_9"] == int(m.sum())
        # avg(l_quantity) counts only non-null quantities
        s, c = int(cols["l_quantity"][m & vq].sum()), int((m & vq).sum())
        q, r = divmod(s * 10**4, c)
        exp_avg = q + (1 if 2 * r >= c else 0)
        assert unscaled(g["col_6"]) == exp_avg


@pytest.mark.parametrize("variant", ["dec", "f64"])
def test_partial_merge_is_transparent(cb, variant):
    """AggregateMode PartialMerge (operator.proto: merge state columns, emit state columns): Partial -> PartialMerge -> Final
    over several partitions gives exactly what Partial -> Final gives."""
    t = cb.tpch
    P = cb.proto
    n = 120_000
    cols = t.gen_lineitem(n, seed=77)
    parts = []
    for lo, hi in [(0, 50_000), (50_000, 90_000), (90_000, n)]:
        tbl = t.lineitem_table({k: v[lo:hi] for k, v in cols.items()}, variant)
        parts.append(run(cb, t.q1_partial_plan(variant), [tbl.to_batches(max_chunksize=8192)]))
    states = pa.concat_tables(parts)
    direct = run(cb, t.q1_final_plan(variant), [states])
    sc = P.scan(t.q1_state_fields(variant), source="shuffle")
    merge_plan = P.hash_agg(sc, [P.bound(0, P.STRING), P.bound(1, P.STRING)], t.q1_aggs(variant, bound=False), P.PARTIAL_MERGE)
    merged = run(cb, merge_plan, [pa.concat_tables(parts[:2])])            # two partitions pre-merged ...
    assert merged.schema.types == parts[0].schema.types
    via_merge = run(cb, t.q1_final_plan(variant), [pa.concat_tables([merged, parts[2]])])   # ... then finalised with the third
    a, b = q1_groups(direct), q1_groups(via_merge)
    assert a.keys() == b.keys()
    for k in a:
        for c in a[k]:
            if variant == "f64" and isinstance(a[k][c], float):
                assert math.isclose(a[k][c], b[k][c], rel_tol=1e-15), (k, c)    # double-double partial sums re-rounded once more
            else:
                assert a[k][c] == b[k][c], (k, c)
