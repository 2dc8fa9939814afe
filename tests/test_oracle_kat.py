"""Pin the CPU oracle against the reference's own in-file known-answer tests.

Each test names the reference file:line holding the vector (paths under native/ of
apache/datafusion-comet).  These run on CPU (`-m "not gpu"`).
"""
import numpy as np
import pytest

LEGACY, TRY, ANSI = 0, 1, 2
ADD, SUB, MUL = 0, 1, 2


def u32(xs):
    return [x & 0xFFFFFFFF for x in xs]


# ---- murmur3: spark-expr/src/hash_funcs/murmur3.rs:208-280 -------------------------------------
def test_murmur3_i8(oracle):  # murmur3.rs:208-213
    h = oracle.murmur3_column("i8", [1, 0, -1, 127, -128])
    assert list(h) == [0xDEA578E3, 0x379FAE8F, 0xA0590E3D, 0x43B4D8ED, 0x422A1365]


def test_murmur3_i32(oracle):  # murmur3.rs:216-221
    h = oracle.murmur3_column("i32", [1, 0, -1, 2**31 - 1, -(2**31)])
    assert list(h) == [0xDEA578E3, 0x379FAE8F, 0xA0590E3D, 0x07FB67E7, 0x2B1F0FC6]


def test_murmur3_i64(oracle):  # murmur3.rs:224-229
    h = oracle.murmur3_column("i64", [1, 0, -1, 2**63 - 1, -(2**63)])
    assert list(h) == [0x99F0149D, 0x9C67B85D, 0xC8008529, 0xA05B5D7B, 0xCD1E64FB]


def test_murmur3_f32(oracle):  # murmur3.rs:232-247
    vals = np.array([1.0, 0.0, -0.0, -1.0, 99999999999.99999999999, -99999999999.99999999999], dtype=np.float32)
    h = oracle.murmur3_column("f32", vals)
    assert list(h) == [0xE434CC39, 0x379FAE8F, 0x379FAE8F, 0xDC0DA8EB, 0xCBDC340F, 0xC0361C86]


def test_murmur3_f64(oracle):  # murmur3.rs:250-265
    vals = np.array([1.0, 0.0, -0.0, -1.0, 99999999999.99999999999, -99999999999.99999999999])
    h = oracle.murmur3_column("f64", vals)
    assert list(h) == [0xE4876492, 0x9C67B85D, 0x9C67B85D, 0x13D81357, 0xB87E1595, 0xA0EEF9F9]


def test_murmur3_str(oracle):  # murmur3.rs:268-280
    inp = ["hello", "bar", "", "😁", "天地", "a", "ab", "abc", "abcd", "abcde"]
    exp = [3286402344, 2486176763, 142593372, 885025535, 2395000894, 1485273170, 0xFA37157B, 1322437556,
           0xE860E5CC, 814637928]
    assert list(oracle.murmur3_strings(inp)) == exp


def test_murmur3_null_leaves_hash(oracle):  # hash_funcs/utils.rs:38-42
    h = oracle.murmur3_column("i32", [1, 5, 1], valid=[1, 0, 1])
    assert h[1] == 42 and h[0] == h[2] == 0xDEA578E3


def test_murmur3_small_decimal_is_i64(oracle):  # hash_funcs/utils.rs:159-196,726-728
    d = oracle.dec_from_ints([1, 0, -1])
    assert list(oracle.murmur3_column("dec_small", d)) == [0x99F0149D, 0x9C67B85D, 0xC8008529]


def test_murmur3_large_decimal_16_bytes(oracle):  # hash_funcs/utils.rs:199-226
    d = oracle.dec_from_ints([1, -1])
    h = oracle.murmur3_column("dec_large", d)
    assert h[0] == oracle.murmur3_bytes((1).to_bytes(16, "little", signed=True))
    assert h[1] == oracle.murmur3_bytes((-1).to_bytes(16, "little", signed=True))


def test_murmur3_chain_two_columns(oracle):  # utils.rs:573-580 chained seed
    h = oracle.murmur3_column("i32", [7, 8])
    h2 = oracle.murmur3_column("i64", [1, 2], hashes=h.copy())
    for i, (a, b) in enumerate([(7, 1), (8, 2)]):
        s = oracle.murmur3_bytes(int(a).to_bytes(4, "little", signed=True), 42)
        assert h2[i] == oracle.murmur3_bytes(int(b).to_bytes(8, "little", signed=True), s)


def test_pmod(oracle):  # shuffle/src/comet_partitioning.rs:63-71
    hs = [0x99F0149D, 0x9C67B85D, 0xC8008529, 0xA05B5D7B, 0xCD1E64FB]
    assert [oracle.pmod(h, 200) for h in hs] == [69, 5, 193, 171, 115]


def test_partition_rows_stable(oracle):  # shuffle/src/partitioners/multi_partition.rs:54-99
    hs = np.array([0x99F0149D, 0x9C67B85D, 0xC8008529, 0xA05B5D7B, 0xCD1E64FB, 0x99F0149D], dtype=np.uint32)
    pids, starts, idx = oracle.partition_rows(hs, 4)
    assert list(pids) == [oracle.pmod(h, 4) for h in hs]
    for p in range(4):
        seg = list(idx[starts[p]:starts[p + 1]])
        assert seg == sorted(seg) and all(pids[i] == p for i in seg)


# ---- wide decimal: spark-expr/src/math_funcs/wide_decimal_binary_expr.rs:399-560 ----------------
def _wide(oracle, op, l, s1, r, s2, p, s, mode=LEGACY):
    lv = [x is not None for x in l]
    rv = [x is not None for x in r]
    out, outv = oracle.wide_decimal(op, oracle.dec_from_ints(l), lv, s1, oracle.dec_from_ints(r), rv, s2, p, s, mode)
    return oracle.dec_to_ints(out, outv)


def test_wide_add_same_scale(oracle):  # :399-414
    assert _wide(oracle, ADD, [1000000000, 2500000000], 10, [2000000000, 7500000000], 10, 38, 10) == [3000000000, 10000000000]


def test_wide_subtract_same_scale(oracle):  # :417-430
    assert _wide(oracle, SUB, [5000, 1000], 2, [3000, 2000], 2, 38, 2) == [2000, -1000]


def test_wide_add_different_scales(oracle):  # :433-446
    assert _wide(oracle, ADD, [150], 2, [2500], 4, 38, 4) == [17500]


def test_wide_mul_scale_reduction(oracle):  # :449-464
    assert _wide(oracle, MUL, [100000], 5, [200000], 5, 38, 6) == [2000000]


def test_wide_mul_half_up(oracle):  # :467-483
    assert _wide(oracle, MUL, [15], 1, [15], 1, 38, 1) == [23]


def test_wide_mul_half_up_negative(oracle):  # :486-500
    assert _wide(oracle, MUL, [-15], 1, [15], 1, 38, 1) == [-23]


def test_wide_overflow_legacy_null(oracle):  # :503-509
    assert _wide(oracle, ADD, [5], 0, [5], 0, 1, 0) == [None]


def test_wide_overflow_ansi_error(oracle):  # :512-516
    with pytest.raises(oracle.OracleError):
        _wide(oracle, ADD, [5], 0, [5], 0, 1, 0, ANSI)


def test_wide_null_propagation(oracle):  # :519-525
    assert _wide(oracle, ADD, [100, None], 2, [None, 200], 2, 38, 2) == [None, None]


def test_wide_zeros(oracle):  # :528-533
    assert _wide(oracle, MUL, [0], 10, [0], 10, 38, 10) == [0]


def test_wide_max_precision(oracle):  # :536-543
    m = 10**38 - 1
    assert _wide(oracle, ADD, [m], 0, [0], 0, 38, 0) == [m]


def test_wide_add_scale_up(oracle):  # :546-562
    assert _wide(oracle, ADD, [150], 2, [25], 2, 38, 4) == [17500]


def test_wide_sub_scale_up(oracle):  # :565-579
    assert _wide(oracle, SUB, [300], 2, [100], 2, 38, 4) == [20000]


def test_wide_scalar_pattern(oracle):  # :592-625  0.95 * 100.00 -> 95.00 at scale 2
    assert _wide(oracle, MUL, [95], 2, [10000], 2, 38, 2) == [9500]


def test_wide_matches_python_bigint(oracle):
    rng = np.random.default_rng(7)
    for op in (ADD, SUB, MUL):
        l = [int(rng.integers(-10**18, 10**18)) * int(rng.integers(1, 10**15)) for _ in range(300)]
        r = [int(rng.integers(-10**18, 10**18)) * int(rng.integers(1, 10**4)) for _ in range(300)]
        s1, s2, p, s = 6, 4, 38, 6
        got = _wide(oracle, op, l, s1, r, s2, p, s)
        for a, b, g in zip(l, r, got):
            if op == MUL:
                raw, nat = a * b, s1 + s2
            else:
                ms = max(s1, s2)
                x, y = a * 10**(ms - s1), b * 10**(ms - s2)
                raw, nat = (x + y if op == ADD else x - y), ms
            d = nat - s
            if d > 0:
                q, rem = divmod(abs(raw), 10**d)
                if rem * 2 >= 10**d:
                    q += 1
                res = q if raw >= 0 else -q
            else:
                res = raw * 10**(-d)
            exp = res if abs(res) <= 10**p - 1 else None
            assert g == exp


# ---- DecimalRescaleCheckOverflow: math_funcs/internal/decimal_rescale_check.rs:301-396 ----------
def _rescale(oracle, vals, s_in, p_out, s_out, fail=False):
    v = [x is not None for x in vals]
    out, outv = oracle.decimal_rescale_check(oracle.dec_from_ints(vals), v, s_in, p_out, s_out, fail)
    return oracle.dec_to_ints(out, outv)


def test_rescale_scale_up(oracle):  # :302-309
    assert _rescale(oracle, [150, -300], 2, 10, 4) == [15000, -30000]


def test_rescale_half_up(oracle):  # :312-323
    assert _rescale(oracle, [12350, 12349, -12350], 4, 10, 2) == [124, 123, -124]


def test_rescale_precision_only(oracle):  # :326-333
    assert _rescale(oracle, [999, 1000], 0, 3, 0) == [999, None]


def test_rescale_overflow_legacy(oracle):  # :336-343
    assert _rescale(oracle, [10], 0, 3, 2) == [None]


def test_rescale_overflow_ansi(oracle):  # :346-350
    with pytest.raises(oracle.OracleError):
        _rescale(oracle, [10], 0, 3, 2, True)


def test_rescale_overflow_with_nulls(oracle):  # :353-363
    assert _rescale(oracle, [150, 10_000, None, 250], 2, 4, 2) == [150, None, None, 250]


def test_rescale_all_overflow(oracle):  # :366-375
    assert _rescale(oracle, [10_000, 20_000, 30_000], 2, 4, 2) == [None, None, None]


def test_rescale_boundary(oracle):  # :378-386
    assert _rescale(oracle, [9999, 10_000], 0, 4, 0) == [9999, None]


# ---- CheckOverflow: math_funcs/internal/checkoverflow.rs:305-330 --------------------------------
def test_check_overflow_legacy(oracle):
    out, outv = oracle.check_overflow(oracle.dec_from_ints([999, 1000, -999, -1000]), None, 3, False)
    assert oracle.dec_to_ints(out, outv) == [999, None, -999, None]


def test_check_overflow_ansi(oracle):
    with pytest.raises(oracle.OracleError):
        oracle.check_overflow(oracle.dec_from_ints([1000]), None, 3, True)


# ---- SumDecimal: agg_funcs/sum_decimal.rs:732-801 -----------------------------------------------
def test_sum_decimal_update_with_filter(oracle):  # :732-754
    acc = oracle.SumDecimalGroups(1, 10)
    acc.update(oracle.dec_from_ints([100, 200, 300, 400]), None, [0, 0, 0, 0], filt=[1, 0, 1, 0])
    out, outv = acc.evaluate()
    assert oracle.dec_to_ints(out, outv) == [400]


def test_sum_decimal_filter_null_excluded(oracle):  # :757-778 (NULL filter entry == excluded)
    acc = oracle.SumDecimalGroups(1, 10)
    acc.update(oracle.dec_from_ints([10, 20, 30]), None, [0, 0, 0], filt=[1, 0, 1])
    out, outv = acc.evaluate()
    assert oracle.dec_to_ints(out, outv) == [40]


def test_sum_decimal_acc_merge_multi_row(oracle):  # :781-801
    acc = oracle.SumDecimalAcc(10)
    acc.merge(oracle.dec_from_ints([100, 200, 0, 300]), [1, 1, 0, 1], [0, 0, 1, 0], None)
    out, outv = acc.evaluate()
    assert oracle.dec_to_ints(out, outv) == [600]


def test_sum_decimal_overflow_sticky(oracle):  # sum_decimal.rs:418-439
    acc = oracle.SumDecimalGroups(2, 3)
    acc.update(oracle.dec_from_ints([999, 1, -500, 5]), None, [0, 0, 0, 1])
    out, outv = acc.evaluate()
    assert oracle.dec_to_ints(out, outv) == [None, 5]
    s, sv, e = acc.state()
    assert list(sv) == [0, 1] and list(e) == [0, 0]


def test_sum_decimal_empty_group_is_null(oracle):  # sum_decimal.rs:477-490
    acc = oracle.SumDecimalGroups(2, 10)
    acc.update(oracle.dec_from_ints([1]), None, [1])
    out, outv = acc.evaluate()
    assert oracle.dec_to_ints(out, outv) == [None, 1]


def test_sum_decimal_ansi_error(oracle):
    acc = oracle.SumDecimalGroups(1, 3, ANSI)
    with pytest.raises(oracle.OracleError):
        acc.update(oracle.dec_from_ints([999, 1]), None, [0, 0])


# ---- AvgDecimal: agg_funcs/avg_decimal.rs:597-689 -----------------------------------------------
def test_avg_decimal_half_up(oracle):
    # d(12,2) input -> sum d(22,2), result d(16,6): avg(1.00, 2.00, 2.00) = 1.666667
    acc = oracle.AvgDecimalGroups(1, 22, 2, 16, 6)
    acc.update(oracle.dec_from_ints([100, 200, 200]), None, [0, 0, 0])
    out, outv = acc.evaluate()
    assert oracle.dec_to_ints(out, outv) == [1666667]
    acc = oracle.AvgDecimalGroups(1, 22, 2, 16, 6)
    acc.update(oracle.dec_from_ints([-100, -200, -200]), None, [0, 0, 0])
    out, outv = acc.evaluate()
    assert oracle.dec_to_ints(out, outv) == [-1666667]


def test_avg_decimal_empty_null(oracle):
    acc = oracle.AvgDecimalGroups(2, 22, 2, 16, 6)
    acc.update(oracle.dec_from_ints([100]), [0], [0])
    out, outv = acc.evaluate()
    assert oracle.dec_to_ints(out, outv) == [None, None]


def test_avg_decimal_merge(oracle):
    a = oracle.AvgDecimalGroups(1, 22, 2, 16, 6)
    a.merge(oracle.dec_from_ints([100, 300]), [1, 1], [1, 2], [1, 1], [0, 0])
    out, outv = a.evaluate()
    assert oracle.dec_to_ints(out, outv) == [1333333]


# ---- SumInt: agg_funcs/sum_int.rs:918-990 -------------------------------------------------------
def test_sum_int_legacy_filter(oracle):  # :919-929
    acc = oracle.SumIntGroups(1)
    acc.update([1, 2, 3, 4, 5], None, [0] * 5, filt=[1, 0, 1, 0, 1])
    assert acc.sums[0] == 9 and acc.sums_valid[0] == 1


def test_sum_int_ansi_filter(oracle):  # :950-960
    acc = oracle.SumIntGroups(2, ANSI)
    acc.update([10, 20, 30, 40], None, [0, 1, 0, 1], filt=[1, 1, 0, 1])
    assert list(acc.sums) == [10, 60]


def test_sum_int_try_filter(oracle):  # :964-973
    acc = oracle.SumIntGroups(1, TRY)
    acc.update([1, 2, 3, 4, 5], None, [0] * 5, filt=[1, 0, 1, 0, 1])
    assert acc.sums[0] == 9


def test_sum_int_legacy_wraps(oracle):  # sum_int.rs:432 add_wrapping
    acc = oracle.SumIntGroups(1)
    acc.update([2**63 - 1, 1], None, [0, 0])
    assert acc.sums[0] == -(2**63)


def test_sum_int_ansi_overflow(oracle):
    acc = oracle.SumIntGroups(1, ANSI)
    with pytest.raises(oracle.OracleError):
        acc.update([2**63 - 1, 1], None, [0, 0])


def test_sum_int_all_null_is_null(oracle):  # sums stay None until first non-null
    acc = oracle.SumIntGroups(1)
    acc.update([1, 2], [0, 0], [0, 0])
    assert acc.sums_valid[0] == 0


# ---- checked arithmetic: math_funcs/checked_arithmetic.rs:53-128 --------------------------------
def test_int_arith_modes(oracle):
    out, outv = oracle.int_arith(0, 32, [2**31 - 1, 1], None, [1, 1], None, LEGACY)
    assert list(out) == [-(2**31), 2] and list(outv) == [1, 1]
    out, outv = oracle.int_arith(0, 32, [2**31 - 1, 1], None, [1, 1], None, TRY)
    assert list(outv) == [0, 1] and out[1] == 2
    with pytest.raises(oracle.OracleError):
        oracle.int_arith(2, 64, [2**62], None, [4], None, ANSI)


# ---- exact f64 sum (yardstick for the 1-ULP bar) -------------------------------------------------
def test_sum_f64_exact_against_fsum(oracle):
    import math
    rng = np.random.default_rng(3)
    v = rng.standard_normal(20000) * 10.0 ** rng.integers(-20, 20, 20000)
    g = rng.integers(0, 3, 20000)
    out = oracle.sum_f64_exact(v, None, g, 3)
    for k in range(3):
        assert out[k] == math.fsum(v[g == k])


# ---- TPC-H golden *types* (values need dbgen data; see SURVEY 8c) --------------------------------
def test_q1_pipeline_small(oracle):
    # 3 rows, one group: check the d(12,2) expression tree scales of SURVEY 8(a)
    qty = oracle.dec_from_ints([1700, 3600, 800])
    price = oracle.dec_from_ints([2116823, 4598616, 1395228])
    disc = oracle.dec_from_ints([4, 9, 10])
    tax = oracle.dec_from_ints([2, 6, 2])
    ship = np.array([9568, 9598, 9526], dtype=np.int32)
    rf = np.zeros(3, dtype=np.uint8)
    ls = np.zeros(3, dtype=np.uint8)
    rows = oracle.q1_dec(qty, price, disc, tax, ship, rf, ls, 1, 1, 10471, 2)
    r = rows[0]
    dp = [2116823 * 96, 4598616 * 91, 1395228 * 90]
    ch = [dp[0] * 102, dp[1] * 106, dp[2] * 102]
    assert r["sum_qty"] == 6100 and r["sum_base"] == sum([2116823, 4598616, 1395228])
    assert r["sum_disc_price"] == sum(dp) and r["sum_charge"] == sum(ch)
    assert r["count"] == 3
    # avg qty = 61.00/3 = 20.333333 at scale 6
    assert r["avg_qty"] == 20333333


# ---- whole-pipeline baselines vs plain python ---------------------------------------------------
def _lineitem(n, seed):
    import sys, os
    from comet_b200 import tpch
    return tpch, tpch.gen_lineitem(n, seed=seed)


@pytest.mark.parametrize("threads", [1, 3])
def test_q6_dec_pipeline(oracle, threads):
    tpch, c = _lineitem(20000, 5)
    d = oracle.dec_from_i64
    got = oracle.q6_dec(d(c["l_quantity"]), d(c["l_extendedprice"]), d(c["l_discount"]), c["l_shipdate"], tpch.DATE_1994_01_01,
                        tpch.DATE_1995_01_01, 5, 7, 2400, threads)
    m = (c["l_shipdate"] >= tpch.DATE_1994_01_01) & (c["l_shipdate"] < tpch.DATE_1995_01_01) & (c["l_discount"] >= 5) & \
        (c["l_discount"] <= 7) & (c["l_quantity"] < 2400)
    assert got == int((c["l_extendedprice"][m].astype(object) * c["l_discount"][m].astype(object)).sum())


def test_q6_f64_and_config1_pipelines(oracle):
    import math
    tpch, c = _lineitem(30000, 6)
    q, p, dsc = (c[k].astype(np.float64) / 100.0 for k in ("l_quantity", "l_extendedprice", "l_discount"))
    got = oracle.q6_f64(q, p, dsc, c["l_shipdate"], tpch.DATE_1994_01_01, tpch.DATE_1995_01_01, 0.05, 0.07, 24.0, 1)
    m = (c["l_shipdate"] >= tpch.DATE_1994_01_01) & (c["l_shipdate"] < tpch.DATE_1995_01_01) & (dsc >= 0.05) & (dsc <= 0.07) & (q < 24.0)
    assert abs(got - math.fsum((p * dsc)[m])) <= 1e-9 * abs(got)
    out = oracle.filter_project_f64(q, p, c["l_shipdate"], tpch.DATE_1998_09_02, 3)
    keep = c["l_shipdate"] < tpch.DATE_1998_09_02
    assert (out == (q * p)[keep]).all()
    d = oracle.dec_from_i64
    o, ov = oracle.filter_project_dec(d(c["l_quantity"]), d(c["l_extendedprice"]), c["l_shipdate"], tpch.DATE_1998_09_02, 2)
    assert oracle.dec_to_ints(o[:50]) == [int(a) * int(b) for a, b in zip(c["l_quantity"][keep][:50], c["l_extendedprice"][keep][:50])]
    assert ov.all() and o.shape[0] == int(keep.sum())


def test_q1_dec_threads_agree(oracle):
    tpch, c = _lineitem(50000, 8)
    d = oracle.dec_from_i64
    args = (d(c["l_quantity"]), d(c["l_extendedprice"]), d(c["l_discount"]), d(c["l_tax"]), c["l_shipdate"], c["l_returnflag"],
            c["l_linestatus"], 3, 2, tpch.Q1_CUTOFF)
    a, b = oracle.q1_dec(*args, 1), oracle.q1_dec(*args, 5)
    assert a == b
    keep = c["l_shipdate"] <= tpch.Q1_CUTOFF
    k0 = keep & (c["l_returnflag"] == 0) & (c["l_linestatus"] == 0)
    assert a[0]["sum_qty"] == int(c["l_quantity"][k0].sum()) and a[0]["count"] == int(k0.sum())


# ---- more of checked_arithmetic.rs's own tests (:266-340) --------------------------------------------------------------------------
def test_checked_add_propagates_nulls(oracle):  # :266-273
    out, outv = oracle.int_arith(0, 32, [1, 0, 3, 0], [1, 0, 1, 0], [10, 20, 0, 0], [1, 1, 0, 0], ANSI)
    assert list(outv) == [1, 0, 0, 0] and out[0] == 11


def test_checked_sub_and_mul_overflow_try(oracle):  # :289-297
    out, outv = oracle.int_arith(1, 32, [-(2**31), 5], None, [1, 3], None, TRY)
    assert list(outv) == [0, 1] and out[1] == 2
    out, outv = oracle.int_arith(2, 32, [2**31 - 1, 5], None, [2, 3], None, TRY)
    assert list(outv) == [0, 1] and out[1] == 15


def test_null_row_with_garbage_value_does_not_error_in_ansi_mode(oracle):  # :322-340
    out, outv = oracle.int_arith(0, 32, [2**31 - 1, 1], [0, 1], [1, 1], None, ANSI)     # slot 0 is NULL and holds i32::MAX
    assert list(outv) == [0, 1] and out[1] == 2 and out[0] == 0


def test_checked_div_by_zero_through_the_expression_interpreter():  # :300-319; tests/exprs.py is what the GPU expression tests compare with
    import exprs as E
    from comet_b200 import proto as P
    cols = [(np.array([1.0, 8.0]), np.array([True, True])), (np.array([0.0, 2.0]), np.array([True, True]))]
    a, b = E.Col(0, P.DOUBLE), E.Col(1, P.DOUBLE)
    v, valid = E.Arith("divide", a, b, P.DOUBLE, E.TRY).eval(cols)
    assert list(valid) == [False, True] and v[1] == 4.0
    with pytest.raises(E.AnsiError):
        E.Arith("divide", a, b, P.DOUBLE, E.ANSI).eval(cols)
    v, valid = E.Arith("divide", a, b, P.DOUBLE).eval(cols)                               # Legacy: IEEE
    assert list(valid) == [True, True] and np.isinf(v[0]) and v[1] == 4.0


# ---- CheckOverflow array vectors: math_funcs/internal/checkoverflow.rs:417-512 --------------------------------------------------------
def _co(oracle, vals, precision, ansi=False):
    a = oracle.dec_from_ints([0 if v is None else v for v in vals])
    av = np.array([v is not None for v in vals], dtype=np.uint8)
    out, outv = oracle.check_overflow(a, av, precision, ansi)
    return oracle.dec_to_ints(out, outv)


def test_check_overflow_array_vectors(oracle):
    assert _co(oracle, [999, 12, None, 5], 3) == [999, 12, None, 5]                  # :417-427 nothing overflows, NULLs kept
    assert _co(oracle, [999, 1000, None, 5], 3) == [999, None, None, 5]              # :430-439
    assert _co(oracle, [999, None, 5], 3, ansi=True) == [999, None, 5]               # :442-449
    assert _co(oracle, [-1000, 5], 3) == [None, 5]                                   # :459-465 the lower bound is its own branch
    assert _co(oracle, [None, None, None], 3) == [None, None, None]                  # :480-487
    assert _co(oracle, [1000, 5000, -2000], 3) == [None, None, None]                 # :490-495
    assert _co(oracle, [999, 9999], 3) == [999, None]                                # :505-511 off-by-one on the bound
    for bad in ([999, 1000], [5, -1000], [1000, 5000]):                              # :452-456, :468-477, :498-502 ANSI raises on either side
        with pytest.raises(oracle.OracleError):
            _co(oracle, bad, 3, ansi=True)


# ---- the rest of sum_int.rs's own tests (:933-947, :977-1015) ---------------------------------------------------------------------
def test_sum_int_filter_null_is_exclude_and_no_filter(oracle):
    acc = oracle.SumIntGroups(1)                       # :933-947: a NULL filter entry excludes the row (filter passed as "true AND valid")
    acc.update([10, 20, 30], None, [0, 0, 0], filt=[1, 0, 1])
    assert acc.sums[0] == 40 and acc.sums_valid[0] == 1
    acc = oracle.SumIntGroups(1)                       # :977-988
    acc.update([1, 2, 3], None, [0, 0, 0])
    assert acc.sums[0] == 6


def test_sum_int_merge_consumes_every_state_row(oracle):  # :995-1015: merging partial sums = summing the non-NULL state rows, all of them
    acc = oracle.SumIntGroups(1)
    acc.update([1, 2, 0, 3], [1, 1, 0, 1], [0, 0, 0, 0])
    assert acc.sums[0] == 6
    acc = oracle.SumIntGroups(1, ANSI)
    acc.update([10, 20, 0, 30], [1, 1, 0, 1], [0, 0, 0, 0])
    assert acc.sums[0] == 60
