"""The range-specialised dense aggregate kernels at their bounds.  A decimal aggregate pipeline first runs a kernel that assumes its
inputs fit the declared precision (TYPE), then kernels specialised to the bits observed so far plus two (TIGHT); every launch checks
its assumption through the value masks and is re-run one level wider (TIGHT -> TYPE -> SAFE, the fully checked kernel) when the
input breaks it.  Each test asserts which levels ran (cb200_stats.agg_range_levels) and how many launches were discarded
(agg_range_reruns), so it proves it exercised the path it names, and compares the answer with tests/aggref.py or a closed form.
"""
import threading

import numpy as np
import pyarrow as pa
import pytest

import aggref as R
import exprs as E
from sources import device_table, scan_of, write_parquet

pytestmark = pytest.mark.gpu

P = E.P
TIGHT, TYPE, SAFE = 1, 2, 4
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
KEYS = ["a", "b", "c"]


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def dec_raw(vals, p, s, valid=None):
    """exact two's-complement i128 values (past the precision too) as an Arrow decimal128(p, s); NULL slots keep their value"""
    n = len(vals)
    raw = np.empty((n, 2), dtype=np.uint64)
    for i, v in enumerate(vals):
        u = v & (2**128 - 1)
        raw[i, 0], raw[i, 1] = u & (2**64 - 1), u >> 64
    bufs = [None if valid is None else pa.py_buffer(np.packbits(np.asarray(valid, dtype=bool), bitorder="little").tobytes()),
            pa.py_buffer(raw.tobytes())]
    return pa.Array.from_buffers(pa.decimal128(p, s), n, bufs, null_count=-1 if valid is not None else 0)


def keys_of(codes):
    return pa.DictionaryArray.from_arrays(pa.array(np.asarray(codes, dtype=np.int8)), pa.array(KEYS))


def run_stats(cb, plan, inputs, chunk_rows=None, fresh=True):
    """-> (result, cb200_stats).  fresh: forget the range profiles earlier plans left, so the levels do not depend on test order"""
    if fresh:
        cb.native.reset_range_profiles()
    cfg = {"spark.comet.b200.chunkRows": str(chunk_rows)} if chunk_rows else None
    with cb.native.Plan(plan, inputs, config=cfg) as p:
        out = p.collect()
        st = p.stats()
    return out, st


def run(cb, plan, inputs, chunk_rows=None, fresh=True):
    out, st = run_stats(cb, plan, inputs, chunk_rows, fresh)
    return out, st["agg_range_levels"], st["agg_range_reruns"]


def check_partial(out, tbl, dts, aggs):
    got = dict((k, st) for k, st in R.state_rows_of(out, 1, aggs, [dts[0]] + R.state_schema([], aggs)))
    want = {k: [tuple(s) for s in v] for k, v in R.partial(tbl, dts, [0], aggs).items()}
    assert {k: [tuple(s) for s in v] for k, v in got.items()} == want


# ---- the ladder, driven by data ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ladder_batches():
    """four batches of one decimal(18,2) column: k = 20 bits; exactly k + 2 bits; k + 5 bits (past TIGHT's k + 2 + 2); past the
    precision (10^18, -10^18 - 1 and 64-bit values: the TYPE kernel assumes 60 bits).  Values of 2^127 would leave the SUM certificate
    nothing to prove (n x 2^127 may wrap the 128-bit total), which test_sum_certificate_at_its_edge covers."""
    rng = np.random.default_rng(1)
    n, k = 5000, 20
    out = []
    for extremes in ([(1 << k) - 1, -(1 << k)], [(1 << (k + 2)) - 1, -(1 << (k + 2))], [1 << (k + 4), -(1 << (k + 4))],
                     [10**18, -(10**18) - 1, 1 << 62, I64_MIN - 5]):
        vals = [int(x) for x in rng.integers(-(1 << k), 1 << k, n)]
        for j, v in enumerate(extremes):
            vals[[0, n - 1, 2500, 4000][j]] = v
        out.append(pa.table({"k": keys_of(rng.integers(0, 3, n)), "v": dec_raw(vals, 18, 2)}))
    return out


@pytest.mark.parametrize("upto,levels,reruns", [(1, TYPE, 0), (2, TYPE | TIGHT, 0), (3, TYPE | TIGHT, 1), (4, TYPE | TIGHT | SAFE, 3)])
def test_the_ladder_driven_by_data(cb, oracle, ladder_batches, upto, levels, reruns):
    """batch 1 observes k bits and runs at TYPE; batch 2 sits exactly at k + 2 bits and is accepted at TIGHT; batch 3 breaks TIGHT once
    and runs at TYPE; batch 4 breaks TIGHT and TYPE and runs SAFE"""
    dts = [P.STRING, P.DECIMAL(18, 2)]
    aggs = [R.Agg("sum", E.Col(1, dts[1]), P.DECIMAL(28, 2)), R.Agg("count", E.Col(1, dts[1]))]
    batches = ladder_batches[:upto]
    out, lv, rr = run(cb, R.partial_plan(dts, [0], aggs), [[b for t in batches for b in t.to_batches()]], chunk_rows=5000)
    assert (lv, rr) == (levels, reruns)
    check_partial(out, pa.concat_tables(batches), dts, aggs)


# ---- 8-byte storage holding INT64_MIN: -x and x * -1 are 2^63 -------------------------------------------------------------------
SOURCES = ["arrow16", "device16", "device8", "parquet-int64", "parquet-flba"]


def source(cb, kind, tbl, dts, tmp_path=None, batch=4096):
    """the scan and inputs of `tbl` in one decimal storage: 16-byte Arrow batches of `batch` rows, a device table with 16- or 8-byte
    decimals, or Parquet with INT32 / INT64 (store_decimal_as_integer) or FLBA decimals"""
    names = tbl.column_names
    if kind == "arrow16":
        return P.scan(dts), [tbl.to_batches(max_chunksize=batch)]
    if kind.startswith("device"):
        return P.scan(dts), [device_table(cb, tbl, dts, dec8=tuple(names[1:]) if kind == "device8" else ())]
    path = str(tmp_path / f"{kind}.parquet")
    cols = {k: (tbl.column(k).combine_chunks(), dt) for k, dt in zip(names, dts)}
    write_parquet(path, cols, kind in ("parquet-int32", "parquet-int64"))
    scan, _ = scan_of(cb, cols, names, path)
    return scan, []


def int64_edge_table(n=3000, seed=2, nulls=False):
    rng = np.random.default_rng(seed)
    vals = [int(x) for x in rng.integers(-10**17, 10**17, n)]
    codes = rng.integers(0, 3, n)
    vals[0], vals[n - 1], vals[n // 2] = I64_MIN, I64_MAX, I64_MIN + 1
    valid = None
    if nulls:
        valid = rng.random(n) > 0.2
        valid[[0, n - 1, n // 2]] = True
    return pa.table({"sd": keys_of(codes), "v": dec_raw(vals, 18, 0, valid)})


@pytest.mark.parametrize("kind", SOURCES)
def test_negating_int64_min_in_every_storage(cb, oracle, tmp_path, kind):
    """decimal(18,0) holding INT64_MIN (past its precision, read as-is): the TYPE kernel's assumption fails and the SAFE kernel must
    negate in 128 bits -- -x and x * CAST(-1 AS decimal(1,0)) are +2^63, inside their result types, so no check hides a wrap"""
    dts = [P.STRING, P.DECIMAL(18, 0)]
    x = E.Col(1, dts[1])
    times = E.Arith("multiply", x, E.Lit(-1, P.DECIMAL(1, 0)), P.DECIMAL(20, 0))
    aggs = [R.Agg("sum", E.Neg(x), P.DECIMAL(38, 0)), R.Agg("sum", times, P.DECIMAL(38, 0)), R.Agg("sum", x, P.DECIMAL(38, 0))]
    tbl = int64_edge_table(nulls=True)
    scan, inputs = source(cb, kind, tbl, dts, tmp_path)
    plan = P.hash_agg(scan, [P.bound(0, P.STRING)], [a.proto() for a in aggs], P.PARTIAL)
    out, lv, rr = run(cb, plan, inputs, chunk_rows=1 << 20)
    assert (lv, rr) == (SAFE, 1)
    check_partial(out, tbl, dts, aggs)


@pytest.mark.parametrize("kind", SOURCES)
def test_min_max_at_the_int64_limits(cb, oracle, tmp_path, kind):
    """MIN / MAX keep 64-bit keys: INT64_MIN / INT64_MAX themselves are exact in every storage"""
    dts = [P.STRING, P.DECIMAL(18, 0)]
    x = E.Col(1, dts[1])
    aggs = [R.Agg("min", x, dts[1]), R.Agg("max", x, dts[1])]
    tbl = int64_edge_table(seed=3)
    scan, inputs = source(cb, kind, tbl, dts, tmp_path)
    out, lv, rr = run(cb, P.hash_agg(scan, [P.bound(0, P.STRING)], [a.proto() for a in aggs], P.PARTIAL), inputs, chunk_rows=1 << 20)
    assert (lv, rr) == (SAFE, 1)
    check_partial(out, tbl, dts, aggs)


def test_min_max_of_a_value_past_64_bits_is_refused(cb, oracle):
    """a 16-byte decimal(18,0) carrying 2^63 or -2^63 - 1 reaches the SAFE kernel; comparing it by its low word would give a wrong
    MIN / MAX, so the plan is refused"""
    dts = [P.STRING, P.DECIMAL(18, 0)]
    x = E.Col(1, dts[1])
    aggs = [R.Agg("min", x, dts[1]), R.Agg("max", x, dts[1])]
    for bad in (1 << 63, -(1 << 63) - 1, 1 << 100):
        vals = [5, -7, bad, 11]
        tbl = pa.table({"sd": keys_of([0, 0, 1, 1]), "v": dec_raw(vals, 18, 0)})
        with pytest.raises(cb.native.Unsupported, match="64 bits"):
            run(cb, R.partial_plan(dts, [0], aggs), [tbl.to_batches()])
    # a NULL slot carrying such a value is not an input
    tbl = pa.table({"sd": keys_of([0, 0, 1, 1]), "v": dec_raw([5, -7, 1 << 63, 11], 18, 0, [True, True, False, True])})
    out, lv, rr = run(cb, R.partial_plan(dts, [0], aggs), [tbl.to_batches()])
    assert (lv, rr) == (TYPE, 0)
    check_partial(out, tbl, dts, aggs)


def test_errors_of_a_discarded_launch_are_dropped(cb, oracle):
    """COUNT(x / y) in ANSI mode, y decimal(38,0): after a batch of small divisors the TIGHT kernel holds y in 64 bits, so a divisor of
    2^64 reads as 0.  That launch breaks its assumption and is discarded with its DIVIDE_BY_ZERO; the TYPE re-run divides exactly."""
    rng = np.random.default_rng(9)
    n = 4000
    dts = [P.STRING, P.DECIMAL(12, 2), P.DECIMAL(38, 0)]
    q = E.Arith("divide", E.Col(1, dts[1]), E.Col(2, dts[2]), P.DECIMAL(38, 6), E.ANSI)
    aggs = [R.Agg("count", q)]
    tables = []
    for big in (None, 1 << 64):
        y = [int(v) for v in rng.integers(1, 1000, n)]
        if big:
            y[n // 3] = big
        tables.append(pa.table({"sd": keys_of(rng.integers(0, 3, n)), "x": dec_raw([int(v) for v in rng.integers(-10**9, 10**9, n)], 12, 2),
                                "y": dec_raw(y, 38, 0)}))
    out, lv, rr = run(cb, R.partial_plan(dts, [0], aggs), [[b for t in tables for b in t.to_batches()]], chunk_rows=n)
    assert (lv, rr) == (TYPE, 1)
    check_partial(out, pa.concat_tables(tables), dts, aggs)


# ---- NULL slots carrying huge garbage -------------------------------------------------------------------------------------------
def test_null_slots_with_huge_garbage_change_nothing(cb, oracle):
    rng = np.random.default_rng(4)
    n = 20000
    vals = [int(x) for x in rng.integers(-1000, 1000, n)]
    valid = rng.random(n) > 0.3
    for i in np.flatnonzero(~valid)[:500]:
        vals[i] = int(rng.choice([(1 << 127) - 1, -(1 << 127), 10**30, I64_MIN]))
    tbl = pa.table({"sd": keys_of(rng.integers(0, 3, n)), "v": dec_raw(vals, 12, 2, valid)})
    dts = [P.STRING, P.DECIMAL(12, 2)]
    x = E.Col(1, dts[1])
    aggs = [R.Agg("sum", x, P.DECIMAL(22, 2)), R.Agg("min", x, dts[1]), R.Agg("max", x, dts[1]),
            R.Agg("sum", E.CheckOverflow(E.Arith("multiply", x, E.Lit(10**9, P.DECIMAL(10, 0)), P.DECIMAL(23, 2)), P.DECIMAL(23, 2), True),
                  P.DECIMAL(33, 2))]
    out, lv, rr = run(cb, R.partial_plan(dts, [0], aggs), [tbl.to_batches(max_chunksize=5000)], chunk_rows=5000)
    assert rr == 0 and lv == TYPE | TIGHT
    check_partial(out, tbl, dts, aggs)


# ---- violations at launch edges -------------------------------------------------------------------------------------------------
SAMPLE = 1 << 20


@pytest.mark.parametrize("at,levels,reruns,p", [(0, TYPE | TIGHT, 0, 18), (SAMPLE - 1, TYPE | TIGHT, 0, 18), (SAMPLE, TYPE, 1, 18),
                                               ("last", TYPE, 1, 15)])
def test_violation_at_the_sample_edges(cb, at, levels, reruns, p):
    """a batch over 2 Mi rows: the first 1 Mi rows run at TYPE and measure the ranges, the rest at TIGHT.  One value of 2^45 in the
    sample (its first or last row) is seen before the bulk launch; on the first row after the sample or the batch's last row it
    breaks the bulk launch once."""
    n = 2 * SAMPLE + 12345
    rng = np.random.default_rng(5)
    v = rng.integers(-5000, 5000, n)
    codes = rng.integers(0, 3, n)
    i = n - 1 if at == "last" else at
    v[i] = 1 << 45
    raw = np.empty((n, 2), dtype=np.int64)
    raw[:, 0], raw[:, 1] = v, v >> 63
    tbl = pa.table({"sd": keys_of(codes), "v": pa.Array.from_buffers(pa.decimal128(p, 2), n, [None, pa.py_buffer(raw.tobytes())])})
    dts = [P.STRING, P.DECIMAL(p, 2)]
    aggs = [R.Agg("sum", E.Col(1, dts[1]), P.DECIMAL(28, 2)), R.Agg("count", E.Col(1, dts[1]))]
    out, lv, rr = run(cb, R.partial_plan(dts, [0], aggs), [[tbl.combine_chunks().to_batches()[0]]], chunk_rows=1 << 26)
    assert (lv, rr) == (levels, reruns)
    got = {r["col_0"]: (int(r["col_1"].scaleb(2)), r["col_2"], r["col_3"]) for r in out.to_pylist()}
    assert got == {KEYS[g]: (int(v[codes == g].sum()), False, int((codes == g).sum())) for g in range(3)}


def test_violation_in_the_second_sub_launch(cb):
    """a batch longer than one launch may scan (num_sms x threads x 2^14 rows: 553,648,128 on a 132-SM H100 at 256 threads) is split;
    a value past TIGHT's assumption in the second sub-launch re-runs only that one.  600 M 8-byte rows generated on the device."""
    import torch
    n = 600_000_000
    v = torch.arange(n, dtype=torch.int64, device="cuda")
    v.remainder_(1000)
    v[n - 1] = 1 << 50
    torch.cuda.synchronize()
    t = cb.native.DeviceTable(n)
    t.add(P.DECIMAL(18, 0), v.data_ptr(), 8, keep=v)
    plan = P.hash_agg(P.scan([P.DECIMAL(18, 0)]), [], [P.agg_sum(P.bound(0, P.DECIMAL(18, 0)), P.DECIMAL(38, 0))], P.PARTIAL)
    out, lv, rr = run(cb, plan, [t], chunk_rows=1 << 30)
    q, r = divmod(n, 1000)
    want = q * 499500 + r * (r - 1) // 2 - (n - 1) % 1000 + (1 << 50)
    assert (lv, rr) == (TYPE | TIGHT, 1)
    assert int(out.column(0)[0].as_py().scaleb(0)) == want
    del t, v
    torch.cuda.empty_cache()


# ---- the range profile shared between plans -------------------------------------------------------------------------------------
def _profile_table(n, lo, hi, seed):
    rng = np.random.default_rng(seed)
    v = rng.integers(lo, hi, n)
    codes = rng.integers(0, 3, n)
    raw = np.empty((n, 2), dtype=np.int64)
    raw[:, 0], raw[:, 1] = v, v >> 63
    return pa.table({"sd": keys_of(codes), "v": pa.Array.from_buffers(pa.decimal128(17, 3), n, [None, pa.py_buffer(raw.tobytes())])}), v, codes


def test_range_profile_shared_between_plans(cb):
    """plan A (small values, > 2 Mi rows) leaves its ranges for the next plan with the same pipeline; plan B starts from them with
    larger values, so its first launch is re-run -- and both are exact, also when the two run from two threads"""
    dts = [P.STRING, P.DECIMAL(17, 3)]
    aggs = [R.Agg("sum", E.Col(1, dts[1]), P.DECIMAL(27, 3))]
    plan = R.partial_plan(dts, [0], aggs)
    n = 2 * SAMPLE + 999
    a, va, ca = _profile_table(n, -100, 100, 6)
    b, vb, cbk = _profile_table(n, -(1 << 40), 1 << 40, 7)

    def check(out, v, codes):
        got = {r["col_0"]: int(r["col_1"].scaleb(3)) for r in out.to_pylist()}
        assert got == {KEYS[g]: int(v[codes == g].sum()) for g in range(3)}

    out, lv, rr = run(cb, plan, [[a.combine_chunks().to_batches()[0]]], chunk_rows=1 << 26)
    assert (lv, rr) == (TYPE | TIGHT, 0)
    check(out, va, ca)
    out, lv, rr = run(cb, plan, [[b.combine_chunks().to_batches()[0]]], chunk_rows=1 << 26, fresh=False)
    assert (lv, rr) == (TYPE, 1)
    check(out, vb, cbk)
    errs = []

    def go(tbl, v, codes):
        try:
            for _ in range(2):
                check(run(cb, plan, [[tbl.combine_chunks().to_batches()[0]]], chunk_rows=1 << 26, fresh=False)[0], v, codes)
        except Exception as e:  # noqa: BLE001 -- reported by the main thread
            errs.append(e)
    th = [threading.Thread(target=go, args=x) for x in ((a, va, ca), (b, vb, cbk))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs


# ---- the per-group SUM certificate at its edge ----------------------------------------------------------------------------------
def row_order_sum(vals, p):
    """SumDecimal row by row: NULL for good once a prefix leaves decimal(p)"""
    s = 0
    for v in vals:
        s += v
        if abs(s) >= 10**p:
            return None
    return s


REFUSE, ANSI_ERROR = "refuse", "ansi"


@pytest.mark.parametrize("vals,mode,expect", [
    ([-1] * 9999, E.LEGACY, -9999),            # -1 has a 0-bit mask: B = 1, addends in [-1, 0]; n x B = 10^4 - 1: certified, exact
    ([-1] * 10000, E.LEGACY, None),            # total out of decimal(4): every row order overflows -> NULL
    ([-1] * 9999 + [0], E.LEGACY, REFUSE),     # n x B = 10^4 with a total that fits: nothing proved -> refused (row order: -9999)
    ([1] * 10000, E.LEGACY, None),             # +1 has a 1-bit mask: B = 2 ... total out of range -> NULL
    ([1] * 9999, E.LEGACY, REFUSE),            # ... n x B = 19998 with a total that fits -> refused (row order: 9999)
    ([1] * 9999 + [1, -1], E.LEGACY, REFUSE),  # the row order decides (NULL in this order, 9999 in others) -> refused
    ([-1] * 9999, E.ANSI, -9999),
    ([-1] * 10000, E.ANSI, ANSI_ERROR),        # every row order overflows in ANSI mode -> ARITHMETIC_OVERFLOW
])
def test_sum_certificate_at_its_edge(cb, vals, mode, expect):
    """SUM into decimal(4,0) at n x B = 10^p - 1 and one step past: the exact total, NULL, ARITHMETIC_OVERFLOW, or the refusal of a
    result the certificate cannot prove (error 12) -- never a different number.  Numbers agree with the row-order oracle."""
    tbl = pa.table({"v": dec_raw(vals, 4, 0)})
    plan = P.hash_agg(P.scan([P.DECIMAL(4, 0)]), [], [P.agg_sum(P.bound(0, P.DECIMAL(4, 0)), P.DECIMAL(4, 0), mode)], P.PARTIAL)
    if expect in (REFUSE, ANSI_ERROR):
        with pytest.raises(cb.native.CometB200Error) as ei:
            run(cb, plan, [tbl.to_batches()])
        if expect == REFUSE:
            assert "depends on the row order" in str(ei.value)       # ExecError 12, reported as a Spark error
        else:
            assert ei.value.error_class == "ARITHMETIC_OVERFLOW"
        return
    assert expect == row_order_sum(vals, 4)
    out, lv, rr = run(cb, plan, [tbl.to_batches()])
    assert (lv, rr) == (TYPE, 0)
    got = out.column(0)[0].as_py()
    assert (None if got is None else int(got.scaleb(0))) == expect


# ---- every assumption-dependent choice at its threshold -------------------------------------------------------------------------
def _max_rows(cb, plan):
    """rows one dense launch may scan: num_sms x threads x 2^14 (agg.cpp run_range), so no thread accumulates more than 2^14 rows"""
    import torch
    src = cb.native.kernel_source(plan)
    threads = int(src.split("#define CB_THREADS ", 1)[1].split("\n", 1)[0])
    return torch.cuda.get_device_properties(0).multi_processor_count * threads * (1 << 14) // 1024 * 1024


def _device_dec(cb, v, width, dt):
    """a device table of one decimal column from an int64 torch tensor, 8 or 16 bytes per value"""
    import torch
    if width == 16:
        w = torch.empty((v.numel(), 2), dtype=torch.int64, device="cuda")
        w[:, 0] = v
        w[:, 1] = v >> 63
        v = w
    torch.cuda.synchronize()
    t = cb.native.DeviceTable(v.shape[0])
    t.add(dt, v.data_ptr(), width, keep=v)
    return t


@pytest.mark.parametrize("width", [16, 8])
@pytest.mark.parametrize("value", [-(1 << 48), (1 << 48) - 1])
def test_wrap_sum_at_its_bound_over_a_full_launch(cb, width, value):
    """64-bit per-thread partial sums are exact while 2^14 rows x 2^k < 2^63, so TIGHT at k = 48 takes the `wrap` accumulator.  One
    launch of exactly num_sms x threads x 2^14 rows, every value at -2^48 (or 2^48 - 1): the largest per-thread partial the kernel may
    build.  The observed 46 bits come from a first plan's range profile, so the whole batch is one TIGHT launch (no sample)."""
    import torch
    d = P.DECIMAL(18, 0)
    plan = P.hash_agg(P.scan([d]), [], [P.agg_sum(P.bound(0, d), P.DECIMAL(38, 0)), P.agg_avg(P.bound(0, d), P.DECIMAL(22, 4), P.DECIMAL(28, 0))],
                      P.PARTIAL)
    m = 2 * SAMPLE + 4096
    a = torch.randint(-(1 << 30), 1 << 30, (m,), dtype=torch.int64, device="cuda")
    a[7] = -(1 << 46)                                                    # 46 observed bits: TIGHT assumes 48 from here on
    out, st = run_stats(cb, plan, [_device_dec(cb, a, width, d)], chunk_rows=1 << 30)
    assert (st["agg_range_levels"], st["agg_range_reruns"]) == (TYPE | TIGHT, 0)
    assert int(out.column(0)[0].as_py().scaleb(0)) == int(a.sum())
    n = _max_rows(cb, plan)
    b = torch.full((n,), value, dtype=torch.int64, device="cuda")
    out, st = run_stats(cb, plan, [_device_dec(cb, b, width, d)], chunk_rows=1 << 30, fresh=False)
    assert (st["agg_range_levels"], st["agg_range_reruns"], st["pipeline_launches"], st["pipeline_rows"]) == (TIGHT, 0, 1, n)
    r = out.to_pylist()[0]
    assert int(r["col_0"].scaleb(0)) == n * value and r["col_1"] is False
    assert int(r["col_2"].scaleb(0)) == n * value and r["col_3"] == n
    del a, b
    torch.cuda.empty_cache()


def _two_batches(rng, n, first, second):
    """two batches of n rows: random values of first[0] / second[0] bits with first[1] / second[1] planted"""
    cols = {}
    for name in first:
        vals = []
        for bits, planted in (first[name], second[name]):
            v = [int(x) for x in rng.integers(-(1 << bits), 1 << bits, n)]
            for j, p in enumerate(planted):
                v[(j * 977 + 13) % n] = p
            vals += v
        cols[name] = vals
    return cols


@pytest.mark.parametrize("kind", ["arrow16", "device16", "device8"])
def test_values_straddling_2_46_in_the_wide_accumulator(cb, oracle, kind):
    """observed 48 bits -> TIGHT assumes 50: past the `wrap` bound, so SUM / AVG take the `wide` accumulator, whose values of
    |v| >= 2^46 escape to the exact 128-bit spill.  The second batch holds both sides of 2^46 and the 50-bit corners."""
    rng = np.random.default_rng(10)
    n = 4096
    e = [(1 << 46) - 1, 1 << 46, (1 << 46) + 1, -(1 << 46), -(1 << 46) - 1, 1 - (1 << 46), (1 << 50) - 1, -(1 << 50), (1 << 49)]
    c = _two_batches(rng, n, {"v": (40, [-(1 << 48), (1 << 48) - 1])}, {"v": (47, e)})
    dts = [P.STRING, P.DECIMAL(18, 0)]
    tbl = pa.table({"sd": keys_of(rng.integers(0, 3, 2 * n)), "v": dec_raw(c["v"], 18, 0)})
    x = E.Col(1, dts[1])
    aggs = [R.Agg("sum", x, P.DECIMAL(38, 0)), R.Agg("avg", x, P.DECIMAL(22, 4), P.DECIMAL(28, 0))]
    scan, inputs = source(cb, kind, tbl, dts)
    out, lv, rr = run(cb, P.hash_agg(scan, [P.bound(0, P.STRING)], [a.proto() for a in aggs], P.PARTIAL), inputs, chunk_rows=n)
    assert (lv, rr) == (TYPE | TIGHT, 0)
    check_partial(out, tbl, dts, aggs)


@pytest.mark.parametrize("kind", ["arrow16", "device16", "device8"])
def test_narrow_add_sub_mul_with_scale_factors(cb, oracle, kind):
    """TIGHT at 56 bits: x (scale 2) + y (scale 0) is x + 100 y with |raw| <= 101 x 2^56 < 2^63, one i64 expression; at 31 bits
    u * w is one i64 multiply (2^62).  Every corner -2^k / 2^k - 1 is in the second batch."""
    rng = np.random.default_rng(11)
    n = 4096
    big, small = [(1 << 56) - 1, -(1 << 56)], [(1 << 31) - 1, -(1 << 31)]
    c = _two_batches(rng, n, {"x": (54, [-(1 << 54)]), "y": (54, [-(1 << 54)]), "u": (29, [-(1 << 29)]), "w": (29, [-(1 << 29)])},
                     {"x": (55, big + big[::-1]), "y": (55, big + big), "u": (30, small + small[::-1]), "w": (30, small + small)})
    d2, d0 = P.DECIMAL(18, 2), P.DECIMAL(18, 0)
    dts = [P.STRING, d2, d0, d2, d0]
    tbl = pa.table({"sd": keys_of(rng.integers(0, 3, 2 * n)), "x": dec_raw(c["x"], 18, 2), "y": dec_raw(c["y"], 18, 0),
                    "u": dec_raw(c["u"], 18, 2), "w": dec_raw(c["w"], 18, 0)})
    x, y, u, w = (E.Col(i, dt) for i, dt in enumerate(dts) if i)
    add, sub = E.Arith("add", x, y, P.DECIMAL(21, 2)), E.Arith("subtract", x, y, P.DECIMAL(21, 2))
    mul = E.Arith("multiply", u, w, P.DECIMAL(37, 2))
    aggs = [R.Agg("sum", add, P.DECIMAL(38, 2)), R.Agg("sum", sub, P.DECIMAL(38, 2)), R.Agg("sum", mul, P.DECIMAL(38, 2))]
    scan, inputs = source(cb, kind, tbl, dts)
    out, lv, rr = run(cb, P.hash_agg(scan, [P.bound(0, P.STRING)], [a.proto() for a in aggs], P.PARTIAL), inputs, chunk_rows=n)
    assert (lv, rr) == (TYPE | TIGHT, 0)
    check_partial(out, tbl, dts, aggs)


LAYOUT_BUG = pytest.mark.xfail(strict=True, raises=Exception, reason=(
    "known bug: in Legacy / TRY a CheckOverflow the range proof elides is never NULL, one that is kept may be; the aggregate's count "
    "slots follow that nullability, so a TYPE launch that keeps the check and a TIGHT launch that elides it get different accumulator "
    "layouts and the second fails with 'accumulator layout changed between launches' (DESIGN section 6)"))


@pytest.mark.parametrize("mode", [pytest.param(E.LEGACY, marks=LAYOUT_BUG), pytest.param(E.TRY, marks=LAYOUT_BUG), E.ANSI])
@pytest.mark.parametrize("past", [False, True])
def test_check_overflow_at_the_precision(cb, oracle, mode, past):
    """CheckOverflow(x + L, decimal(18,0)) with L = -(10^18 - 1 - 2^40): at TIGHT (|x| <= 2^40) the bound is exactly 10^18 - 1, so the
    check is not emitted, and x = -2^40 reaches -(10^18 - 1).  One past (x = -2^40 - 1 -> -10^18; and x = 2^40 / 2^40 + 1 against
    L' = -L -> 10^18 - 1 / 10^18) breaks TIGHT, and the TYPE kernel keeps the check: NULL in Legacy / TRY, ARITHMETIC_OVERFLOW in ANSI."""
    rng = np.random.default_rng(12)
    n = 4096
    k, lim = 40, 10**18 - 1
    d = P.DECIMAL(18, 0)
    second = [-(1 << k), (1 << k) - 1] + ([-(1 << k) - 1, 1 << k, (1 << k) + 1] if past else [])
    c = _two_batches(rng, n, {"v": (k - 3, [-(1 << (k - 2))])}, {"v": (k - 1, second)})
    tbl = pa.table({"sd": keys_of(rng.integers(0, 3, 2 * n)), "v": dec_raw(c["v"], 18, 0)})
    dts = [P.STRING, d]
    x = E.Col(1, d)
    aggs = [R.Agg("sum", E.CheckOverflow(E.Arith("add", x, E.Lit(L, d), P.DECIMAL(19, 0), mode), d, mode == E.ANSI), P.DECIMAL(38, 0))
            for L in (-(lim - (1 << k)), lim - (1 << k))]
    plan = R.partial_plan(dts, [0], aggs)
    if past and mode == E.ANSI:
        with pytest.raises(E.AnsiError):
            R.partial(tbl, dts, [0], aggs)
        with pytest.raises(cb.native.CometB200Error) as ei:
            run(cb, plan, [tbl.to_batches(max_chunksize=n)], chunk_rows=n)
        assert ei.value.error_class == "ARITHMETIC_OVERFLOW"
        return
    out, lv, rr = run(cb, plan, [tbl.to_batches(max_chunksize=n)], chunk_rows=n)
    assert (lv, rr) == ((TYPE, 1) if past else (TYPE | TIGHT, 0))
    check_partial(out, tbl, dts, aggs)


@pytest.mark.parametrize("lit", [(1 << 63) - 1, -((1 << 63) - 1), 1 << 63, -(1 << 63)])
def test_decimal_literals_near_2_63(cb, oracle, lit):
    """a decimal literal is one 64-bit value below 2^63 and a 128-bit one from it on; x + L is a wide decimal add"""
    rng = np.random.default_rng(13)
    n = 4096
    vals = [int(v) for v in rng.integers(-10**17, 10**17, n)]
    vals[5], vals[6] = 10**18 - 1, -(10**18 - 1)
    tbl = pa.table({"sd": keys_of(rng.integers(0, 3, n)), "v": dec_raw(vals, 18, 0)})
    dts = [P.STRING, P.DECIMAL(18, 0)]
    add = E.Arith("add", E.Col(1, dts[1]), E.Lit(lit, P.DECIMAL(38, 0)), P.DECIMAL(38, 0))
    aggs = [R.Agg("sum", add, P.DECIMAL(38, 0)), R.Agg("count", add)]
    out, lv, rr = run(cb, R.partial_plan(dts, [0], aggs), [tbl.to_batches()])
    assert (lv, rr) == (TYPE, 0)
    check_partial(out, tbl, dts, aggs)


@pytest.mark.parametrize("kind", ["arrow16", "parquet-int32"])
def test_int32_storage_at_its_limits(cb, oracle, tmp_path, kind):
    """decimal(9,0) stored as Parquet INT32 holding INT32_MIN / INT32_MAX (past precision 9): the TYPE kernel assumes 30 bits, the
    SAFE kernel reads the 4-byte values; -x, x * -1, MIN and MAX exact"""
    rng = np.random.default_rng(14)
    n = 3000
    vals = [int(v) for v in rng.integers(-10**8, 10**8, n)]
    vals[0], vals[n - 1], vals[n // 2] = -(1 << 31), (1 << 31) - 1, 1 - (1 << 31)
    tbl = pa.table({"sd": keys_of(rng.integers(0, 3, n)), "v": dec_raw(vals, 9, 0)})
    d = P.DECIMAL(9, 0)
    dts = [P.STRING, d]
    x = E.Col(1, d)
    aggs = [R.Agg("sum", E.Neg(x), P.DECIMAL(38, 0)), R.Agg("sum", E.Arith("multiply", x, E.Lit(-1, P.DECIMAL(1, 0)), P.DECIMAL(11, 0)),
                                                            P.DECIMAL(38, 0)),
            R.Agg("min", x, d), R.Agg("max", x, d)]
    scan, inputs = source(cb, kind, tbl, dts, tmp_path)
    out, lv, rr = run(cb, P.hash_agg(scan, [P.bound(0, P.STRING)], [a.proto() for a in aggs], P.PARTIAL), inputs, chunk_rows=1 << 20)
    assert (lv, rr) == (SAFE, 1)
    check_partial(out, tbl, dts, aggs)
