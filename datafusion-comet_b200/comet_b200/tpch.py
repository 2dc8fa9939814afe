"""TPC-H-shaped synthetic lineitem data + the serialized plans of BASELINE.json's configs.

Plans are built exactly as the reference's JVM serde would emit them for
benchmarks/tpc/queries/tpch/q1.sql / q6.sql with the reference's test schema
(spark/src/test/scala/org/apache/spark/sql/TPCH.scala:153-156: money columns DECIMAL(12,2)):
every decimal operation is wrapped in CheckOverflow (DecimalPrecision.scala:43-78), literals carry
their Spark types, aggregate result / state types follow Spark's rules (SURVEY.md section 8a).
The F64 variants use DOUBLE money columns (BASELINE.json wording).

Data generator: SURVEY.md section 8(d) -- deterministic (numpy PCG64, seed 42).
"""
import numpy as np
import pyarrow as pa

from . import proto as P

D12 = P.DECIMAL(12, 2)
DATE_1998_09_02 = 10471  # Config 1 cutoff (BASELINE.json configs[0]: l_shipdate < '1998-09-02')
Q1_CUTOFF = 10493        # Q1: date '1998-12-01' - interval '68 days' = 1998-09-24 (reference benchmarks/tpc/queries/tpch/q1.sql:17)
DATE_1994_01_01 = 8766
DATE_1995_01_01 = 9131
DATE_1995_06_17 = 9298
RETURNFLAGS = ["A", "N", "R"]
LINESTATUS = ["F", "O"]
SHIPMODES = ["REG AIR", "AIR", "RAIL", "SHIP", "TRUCK", "MAIL", "FOB"]                  # TPC-H 4.2.2.13 Modes
SHIPINSTRUCTS = ["DELIVER IN PERSON", "COLLECT COD", "NONE", "TAKE BACK RETURN"]       # TPC-H 4.2.2.13 Instructions


# ---- data -----------------------------------------------------------------------------------------
def gen_lineitem(n, seed=42):
    """numpy columns: money as int64 cents, quantity as int64 units*100 (i.e. d(12,2) unscaled)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    lines = rng.integers(1, 8, size=n // 3 + 8)
    orderkey = np.repeat(np.arange(1, lines.shape[0] + 1, dtype=np.int64), lines)[:n]
    if orderkey.shape[0] < n:
        orderkey = np.concatenate([orderkey, np.full(n - orderkey.shape[0], orderkey[-1] + 1, dtype=np.int64)])
    qty_units = rng.integers(1, 51, size=n).astype(np.int64)
    unit_price = rng.integers(90000, 210001, size=n).astype(np.int64)  # cents per unit
    price = qty_units * unit_price  # cents
    disc = rng.integers(0, 11, size=n).astype(np.int64)  # 0.00 .. 0.10
    tax = rng.integers(0, 9, size=n).astype(np.int64)  # 0.00 .. 0.08
    ship = rng.integers(8036, 10562, size=n).astype(np.int32)
    receipt = ship + rng.integers(1, 31, size=n).astype(np.int32)
    ar = rng.integers(0, 2, size=n).astype(np.uint8) * 2  # A (0) or R (2)
    rf = np.where(receipt <= DATE_1995_06_17, ar, np.uint8(1)).astype(np.uint8)  # else N (1)
    ls = (ship > DATE_1995_06_17).astype(np.uint8)  # F (0) / O (1)
    # ship mode / instruction codes (into SHIPMODES / SHIPINSTRUCTS) from a stream of their own: the columns above do not change
    rng2 = np.random.Generator(np.random.PCG64([seed, 1]))
    mode = rng2.integers(0, len(SHIPMODES), size=n).astype(np.uint8)
    instruct = rng2.integers(0, len(SHIPINSTRUCTS), size=n).astype(np.uint8)
    return dict(l_orderkey=orderkey, l_quantity=qty_units * 100, l_extendedprice=price, l_discount=disc, l_tax=tax,
                l_shipdate=ship, l_returnflag=rf, l_linestatus=ls, l_shipmode=mode, l_shipinstruct=instruct)


def _dec_array(cents, precision=12, scale=2, valid=None):
    lo = np.ascontiguousarray(cents, dtype=np.int64)
    buf = np.empty((lo.shape[0], 2), dtype=np.int64)
    buf[:, 0] = lo
    buf[:, 1] = lo >> 63
    vbuf = None
    if valid is not None:
        vbuf = pa.py_buffer(np.packbits(np.asarray(valid, dtype=bool), bitorder="little").tobytes())
    return pa.Array.from_buffers(pa.decimal128(precision, scale), lo.shape[0], [vbuf, pa.py_buffer(buf.tobytes())])


def lineitem_table(cols, variant="dec", dictionary=True, columns=None):
    """Arrow table in the column order of SCHEMA[variant]."""
    money = (lambda a: _dec_array(a)) if variant == "dec" else (lambda a: pa.array(a.astype(np.float64) / 100.0))

    def flags(codes, values):
        idx = pa.array(codes.astype(np.int8))
        d = pa.DictionaryArray.from_arrays(idx, pa.array(values))
        return d if dictionary else d.cast(pa.string())

    arrays = {
        "l_orderkey": lambda: pa.array(cols["l_orderkey"]),
        "l_quantity": lambda: money(cols["l_quantity"]),
        "l_extendedprice": lambda: money(cols["l_extendedprice"]),
        "l_discount": lambda: money(cols["l_discount"]),
        "l_tax": lambda: money(cols["l_tax"]),
        "l_returnflag": lambda: flags(cols["l_returnflag"], RETURNFLAGS),
        "l_linestatus": lambda: flags(cols["l_linestatus"], LINESTATUS),
        "l_shipmode": lambda: flags(cols["l_shipmode"], SHIPMODES),
        "l_shipinstruct": lambda: flags(cols["l_shipinstruct"], SHIPINSTRUCTS),
        "l_shipdate": lambda: pa.array(cols["l_shipdate"], type=pa.date32()),
    }
    names = columns or ["l_quantity", "l_extendedprice", "l_discount", "l_tax", "l_returnflag", "l_linestatus", "l_shipdate"]
    return pa.table({k: arrays[k]() for k in names})


# ---- plans ----------------------------------------------------------------------------------------
def _money(variant):
    return D12 if variant == "dec" else P.DOUBLE


def _lit_money(cents, variant, precision=12):
    return P.literal(cents, P.DECIMAL(precision, 2)) if variant == "dec" else P.literal(cents / 100.0, P.DOUBLE)


def q1_exprs(variant, qty, price, disc, tax):
    """disc_price / charge expression trees over the given column exprs."""
    if variant == "dec":
        one = P.literal(1, P.DECIMAL(1, 0))
        one_minus = P.check_overflow(P.subtract(one, disc, P.DECIMAL(13, 2)), P.DECIMAL(13, 2))
        disc_price = P.check_overflow(P.multiply(price, one_minus, P.DECIMAL(26, 4)), P.DECIMAL(26, 4))
        one_plus = P.check_overflow(P.add(one, tax, P.DECIMAL(13, 2)), P.DECIMAL(13, 2))
        charge = P.check_overflow(P.multiply(disc_price, one_plus, P.DECIMAL(38, 6)), P.DECIMAL(38, 6))
    else:
        one = P.literal(1.0, P.DOUBLE)
        disc_price = P.multiply(price, P.subtract(one, disc, P.DOUBLE), P.DOUBLE)
        charge = P.multiply(disc_price, P.add(one, tax, P.DOUBLE), P.DOUBLE)
    return disc_price, charge


def q1_aggs(variant, bound=True):
    """The eight Q1 aggregates over the projected columns [qty, price, disc, tax, rf, ls]."""
    m = _money(variant)
    ref = (lambda i, dt: P.bound(i, dt)) if bound else (lambda i, dt: P.unbound(f"c{i}", dt))
    qty, price, disc, tax = ref(0, m), ref(1, m), ref(2, m), ref(3, m)
    disc_price, charge = q1_exprs(variant, qty, price, disc, tax)
    if variant == "dec":
        return [P.agg_sum(qty, P.DECIMAL(22, 2)), P.agg_sum(price, P.DECIMAL(22, 2)), P.agg_sum(disc_price, P.DECIMAL(36, 4)),
                P.agg_sum(charge, P.DECIMAL(38, 6)), P.agg_avg(qty, P.DECIMAL(16, 6), P.DECIMAL(22, 2)),
                P.agg_avg(price, P.DECIMAL(16, 6), P.DECIMAL(22, 2)), P.agg_avg(disc, P.DECIMAL(16, 6), P.DECIMAL(22, 2)),
                P.agg_count([P.literal(1, P.INT32)])]
    return [P.agg_sum(qty, P.DOUBLE), P.agg_sum(price, P.DOUBLE), P.agg_sum(disc_price, P.DOUBLE), P.agg_sum(charge, P.DOUBLE),
            P.agg_avg(qty, P.DOUBLE, P.DOUBLE), P.agg_avg(price, P.DOUBLE, P.DOUBLE), P.agg_avg(disc, P.DOUBLE, P.DOUBLE),
            P.agg_count([P.literal(1, P.INT32)])]


def q1_scan_fields(variant):
    m = _money(variant)
    return [m, m, m, m, P.STRING, P.STRING, P.DATE]


Q1_COLUMNS = ["l_quantity", "l_extendedprice", "l_discount", "l_tax", "l_returnflag", "l_linestatus", "l_shipdate"]


def q1_native_scan(variant, files):
    """NativeScan (operator.proto:141) over Parquet files with the Q1 column projection."""
    fields = list(zip(Q1_COLUMNS, q1_scan_fields(variant), [True] * 7))
    return P.native_scan(fields, fields, files)


def write_lineitem_parquet(cols, path, variant="dec", row_group_size=1 << 20, decimal_as_int=True, columns=None):
    """SURVEY.md 8(d) fixture writer: pyarrow, data page v1, dictionary only for the flag columns, PLAIN numerics,
    uncompressed, decimals as INT64 (Spark's layout) or FIXED_LEN_BYTE_ARRAY."""
    import pyarrow.parquet as pq
    tbl = lineitem_table(cols, variant, dictionary=True, columns=columns or Q1_COLUMNS)
    kw = {}
    if decimal_as_int:
        kw["store_decimal_as_integer"] = True
    pq.write_table(tbl, path, row_group_size=row_group_size, compression="NONE", use_dictionary=["l_returnflag", "l_linestatus"],
                   data_page_version="1.0", write_statistics=True, **kw)
    return path


def q1_partial_plan(variant="dec", cutoff=Q1_CUTOFF, scan=None):
    """Map-stage plan of TPC-H Q1: Scan -> Filter -> Project -> HashAggregate(Partial)."""
    m = _money(variant)
    sc = scan if scan is not None else P.scan(q1_scan_fields(variant))
    ship = P.bound(6, P.DATE)
    flt = P.filter_(sc, P.and_(P.is_not_null(ship), P.lt_eq(ship, P.literal(cutoff, P.DATE))))
    proj = P.projection(flt, [P.bound(0, m), P.bound(1, m), P.bound(2, m), P.bound(3, m), P.bound(4, P.STRING), P.bound(5, P.STRING)])
    return P.hash_agg(proj, [P.bound(4, P.STRING), P.bound(5, P.STRING)], q1_aggs(variant), P.PARTIAL)


def q1_state_fields(variant):
    if variant == "dec":
        return [P.STRING, P.STRING, P.DECIMAL(22, 2), P.BOOL, P.DECIMAL(22, 2), P.BOOL, P.DECIMAL(36, 4), P.BOOL,
                P.DECIMAL(38, 6), P.BOOL, P.DECIMAL(22, 2), P.INT64, P.DECIMAL(22, 2), P.INT64, P.DECIMAL(22, 2), P.INT64, P.INT64]
    return [P.STRING, P.STRING, P.DOUBLE, P.DOUBLE, P.DOUBLE, P.DOUBLE, P.DOUBLE, P.INT64, P.DOUBLE, P.INT64, P.DOUBLE, P.INT64, P.INT64]


def q1_final_plan(variant="dec"):
    """Reduce-stage plan: ShuffleScan(partial state) -> HashAggregate(Final)."""
    sc = P.scan(q1_state_fields(variant), source="shuffle")
    return P.hash_agg(sc, [P.bound(0, P.STRING), P.bound(1, P.STRING)], q1_aggs(variant, bound=False), P.FINAL)


def q6_scan_fields(variant):
    m = _money(variant)
    return [m, m, m, P.DATE]  # quantity, extendedprice, discount, shipdate


def q6_aggs(variant, bound=True):
    m = _money(variant)
    ref = (lambda i, dt: P.bound(i, dt)) if bound else (lambda i, dt: P.unbound(f"c{i}", dt))
    price, disc = ref(0, m), ref(1, m)
    if variant == "dec":
        rev = P.check_overflow(P.multiply(price, disc, P.DECIMAL(25, 4)), P.DECIMAL(25, 4))
        return [P.agg_sum(rev, P.DECIMAL(35, 4))]
    return [P.agg_sum(P.multiply(price, disc, P.DOUBLE), P.DOUBLE)]


Q6_COLUMNS = ["l_quantity", "l_extendedprice", "l_discount", "l_shipdate"]


def q6_predicate(variant):
    m = _money(variant)
    qty, disc, ship = P.bound(0, m), P.bound(2, m), P.bound(3, P.DATE)
    return P.and_(P.and_(P.and_(P.and_(P.gt_eq(ship, P.literal(DATE_1994_01_01, P.DATE)), P.lt(ship, P.literal(DATE_1995_01_01, P.DATE))),
                                P.gt_eq(disc, _lit_money(5, variant))), P.lt_eq(disc, _lit_money(7, variant))),
                  P.lt(qty, _lit_money(2400, variant)))


def q6_native_scan(variant, files, push_filters=True):
    """NativeScan with the Q6 projection; `data_filters` carries the predicate the way Spark pushes it to the scan
    (CometNativeScan.scala: exprToProto(filter, scan.output)) -- the reference prunes row groups with it."""
    fields = list(zip(Q6_COLUMNS, q6_scan_fields(variant), [True] * 4))
    return P.native_scan(fields, fields, files, data_filters=[q6_predicate(variant)] if push_filters else ())


def q6_partial_plan(variant="dec", scan=None):
    """TPC-H Q6: 3-predicate filter + ungrouped SUM(l_extendedprice * l_discount)."""
    m = _money(variant)
    sc = scan if scan is not None else P.scan(q6_scan_fields(variant))
    flt = P.filter_(sc, q6_predicate(variant))
    proj = P.projection(flt, [P.bound(1, m), P.bound(2, m)])
    return P.hash_agg(proj, [], q6_aggs(variant), P.PARTIAL)


def q6_state_fields(variant):
    return [P.DECIMAL(35, 4), P.BOOL] if variant == "dec" else [P.DOUBLE]


def q6_final_plan(variant="dec"):
    sc = P.scan(q6_state_fields(variant), source="shuffle")
    return P.hash_agg(sc, [], q6_aggs(variant, bound=False), P.FINAL)


def config1_scan_fields(variant):
    m = _money(variant)
    return [m, m, P.DATE]  # quantity, extendedprice, shipdate


def config1_plan(variant="dec", cutoff=DATE_1998_09_02):
    """BASELINE.json configs[0]: SELECT l_quantity*l_extendedprice FROM lineitem WHERE l_shipdate < '1998-09-02'."""
    m = _money(variant)
    sc = P.scan(config1_scan_fields(variant))
    ship = P.bound(2, P.DATE)
    flt = P.filter_(sc, P.lt(ship, P.literal(cutoff, P.DATE)))
    if variant == "dec":
        e = P.check_overflow(P.multiply(P.bound(0, m), P.bound(1, m), P.DECIMAL(25, 4)), P.DECIMAL(25, 4))
    else:
        e = P.multiply(P.bound(0, m), P.bound(1, m), P.DOUBLE)
    return P.projection(flt, [e])
