"""The aggregate test matrix: deterministic cases over key types, aggregate functions, special values, batch layouts and the three
accumulation strategies of the aggregate executor (csrc/agg.cpp).  Used by tests/test_gpu_agg_matrix.py (runs them) and
tests/test_agg_matrix_cpu.py (checks that every plan compiles and that the matrix reaches every strategy).

Every case has the same value columns after its key columns:

  v0 i64   with MIN / MAX (the MIN / MAX identity words of the accumulators), -1, NULLs
  v1 f64   NaN, -NaN, NaN with a payload, +-Inf, +-0.0, subnormals, cancellation-heavy values, NULLs
  v2 decimal(12,2) at +-(10^12 - 1)      v7 decimal(18,0) at +-(10^18 - 1)
  v3 i8, v4 i16, v5 i32 with MIN / MAX / -1      v6 timestamp with MIN / MAX / -1      v8 bool (FILTER input)

The first key of row 0 forms a group whose values are all NULL, the key of row 1 a group whose v1 is NaN only."""
import math

import numpy as np
import pyarrow as pa

from comet_b200 import proto as P

import aggref as R
import exprs as E

I8, I16, I32, I64, DBL, BOOL, DATE, TS, STR = P.INT8, P.INT16, P.INT32, P.INT64, P.DOUBLE, P.BOOL, P.DATE, P.TIMESTAMP, P.STRING
D12, D18, D18K = P.DECIMAL(12, 2), P.DECIMAL(18, 0), P.DECIMAL(18, 2)
VALUE_TYPES = [I64, DBL, D12, I8, I16, I32, TS, D18, BOOL]

NAN_PAYLOAD = R.f64_of_bits(0x7FF8000000000ABC)
NEG_NAN = R.f64_of_bits(0xFFF8000000000000)
F64_SPECIAL = [math.nan, NEG_NAN, NAN_PAYLOAD, math.inf, -math.inf, 0.0, -0.0, 5e-324, -2.5e-310, 2.2250738585072014e-308]
F64_CANCEL = [1e16, 1.0, -1e16, 0.5, 3e15, -3e15, 1e-3]

STREAM_CFG = {"spark.comet.b200.streamAgg.minRows": "0"}
TABLE_CFG = {"spark.comet.b200.streamAgg.minRows": "-1"}


def int_pool(bits, rng, k):
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    return [lo, hi, -1, 0, 1] + [int(x) for x in rng.integers(lo, hi, k, endpoint=True)]


def key_pool(dt, rng, k):
    """Distinct key values of type dt, the edges first (-1 is the packed word of the key table's empty slot)."""
    if dt.name == "BOOL":
        return [True, False]
    if dt.name in ("INT8", "INT16", "INT32", "DATE"):
        pool = int_pool({"INT8": 8, "INT16": 16}.get(dt.name, 32), rng, k)
    elif dt.name in ("INT64", "TIMESTAMP"):
        pool = int_pool(64, rng, k)
    elif dt.name == "DECIMAL":
        m = 10 ** dt.precision - 1
        pool = [-m, m, -1, 0, 1] + [int(x) for x in rng.integers(-10 ** 17, 10 ** 17, k)]
    else:
        pool = [f"key-{i:04d}" for i in range(k)]
    return list(dict.fromkeys(pool))


def value_rows(rng, n):
    """The value columns v0..v8 as Python lists (None = NULL)."""
    def nulls(vals, frac):
        m = rng.random(n) < frac
        return [None if z else v for v, z in zip(vals, m)]
    pick = lambda pool: [pool[int(i)] for i in rng.integers(0, len(pool), n)]
    i64 = pick([R.I64_MIN, R.I64_MAX, -1, 0, 7] + [int(x) for x in rng.integers(-2 ** 62, 2 ** 62, 32)])
    f64 = []
    for _ in range(n):
        r = rng.random()
        if r < 0.08:
            f64.append(F64_SPECIAL[int(rng.integers(0, len(F64_SPECIAL)))])
        elif r < 0.3:
            f64.append(F64_CANCEL[int(rng.integers(0, len(F64_CANCEL)))])
        else:
            f64.append(float(rng.standard_normal() * 10.0 ** int(rng.integers(-3, 8))))
    m12, m18 = 10 ** 12 - 1, 10 ** 18 - 1
    d12 = pick([m12, -m12, -1, 0] + [int(x) for x in rng.integers(-m12, m12, 32)])
    d18 = pick([m18, -m18, -1, 0] + [int(x) for x in rng.integers(-10 ** 17, 10 ** 17, 32)])
    i8, i16, i32 = pick(int_pool(8, rng, 16)), pick(int_pool(16, rng, 16)), pick(int_pool(32, rng, 16))
    ts = pick(int_pool(64, rng, 16))
    b = [bool(x) for x in rng.integers(0, 2, n)]
    return [nulls(i64, 0.05), nulls(f64, 0.05), nulls(d12, 0.05), nulls(i8, 0.05), nulls(i16, 0.05), nulls(i32, 0.05), nulls(ts, 0.05),
            nulls(d18, 0.05), nulls(b, 0.1)]


# ---- aggregate sets (over the value columns, which start at column nk) -------------------------------------------------------------
def aggset(name, nk):
    c = lambda i: E.Col(nk + i, VALUE_TYPES[i])
    v0, v1, v2, v3, v4, v5, v6, v7, v8 = (c(i) for i in range(9))
    A = R.Agg
    if name == "int":
        return [A("count", v0), A("sum", v0, I64), A("min", v0, I64), A("max", v0, I64), A("count", v0, filt=v8), A("sum", v0, I64, filt=v8),
                A("min", v2, D12)]
    if name == "narrow":
        return [A("min", v3, I8), A("max", v3, I8), A("min", v4, I16), A("max", v4, I16), A("min", v5, I32), A("max", v5, I32),
                A("min", v6, TS), A("max", v6, TS), A("sum", v5, I64, mode=R.TRY), A("min", v7, D18), A("max", v7, D18)]
    if name == "f64":
        return [A("sum", v1, DBL), A("avg", v1, DBL), A("min", v1, DBL), A("max", v1, DBL), A("count", v1),
                A("sum", v1, DBL, filt=E.Cmp("gt", v1, E.Lit(0.0, DBL))), A("avg", v1, DBL, filt=v8)]
    if name == "dec":
        return [A("sum", v2, P.DECIMAL(22, 2)), A("avg", v2, P.DECIMAL(16, 6), sum_dt=P.DECIMAL(22, 2), filt=v8), A("max", v2, D12),
                A("sum", v7, P.DECIMAL(28, 0)), A("avg", v7, P.DECIMAL(22, 4), sum_dt=P.DECIMAL(28, 0))]
    if name == "expr":
        tripled = E.Arith("multiply", v2, E.Lit(3, P.DECIMAL(2, 0)), P.DECIMAL(15, 2))          # decimal(15,2)
        pos = E.If(E.Cmp("gt", v5, E.Lit(0, I32)), v5, E.Lit(0, I32))
        as_dec = E.Cast(v5, D12)
        return [A("sum", tripled, P.DECIMAL(25, 2)), A("sum", pos, I64), A("avg", E.Cast(v5, DBL), DBL), A("sum", as_dec, P.DECIMAL(22, 2)),
                A("count", v0, filt=E.IsNull(v1, negate=True)), A("max", tripled, P.DECIMAL(15, 2), filt=E.Cmp("lt", v3, E.Lit(0, I8)))]
    if name == "ansi":
        return [A("sum", v5, I64, mode=R.ANSI), A("sum", v4, I64, mode=R.TRY), A("sum", v3, I64, mode=R.ANSI, filt=v8),
                A("avg", v5, DBL, mode=R.ANSI)]
    raise KeyError(name)


# ---- cases -------------------------------------------------------------------------------------------------------------------------
class Case:
    def __init__(self, name, strategy, keys, aggs, n=3000, batch_rows=1024, chunk=None, offset=0, nullable=True, seed=0, all_valid=False,
                 clustered=False, key_card=60):
        self.name, self.strategy, self.key_specs, self.aggset = name, strategy, keys, aggs
        self.n, self.batch_rows, self.chunk, self.offset, self.nullable = n, batch_rows, chunk, offset, nullable
        self.seed, self.all_valid, self.clustered, self.key_card = seed, all_valid, clustered, key_card
        self._table = None

    def __repr__(self):
        return self.name

    @property
    def key_types(self):
        return [STR if isinstance(k, tuple) else k for k in self.key_specs]

    @property
    def dts(self):
        return self.key_types + VALUE_TYPES

    @property
    def key_cols(self):
        return list(range(len(self.key_specs)))

    @property
    def aggs(self):
        return aggset(self.aggset, len(self.key_specs))

    def config(self):
        cfg = dict(STREAM_CFG if self.strategy == "stream" else TABLE_CFG)
        if self.chunk:
            cfg["spark.comet.b200.chunkRows"] = str(self.chunk)
        return cfg

    def partial_plan(self):
        return R.partial_plan(self.dts, self.key_cols, self.aggs)

    def merge_plan(self, mode=R.FINAL):
        return R.merge_plan(self.key_types, self.aggs, mode)

    def _key_columns(self, rng, n):
        cols = []
        for spec in self.key_specs:
            if isinstance(spec, tuple):      # ("dict", index type, number of values)
                _, idx_t, card = spec
                pool = key_pool(STR, rng, card)
            else:
                pool = key_pool(spec, rng, self.key_card)
            if self.clustered:
                cols.append(pool)
            else:
                cols.append([pool[int(i)] for i in rng.integers(0, len(pool), n)])
        if self.clustered:                   # runs of ~8 equal keys in a row
            combos = [tuple(p[int(rng.integers(0, len(p)))] for p in cols) for _ in range(n // 6 + 1)]
            rows = []
            for t in combos:
                rows += [t] * int(rng.integers(4, 12))
            rows = rows[:n]
            cols = [[r[k] for r in rows] for k in range(len(cols))]
        if self.nullable and n > 0:
            for col in cols:
                for i in rng.integers(0, n, max(1, n // 40)):
                    col[int(i)] = None
        return cols

    def table(self):
        """The input table (already sliced at `offset`, so its buffers start mid-byte when offset % 8 != 0)."""
        if self._table is None:
            rng = np.random.default_rng(self.seed)
            n = self.n + self.offset
            keys = self._key_columns(rng, n)
            vals = value_rows(rng, n)
            if keys and n > self.offset + 1:
                k0 = tuple(k[self.offset] for k in keys)
                k1 = tuple(k[self.offset + 1] for k in keys)
                for i in range(n):
                    kt = tuple(k[i] for k in keys)
                    if kt == k0:
                        for v in vals:
                            v[i] = None              # a group whose values are all NULL
                    elif kt == k1 and vals[1][i] is not None:
                        vals[1][i] = math.nan        # a group whose float values are NaN only
            arrays = []
            for spec, col in zip(self.key_specs, keys):
                if isinstance(spec, tuple):
                    names = sorted({v for v in col if v is not None})
                    pos = {s: j for j, s in enumerate(names)}
                    idx = pa.array([None if v is None else pos[v] for v in col], type=spec[1])
                    arrays.append(pa.DictionaryArray.from_arrays(idx, pa.array(names or ["x"], type=pa.string())))
                else:
                    arrays.append(R.arrow_column(col, spec))
            arrays += [R.arrow_column(v, t) for v, t in zip(vals, VALUE_TYPES)]
            if self.all_valid:
                arrays = [all_valid_bitmap(a) for a in arrays]
            self._table = pa.table(arrays, names=[f"c{i}" for i in range(len(arrays))]).slice(self.offset)
        return self._table

    def batches(self):
        t = self.table()
        if t.num_rows == 0:
            return [pa.RecordBatch.from_arrays([pa.array([], type=f.type) for f in t.schema], schema=t.schema)]
        return t.to_batches(max_chunksize=self.batch_rows)


def all_valid_bitmap(a):
    """The same values with a validity buffer whose bits are all set (instead of none at all)."""
    if a.null_count or pa.types.is_dictionary(a.type) or a.buffers()[0] is not None:
        return a
    bitmap = pa.py_buffer(np.packbits(np.ones(len(a) + a.offset, dtype=np.uint8), bitorder="little").tobytes())
    return pa.Array.from_buffers(a.type, len(a), [bitmap] + a.buffers()[1:], null_count=0, offset=a.offset)


class MigrateCase(Case):
    """A dictionary key with 6 values in the first batches and 300 later: dense first, then the key table (csrc/agg.cpp leave_dense)."""

    def table(self):
        if self._table is None:
            rng = np.random.default_rng(self.seed)
            small = [f"s{i}" for i in range(6)]
            big = [f"b{i:03d}" for i in range(294)] + small
            batches = []
            for bi in range(6):
                names = small if bi < 2 else big
                m = self.batch_rows
                codes = rng.integers(0, len(names), m).astype(np.int32)
                mask = rng.random(m) < 0.03
                keys = pa.DictionaryArray.from_arrays(pa.array(codes, mask=mask), pa.array(names))
                vals = value_rows(rng, m)
                batches.append(pa.RecordBatch.from_arrays([keys] + [R.arrow_column(v, t) for v, t in zip(vals, VALUE_TYPES)],
                                                          names=[f"c{i}" for i in range(10)]))
            self._table = pa.Table.from_batches(batches)
        return self._table

    def batches(self):
        return self.table().to_batches()


def _cases():
    cs = []
    aggsets = ["int", "narrow", "f64", "dec", "expr", "ansi"]
    a = lambda i: aggsets[i % len(aggsets)]
    # key table: every key type the hash path packs, scattered keys
    hash_keys = [[I8], [I16], [I32], [DATE], [I64], [TS], [D18K], [BOOL, I32], [I8, I16, I32, BOOL], [I32, I64], [I64, I32],
                 [I64, I64, DATE, I8]]
    for i, keys in enumerate(hash_keys):
        name = "table-" + "-".join(k.name.lower() if k.name != "DECIMAL" else "dec18" for k in keys)
        for s in (["int", "f64"] if len(keys) == 1 and keys[0].name in ("INT64", "TIMESTAMP", "DECIMAL") else [a(i)]):
            cs.append(Case(f"{name}-{s}", "table", keys, s, seed=100 + i, chunk=[None, 1024, 700, 5000][i % 4], offset=[0, 3, 0, 13][i % 4],
                           nullable=i % 5 != 4))
    # stream: clustered keys, one state row per run
    for i, (keys, s) in enumerate([([I64], "f64"), ([I32], "ansi"), ([DATE, I64], "dec"), ([D18K], "narrow"), ([I16], "expr"), ([TS], "int"),
                                   ([I8, BOOL], "f64")]):
        cs.append(Case(f"stream-{i}-{s}", "stream", keys, s, n=4000, seed=200 + i, clustered=True, chunk=[None, 2048][i % 2], offset=[0, 5][i % 2]))
    # dense: dictionary strings (int8 / int16 / int32 indices) and bool keys, <= 64 groups
    dense = [([("dict", pa.int8(), 20)], "f64"), ([("dict", pa.int16(), 30)], "int"), ([("dict", pa.int32(), 7), BOOL], "dec"), ([BOOL], "narrow"),
             ([("dict", pa.int8(), 12)], "expr"), ([("dict", pa.int16(), 5), BOOL], "ansi"), ([("dict", pa.int32(), 3), ("dict", pa.int8(), 4)], "f64")]
    for i, (keys, s) in enumerate(dense):
        cs.append(Case(f"dense-{i}-{s}", "dense", keys, s, seed=300 + i, chunk=[None, 600][i % 2], offset=[0, 11][i % 2], all_valid=i == 1))
    # dense -> key table mid-stream
    cs.append(MigrateCase("migrate-f64", "migrate", [("dict", pa.int32(), 300)], "f64", seed=400, batch_rows=2000, chunk=2000))
    cs.append(MigrateCase("migrate-int", "migrate", [("dict", pa.int32(), 300)], "int", seed=401, batch_rows=1500, chunk=1500))
    # ungrouped
    for i, s in enumerate(["f64", "dec", "int", "narrow", "ansi", "expr"]):
        cs.append(Case(f"ungrouped-{s}", "ungrouped", [], s, seed=500 + i, chunk=[None, 777][i % 2], offset=[0, 6][i % 2]))
    # layout edges: one row, empty input, a value column with an all-set validity buffer, chunks equal to the batches
    cs.append(Case("one-row-i64", "table", [I64], "f64", n=1, seed=600))
    cs.append(Case("empty-ungrouped", "empty", [], "f64", n=0, seed=601))
    cs.append(Case("empty-ungrouped-dec", "empty", [], "dec", n=0, seed=602))
    cs.append(Case("empty-grouped", "empty", [I64], "int", n=0, seed=603))
    cs.append(Case("all-valid-bitmaps", "table", [I32], "int", nullable=False, all_valid=True, seed=604, chunk=1024))
    return cs


CASES = _cases()
EXPECTED_BITS = {"dense": 1, "table": 2, "stream": 4, "migrate": 1 | 8 | 2, "ungrouped": 1, "empty": 0}
