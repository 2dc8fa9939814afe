"""Distinct-aggregate chains (tests/distinctref.py) over key types, ordinary and distinct aggregate sets, stage 3 orders and batch
layouts.  Used by tests/test_distinct_agg_cpu.py (every plan compiles) and tests/test_gpu_distinct_agg.py (every stage on the device).

Input columns: the outer keys, the distinct column x, then
  y0 decimal(12,2)   y1 i64   y2 f64   y3 i32 (COUNT(DISTINCT x, y3)'s second column)   b bool (FILTER input)"""
import numpy as np
import pyarrow as pa

from comet_b200 import proto as P

import aggcases
import aggref as R
import distinctref as D
import exprs as E

I32, I64, DBL, BOOL, DATE, STR = P.INT32, P.INT64, P.DOUBLE, P.BOOL, P.DATE, P.STRING
D12, D18 = P.DECIMAL(12, 2), P.DECIMAL(18, 2)  # a distinct column is a group key: decimal(p > 18) keys are refused
VALUE_TYPES = [D12, I64, DBL, I32, BOOL]
DICT = ("dict", pa.int16())     # a dictionary-coded string column


def ordinary(name, nk):
    """Ordinary aggregates over the value columns (which start after the outer keys and x)."""
    y0, y1, y2, y3, b = (E.Col(nk + 1 + i, t) for i, t in enumerate(VALUE_TYPES))
    A = R.Agg
    if name == "none":
        return []
    if name == "dec":
        return [A("sum", y0, P.DECIMAL(22, 2)), A("avg", y0, P.DECIMAL(16, 6), sum_dt=P.DECIMAL(22, 2), filt=b), A("min", y0, D12), A("count", y1)]
    if name == "int":
        return [A("sum", y1, I64), A("sum", y3, I64, mode=R.TRY), A("sum", y3, I64, mode=R.ANSI, filt=b), A("max", y1, I64), A("count", y1, filt=b)]
    if name == "f64":
        return [A("sum", y2, DBL), A("avg", y2, DBL), A("min", y2, DBL), A("max", y2, DBL, filt=b)]
    raise KeyError(name)


def distinct(name, xt):
    """Distinct aggregates over x: (kind, dt, sum_dt, eval_mode)."""
    if name == "count":
        return [("count", None, None, R.LEGACY)]
    if xt.name == "DECIMAL":
        p = xt.precision
        return [("count", None, None, R.LEGACY), ("sum", P.DECIMAL(p + 10, 2), None, R.LEGACY), ("avg", P.DECIMAL(p + 4, 6), P.DECIMAL(p + 10, 2), R.LEGACY)]
    return [("count", None, None, R.LEGACY), ("sum", I64, None, R.LEGACY), ("avg", DBL, None, R.LEGACY)]


class Case:
    """bits: the expected cb200_stats.agg_strategies of stages 1-4."""

    def __init__(self, name, keys, x, ordinary_set, distinct_set, bits, n=3000, seed=0, interleave=False, nullable=True, chunk=None,
                 batch_rows=1024, clustered=False, count2=False, offset2=True, key_card=30, x_card=40):
        self.name, self.key_specs, self.x_spec, self.oset, self.dset, self.bits = name, keys, x, ordinary_set, distinct_set, bits
        self.n, self.seed, self.interleave, self.nullable, self.chunk, self.batch_rows = n, seed, interleave, nullable, chunk, batch_rows
        self.clustered, self.count2, self.offset2, self.key_card, self.x_card = clustered, count2, offset2, key_card, x_card
        self._table = None

    def __repr__(self):
        return self.name

    @staticmethod
    def _type(spec):
        return STR if isinstance(spec, tuple) else spec

    @property
    def dts(self):
        return [self._type(k) for k in self.key_specs] + [self._type(self.x_spec)] + VALUE_TYPES

    def chain(self):
        nk = len(self.key_specs)
        xt = self._type(self.x_spec)
        o = ordinary(self.oset, nk)
        d = distinct(self.dset if xt.name not in ("STRING", "BOOL", "DATE") else "count", xt)
        order = None
        if self.interleave:   # distinct and merging aggregates alternate, a distinct one first
            order, oi, di = [], 0, 0
            while oi < len(o) or di < len(d):
                if di < len(d):
                    order.append(("d", di)); di += 1
                if oi < len(o):
                    order.append(("o", oi)); oi += 1
        dcols = [nk, nk + 4] if self.count2 else [nk]
        if self.count2:
            d = [("count", None, None, R.LEGACY)]
        return D.Chain(self.dts, range(nk), dcols, o, d, order)

    def config(self, stage):
        cfg = dict(aggcases.STREAM_CFG if self.clustered and stage == 1 else aggcases.TABLE_CFG)
        if self.chunk:
            cfg["spark.comet.b200.chunkRows"] = str(self.chunk)
        return cfg

    def table(self):
        if self._table is None:
            rng = np.random.default_rng(self.seed)
            n = self.n
            cols = []
            for spec, card in [(k, self.key_card) for k in self.key_specs] + [(self.x_spec, self.x_card)]:
                t = self._type(spec)
                if t.name == "DECIMAL":   # edges of the declared precision, then values that fit it
                    m = 10 ** t.precision - 1
                    pool = list(dict.fromkeys([-m, m, -1, 0, 1] + [int(v) for v in rng.integers(-min(m, 10 ** 17), min(m, 10 ** 17), card)]))
                else:
                    pool = aggcases.key_pool(t, rng, card)
                if self.clustered:
                    vals = [pool[int(i)] for i in np.sort(rng.integers(0, len(pool), n))]
                else:
                    vals = [pool[int(i)] for i in rng.integers(0, len(pool), n)]
                if self.nullable and n:
                    for i in rng.integers(0, n, max(1, n // 30)):
                        vals[int(i)] = None
                cols.append((spec, vals))
            nul = lambda vals: [None if z else v for v, z in zip(vals, rng.random(n) < 0.05)]
            y0 = nul([int(v) for v in rng.integers(-10 ** 11, 10 ** 11, n)])
            y1 = nul([int(v) for v in rng.integers(-2 ** 40, 2 ** 40, n)])
            y2 = nul([float(v) for v in rng.standard_normal(n) * 1e3])
            y3 = nul([int(v) for v in rng.integers(-2 ** 31, 2 ** 31, n)])
            b = nul([bool(v) for v in rng.integers(0, 2, n)])
            if self.key_specs and n > 1:  # the outer key of row 0 forms a group whose values are all NULL
                k0 = tuple(c[1][0] for c in cols[:len(self.key_specs)])
                for i in range(n):
                    if tuple(c[1][i] for c in cols[:len(self.key_specs)]) == k0:
                        y0[i] = y1[i] = y2[i] = y3[i] = cols[-1][1][i] = None
            arrays = []
            for spec, vals in cols:
                if isinstance(spec, tuple):
                    names = sorted({v for v in vals if v is not None}) or ["x"]
                    pos = {s: j for j, s in enumerate(names)}
                    arrays.append(pa.DictionaryArray.from_arrays(pa.array([None if v is None else pos[v] for v in vals], type=spec[1]), pa.array(names)))
                else:
                    arrays.append(R.arrow_column(vals, spec))
            arrays += [R.arrow_column(v, t) for v, t in zip([y0, y1, y2, y3, b], VALUE_TYPES)]
            self._table = pa.table(arrays, names=[f"c{i}" for i in range(len(arrays))])
        return self._table

    def batches(self):
        t = self.table()
        if t.num_rows == 0:
            return [pa.RecordBatch.from_arrays([pa.array([], type=f.type) for f in t.schema], schema=t.schema)]
        return t.to_batches(max_chunksize=self.batch_rows)


T, S, DN = 2, 4, 1   # key table, stream, dense (cb200 agg strategy bits)
CASES = [
    Case("i64-x_i64-dec", [I64], I64, "dec", "all", (T, T, T, T), seed=1),
    Case("i32-x_dec12-int-interleaved", [I32], D12, "int", "all", (T, T, T, T), seed=2, interleave=True, chunk=700),
    Case("date-x_dec18-f64", [DATE], D18, "f64", "all", (T, T, T, T), seed=3, offset2=False),
    Case("dict-x_i32-dec", [DICT], I32, "dec", "all", (T, T, DN, DN), seed=4, key_card=5, interleave=True),
    Case("bool-x_bool-f64", [BOOL], BOOL, "f64", "count", (DN, DN, DN, DN), seed=5),
    Case("i64_bool-x_date-int", [I64, BOOL], DATE, "int", "count", (T, T, T, T), seed=6, nullable=False),
    Case("global-x_i64-int", [], I64, "int", "all", (T, T, DN, DN), seed=7, chunk=500),
    Case("global-x_dec12-dec-interleaved", [], D12, "dec", "all", (T, T, DN, DN), seed=8, interleave=True),
    Case("count2-i64-x_i32_y3-dec", [I64], I32, "dec", "count", (T, T, T, T), seed=9, count2=True),
    Case("stream-i64-x_i32-dec", [I64], I32, "dec", "all", (S, T, T, T), seed=10, clustered=True, n=6000),
    Case("keysonly-i64-x_i32", [I64], I32, "none", "all", (T, T, T, T), seed=11),
    Case("keysonly-dict-x_bool", [DICT], BOOL, "none", "count", (DN, DN, DN, DN), seed=12, key_card=6),
    Case("keysonly-stream-i64-x_i64", [I64], I64, "none", "count", (S, T, T, T), seed=13, clustered=True, n=6000),
    Case("keysonly-global-x_dec18", [], D18, "none", "all", (T, T, DN, DN), seed=14),
    Case("one-row", [I64], I64, "dec", "all", (T, T, T, T), n=1, seed=15),
    Case("empty-grouped", [I64], I64, "int", "all", (0, 0, 0, 0), n=0, seed=16),
    Case("empty-global", [], I64, "f64", "all", (0, 0, 0, DN), n=0, seed=17),   # stage 3 still emits its one ungrouped row
]
