"""A plain CPU reference of the HashAggregate operator, written for clarity rather than speed: the counterpart of tests/exprs.py for
the aggregate operator (tests/test_gpu_agg_matrix.py runs it against the library).

Integer and decimal totals are Python ints, float sums are exact (`fractions.Fraction`, rounded once), and AVG(decimal) goes through
the oracle's `AvgDecimalGroups`, which restates avg_decimal.rs.  Aggregate inputs and FILTER clauses are `exprs.py` nodes evaluated by
that interpreter.

Values are Python objects: int for integers, dates (days), timestamps (microseconds) and unscaled decimals, float for doubles (the
bits, NaN sign and payload included, are kept), bool, str for dictionary strings, and None for NULL.  A group key is the tuple of its
key values.

Rules, one per function (paths are under native/spark-expr/src/agg_funcs/ of the reference):

- FILTER: a row passes when the filter is TRUE; FALSE and NULL both exclude it (sum_decimal.rs:452-458).
- COUNT(x): the number of passing rows whose inputs are all non-NULL.  State: (count).
- SUM(int), Legacy: wrapping i64 sum, NULL while no value was seen (sum_int.rs:107-170).  State: (sum).
  TRY: checked row by row; an overflow makes the sum NULL for good; the state also carries has_all_nulls (sum_int.rs:236-390).
  ANSI: checked row by row; an overflow fails the query (sum_int.rs:176-235).
- SUM(decimal): exact sum; state (sum, is_empty), sum = 0 while empty and NULL after an overflow of the result precision;
  evaluates to NULL when empty or overflowed (sum_decimal.rs:176-369, merge :309-369).
- AVG(decimal): the oracle's AvgDecimalGroups (avg_decimal.rs:410-668).  State: (sum, count), sharing one validity.
- SUM(f64): the exact sum under IEEE special values: any NaN gives NaN, +Inf together with -Inf gives NaN, otherwise any Inf gives
  that Inf; a finite exact sum is rounded once (to +-Inf when it is out of range).  NULL when no value was seen.  State: (sum).
- AVG(f64): state (sum, count) (avg.rs:82-95).  Merging: the grouped accumulator adds every partial sum and count
  (avg.rs:279-309); the ungrouped one skips NULL sums and NULL counts through arrow's null-skipping `sum` (avg.rs:165-175), and its
  Partial emits a NULL sum for a partition that saw no batch (avg.rs:148-153).  This module merges by the ungrouped rule in both
  cases: the grouped reference never emits a NULL partial sum, and Arrow leaves the bytes under a NULL slot unspecified, so the two
  rules agree wherever the grouped one is defined.  Evaluates to NULL when the count is 0, else sum / count (avg.rs:177-188).
- MIN / MAX: NULL when no value was seen.  Floats are ordered by IEEE 754 totalOrder: -NaN < -Inf < ... < -0.0 < +0.0 < ... <
  +Inf < +NaN, NaNs ordered by payload, and the winning value is returned with its exact bits.  The DataFusion / arrow-rs min/max
  sources are not part of the reference tree; this restates the behaviour the library's DESIGN.md section 2 assumes: arrow-rs
  compares floats with `ArrowNativeTypeOp::is_lt` / `is_gt`, which for f32 / f64 are defined through `total_cmp`, and DataFusion's
  min / max accumulators keep the first operand unless the new value compares strictly less (greater).  Under totalOrder two values
  compare equal only when their bits are equal, so which of two equal values is kept cannot be observed.
- Grouping: NULL keys form a group of their own.  An ungrouped aggregate over no rows still emits one row, the state / result of a
  fresh accumulator.
"""
import math
import struct
from fractions import Fraction

import numpy as np
import pyarrow as pa

from comet_b200 import proto as P
from oracle import oracle as O

import exprs as E

LEGACY, TRY, ANSI = E.LEGACY, E.TRY, E.ANSI
PARTIAL, FINAL, PARTIAL_MERGE = P.PARTIAL, P.FINAL, P.PARTIAL_MERGE
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1

INT_TYPES = ("INT8", "INT16", "INT32", "INT64")


class Agg:
    """One aggregate expression.  `arg`: exprs.py node over the Partial's input columns; `dt`: the declared result type (the input
    type for MIN / MAX, the sum type for SUM, the result type for AVG); `sum_dt`: AVG's sum type; `filt`: optional BOOL node."""

    def __init__(self, kind, arg, dt=None, sum_dt=None, mode=LEGACY, filt=None):
        self.kind, self.arg, self.dt, self.sum_dt, self.mode, self.filt = kind, arg, dt, sum_dt, mode, filt
        if kind == "count":
            self.dt = P.INT64
        if kind == "avg" and dt.name != "DECIMAL":
            self.sum_dt = P.DOUBLE

    def proto(self, merge=False):
        """The aggregate as the Partial plan carries it (merge=False) or as a Final / PartialMerge plan does (input by name)."""
        child = P.unbound("s", self.arg.dt) if merge else self.arg.proto()
        f = None if merge or self.filt is None else self.filt.proto()
        if self.kind == "count":
            return P.agg_count([child], f)
        if self.kind == "sum":
            return P.agg_sum(child, self.dt, self.mode, filter_expr=f)
        if self.kind == "avg":
            return P.agg_avg(child, self.dt, self.sum_dt, self.mode, filter_expr=f)
        return (P.agg_min if self.kind == "min" else P.agg_max)(child, self.dt, filter_expr=f)

    def state_types(self):  # plan.cpp agg_state_types
        k, dt = self.kind, self.dt
        if k == "count":
            return [P.INT64]
        if k == "sum":
            if dt.name == "DECIMAL":
                return [dt, P.BOOL]
            if dt.name in INT_TYPES:
                return [P.INT64, P.BOOL] if self.mode == TRY else [P.INT64]
            return [dt]
        if k == "avg":
            return [self.sum_dt, P.INT64]
        return [dt]

    def result_type(self):
        if self.kind == "count":
            return P.INT64
        if self.kind == "avg":
            return self.dt if self.dt.name == "DECIMAL" else P.DOUBLE
        return self.dt

    @property
    def f64_sum(self):
        """SUM(f64) / AVG(f64): double-double on the device, exact here."""
        return (self.kind == "avg" and self.dt.name != "DECIMAL") or (self.kind == "sum" and self.dt.name == "DOUBLE")


def partial_plan(in_types, key_cols, aggs):
    return P.hash_agg(P.scan(in_types), [P.bound(k, in_types[k]) for k in key_cols], [a.proto() for a in aggs], PARTIAL)


def state_schema(key_types, aggs):
    out = list(key_types)
    for a in aggs:
        out += a.state_types()
    return out


def merge_plan(key_types, aggs, mode=FINAL):
    """A Final or PartialMerge aggregate over a state batch (group keys first, then every aggregate's state columns)."""
    return P.hash_agg(P.scan(state_schema(key_types, aggs), source="shuffle"), [P.bound(k, t) for k, t in enumerate(key_types)],
                      [a.proto(merge=True) for a in aggs], mode)


# ---- Arrow -> Python values -----------------------------------------------------------------------------------------------------
def f64_bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def f64_of_bits(b):
    return struct.unpack("<d", struct.pack("<Q", b))[0]


def total_key(x):
    """IEEE 754 totalOrder as a signed integer (the same map as cb::f64_total_key)."""
    b = f64_bits(x)
    s = b - (1 << 64) if b >> 63 else b
    return s ^ 0x7FFFFFFFFFFFFFFF if s < 0 else s


def pyvalues(arr, dt):
    """One Arrow column -> list of Python values (None for NULL)."""
    if isinstance(arr, pa.ChunkedArray):  # chunk by chunk: dictionary chunks may carry different dictionaries
        return [v for c in arr.chunks for v in pyvalues(c, dt)]
    n = len(arr)
    valid = arr.is_valid().to_numpy(zero_copy_only=False) if arr.null_count else np.ones(n, dtype=bool)
    if pa.types.is_dictionary(arr.type):
        idx = arr.indices.to_numpy(zero_copy_only=False)
        d = arr.dictionary.to_pylist()
        return [d[int(i)] if ok else None for i, ok in zip(idx, valid)]
    if dt.name == "DOUBLE":
        v = np.frombuffer(arr.buffers()[1], dtype=np.float64)[arr.offset:arr.offset + n]
        return [float(x) if ok else None for x, ok in zip(v, valid)]
    if dt.name == "DECIMAL":
        v = np.frombuffer(arr.buffers()[1], dtype=np.uint64)[2 * arr.offset:2 * (arr.offset + n)].reshape(-1, 2)
        return O.dec_to_ints(v, valid)
    if dt.name in ("DATE", "TIMESTAMP"):
        arr = arr.view(pa.int32() if dt.name == "DATE" else pa.int64())
    out = arr.to_pylist()
    return out


def exprs_columns(table, dts):
    """A table -> the column form exprs.py evaluates: (values, valid) per column; strings as object arrays."""
    cols = []
    for c, dt in zip(table.columns, dts):
        vals = pyvalues(c, dt)
        valid = np.array([v is not None for v in vals], dtype=bool)
        if dt.name == "DECIMAL":
            cols.append((O.dec_from_ints(vals), valid))
        elif dt.name == "DOUBLE":
            cols.append((np.array([0.0 if v is None else v for v in vals], dtype=np.float64), valid))
        elif dt.name == "BOOL":
            cols.append((np.array([bool(v) for v in vals], dtype=bool), valid))
        elif dt.name == "STRING":
            cols.append((np.array(vals, dtype=object), valid))
        else:
            cols.append((np.array([0 if v is None else v for v in vals], dtype=np.int64), valid))
    return cols


def node_values(node, cols):
    """Evaluate an exprs.py node -> list of Python values (None for NULL)."""
    v, valid = node.eval(cols)
    valid = np.asarray(valid, dtype=bool)
    dt = node.dt
    if dt.name == "DECIMAL":
        return O.dec_to_ints(v, valid)
    if dt.name == "DOUBLE":
        return [float(x) if ok else None for x, ok in zip(np.asarray(v, dtype=np.float64), valid)]
    if dt.name == "BOOL":
        return [bool(x) if ok else None for x, ok in zip(v, valid)]
    return [int(x) if ok else None for x, ok in zip(v, valid)]


# ---- exact float arithmetic -------------------------------------------------------------------------------------------------------
class ExactF64:
    """The exact sum of doubles under IEEE special-value rules."""

    def __init__(self):
        self.total, self.nan, self.pinf, self.ninf = Fraction(0), False, False, False

    def add(self, x):
        if math.isnan(x):
            self.nan = True
        elif x == math.inf:
            self.pinf = True
        elif x == -math.inf:
            self.ninf = True
        else:
            self.total += Fraction(x)

    def special(self):
        """NaN / +-Inf when the inputs decide the result by themselves, else None."""
        if self.nan or (self.pinf and self.ninf):
            return math.nan
        if self.pinf or self.ninf:
            return math.inf if self.pinf else -math.inf
        return None

    def value(self):
        s = self.special()
        return s if s is not None else round_fraction(self.total)

    def divided(self, n):
        s = self.special()
        return s if s is not None else round_fraction(self.total / n)


def round_fraction(q):
    try:
        return float(q)          # correctly rounded
    except OverflowError:
        return math.inf if q > 0 else -math.inf


# ---- per-group accumulation -------------------------------------------------------------------------------------------------------
def _wrap64(x):
    return ((x + (1 << 63)) % (1 << 64)) - (1 << 63)


class _AnsiOverflow(Exception):
    pass


def _partial_state(a, vals):
    """State of one aggregate over the values of one group (the passing, non-NULL inputs in row order)."""
    k, dt = a.kind, a.dt
    n = len(vals)
    if k == "count":
        return (n,)
    if k in ("min", "max"):
        if not vals:
            return (None,)
        if dt.name == "DOUBLE":
            pick = min if k == "min" else max
            return (pick(vals, key=total_key),)
        return ((min if k == "min" else max)(vals),)
    if k == "sum" and dt.name == "DECIMAL":
        s = sum(vals)
        return (0, True) if n == 0 else ((s, False) if abs(s) < 10 ** dt.precision else (None, False))
    if k == "sum" and dt.name in INT_TYPES:
        if a.mode == LEGACY:
            return (_wrap64(sum(vals)) if n else None,)
        s, ovf = 0, False
        for v in vals:                      # row-ordered add_checked
            s += v
            if not I64_MIN <= s <= I64_MAX:
                ovf = True
                break
        if a.mode == ANSI:
            if ovf:
                raise _AnsiOverflow()
            return (s if n else None,)
        return (None, False) if ovf else (s, n == 0)
    if a.f64_sum:
        acc = ExactF64()
        for v in vals:
            acc.add(float(v))
        if k == "sum":
            return (acc.value() if n else None,)
        # grouped reference: (0.0, 0) for a group without values.  The ungrouped reference's Partial emits (NULL, 0) when it saw
        # no batch (avg.rs:148-153); the library emits (0.0, 0) there as well (DESIGN.md section 6), with the same Final result.
        return (acc.value() if n else 0.0, n)
    raise AssertionError(k)


def _merge_state(a, states):
    """Merge state tuples of one group: the state of the merged accumulator (the Partial -> PartialMerge step)."""
    k, dt = a.kind, a.dt
    if k == "count":
        return (sum(s[0] for s in states if s[0] is not None),)
    if k in ("min", "max"):
        vs = [s[0] for s in states if s[0] is not None]
        return _partial_state(a, vs)
    if k == "sum" and dt.name == "DECIMAL":  # sum_decimal.rs:309-369
        if any(not e and s is None for s, e in states):
            return (None, False)
        if all(e for _, e in states):
            return (0, True)
        return _partial_state(a, [s for s, e in states if not e])
    if k == "sum" and dt.name in INT_TYPES:
        if a.mode == TRY:                   # sum_int.rs:331-389
            if any(not e and s is None for s, e in states):
                return (None, False)
            if all(e for _, e in states):
                return (0, True)
            return _partial_state(a, [s for s, e in states if not e])
        vs = [s[0] for s in states if s[0] is not None]
        return _partial_state(a, vs)
    if a.f64_sum:
        if k == "sum":
            return _partial_state(a, [s[0] for s in states if s[0] is not None])
        acc = ExactF64()
        for s, _ in states:
            if s is not None:
                acc.add(s)
        return (acc.value(), sum(c for _, c in states if c is not None))
    raise AssertionError(k)


def _evaluate(a, state):
    k, dt = a.kind, a.dt
    if k in ("count", "min", "max"):
        return state[0]
    if k == "sum" and dt.name == "DECIMAL":
        s, empty = state
        return None if empty else s
    if k == "sum" and dt.name in INT_TYPES:
        if a.mode == TRY:
            s, empty = state
            return None if empty else s
        return state[0]
    if k == "sum":
        return state[0]
    raise AssertionError(k)


class _AvgF64Final:
    """AVG(f64) evaluation needs the exact sum, not its rounded state: kept apart so the mean is rounded once."""

    def __init__(self):
        self.acc, self.n = ExactF64(), 0

    def add_state(self, s, c):
        if s is not None:
            self.acc.add(s)
        if c is not None:
            self.n += c

    def add_value(self, v):
        self.acc.add(float(v))
        self.n += 1

    def result(self):
        return None if self.n == 0 else self.acc.divided(self.n)


# ---- the operator -----------------------------------------------------------------------------------------------------------------
class Groups:
    """Group keys in first-occurrence order and per-group row lists."""

    def __init__(self):
        self.index, self.keys = {}, []

    def gid(self, key):
        g = self.index.get(key)
        if g is None:
            g = self.index[key] = len(self.keys)
            self.keys.append(key)
        return g


def _input_rows(table, dts, key_cols, aggs):
    """Per aggregate: (group id of every row, passing non-NULL input value or a skip marker) plus the groups."""
    cols = exprs_columns(table, dts)
    n = table.num_rows
    key_vals = [pyvalues(table.column(k), dts[k]) for k in key_cols]
    groups = Groups()
    gids = [groups.gid(tuple(kv[i] for kv in key_vals)) for i in range(n)]
    per_agg = []
    for a in aggs:
        vals = node_values(a.arg, cols) if n else []
        if a.filt is not None and n:
            fv = node_values(a.filt, cols)
            vals = [v if f is True else None for v, f in zip(vals, fv)]
        per_agg.append(vals)
    return groups, gids, per_agg


def partial(table, dts, key_cols, aggs):
    """Partial aggregate: {key tuple: [state tuple per aggregate]}.  Raises exprs.AnsiError for an ANSI overflow."""
    groups, gids, per_agg = _input_rows(table, dts, key_cols, aggs)
    if not key_cols and not groups.keys:
        groups.gid(())
    out = {}
    for ai, a in enumerate(aggs):
        rows = [[] for _ in groups.keys]
        for g, v in zip(gids, per_agg[ai]):
            if v is not None:
                rows[g].append(v)
        if a.kind == "avg" and a.dt.name == "DECIMAL":
            st, _ = _avg_decimal(a, rows)
        else:
            try:
                st = [_partial_state(a, r) for r in rows]
            except _AnsiOverflow:
                raise E.AnsiError()
        for key, s in zip(groups.keys, st):
            out.setdefault(key, [None] * len(aggs))[ai] = s
    return out


def _avg_decimal(a, rows, states=None):
    """AVG(decimal) through the oracle's AvgDecimalGroups: states of `rows` (Partial) or of merged `states` (list per group)."""
    ng = len(rows) if rows is not None else len(states)
    acc = O.AvgDecimalGroups(max(ng, 1), a.sum_dt.precision, a.sum_dt.scale, a.dt.precision, a.dt.scale, a.mode)
    if rows is not None:
        vals = [v for r in rows for v in r]
        gidx = np.array([g for g, r in enumerate(rows) for _ in r], dtype=np.int64)
        if vals:
            acc.update(O.dec_from_ints(vals), np.ones(len(vals), dtype=np.uint8), gidx)
    else:
        flat = [(g, s) for g, ss in enumerate(states) for s in ss]
        if flat:
            sums = O.dec_from_ints([s[0] for _, s in flat])
            sv = np.array([s[0] is not None for _, s in flat], dtype=np.uint8)
            cnt = np.array([0 if s[1] is None else s[1] for _, s in flat], dtype=np.int64)
            cv = np.array([s[1] is not None for _, s in flat], dtype=np.uint8)
            acc.merge(sums, sv, cnt, cv, np.array([g for g, _ in flat], dtype=np.int64))
    sums, counts, nn = acc.state()
    return [(O.dec_to_ints(sums[g:g + 1])[0] if nn[g] else None, int(counts[g]) if nn[g] else None) for g in range(ng)], acc


def merge(state_rows, aggs):
    """Merge state rows [(key, [state per aggregate])...] -> {key: [merged state per aggregate]} (PartialMerge)."""
    by_key = {}
    for key, st in state_rows:
        by_key.setdefault(key, []).append(st)
    out = {}
    keys = list(by_key)
    for ai, a in enumerate(aggs):
        if a.kind == "avg" and a.dt.name == "DECIMAL":
            st, _ = _avg_decimal(a, None, [[s[ai] for s in by_key[k]] for k in keys])
        else:
            st = [_merge_state(a, [s[ai] for s in by_key[k]]) for k in keys]
        for k, s in zip(keys, st):
            out.setdefault(k, [None] * len(aggs))[ai] = s
    return out


def final(state_rows, aggs, ungrouped=False):
    """Final aggregate over state rows [(key, [state per aggregate])...] -> {key: [result per aggregate]}."""
    by_key = {}
    for key, st in state_rows:
        by_key.setdefault(key, []).append(st)
    if ungrouped and not by_key:
        by_key[()] = []
    keys = list(by_key)
    out = {k: [None] * len(aggs) for k in keys}
    for ai, a in enumerate(aggs):
        if a.kind == "avg" and a.dt.name == "DECIMAL":
            _, acc = _avg_decimal(a, None, [[s[ai] for s in by_key[k]] for k in keys])
            res, ok = acc.evaluate()
            for g, k in enumerate(keys):
                out[k][ai] = O.dec_to_ints(res[g:g + 1])[0] if ok[g] else None
            continue
        for k in keys:
            sts = [s[ai] for s in by_key[k]]
            if a.kind == "avg":
                f = _AvgF64Final()
                for s, c in sts:
                    f.add_state(s, c)
                out[k][ai] = f.result()
            elif not sts:
                out[k][ai] = _evaluate(a, _partial_state(a, []))
            else:
                out[k][ai] = _evaluate(a, _merge_state(a, sts))
    return out


def aggregate(table, dts, key_cols, aggs):
    """Partial -> Final in one step: {key: [result per aggregate]} with AVG(f64) rounded once from the exact mean."""
    st = partial(table, dts, key_cols, aggs)
    res = final([(k, v) for k, v in st.items()], aggs, ungrouped=not key_cols)
    groups, gids, per_agg = _input_rows(table, dts, key_cols, aggs)
    for ai, a in enumerate(aggs):
        if a.kind == "avg" and a.dt.name != "DECIMAL":
            fs = {k: _AvgF64Final() for k in res}
            for g, v in zip(gids, per_agg[ai]):
                if v is not None:
                    fs[groups.keys[g]].add_value(v)
            for k in res:
                res[k][ai] = fs[k].result()
    return res


# ---- state batches ----------------------------------------------------------------------------------------------------------------
def state_rows_of(table, n_keys, aggs, dts):
    """A state batch (library output or `state_batch`) -> [(key, [state per aggregate])...]."""
    cols = [pyvalues(table.column(i), dts[i]) for i in range(table.num_columns)]
    out = []
    for r in range(table.num_rows):
        key = tuple(cols[k][r] for k in range(n_keys))
        at, st = n_keys, []
        for a in aggs:
            w = len(a.state_types())
            st.append(tuple(cols[at + j][r] for j in range(w)))
            at += w
        out.append((key, st))
    return out


_GARBAGE = {"DOUBLE": [math.nan, -math.inf, 1e300, f64_of_bits(0xFFF0000000000ABC)], "INT64": [I64_MIN, -1, 0x5A5A5A5A5A5A5A5A],
            "BOOL": [True, False]}


def arrow_column(vals, dt, garbage_seed=None):
    """Python values -> an Arrow array of `dt`.  With `garbage_seed`, every NULL slot holds nonzero bytes (NaN, +-Inf, large
    integers): Arrow leaves NULL slots unspecified, so a consumer that reads them is wrong."""
    n = len(vals)
    valid = [v is not None for v in vals]
    if dt.name in ("DECIMAL", "DOUBLE", "INT64", "INT32", "INT16", "INT8", "DATE", "TIMESTAMP") and garbage_seed is not None and not all(valid):
        rng = np.random.default_rng(garbage_seed)
        if dt.name == "DECIMAL":
            raw = O.dec_from_ints([v if v is not None else int(rng.integers(1, 1 << 62)) * (1 << 64) + 7 for v in vals])
            data = raw.tobytes()
        elif dt.name == "DOUBLE":
            g = _GARBAGE["DOUBLE"]
            data = np.array([v if v is not None else g[i % len(g)] for i, v in enumerate(vals)], dtype=np.float64).tobytes()
        else:
            np_t = {"INT64": np.int64, "TIMESTAMP": np.int64, "INT32": np.int32, "DATE": np.int32, "INT16": np.int16, "INT8": np.int8}[dt.name]
            fill = {np.int64: 0x5A5A5A5A5A5A5A5A, np.int32: 0x5A5A5A5A, np.int16: 0x5A5A, np.int8: 0x5A}[np_t]
            data = np.array([v if v is not None else fill for v in vals], dtype=np_t).tobytes()
        bitmap = np.packbits(np.array(valid, dtype=np.uint8), bitorder="little").tobytes()
        return pa.Array.from_buffers(arrow_type(dt), n, [pa.py_buffer(bitmap), pa.py_buffer(data)], null_count=n - sum(valid))
    if dt.name == "DECIMAL":
        import decimal
        ctx = decimal.Context(prec=60)
        return pa.array([None if v is None else decimal.Decimal(v).scaleb(-dt.scale, context=ctx) for v in vals], type=arrow_type(dt))
    if dt.name == "DOUBLE":
        data = np.array([0.0 if v is None else v for v in vals], dtype=np.float64)
        return pa.array(data, mask=np.array([not x for x in valid]) if not all(valid) else None)
    if dt.name in ("DATE", "TIMESTAMP"):
        base = pa.array(vals, type=pa.int32() if dt.name == "DATE" else pa.int64())
        return base.view(arrow_type(dt))
    return pa.array(vals, type=arrow_type(dt))


def arrow_type(dt):
    return {"BOOL": pa.bool_(), "INT8": pa.int8(), "INT16": pa.int16(), "INT32": pa.int32(), "INT64": pa.int64(), "DOUBLE": pa.float64(),
            "STRING": pa.string(), "DATE": pa.date32(), "TIMESTAMP": pa.timestamp("us", tz="UTC")}.get(dt.name) or pa.decimal128(dt.precision, dt.scale)


def state_batch(state_rows, key_types, aggs, garbage_seed=None):
    """[(key, [state per aggregate])...] -> a state RecordBatch in the layout a Final aggregate reads."""
    types = state_schema(key_types, aggs)
    cols = [[] for _ in types]
    for key, st in state_rows:
        vals = list(key) + [x for s in st for x in s]
        for c, v in zip(cols, vals):
            c.append(v)
    arrays = [arrow_column(c, t, garbage_seed) for c, t in zip(cols, types)]
    return pa.RecordBatch.from_arrays(arrays, names=[f"s{i}" for i in range(len(arrays))])
