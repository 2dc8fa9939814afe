"""GPU parity of the expression layer (csrc/codegen.cpp) against the interpreter of tests/exprs.py, for every column type, source
layout and evaluation mode the code generator handles:

  - a wide table: every integer width at MIN / MAX / -1 / 0, Float32 and Float64 NaNs (quiet, signalling, payloads, both signs),
    +-Inf, +-0.0, subnormals, FLT_MAX and integers above 2^24, timestamps at the i64 edges, booleans, dates and decimals stored in
    4, 8 and 16 bytes at +-(10^p - 1) and at HALF_UP ties -- all with NULLs;
  - four sources of that table: an Arrow stream sliced at offset 3 (validity and boolean bitmaps that start mid-byte), a device table
    with 8-byte decimals, and Parquet with decimals stored as INT32 / INT64 or as FLBA (Parquet has no boolean column here);
  - hand-written expression lists (Float32 arithmetic, comparisons and IN; integer arithmetic in LEGACY / TRY / ANSI; every accepted
    cast; narrow-decimal arithmetic) and a few hundred seeded random expression trees;
  - ANSI errors inside grouped aggregates with the key-table and the stream strategies.

Every output is compared bit for bit (floats by their bits, NaN payloads included) with its validity.  A plan must raise exactly
when the interpreter raises, with an error class the interpreter raised.  tests/test_expr_matrix_cpu.py compiles every plan built
here on a machine without a GPU."""
import numpy as np
import pyarrow as pa
import pytest

import exprs as E
from comet_b200 import proto as P
from oracle import oracle as O
from sources import device_table, scan_of, write_parquet

pytestmark = pytest.mark.gpu

I8, I16, I32, I64, F32, F64, TS, BOOL, DATE = P.INT8, P.INT16, P.INT32, P.INT64, P.FLOAT, P.DOUBLE, P.TIMESTAMP, P.BOOL, P.DATE
D9, D18, D18S, D38 = P.DECIMAL(9, 2), P.DECIMAL(18, 0), P.DECIMAL(18, 1), P.DECIMAL(38, 4)
INT_BITS = {"INT8": 8, "INT16": 16, "INT32": 32, "INT64": 64}

N = 6000
OFFSET = 3            # the Arrow source is sliced here: its bitmaps start mid-byte
BATCH = 1000
CHUNK = 2500          # not a multiple of BATCH
SOURCES = ["arrow", "device", "parquet-int", "parquet-flba"]

F32_SPECIAL = np.array([0x7FC00000, 0xFFC00000, 0x7FC0BEEF, 0x7F800001, 0xFFA00123, 0x7F800000, 0xFF800000, 0x00000000, 0x80000000,
                        0x00000001, 0x807FFFFF, 0x7F7FFFFF, 0xFF7FFFFF, 0x4B800001, 0x4C000003, 0xCB7FFFFF, 0x3F800000],
                       dtype=np.uint32).view(np.float32)  # NaNs, +-Inf, +-0, subnormals, +-FLT_MAX, 2^24 + 2, 2^25 + 12, -(2^24 - 1), 1
F64_SPECIAL = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF8DEADBEEF0001, 0x7FF0000000000001, 0x7FF0000000000000,
                        0xFFF0000000000000, 0, 0x8000000000000000, 1, 0x800FFFFFFFFFFFFF, 0x7FEFFFFFFFFFFFFF], dtype=np.uint64).view(np.float64)
DEC_TIES = [5, -5, 15, -15, 25, -25, 149, -150, 250, -250]   # HALF_UP ties one and two digits down, both signs

# name -> type, in column order
COLUMNS = {"i8": I8, "i16": I16, "i32": I32, "i64": I64, "f32": F32, "g32": F32, "f64": F64, "g64": F64, "ts": TS, "date": DATE,
           "d9": D9, "d18": D18, "d18s": D18S, "d38": D38, "b": BOOL}


def _specials(rng, n, base, specials, start=OFFSET):
    """base with the specials from row `start` on (the first rows of the sliced table) and again at random rows"""
    v = np.array(base)
    v[start:start + len(specials)] = specials
    v[rng.choice(np.arange(start + len(specials), n), len(specials), replace=False)] = specials
    return v


def _int_values(rng, n, bits):
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    dt = {8: np.int8, 16: np.int16, 32: np.int32, 64: np.int64}[bits]
    small = rng.integers(-100, 100, n)                       # a third of the rows small: arithmetic that does not overflow
    big = rng.integers(lo, hi, n, endpoint=True, dtype=np.int64)
    base = np.where(rng.random(n) < 0.33, small, big).astype(dt)
    return _specials(rng, n, base, np.array([lo, hi, -1, 0, 1, lo + 1, hi - 1, 2], dtype=dt))


def _dec_values(rng, n, p):
    m = 10 ** p - 1
    if p <= 18:
        base = np.where(rng.random(n) < 0.5, rng.integers(-m, m, n, endpoint=True), rng.integers(-1000, 1000, n))
        return [int(x) for x in _specials(rng, n, base, np.array([m, -m, 0, -1, 1] + DEC_TIES, dtype=np.int64))]
    vals = [int(a) * 10 ** 20 + int(b) for a, b in zip(rng.integers(-10 ** 18, 10 ** 18, n), rng.integers(0, 10 ** 18, n))]
    vals[OFFSET:OFFSET + 5 + len(DEC_TIES)] = [m, -m, 0, -1, 1] + DEC_TIES
    return vals


def _dec_array(vals, p, s, mask):
    words = O.dec_from_ints(vals)
    validity = pa.py_buffer(np.packbits(~mask, bitorder="little"))
    return pa.Array.from_buffers(pa.decimal128(p, s), len(vals), [validity, pa.py_buffer(words.tobytes())], null_count=int(mask.sum()))


def make_table(seed=0):
    """-> (pyarrow table of COLUMNS sliced at OFFSET, interpreter columns {name: (values, valid)})"""
    rng = np.random.default_rng(seed)
    n = N + OFFSET
    mask = lambda: rng.random(n) < 0.1
    arrays, cols = {}, {}
    for name, dt in COLUMNS.items():
        m = mask()
        m[OFFSET:OFFSET + 3] = False                          # the leading specials are valid in the sliced table too
        if dt.name in INT_BITS:
            v = _int_values(rng, n, INT_BITS[dt.name])
            arrays[name], cols[name] = pa.array(v, mask=m), (v.astype(np.int64), ~m)
        elif dt.name == "FLOAT":
            v = _specials(rng, n, (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 6, n)).astype(np.float32), np.roll(F32_SPECIAL, 3 * (name == "g32")))
            arrays[name], cols[name] = pa.array(v, mask=m), (v, ~m)
        elif dt.name == "DOUBLE":
            v = _specials(rng, n, rng.standard_normal(n) * 10.0 ** rng.integers(-3, 6, n), np.roll(F64_SPECIAL, 4 * (name == "g64")))
            arrays[name], cols[name] = pa.array(v, mask=m), (v, ~m)
        elif dt.name == "TIMESTAMP":
            v = _int_values(rng, n, 64)
            arrays[name], cols[name] = pa.array(v, type=pa.timestamp("us"), mask=m), (v.astype(np.int64), ~m)
        elif dt.name == "DATE":
            v = rng.integers(-30000, 30000, n).astype(np.int32)
            arrays[name], cols[name] = pa.array(v, type=pa.date32(), mask=m), (v.astype(np.int64), ~m)
        elif dt.name == "BOOL":
            v = rng.random(n) < 0.5
            arrays[name], cols[name] = pa.array(v, mask=m), (v, ~m)
        else:
            v = _dec_values(rng, n, dt.precision)
            arrays[name], cols[name] = _dec_array(v, dt.precision, dt.scale, m), (O.dec_from_ints(v), ~m)
    tbl = pa.table(arrays).slice(OFFSET)
    cols = {k: (np.asarray(v)[OFFSET:], np.asarray(ok)[OFFSET:]) for k, (v, ok) in cols.items()}
    return tbl, cols


def source_names(source):
    return [k for k in COLUMNS if not (source.startswith("parquet") and k == "b")]


class Cols:
    """Column references of one source's column order: cols.f32 -> E.Col(index of f32, FLOAT)"""

    def __init__(self, names):
        self.names = names

    def __getattr__(self, name):
        if name not in self.names:
            raise KeyError(name)
        return E.Col(self.names.index(name), COLUMNS[name])


def L(v, dt):
    return E.Lit(v, dt)


# ---- sources ------------------------------------------------------------------------------------------------------------------------
_TABLES = {}


def table(seed=0):
    if seed not in _TABLES:
        _TABLES[seed] = make_table(seed)
    return _TABLES[seed]


def source_input(cb, source, tmp_path, seed=0):
    """-> (scan node, inputs, column names) of one source of the table"""
    tbl, _ = table(seed)
    names = source_names(source)
    types = [COLUMNS[k] for k in names]
    if source == "arrow":
        return P.scan(types), [tbl.to_batches(max_chunksize=BATCH)], names
    if source == "device":
        return P.scan(types), [device_table(cb, tbl, types, dec8=("d9", "d18", "d18s"))], names
    path = str(tmp_path / f"{source}-{seed}.parquet")
    cols = {k: (tbl.column(k).combine_chunks(), COLUMNS[k]) for k in names}
    write_parquet(path, cols, source == "parquet-int")
    scan, _ = scan_of(cb, cols, names, path)
    return scan, [], names


def plan_of(scan, pred, outs):
    node = scan if pred is None else P.filter_(scan, pred.proto())
    return P.projection(node, [o.proto() for o in outs])


def run(cb, node, inputs):
    with cb.native.Plan(node, inputs, config={"spark.comet.b200.chunkRows": str(CHUNK)}) as p:
        return p.collect()


def interp(pred, outs, cols_by_name, names):
    """the interpreter's (kept-row count, [(values, valid)] or the AnsiError of each output)"""
    cols = [cols_by_name[k] for k in names]
    keep = np.ones(N, dtype=bool)
    if pred is not None:
        pv, pvalid = pred.eval(cols)
        keep = np.asarray(pv, dtype=bool) & np.asarray(pvalid, dtype=bool)
    kept = [(np.asarray(v)[keep], np.asarray(ok)[keep]) for v, ok in cols]
    res = []
    for o in outs:
        try:
            res.append(o.eval(kept))
        except E.AnsiError as ex:
            res.append(ex)
    return int(keep.sum()), res


def column_values(col, dt):
    """one result column -> (values as the interpreter holds them, valid)"""
    col = col.combine_chunks() if isinstance(col, pa.ChunkedArray) else col
    n, off = len(col), col.offset
    valid = np.asarray(col.is_valid()) if col.null_count else np.ones(n, dtype=bool)
    if dt.name == "BOOL":
        return np.asarray(col.fill_null(False)), valid
    if dt.name == "DECIMAL":
        return np.frombuffer(col.buffers()[1], dtype=np.uint64)[2 * off:2 * (off + n)].reshape(-1, 2), valid
    np_dt = {"FLOAT": np.float32, "DOUBLE": np.float64, "INT8": np.int8, "INT16": np.int16, "INT32": np.int32, "DATE": np.int32,
             "INT64": np.int64, "TIMESTAMP": np.int64}[dt.name]
    return np.frombuffer(col.buffers()[1], dtype=np_dt)[off:off + n], valid


def assert_output(j, got_col, want, dt, what=""):
    v, valid = want
    valid = np.asarray(valid, dtype=bool)
    g, gvalid = column_values(got_col, dt)
    bad = np.nonzero(gvalid != valid)[0]
    assert bad.size == 0, f"{what} output {j}: validity differs at {bad.size} rows, first row {bad[0]} got {gvalid[bad[0]]}"
    if dt.name == "DECIMAL":
        gv, ev = g[valid], np.asarray(v)[valid]
        bad = np.nonzero((gv != ev).any(axis=1))[0]
        assert bad.size == 0, f"{what} output {j}: {bad.size} rows differ, first got {O.dec_to_ints(gv[bad[:1]])} want {O.dec_to_ints(ev[bad[:1]])}"
    elif dt.name in ("FLOAT", "DOUBLE"):
        w = np.uint32 if dt.name == "FLOAT" else np.uint64
        gb = np.ascontiguousarray(g[valid]).view(w)
        eb = np.ascontiguousarray(np.asarray(v, dtype=np.float32 if dt.name == "FLOAT" else np.float64)[valid]).view(w)
        bad = np.nonzero(gb != eb)[0]
        assert bad.size == 0, f"{what} output {j}: {bad.size} rows differ, first got {gb[bad[0]]:#x} want {eb[bad[0]]:#x}"
    else:
        gv, ev = g[valid].astype(np.int64), np.asarray(v)[valid].astype(np.int64)
        bad = np.nonzero(gv != ev)[0]
        assert bad.size == 0, f"{what} output {j}: {bad.size} rows differ, first got {gv[bad[0]]} want {ev[bad[0]]}"


MAX_OUTPUTS = 12


def groups(outs):
    return [outs[i:i + MAX_OUTPUTS] for i in range(0, len(outs), MAX_OUTPUTS)]


def check(cb, source, tmp_path, build, pred=None, seed=0, what=""):
    """build(Cols) -> outputs (or (predicate, outputs)); runs them over one source and compares with the interpreter"""
    scan, inputs, names = source_input(cb, source, tmp_path, seed)
    c = Cols(names)
    outs = build(c)
    if isinstance(outs, tuple):
        pred, outs = outs
    if len(outs) > MAX_OUTPUTS:                               # a fused projection emits at most 16 columns
        return [check(cb, source, tmp_path, lambda c, g=g: (pred, g), seed=seed, what=what) for g in groups(outs)][-1]
    n_keep, want = interp(pred, outs, table(seed)[1], names)
    errors = [w for w in want if isinstance(w, E.AnsiError)]
    node = plan_of(scan, pred, outs)
    if errors:
        with pytest.raises(cb.native.CometB200Error) as ei:
            run(cb, node, inputs)
        classes = set().union(*(e.classes for e in errors))
        assert ei.value.error_class in classes, f"{what}: device raised {ei.value.error_class!r}, the interpreter {classes}"
        return ei.value.error_class
    res = run(cb, node, inputs)
    assert (res.num_rows if res is not None else 0) == n_keep, what
    for j, (o, w) in enumerate(zip(outs, want)):
        assert_output(j, res.column(j), w, o.dt, what)
    return None


# ---- expression lists -----------------------------------------------------------------------------------------------------------------
NAN, INF = float("nan"), float("inf")


def f32_arith(c, mode=E.LEGACY):
    f, g = c.f32, c.g32
    out = [E.Arith(op, f, g, F32, mode) for op in ("add", "subtract", "multiply", "divide")]
    out += [E.Arith("add", f, L(NAN, F32), F32, mode), E.Arith("multiply", f, L(INF, F32), F32, mode), E.Arith("subtract", f, f, F32, mode),
            E.Arith("divide", g, L(0.0, F32), F32, mode), E.Arith("multiply", f, L(-0.0, F32), F32, mode), E.Neg(f), E.Neg(E.Arith("add", g, f, F32, mode)),
            E.Arith("add", E.Arith("multiply", f, f, F32, mode), L(3.0e38, F32), F32, mode)]
    return out


def f32_compare(c):
    f, g = c.f32, c.g32
    out = [E.Cmp(op, f, L(NAN, F32)) for op in ("eq", "neq", "lt", "lt_eq", "gt", "gt_eq")]
    out += [E.Cmp(op, f, L(-0.0, F32)) for op in ("eq", "lt", "gt_eq")] + [E.Cmp("eq", f, L(0.0, F32)), E.Cmp("lt", f, g), E.Cmp("eq", f, g),
                                                                          E.Cmp("gt", f, L(-NAN, F32)), E.Cmp("lt", L(-NAN, F32), f)]
    return out


def in_lists(c, dt):
    f = c.f32 if dt is F32 else c.f64
    return [E.In(f, [L(NAN, dt)]), E.In(f, [L(-0.0, dt)]), E.In(f, [L(0.0, dt), L(None, dt)]), E.In(f, [L(NAN, dt), L(-0.0, dt)], negated=True),
            E.In(f, [L(-NAN, dt), L(INF, dt)]), E.In(f, [L(1.0, dt), L(None, dt)], negated=True), E.In(f, [L(None, dt)]),
            E.In(f, [L(-INF, dt), L(0.0, dt), L(1.0, dt)])]


def int_cols(c):
    return [(c.i8, I8), (c.i16, I16), (c.i32, I32), (c.i64, I64)]


def int_arith(c, mode):
    out = []
    for x, dt in int_cols(c):
        w = INT_BITS[dt.name]
        mx = (1 << (w - 1)) - 1
        out += [E.Arith("add", x, x, dt, mode), E.Arith("subtract", x, L(mx, dt), dt, mode), E.Arith("multiply", x, x, dt, mode), E.Neg(x)]
        if mode != E.LEGACY:
            out += [E.Arith("divide", x, L(-1, dt), dt, mode), E.Arith("divide", L(7, dt), x, dt, mode)]
    return out


def widening_casts(c, mode=E.LEGACY):
    out = []
    ints = int_cols(c)
    for i, (x, dt) in enumerate(ints):
        out += [E.Cast(x, t, mode) for _, t in ints[i + 1:]] + [E.Cast(x, F32, mode), E.Cast(x, F64, mode)]
    return out + [E.Cast(c.f32, F64, mode), E.Cast(c.g32, F64, mode)]


def decimal_casts(c, mode=E.LEGACY):
    return [E.Cast(c.i8, P.DECIMAL(3, 0), mode), E.Cast(c.i8, P.DECIMAL(3, 1), mode), E.Cast(c.i16, P.DECIMAL(5, 0), mode), E.Cast(c.i16, P.DECIMAL(6, 2), mode),
            E.Cast(c.i32, P.DECIMAL(10, 0), mode), E.Cast(c.i32, P.DECIMAL(9, 0), mode), E.Cast(c.i64, P.DECIMAL(19, 0), mode), E.Cast(c.i64, P.DECIMAL(18, 0), mode),
            E.Cast(c.i64, P.DECIMAL(38, 18), mode), E.Cast(c.d18s, D18, mode), E.Cast(c.d9, P.DECIMAL(8, 1), mode), E.Cast(c.d9, P.DECIMAL(7, 0), mode),
            E.Cast(c.d18, P.DECIMAL(20, 2), mode), E.Cast(c.d38, P.DECIMAL(38, 2), mode), E.Cast(c.d38, P.DECIMAL(20, 0), mode), E.Cast(c.d18, P.DECIMAL(17, 0), mode)]


def narrow_decimals(c):
    d9, d18, d18s = c.d9, c.d18, c.d18s
    return [E.Arith("add", d18, d18s, P.DECIMAL(20, 1)), E.Arith("subtract", d18s, d18, P.DECIMAL(20, 1)), E.Arith("add", d9, d9, P.DECIMAL(10, 2)),
            E.Arith("multiply", d9, d9, P.DECIMAL(19, 4)), E.Arith("multiply", d18, d9, P.DECIMAL(28, 2)), E.Arith("subtract", d9, d18, P.DECIMAL(21, 2)),
            E.CheckOverflow(E.Arith("add", d9, d9, P.DECIMAL(10, 2)), P.DECIMAL(10, 2)), E.CheckOverflow(E.Arith("add", d9, d9, P.DECIMAL(10, 2)), P.DECIMAL(9, 2)),
            E.CheckOverflow(E.Cast(d18s, D18), D18), E.Neg(d18), E.Neg(d9),
            E.Cmp("lt", d18, E.Neg(d18)), E.Cmp("eq", d9, L(-5, D9)), E.In(d18, [L(10 ** 18 - 1, D18), L(-1, D18), L(None, D18)]),
            E.In(d9, [L(5, D9), L(-(10 ** 9 - 1), D9)], negated=True), E.Cmp("gt_eq", c.d38, L(-5, D38))]


def temporal_and_bool(c):
    ts, b, d = c.ts, c.b, c.date
    mn, mx = -(1 << 63), (1 << 63) - 1
    return [ts, b, E.Cmp("eq", ts, L(mn, TS)), E.Cmp("lt", ts, L(mx, TS)), E.In(ts, [L(mn, TS), L(mx, TS), L(None, TS)]), E.If(b, ts, L(mx, TS)),
            E.Not(b), E.Logic("and", b, E.Cmp("gt", d, L(0, DATE))), E.Logic("or", E.Not(b), E.IsNull(ts)), E.If(b, c.f32, E.Neg(c.f32)),
            E.CaseWhen([b, E.Cmp("lt", ts, L(0, TS))], [c.i16, E.Neg(c.i16)]), E.IsNull(b, negate=True), E.Cast(b, BOOL), E.Cast(ts, TS)]


LISTS = {
    "f32-legacy": lambda c: f32_arith(c),
    "f32-try": lambda c: f32_arith(c, E.TRY),
    "f32-compare": f32_compare,
    "f32-in": lambda c: in_lists(c, F32),
    "f64-in": lambda c: in_lists(c, F64),
    "int-legacy": lambda c: int_arith(c, E.LEGACY),
    "int-try": lambda c: int_arith(c, E.TRY),
    "casts-widening": widening_casts,
    "casts-decimal": decimal_casts,
    "narrow-decimals": narrow_decimals,
    "temporal-bool": temporal_and_bool,
}


def lists_for(source):
    return [k for k in LISTS if not (source.startswith("parquet") and k == "temporal-bool")]


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


@pytest.mark.parametrize("source", SOURCES)
def test_expression_lists(cb, tmp_path, source):
    """every hand-written list over one source, without and with a filter in front"""
    for name in lists_for(source):
        check(cb, source, tmp_path, LISTS[name], what=f"{source} {name}")
    pred = lambda c: E.Logic("or", E.Cmp("lt", c.f32, L(0.5, F32)), E.IsNull(c.i32))
    for name in ("f32-legacy", "int-try", "narrow-decimals"):
        check(cb, source, tmp_path, lambda c, n=name: (pred(c), LISTS[n](c)), what=f"{source} {name} filtered")


def test_float32_in_compares_bits(cb, tmp_path):
    """x IN (NaN) is TRUE for the NaN with those bits, 0.0 IN (-0.0) is FALSE: totalOrder equality, as comparisons and Float64 IN"""
    tbl, cols = table()
    f = cols["f32"][0].view(np.uint32)
    assert (f == 0x7FC00000).any() and (f == 0).any() and (f == 0x80000000).any()
    check(cb, "arrow", tmp_path, lambda c: [E.In(c.f32, [L(NAN, F32)]), E.In(c.f32, [L(-0.0, F32)]), E.In(c.f32, [L(0.0, F32)])])


@pytest.mark.parametrize("dt", ["INT8", "INT16", "INT32", "INT64"])
def test_integer_ansi_errors(cb, tmp_path, dt):
    """ANSI add / sub / mul / neg overflow and division by zero raise their error class; the same expressions under a filter that keeps
    only safe rows do not raise and match the interpreter"""
    name = {"INT8": "i8", "INT16": "i16", "INT32": "i32", "INT64": "i64"}[dt]
    t = getattr(P, dt)
    mx = (1 << (INT_BITS[dt] - 1)) - 1
    cases = [(lambda x: E.Arith("add", x, x, t, E.ANSI), E.OVERFLOW), (lambda x: E.Arith("subtract", x, L(mx, t), t, E.ANSI), E.OVERFLOW),
             (lambda x: E.Arith("multiply", x, x, t, E.ANSI), E.OVERFLOW), (lambda x: E.Neg(x, fail=True), E.OVERFLOW),
             (lambda x: E.Arith("divide", L(7, t), x, t, E.ANSI), E.DIVIDE_BY_ZERO), (lambda x: E.Arith("divide", x, L(-1, t), t, E.ANSI), E.OVERFLOW)]
    for k, (mk, cls) in enumerate(cases):
        got = check(cb, "arrow", tmp_path, lambda c: [mk(getattr(c, name))], what=f"{dt} ANSI case {k}")
        assert got == cls, (dt, k, got)
    safe = lambda c: E.Logic("and", E.Cmp("gt", getattr(c, name), L(0, t)), E.Cmp("lt", getattr(c, name), L(8, t)))
    assert check(cb, "arrow", tmp_path, lambda c: (safe(c), [mk(getattr(c, name)) for mk, _ in cases])) is None


def test_ansi_casts_and_float_division(cb, tmp_path):
    """ANSI int -> decimal and decimal -> decimal casts raise only when a value leaves the precision; ANSI float division by zero"""
    assert check(cb, "device", tmp_path, lambda c: decimal_casts(c, E.ANSI)[:1] + [E.Cast(c.i64, P.DECIMAL(19, 0), E.ANSI),
                                                                                   E.Cast(c.d18s, P.DECIMAL(19, 1), E.ANSI)]) is None
    for k, mk in enumerate([lambda c: E.Cast(c.i8, P.DECIMAL(3, 1), E.ANSI), lambda c: E.Cast(c.d9, P.DECIMAL(7, 0), E.ANSI),
                            lambda c: E.Cast(c.i64, P.DECIMAL(18, 0), E.ANSI), lambda c: E.Cast(c.d38, P.DECIMAL(20, 0), E.ANSI)]):
        assert check(cb, "parquet-int", tmp_path, lambda c: [mk(c)], what=f"ansi cast {k}") == E.OVERFLOW
    assert check(cb, "arrow", tmp_path, lambda c: [E.Arith("divide", c.f32, c.g32, F32, E.ANSI)]) == E.DIVIDE_BY_ZERO
    assert check(cb, "arrow", tmp_path, lambda c: [E.Arith("divide", c.f32, L(-2.0, F32), F32, E.ANSI), E.Arith("divide", c.f64, L(0.5, F64), F64, E.ANSI)]) is None


def test_int64_add_at_the_edge_of_the_64_bit_form(cb, tmp_path):
    """decimal(18,0) + decimal(18,1) stored as Parquet INT64: +-(10^18 - 1) on both sides needs more than 64 bits after the rescale"""
    tbl, cols = table()
    d18, d18s = O.dec_to_ints(cols["d18"][0][:1]), O.dec_to_ints(cols["d18s"][0][:1])
    assert d18 == d18s == [10 ** 18 - 1]
    check(cb, "parquet-int", tmp_path, lambda c: [E.Arith("add", c.d18, c.d18s, P.DECIMAL(20, 1)), E.Arith("subtract", E.Neg(c.d18s), c.d18, P.DECIMAL(20, 1))])


# ---- random expression trees ----------------------------------------------------------------------------------------------------------
class Gen:
    """A seeded, type-correct generator of exprs.py trees of depth <= 4.  family: None (no ANSI), "overflow" (ANSI arithmetic,
    negation and casts) or "divide" (ANSI division only), so a raising plan fails for one kind of reason."""
    NUM = [I8, I16, I32, I64, F32, F64]
    DEC = [D9, D18, D18S]

    def __init__(self, rng, names, family=None):
        self.rng, self.c, self.family = rng, Cols(names), family
        self.names = names

    def pick(self, xs):
        return xs[int(self.rng.integers(0, len(xs)))]

    def mode(self, kind):
        m = self.pick([E.LEGACY, E.TRY, E.TRY])
        if self.family == kind and self.rng.random() < 0.6:
            m = E.ANSI
        return m

    def col_of(self, dt):
        return [k for k in self.names if COLUMNS[k] == dt]

    def lit(self, dt):
        if self.rng.random() < 0.1:
            return L(None, dt)
        if dt.name in INT_BITS:
            w = INT_BITS[dt.name]
            return L(int(self.pick([-(1 << (w - 1)), (1 << (w - 1)) - 1, -1, 0, 1, 2, 7, -3])), dt)
        if dt.name in ("FLOAT", "DOUBLE"):
            return L(self.pick([NAN, -NAN, INF, -INF, 0.0, -0.0, 1.5, -2.0, 3.0e38 if dt is F32 else 1e308]), dt)
        if dt.name == "DECIMAL":
            m = 10 ** dt.precision - 1
            return L(self.pick([m, -m, 0, -5, 5, 12345]), dt)
        if dt.name == "TIMESTAMP":
            return L(self.pick([-(1 << 63), (1 << 63) - 1, 0]), dt)
        if dt.name == "DATE":
            return L(int(self.rng.integers(-30000, 30000)), dt)
        return L(bool(self.rng.integers(0, 2)), dt)

    def leaf(self, dt):
        cs = self.col_of(dt)
        if cs and self.rng.random() < 0.75:
            return getattr(self.c, self.pick(cs))
        return self.lit(dt)

    def gen(self, dt, depth):
        if depth <= 1 or self.rng.random() < 0.2:
            return self.leaf(dt)
        d = depth - 1
        r = self.rng.random()
        if dt.name == "BOOL":
            if r < 0.4:
                t = self.pick(self.NUM + self.DEC + [TS, DATE])
                return E.Cmp(self.pick(["eq", "neq", "lt", "lt_eq", "gt", "gt_eq"]), self.gen(t, d), self.gen(t, d))
            if r < 0.6:
                return E.Logic(self.pick(["and", "or"]), self.gen(BOOL, d), self.gen(BOOL, d))
            if r < 0.7:
                return E.Not(self.gen(BOOL, d))
            if r < 0.8:
                return E.IsNull(self.gen(self.pick(self.NUM + self.DEC), d), negate=bool(self.rng.integers(0, 2)))
            if r < 0.9:
                t = self.pick(self.NUM + [D9, D18, TS])
                return E.In(self.gen(t, d), [self.lit(t) for _ in range(int(self.rng.integers(1, 4)))], negated=bool(self.rng.integers(0, 2)))
            return E.If(self.gen(BOOL, d), self.gen(BOOL, d), self.gen(BOOL, d))
        if dt.name in ("TIMESTAMP", "DATE"):
            return E.If(self.gen(BOOL, d), self.gen(dt, d), self.gen(dt, d)) if r < 0.5 else self.leaf(dt)
        if dt.name == "DECIMAL":
            if r < 0.25:
                return E.Neg(self.gen(dt, d))
            if r < 0.45:
                return E.If(self.gen(BOOL, d), self.gen(dt, d), self.gen(dt, d))
            if r < 0.65:
                src = self.pick([x for x in self.DEC if x != dt] + [D38])
                return E.Cast(self.gen(src, d), dt, self.mode("overflow"))
            if r < 0.8:
                src = self.pick([I8, I16, I32, I64])
                return E.Cast(self.gen(src, d), dt, self.mode("overflow"))
            a, b = self.gen(self.pick(self.DEC), d), self.gen(self.pick(self.DEC), d)
            op = self.pick(["add", "subtract", "multiply"])
            ar = E.Arith(op, a, b, P.DECIMAL(38, 0))
            return E.Cast(ar, dt, self.mode("overflow"))
        # integers and floats
        if r < 0.45:
            op = self.pick(["add", "subtract", "multiply", "divide"])
            mode = self.mode("divide" if op == "divide" else "overflow")
            if op == "divide" and mode == E.LEGACY and dt.name in INT_BITS:
                mode = E.TRY                                  # Legacy integer division by zero fails the query with an Arrow error
            if dt.name in ("FLOAT", "DOUBLE") and op != "divide" and mode == E.ANSI:
                mode = E.LEGACY
            return E.Arith(op, self.gen(dt, d), self.gen(dt, d), dt, mode)
        if r < 0.6:
            return E.Neg(self.gen(dt, d), fail=dt.name in INT_BITS and self.family == "overflow" and self.rng.random() < 0.3)
        if r < 0.8:
            return E.If(self.gen(BOOL, d), self.gen(dt, d), self.gen(dt, d))
        narrower = {"INT16": [I8], "INT32": [I8, I16], "INT64": [I8, I16, I32], "FLOAT": [I8, I16, I32, I64], "DOUBLE": [I8, I16, I32, I64, F32]}.get(dt.name)
        if narrower:
            return E.Cast(self.gen(self.pick(narrower), d), dt)
        return self.leaf(dt)


FUZZ_PLANS = 24          # x 12 outputs = 288 trees
FUZZ_OUTPUTS = 12


def fuzz_plan(k, names):
    """-> (predicate or None, outputs) of random plan k: a third of the plans may hold ANSI expressions, half have a filter"""
    rng = np.random.default_rng(1000 + k)
    family = [None, None, "overflow", None, "divide", None][k % 6]
    g = Gen(rng, names, family)
    pg = Gen(rng, names)
    pred = E.Logic(pg.pick(["and", "or"]), pg.gen(BOOL, 4), E.IsNull(getattr(pg.c, pg.pick(names)))) if k % 2 else None   # reads a column
    types = Gen.NUM + Gen.DEC + [BOOL, TS, DATE]
    n_out = FUZZ_OUTPUTS if family is None else 4
    outs = [getattr(g.c, g.pick(names))] + [g.gen(g.pick(types), 4) for _ in range(n_out - 1)]   # one column: a plan always reads input
    if family is not None:                                                                       # and an ANSI node at the root
        t = g.pick([I8, I16, I32, I64])
        outs[1] = E.Arith("divide" if family == "divide" else g.pick(["add", "subtract", "multiply"]), g.gen(t, 3), g.gen(t, 3), t, E.ANSI)
    return pred, outs


def fuzz_source(k):
    return ["arrow", "device", "parquet-int", "parquet-flba"][k % 4]


@pytest.mark.parametrize("k", range(FUZZ_PLANS))
def test_random_expression_trees(cb, tmp_path, k):
    source = fuzz_source(k)
    pred, outs = fuzz_plan(k, source_names(source))
    check(cb, source, tmp_path, lambda c: (pred, outs), what=f"fuzz plan {k} on {source}")


# ---- errors inside aggregate pipelines ------------------------------------------------------------------------------------------------
def agg_table(n=20000, seed=5):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 300, n)
    k = np.sort(k) if seed % 2 else k
    a = _int_values(rng, n, 32)
    z = rng.integers(0, 3, n).astype(np.int32)                    # zeros: an ANSI division by zero wherever it is evaluated
    f = _specials(rng, n, (rng.standard_normal(n) * 1e3).astype(np.float32), F32_SPECIAL[[2, 5, 7, 8, 9, 11, 13, 14, 16]], 0)
    m = rng.random(n) < 0.08
    return pa.table({"k": pa.array(k, pa.int64()), "a": pa.array(a, mask=m), "z": pa.array(z), "f": pa.array(f, mask=rng.random(n) < 0.08)})


AGG_TYPES = [I64, I32, I32, F32]


def agg_run(cb, aggs, cfg, tbl, stream, pred=None):
    """Partial (over a Filter when pred is given, fused into the aggregate pipeline) -> Final"""
    import aggref as R
    tbl = tbl.sort_by("k") if stream else tbl
    child = P.scan(AGG_TYPES) if pred is None else P.filter_(P.scan(AGG_TYPES), pred.proto())
    partial = P.hash_agg(child, [P.bound(0, I64)], [a.proto() for a in aggs], R.PARTIAL)
    with cb.native.Plan(partial, [tbl.to_batches(max_chunksize=4096)], config=cfg) as p:
        state = p.collect()
        bits = p.stats()["agg_strategies"]
    with cb.native.Plan(R.merge_plan([I64], aggs), [state]) as p:
        res = p.collect()
    return res, bits


def agg_result(res, aggs):
    import aggref as R
    cols = [R.pyvalues(res.column(i), t) for i, t in enumerate([I64] + [x.result_type() for x in aggs])]
    return {(r[0],): list(r[1:]) for r in zip(*cols)}


@pytest.mark.parametrize("strategy", ["table", "stream"])
def test_ansi_errors_in_aggregate_pipelines(cb, strategy):
    """Hash-aggregate pipelines evaluate every row slot, rows past the tile's end and rows the filter removes included: an ANSI error
    fires only for rows the Filter keeps and only in the IF branch a row takes"""
    import aggcases
    import aggref as R
    cfg = aggcases.STREAM_CFG if strategy == "stream" else aggcases.TABLE_CFG
    tbl = agg_table(seed=5 if strategy == "table" else 6)
    tbl = tbl.sort_by("k") if strategy == "stream" else tbl
    a, z = E.Col(1, I32), E.Col(2, I32)
    twice = E.Arith("add", a, a, I32, E.ANSI)
    safe = E.Logic("and", E.Cmp("gt", a, L(-1000, I32)), E.Cmp("lt", a, L(1000, I32)))
    div = E.If(E.Cmp("eq", z, L(0, I32)), L(0, I32), E.Arith("divide", a, z, I32, E.ANSI))
    aggs = [R.Agg("sum", twice, I64), R.Agg("count", twice), R.Agg("sum", div, I64), R.Agg("max", twice, I32)]
    res, bits = agg_run(cb, aggs, cfg, tbl, False, pred=safe)
    assert bits == aggcases.EXPECTED_BITS[strategy]
    sv, svalid = safe.eval(R.exprs_columns(tbl, AGG_TYPES))
    kept = tbl.filter(pa.array(np.asarray(sv, bool) & np.asarray(svalid, bool)))
    assert 0 < kept.num_rows < tbl.num_rows
    exp = R.aggregate(kept, AGG_TYPES, [0], aggs)
    assert agg_result(res, aggs) == {k: list(v) for k, v in exp.items()}
    with pytest.raises(cb.native.CometB200Error) as ei:                 # without the filter the doubled MIN / MAX overflow
        agg_run(cb, [R.Agg("sum", twice, I64)], cfg, tbl, False)
    assert ei.value.error_class == "ARITHMETIC_OVERFLOW"
    with pytest.raises(E.AnsiError):
        R.aggregate(tbl, AGG_TYPES, [0], [R.Agg("sum", twice, I64)])
    with pytest.raises(cb.native.CometB200Error) as ei:                 # the division taken on every row
        agg_run(cb, [R.Agg("sum", E.Arith("divide", a, z, I32, E.ANSI), I64)], cfg, tbl, False)
    assert ei.value.error_class == "DIVIDE_BY_ZERO"


@pytest.mark.parametrize("strategy", ["table", "stream"])
def test_float32_value_column_aggregates(cb, strategy):
    """SUM / AVG of a Float32 column into DOUBLE and MIN / MAX of it widened to DOUBLE, NaNs and infinities among the values"""
    import aggcases
    import aggref as R
    cfg = aggcases.STREAM_CFG if strategy == "stream" else aggcases.TABLE_CFG
    tbl = agg_table(seed=7 if strategy == "table" else 8)
    f = E.Col(3, F32)
    aggs = [R.Agg("sum", f, F64), R.Agg("avg", f, F64), R.Agg("min", E.Cast(f, F64), F64), R.Agg("max", E.Cast(f, F64), F64), R.Agg("count", f)]
    res, bits = agg_run(cb, aggs, cfg, tbl, strategy == "stream")
    assert bits == aggcases.EXPECTED_BITS[strategy]
    stbl = tbl.sort_by("k") if strategy == "stream" else tbl
    exp = R.aggregate(stbl, AGG_TYPES, [0], aggs)
    cols = [R.pyvalues(res.column(i), t) for i, t in enumerate([I64] + [x.result_type() for x in aggs])]
    got = {(r[0],): r[1:] for r in zip(*cols)}
    assert set(got) == set(exp)
    import math
    for key, e in exp.items():
        g = got[key]
        for i in (0, 1):                                          # double-double sums: within 1 (SUM) / 2 (AVG) ULP, non-finite by class
            if e[i] is None or not math.isfinite(e[i]):
                assert (g[i] is None and e[i] is None) or (math.isnan(g[i]) and math.isnan(e[i])) or g[i] == e[i], (key, i, g[i], e[i])
            else:
                assert abs(g[i] - e[i]) <= (i + 1) * math.ulp(e[i]), (key, i, g[i], e[i])
        for i in (2, 3, 4):
            assert R.f64_bits(g[i]) == R.f64_bits(e[i]) if isinstance(e[i], float) else g[i] == e[i], (key, i, g[i], e[i])
