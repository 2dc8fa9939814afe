"""High-cardinality cases of the hash aggregate (csrc/agg.cpp: key table growth, id ranges, reserved rows, stream state) and a
vectorised reference for them.  Used by tests/test_gpu_agg_scale.py (runs them) and tests/test_agg_scale_cpu.py (pins the reference
against tests/aggref.py on slices and compiles every plan).

tests/aggref.py works on Python ints and exact fractions: right, but too slow for 10^6 groups.  Here a column is a pair of numpy
arrays (values, validity), groups come from np.unique over the key columns (a NULL key value is its own value), and every aggregate
is a segmented reduction over the rows sorted by group.  Integer and decimal totals are exact int64 sums (the data keeps every
group's total far below 2^63); f64 sums are checked in every group against an error bound of the naive sum and, in a deterministic
sample of groups, within 1 ULP of the correctly rounded sum (math.fsum), the bound tests/test_gpu_agg_matrix.py uses.

Every case has the same value columns after its key columns, and the same aggregates over them (AGGS):
  v0 i64 (NULLs)   v1 decimal(12,2) (NULLs)   v2 f64 (NULLs, rare NaN / +-Inf)   v3 bool (the FILTER input, NULLs)"""
import math
from fractions import Fraction

import numpy as np
import pyarrow as pa

from comet_b200 import proto as P

import aggref as R
import exprs as E

I8, I32, I64, DBL, BOOL, DATE, STR = P.INT8, P.INT32, P.INT64, P.DOUBLE, P.BOOL, P.DATE, P.STRING
D12, D18, D22, D16_6 = P.DECIMAL(12, 2), P.DECIMAL(18, 0), P.DECIMAL(22, 2), P.DECIMAL(16, 6)
VALUE_TYPES = [I64, D12, DBL, BOOL]

STREAM_CFG = {"spark.comet.b200.streamAgg.minRows": "0"}
TABLE_CFG = {"spark.comet.b200.streamAgg.minRows": "-1"}

# per aggregate: (reduction, value column, filtered by v3)
KINDS = [("sum", 0, False), ("count", 0, False), ("min", 0, False), ("max", 0, False), ("sum_dec", 1, False), ("avg_dec", 1, False),
         ("min", 1, False), ("max", 1, False), ("sum_f64", 2, False), ("avg_f64", 2, False), ("count_star", None, False), ("sum", 0, True)]


# A merging (Final / PartialMerge) hash aggregate stages every state column of a chunk in shared memory, which holds about nine of
# them beside a 64-bit key: the twelve aggregates run as two plans over the same input (MERGE_SETS).  A Partial takes all twelve.
SETS = {"int-dec": [0, 1, 2, 3, 4, 5, 10], "dec-f64": [6, 7, 8, 9, 11], "all": list(range(12))}
MERGE_SETS = ["int-dec", "dec-f64"]


def aggs(nk, aggset=None):
    """SUM / COUNT / MIN / MAX of i64, SUM / AVG / MIN / MAX of decimal(12,2), SUM / AVG of f64, COUNT(*), SUM(i64) FILTER (v3);
    with `aggset`, the ones of SETS[aggset]."""
    full = _aggs(nk)
    return full if aggset is None else [full[i] for i in SETS[aggset]]


def _aggs(nk):
    i64, dec, f64, flag = E.Col(nk, I64), E.Col(nk + 1, D12), E.Col(nk + 2, DBL), E.Col(nk + 3, BOOL)
    A = R.Agg
    return [A("sum", i64, I64), A("count", i64), A("min", i64, I64), A("max", i64, I64), A("sum", dec, D22),
            A("avg", dec, D16_6, sum_dt=D22), A("min", dec, D12), A("max", dec, D12), A("sum", f64, DBL), A("avg", f64, DBL),
            A("count", E.Lit(1, I32)), A("sum", i64, I64, filt=flag)]


class Col:
    """One column: dt, values (int64 for integers, dates and unscaled decimals; float64; bool; int64 codes into `names` for a
    string), validity."""

    def __init__(self, dt, values, valid=None, names=None):
        self.dt, self.values, self.names = dt, values, names
        self.valid = np.ones(len(values), dtype=bool) if valid is None else valid

    def __len__(self):
        return len(self.values)

    def slice(self, lo, hi):
        return Col(self.dt, self.values[lo:hi], self.valid[lo:hi], self.names)

    def take(self, idx):
        return Col(self.dt, self.values[idx], self.valid[idx], self.names)


# ---- Arrow <-> numpy -----------------------------------------------------------------------------------------------------------------
_NP = {"INT64": np.int64, "TIMESTAMP": np.int64, "INT32": np.int32, "DATE": np.int32, "INT16": np.int16, "INT8": np.int8, "DOUBLE": np.float64}


def arrow(col, names=None):
    """Col -> Arrow array (a string column becomes a dictionary array over `names`, default the column's own)."""
    n, ok = len(col), col.valid
    mask = None if ok.all() else ~ok
    name = col.dt.name
    if name == "DECIMAL":
        w = np.empty((n, 2), dtype=np.int64)
        w[:, 0] = col.values
        w[:, 1] = col.values >> 63
        bitmap = None if mask is None else pa.py_buffer(np.packbits(ok, bitorder="little").tobytes())
        return pa.Array.from_buffers(pa.decimal128(col.dt.precision, col.dt.scale), n, [bitmap, pa.py_buffer(w.tobytes())],
                                     null_count=int(n - ok.sum()))
    if name == "STRING":
        return pa.DictionaryArray.from_arrays(pa.array(col.values.astype(np.int32), mask=mask), pa.array(names or col.names))
    if name == "BOOL":
        return pa.array(col.values.astype(bool), mask=mask)
    arr = pa.array(col.values.astype(_NP[name]), mask=mask)
    return arr.view(pa.date32()) if name == "DATE" else arr


def table(cols):
    return pa.table([arrow(c) for c in cols], names=[f"c{i}" for i in range(len(cols))])


def from_arrow(arr, dt, names=None):
    """Arrow array -> Col (decimals must fit 64 bits; strings become codes into `names`, -1 for a string not in it)."""
    if isinstance(arr, pa.ChunkedArray):
        parts = [from_arrow(c, dt, names) for c in arr.chunks]
        if not parts:
            return Col(dt, np.zeros(0, dtype=np.int64), np.zeros(0, dtype=bool), names)
        return Col(dt, np.concatenate([p.values for p in parts]), np.concatenate([p.valid for p in parts]), names)
    n, off = len(arr), arr.offset
    valid = arr.is_valid().to_numpy(zero_copy_only=False) if arr.null_count else np.ones(n, dtype=bool)
    name = dt.name
    if pa.types.is_dictionary(arr.type) or name == "STRING":
        code = {s: i for i, s in enumerate(names)}
        strs = arr.to_pylist()
        return Col(dt, np.array([-1 if s is None else code.get(s, -1) for s in strs], dtype=np.int64), valid, names)
    if name == "DECIMAL":
        w = np.frombuffer(arr.buffers()[1], dtype=np.int64)[2 * off:2 * (off + n)].reshape(-1, 2)
        assert ((w[:, 1] == w[:, 0] >> 63) | ~valid).all(), "a decimal that does not fit 64 bits"
        return Col(dt, w[:, 0].copy(), valid)
    if name == "BOOL":
        return Col(dt, arr.fill_null(False).to_numpy(zero_copy_only=False).astype(bool), valid)
    v = np.frombuffer(arr.buffers()[1], dtype=_NP[name])[off:off + n]
    return Col(dt, v.astype(np.float64 if name == "DOUBLE" else np.int64), valid)


def key_matrix(keys):
    """Key columns -> int64 matrix, two columns per key (validity, value or 0 under NULL): equal rows = equal group keys."""
    m = np.zeros((len(keys[0]), 2 * len(keys)), dtype=np.int64)
    for i, k in enumerate(keys):
        m[:, 2 * i] = k.valid
        m[:, 2 * i + 1] = np.where(k.valid, k.values, 0)
    return m


def row_ids(m):
    """dense ids of the distinct rows of an int64 matrix (equal rows, equal ids): one 1-D np.unique per column, each folding the
    column into the ids of the columns before it (np.unique(axis=0) sorts whole rows and is several times slower)"""
    ids = np.zeros(len(m), dtype=np.int64)
    for c in range(m.shape[1]):
        cu, ci = np.unique(m[:, c], return_inverse=True)
        ids = np.unique(ids * len(cu) + ci.reshape(-1), return_inverse=True)[1].reshape(-1)
    return ids


def segments(gidx, ng):
    """rows sorted by group, the first sorted row of every group, rows per group"""
    order = np.argsort(gidx, kind="stable")
    counts = np.bincount(gidx, minlength=ng)
    starts = np.zeros(ng, dtype=np.int64)
    np.cumsum(counts[:-1], out=starts[1:])
    return order, starts, counts


def seg_reduce(ufunc, vals, order, starts, counts, identity):
    """one reduction per group; a group without rows gets `identity`"""
    if len(order) == 0:
        return np.full(len(starts), identity, dtype=vals.dtype)
    out = ufunc.reduceat(vals[order], np.minimum(starts, len(order) - 1))
    out[counts == 0] = identity
    return out


I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def f64_class(x):
    """0 finite, 1 NaN, 2 +Inf, 3 -Inf"""
    return np.where(np.isnan(x), 1, np.where(x == np.inf, 2, np.where(x == -np.inf, 3, 0)))


class F64Sums:
    """Per group: the naive sum of the finite addends, their absolute sum, their count, and the IEEE class of the exact sum."""

    def __init__(self, vals, incl, gidx, ng, seg):
        self.vals, self.incl, self.seg = vals, incl, seg
        finite = incl & np.isfinite(vals)
        self.naive = np.bincount(gidx, weights=np.where(finite, vals, 0.0), minlength=ng)
        self.absum = np.bincount(gidx, weights=np.where(finite, np.abs(vals), 0.0), minlength=ng)
        self.n = np.bincount(gidx, weights=incl, minlength=ng).astype(np.int64)
        nan = np.bincount(gidx, weights=incl & np.isnan(vals), minlength=ng) > 0
        pinf = np.bincount(gidx, weights=incl & (vals == np.inf), minlength=ng) > 0
        ninf = np.bincount(gidx, weights=incl & (vals == -np.inf), minlength=ng) > 0
        self.cls = np.where(nan | (pinf & ninf), 1, np.where(pinf, 2, np.where(ninf, 3, 0)))

    def tolerance(self):
        """bound on |naive - exact| (bincount adds in row order: (n - 1) roundings of partial sums <= absum)"""
        eps = np.finfo(np.float64).eps
        return eps * (self.n + 2) * self.absum + 4 * np.spacing(np.abs(self.naive))

    def addends(self, g):
        order, starts, counts = self.seg
        rows = order[starts[g]:starts[g] + counts[g]]
        return self.vals[rows[self.incl[rows]]]


class Ref:
    """The expected Partial state and Final result of AGGS for one input: key columns and the four value columns."""

    def __init__(self, keys, vals, special_keys=()):
        self.keys, self.vals = keys, vals
        self.key_types = [k.dt for k in keys]
        self.names = next((k.names for k in keys if k.dt.name == "STRING"), None)
        self.aggs = aggs(len(keys))
        m = key_matrix(keys)
        self.gidx = row_ids(m)
        ng = self.ng = int(self.gidx.max()) + 1 if len(m) else 0
        self.kuniq = np.zeros((ng, m.shape[1]), dtype=np.int64)
        self.kuniq[self.gidx] = m
        order, starts, counts = self.seg = segments(self.gidx, ng)
        flag = vals[3].values & vals[3].valid
        self.state, self.result, self.f64 = [], [], {}
        for ai, (kind, vc, filt) in enumerate(KINDS):
            if vc is None:
                incl = np.ones(len(self.gidx), dtype=bool)
            else:
                incl = vals[vc].valid & (flag if filt else True)
            n = np.bincount(self.gidx, weights=incl, minlength=ng).astype(np.int64)
            has = n > 0
            if kind in ("sum", "sum_dec", "avg_dec"):
                s = seg_reduce(np.add, np.where(incl, vals[vc].values, 0), order, starts, counts, 0)
                bound = np.bincount(self.gidx, weights=np.abs(np.where(incl, vals[vc].values, 0)).astype(np.float64), minlength=ng)
                assert (bound < 2.0 ** 62).all(), "a group total near 2^63: the int64 reference would wrap"
                if kind == "sum":
                    self.state.append([(s, has)])
                    self.result.append((s, has))
                elif kind == "sum_dec":
                    self.state.append([(s, np.ones(ng, dtype=bool)), (~has, np.ones(ng, dtype=bool))])
                    self.result.append((s, has))
                else:
                    self.state.append([(s, np.ones(ng, dtype=bool)), (n, np.ones(ng, dtype=bool))])
                    self.result.append((avg_decimal(s, n), has))
            elif kind in ("count", "count_star"):
                self.state.append([(n, np.ones(ng, dtype=bool))])
                self.result.append((n, np.ones(ng, dtype=bool)))
            elif kind in ("min", "max"):
                ident = I64_MAX if kind == "min" else I64_MIN
                v = seg_reduce(np.minimum if kind == "min" else np.maximum, np.where(incl, vals[vc].values, ident), order, starts, counts, ident)
                self.state.append([(v, has)])
                self.result.append((v, has))
            else:
                fs = self.f64[ai] = F64Sums(vals[vc].values, incl, self.gidx, ng, self.seg)
                if kind == "sum_f64":
                    self.state.append([(fs.naive, has)])
                    self.result.append((fs.naive, has))
                else:
                    self.state.append([(np.where(has, fs.naive, 0.0), np.ones(ng, dtype=bool)), (n, np.ones(ng, dtype=bool))])
                    self.result.append((fs.naive / np.maximum(n, 1), has))
        # a deterministic sample of groups whose f64 sums are checked exactly: every k-th group and the named keys
        sample = set(range(0, ng, max(1, ng // 300)))
        if special_keys:
            named = [Col(k.dt, np.array([0 if x is None else x for x in col], dtype=np.int64), np.array([x is not None for x in col]), k.names)
                     for k, col in zip(keys, zip(*special_keys))]
            sample |= set(self.locate(named).tolist())
        self.sample = sorted(sample)

    # ---- library output -> reference groups ------------------------------------------------------------------------------------------
    def locate(self, out_keys):
        """reference group of every output row; asserts that the input has every key the output holds"""
        m = key_matrix(out_keys)
        ids = row_ids(np.vstack([self.kuniq, m]))
        back = np.full(int(ids.max()) + 1, -1, dtype=np.int64)
        back[ids[:self.ng]] = np.arange(self.ng)
        g = back[ids[self.ng:]]
        extra = np.flatnonzero(g < 0)
        assert len(extra) == 0, f"{len(extra)} output rows with keys the input does not have, first (key matrix rows) {m[extra[:3]].tolist()}"
        return g

    def out_cols(self, tbl, types):
        return [from_arrow(tbl.column(i), t, self.names) for i, t in enumerate(types)]


def avg_decimal(s, n):
    """AVG(decimal(12,2)) as decimal(16,6): the mean rounded half away from zero at scale 6 (tests/aggref.py / AvgDecimalGroups)."""
    n1 = np.maximum(n, 1)
    assert (np.abs(s) < 2 ** 58 // 10 ** 4).all()
    q = (2 * np.abs(s) * 10 ** 4 + n1) // (2 * n1)
    return np.where(s < 0, -q, q)


def partial_plan(key_types, aggset):
    return R.partial_plan(list(key_types) + VALUE_TYPES, list(range(len(key_types))), aggs(len(key_types), aggset))


def merge_plan(key_types, aggset, mode=R.FINAL):
    return R.merge_plan(list(key_types), aggs(len(key_types), aggset), mode)


def state_types(aggs_):
    return [t for a in aggs_ for t in a.state_types()]


# ---- comparisons -------------------------------------------------------------------------------------------------------------------
def _valid(got_ok, exp_ok, what, keys_of):
    bad = np.flatnonzero(got_ok != exp_ok)
    assert len(bad) == 0, f"{what}: validity differs in {len(bad)} groups, first {keys_of(bad[:3])}: got {got_ok[bad[:3]]}, want {exp_ok[bad[:3]]}"


def _exact(got_v, got_ok, exp_v, exp_ok, what, keys_of):
    _valid(got_ok, exp_ok, what, keys_of)
    bad = np.flatnonzero(exp_ok & (got_v != exp_v))
    assert len(bad) == 0, f"{what}: {len(bad)} groups differ, first {keys_of(bad[:3])}: got {got_v[bad[:3]]}, want {exp_v[bad[:3]]}"


def _f64_close(got, ok, fs, exp, tol, what, keys_of):
    """class per group and |got - naive| <= tol for the finite ones"""
    cls = f64_class(got)
    bad = np.flatnonzero(ok & (cls != fs.cls))
    assert len(bad) == 0, f"{what}: IEEE class differs in {len(bad)} groups, first {keys_of(bad[:3])}: got {got[bad[:3]]}, class {fs.cls[bad[:3]]}"
    fin = ok & (fs.cls == 0)
    bad = np.flatnonzero(fin & ~(np.abs(got - exp) <= tol))
    assert len(bad) == 0, f"{what}: {len(bad)} groups off by more than the bound, first {keys_of(bad[:3])}: got {got[bad[:3]]}, want {exp[bad[:3]]} +- {tol[bad[:3]]}"


def check(out, ref, stage, kind, aggset, fed=None, unique=True):
    """Compare a library output table with the reference, group by group.

    kind "state": a Partial / PartialMerge state batch (a key may repeat unless `unique`: repeated rows are merged first, each float
    sum allowed its own 1 ULP); kind "result": a Final result (every key once).  `fed`: the state table the stage merged (None: the
    stage read rows), whose float sums the exactly checked sample is measured against.  Returns the number of output rows."""
    nk = len(ref.keys)
    sel = SETS[aggset]
    set_aggs = [ref.aggs[i] for i in sel]
    types = ref.key_types + (state_types(set_aggs) if kind == "state" else [a.result_type() for a in set_aggs])
    assert out is not None and out.num_columns == len(types), f"{stage}: {None if out is None else out.num_columns} columns, want {len(types)}"
    cols = ref.out_cols(out, types)
    g = ref.locate(cols[:nk])
    rows_per = np.bincount(g, minlength=ref.ng)
    missing = np.flatnonzero(rows_per == 0)
    keys_of = lambda idx: [tuple(r) for r in ref.kuniq[np.asarray(idx, dtype=np.int64)]]
    assert len(missing) == 0, f"{stage}: {len(missing)} groups missing, first {keys_of(missing[:3])}"
    if unique or kind == "result":
        dup = np.flatnonzero(rows_per > 1)
        assert len(dup) == 0, f"{stage}: {len(dup)} keys emitted more than once, first {keys_of(dup[:3])}"
    order, starts, counts = segments(g, ref.ng)
    fed_groups = None
    if fed is not None:
        fcols = ref.out_cols(fed, ref.key_types + state_types(set_aggs))
        fed_groups = (ref.locate(fcols[:nk]), fcols)
    at = nk
    for si, ai in enumerate(sel):
        k, vc, filt = KINDS[ai]
        what = f"{stage}: aggregate {ai} ({k}{' FILTER' if filt else ''})"
        width = len(ref.aggs[ai].state_types()) if kind == "state" else 1
        got = cols[at:at + width]
        if kind == "state":
            merged = []
            for j, c in enumerate(got):
                is_f = c.dt.name == "DOUBLE"
                is_empty = k == "sum_dec" and j == 1
                if k in ("min", "max"):
                    ident = I64_MAX if k == "min" else I64_MIN
                    v = seg_reduce(np.minimum if k == "min" else np.maximum, np.where(c.valid, c.values, ident), order, starts, counts, ident)
                elif is_empty:
                    v = seg_reduce(np.logical_and, c.values | ~c.valid, order, starts, counts, True)
                else:
                    v = seg_reduce(np.add, np.where(c.valid, c.values, 0.0 if is_f else 0), order, starts, counts, 0)
                ok = seg_reduce(np.logical_or, c.valid, order, starts, counts, False)
                merged.append((v, ok))
            exp = ref.state[ai]
            for j, ((gv, gok), (ev, eok)) in enumerate(zip(merged, exp)):
                if got[j].dt.name == "DOUBLE":
                    fs = ref.f64[ai]
                    slack = seg_reduce(np.add, np.where(got[j].valid & np.isfinite(got[j].values), np.spacing(np.abs(got[j].values)), 0.0),
                                       order, starts, counts, 0.0) * (rows_per > 1)
                    _valid(gok, eok, what, keys_of)
                    _f64_close(gv, gok, fs, ev, fs.tolerance() + slack, what, keys_of)
                    _f64_sample(ref, ai, si, set_aggs, gv, gok, slack, fed_groups, False, what)
                else:
                    _exact(gv, gok, ev, eok, what + f" state column {j}", keys_of)
        else:
            c = got[0]
            v, ok = c.values[order], c.valid[order]
            ev, eok = ref.result[ai]
            if c.dt.name == "DOUBLE":
                fs = ref.f64[ai]
                _valid(ok, eok, what, keys_of)
                tol = fs.tolerance() if k == "sum_f64" else fs.tolerance() / np.maximum(fs.n, 1) + 4 * np.spacing(np.abs(ev))
                _f64_close(v, ok, fs, ev, tol, what, keys_of)
                _f64_sample(ref, ai, si, set_aggs, v, ok, np.zeros(ref.ng), fed_groups, k == "avg_f64", what)
            else:
                _exact(v, ok, ev, eok, what, keys_of)
        at += width
    return out.num_rows


def _f64_sample(ref, ai, si, set_aggs, got, ok, slack, fed_groups, mean, what):
    """The sampled groups: a sum within 1 ULP (+ slack) of the correctly rounded sum of what the stage added -- the input values, or
    the float sums of the states it merged; a mean within 2 ULP of the correctly rounded exact quotient of that sum by the count."""
    fs = ref.f64[ai]
    if fed_groups is not None:
        fg, fcols = fed_groups
        at = len(ref.keys) + sum(len(a.state_types()) for a in set_aggs[:si])
        col = fcols[at]
        cnt = fcols[at + 1] if mean else None
        forder, fstarts, fcounts = segments(fg, ref.ng)
    for g in ref.sample:
        if not ok[g] or fs.cls[g] != 0:
            continue
        if fed_groups is None:
            add = fs.addends(g)
            n = len(add)
        else:
            rows = forder[fstarts[g]:fstarts[g] + fcounts[g]]
            add = col.values[rows[col.valid[rows]]]
            n = int(cnt.values[rows].sum()) if mean else 0
        if not np.isfinite(add).all():
            continue
        if mean:
            exact = float(sum((Fraction(float(x)) for x in add), Fraction(0)) / n)
            tol = 2 * math.ulp(exact)
        else:
            exact = math.fsum(add.tolist())
            tol = math.ulp(exact) + slack[g]
        assert abs(got[g] - exact) <= tol, f"{what}: group {tuple(ref.kuniq[g])}: got {got[g]!r}, want {exact!r} (tolerance {tol!r})"




# ---- data -----------------------------------------------------------------------------------------------------------------------
def value_cols(rng, n, null_frac=0.05):
    """v0 i64 in +-2^40, v1 decimal(12,2) unscaled in +-10^9 (with the type's edges +-(10^12 - 1) now and then), v2 f64 over many
    magnitudes with NaN / +Inf / -Inf at one row in a thousand, v3 bool; NULLs in each"""
    nulls = lambda: rng.random(n) >= null_frac
    i64 = rng.integers(-2 ** 40, 2 ** 40, n)
    dec = rng.integers(-10 ** 9, 10 ** 9, n)
    edge = rng.random(n) < 0.001
    dec[edge] = np.where(rng.random(int(edge.sum())) < 0.5, -(10 ** 12 - 1), 10 ** 12 - 1)
    f64 = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 7, n)
    sp = rng.random(n) < 0.001
    f64[sp] = np.array([np.nan, np.inf, -np.inf])[rng.integers(0, 3, int(sp.sum()))]
    return [Col(I64, i64, nulls()), Col(D12, dec, nulls()), Col(DBL, f64, nulls()), Col(BOOL, rng.random(n) < 0.5, nulls())]


def scattered(idx):
    """distinct ids -> distinct int64 keys spread over the whole range (never -1: the empty-slot word, tested on purpose elsewhere)"""
    k = (np.asarray(idx, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(12345)).view(np.int64)
    return np.where(k == -1, 7, k)


class Data:
    """One input: key columns, value columns, its batches' row count and the keys whose float results the check always samples."""

    def __init__(self, name, keys, vals, batch_rows=8192, special_keys=(), batches=None):
        self.name, self.keys, self.vals, self.batch_rows, self.special_keys = name, keys, vals, batch_rows, special_keys
        self._batches, self._ref, self._table = batches, None, None

    def __repr__(self):
        return self.name

    @property
    def cols(self):
        return self.keys + self.vals

    @property
    def dts(self):
        return [c.dt for c in self.cols]

    @property
    def key_types(self):
        return [k.dt for k in self.keys]

    @property
    def n(self):
        return len(self.vals[0])

    def ref(self):
        if self._ref is None:
            self._ref = Ref(self.keys, self.vals, self.special_keys)
        return self._ref

    def table(self):
        if self._table is None:
            self._table = table(self.cols)
        return self._table

    def batches(self):
        if self._batches is not None:
            return self._batches(self)
        return self.table().to_batches(max_chunksize=self.batch_rows)

    def partial_plan(self, aggset):
        return partial_plan(self.key_types, aggset)

    def merge_plan(self, aggset, mode=R.FINAL):
        return merge_plan(self.key_types, aggset, mode)

    def slice(self, lo, hi):
        return Data(f"{self.name}[{lo}:{hi}]", [k.slice(lo, hi) for k in self.keys], [v.slice(lo, hi) for v in self.vals])


def growth(seed=1, n=2_000_000, pool=1_150_000):
    """case 1: one int64 key, ~10^6 distinct keys over 2 * 10^6 rows in scattered order, NULL keys now and then"""
    rng = np.random.default_rng(seed)
    k = scattered(rng.integers(0, pool, n))
    return Data("growth", [Col(I64, k, rng.random(n) >= 0.001)], value_cols(rng, n), batch_rows=4096)


def crossing(distinct, seed=2):
    """case 2: `distinct` keys over 2 * distinct rows, each key's first row anywhere, so new keys keep arriving in every chunk.  The
    distinct counts bracket 32 768, 65 536 and 131 072; where the key table doubles is set by the ids handed out plus the incoming
    chunk (KeyTable::ensure), so a pair may double it at the same chunk -- each input grows it past its first 65 536 slots or
    right up to them, and is checked group by group."""
    rng = np.random.default_rng(seed + distinct)
    ids = rng.permutation(np.concatenate([np.arange(distinct), rng.integers(0, distinct, distinct)]))
    n = len(ids)
    return Data(f"crossing-{distinct}", [Col(I64, scattered(ids))], value_cols(rng, n), batch_rows=8192)


def reserved(early, seed=3, n=600_000):
    """case 3: the NULL key and the key -1 (the empty-slot word of the key table) in the first chunk and again after several
    growths (early), or for the first time only after growths (late)"""
    rng = np.random.default_rng(seed + early)
    k = scattered(rng.integers(0, n // 2, n))
    valid = np.ones(n, dtype=bool)
    null_rows = [3, 7, 100, 451_003, 590_017] if early else [400_001, 400_002, 555_555]
    neg_rows = [1, 5, 4000, 450_000, 599_999] if early else [420_000, 420_001, 598_765]
    valid[null_rows] = False
    k[neg_rows] = -1
    return Data(f"reserved-{'early' if early else 'late'}", [Col(I64, k, valid)], value_cols(rng, n), batch_rows=8192,
                special_keys=[(None,), (-1,)])


def all_new(seed=4, n=150_000):
    """case 4: every row its own key"""
    rng = np.random.default_rng(seed)
    return Data("all-new", [Col(I64, scattered(rng.permutation(n)))], value_cols(rng, n), batch_rows=1024)


WIDE = {"i64-i64": [I64, I64], "i64-i32-date-i8": [I64, I32, DATE, I8], "dec18-i64": [D18, I64]}


def wide(which, seed=5, n=1_000_000, base=600_000):
    """case 5: multi-word keys, ~5 * 10^5 groups, NULLs in every key column"""
    rng = np.random.default_rng(seed + len(which))
    pick = rng.integers(0, base, n)
    keys = []
    for dt in WIDE[which]:
        lo, hi = {"INT64": (-2 ** 63, 2 ** 63 - 1), "INT32": (-2 ** 31, 2 ** 31 - 1), "DATE": (-30_000, 30_000), "INT8": (-128, 127),
                  "DECIMAL": (-10 ** 18 + 1, 10 ** 18 - 1)}[dt.name]
        pool = rng.integers(lo, hi, base, endpoint=True)
        if dt.name == "INT8":                     # a narrow component: the other components must tell the groups apart
            pool = pool % 7 - 3
        keys.append(Col(dt, pool[pick], rng.random(n) >= 0.02))
    return Data(f"wide-{which}", keys, value_cols(rng, n), batch_rows=16384)


def hot_cold(seed=6, cold=1_000_000, hot_rows=120_000):
    """case 6: 10 % of the rows on 8 keys, spread over every batch, among 10^6 cold keys"""
    rng = np.random.default_rng(seed)
    ids = np.concatenate([np.arange(cold), rng.integers(0, cold, 80_000), cold + rng.integers(0, 8, hot_rows)])
    ids = rng.permutation(ids)
    return Data("hot-cold", [Col(I64, scattered(ids))], value_cols(rng, len(ids)), batch_rows=16384,
                special_keys=[(int(scattered([cold + h])[0]),) for h in range(8)])


def skewed(few_first, seed=7, n=1_000_000):
    """estimate-breaking inputs for the DeviceTable sizing: 30 % of the rows over 1000 keys then every row new (few_first), or the
    reverse"""
    rng = np.random.default_rng(seed + few_first)
    a = int(0.3 * n)
    few = rng.integers(0, 1000, a if few_first else n - a)
    many = 1000 + rng.permutation(n - a if few_first else a)
    ids = np.concatenate([few, many] if few_first else [many, few])
    return Data(f"skewed-{'few-first' if few_first else 'many-first'}", [Col(I64, scattered(ids), rng.random(n) >= 0.001)],
                value_cols(rng, n))


def clustered(seed=8, n_head=1_100_000, n_tail=2_200_000, name="clustered"):
    """case 8: runs of 8 equal keys, then every row its own key, NULL keys in both parts.  In one batch, the stream strategy samples
    the first 2^20 rows (runs of 8) and sizes for twice that; the tail's runs overflow it, so the launch is discarded and repeated.
    clustered_slices: the same shape read in 2^18-row DeviceTable slices, sized from the rows still to come."""
    rng = np.random.default_rng(seed)
    k = np.concatenate([scattered(np.repeat(np.arange(n_head // 8), 8)), scattered(10 ** 9 + np.arange(n_tail))])
    valid = np.ones(len(k), dtype=bool)
    valid[5:9] = False
    valid[n_head + 10:n_head + 12] = False
    return Data(name, [Col(I64, k, valid)], value_cols(rng, len(k)), special_keys=[(None,)])


def clustered_slices():
    return clustered(seed=10, n_head=400_000, n_tail=1_100_000, name="clustered-slices")


def migrate(seed=9, small_batches=2, big_batches=14, rows=20_000, big=100_000):
    """case 9: a dictionary key with 6 values in the first batches (dense) and 10^5 later (key table, several growths)"""
    rng = np.random.default_rng(seed)
    names = [f"s{i}" for i in range(6)] + [f"b{i:06d}" for i in range(big - 6)]
    codes = np.concatenate([rng.integers(0, 6, rows * small_batches), rng.integers(0, big, rows * big_batches)])
    n = len(codes)
    key = Col(STR, codes, rng.random(n) >= 0.01, names)
    vals = value_cols(rng, n)

    def batches(d):
        out = []
        for b in range(small_batches + big_batches):
            lo, hi = b * rows, (b + 1) * rows
            cols = [arrow(key.slice(lo, hi), names[:6] if b < small_batches else names)] + [arrow(v.slice(lo, hi)) for v in vals]
            out.append(pa.RecordBatch.from_arrays(cols, names=[f"c{i}" for i in range(len(cols))]))
        return out
    return Data("migrate", [key], vals, batch_rows=rows, batches=batches)


KEY_SETS = [[I64], [STR]] + list(WIDE.values())
CROSSINGS = [32_700, 32_840, 65_480, 65_600, 131_000, 131_150]


def all_data():
    """(name, generator) of every input of the GPU suite; each input is built when its generator is called"""
    out = [("growth", growth), ("all-new", all_new), ("hot-cold", hot_cold), ("clustered", clustered), ("clustered-slices", clustered_slices),
           ("migrate", migrate)]
    out += [(f"crossing-{d}", lambda d=d: crossing(d)) for d in CROSSINGS]
    out += [(f"reserved-{'early' if e else 'late'}", lambda e=e: reserved(e)) for e in (True, False)]
    out += [(f"wide-{w}", lambda w=w: wide(w)) for w in WIDE]
    out += [(f"skewed-{'few-first' if f else 'many-first'}", lambda f=f: skewed(f)) for f in (True, False)]
    return out
