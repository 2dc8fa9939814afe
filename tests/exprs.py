"""Expression ASTs that serialise to the reference's plan IR AND evaluate on the CPU through the oracle --
the harness of the generic projection / filter parity tests (tests/test_gpu_exprs.py).

Evaluation is operator-at-a-time over whole columns, one array per node, i.e. exactly how the reference's
PhysicalExpr::evaluate works (SURVEY.md 3C)."""
import numpy as np

from comet_b200 import proto as P
from oracle import oracle as O

LEGACY, TRY, ANSI = 0, 1, 2


OVERFLOW, DIVIDE_BY_ZERO = "ARITHMETIC_OVERFLOW", "DIVIDE_BY_ZERO"


class AnsiError(Exception):
    """A Spark error in ANSI mode.  `classes`: the error classes of the failing rows (a batch may fail for more than one reason)."""

    def __init__(self, *classes):
        super().__init__(*classes)
        self.classes = set(classes) or {OVERFLOW}


def _valid_and(a, b):
    return a & b


class Node:
    dt = None


class Col(Node):
    def __init__(self, i, dt):
        self.i, self.dt = i, dt

    def proto(self):
        return P.bound(self.i, self.dt)

    def eval(self, cols):
        return cols[self.i]


class Lit(Node):
    def __init__(self, v, dt):
        self.v, self.dt = v, dt

    def proto(self):
        return P.literal(self.v, self.dt)

    def eval(self, cols):
        n = len(cols[0][1])
        valid = np.full(n, self.v is not None)
        if self.dt.name == "DECIMAL":
            return O.dec_from_ints([self.v or 0] * n), valid
        np_dt = {"INT8": np.int64, "INT16": np.int64, "INT32": np.int64, "INT64": np.int64, "DATE": np.int64, "TIMESTAMP": np.int64, "DOUBLE": np.float64,
                 "FLOAT": np.float32, "BOOL": np.bool_}[self.dt.name]
        return np.full(n, self.v if self.v is not None else 0, dtype=np_dt), valid


def _int_width(dt):
    return {"INT8": 8, "INT16": 16, "INT32": 32, "INT64": 64}[dt.name]


class ArrowError(Exception):
    """arrow-arith failed the query (Legacy-mode checked division)"""


class Arith(Node):
    """Add / Subtract / Multiply / Divide with the planner's lowering rules (planner.rs:976-1131)."""

    def __init__(self, op, l, r, ret, mode=LEGACY):
        self.op, self.l, self.r, self.ret, self.mode = op, l, r, ret, mode
        lt, rt = l.dt, r.dt
        if op == "divide":
            self.wide = False
            self.dt = ret
        elif lt.name == "DECIMAL":
            if op == "multiply":
                self.wide = lt.precision + rt.precision >= 38
            else:
                self.wide = max(lt.scale, rt.scale) + max(lt.precision - lt.scale, rt.precision - rt.scale) >= 38
            if self.wide:
                self.dt = ret
            elif op == "multiply":
                self.dt = P.DECIMAL(min(lt.precision + rt.precision + 1, 38), lt.scale + rt.scale)
            else:
                rs = max(lt.scale, rt.scale)
                self.dt = P.DECIMAL(min(rs + max(lt.precision - lt.scale, rt.precision - rt.scale) + 1, 38), rs)
        else:
            self.dt = ret

    def proto(self):
        return getattr(P, self.op)(self.l.proto(), self.r.proto(), self.ret, self.mode)

    def eval_divide(self, a, av, b, bv):
        lt, rt = self.l.dt, self.r.dt
        av, bv = np.asarray(av, dtype=bool), np.asarray(bv, dtype=bool)
        if lt.name == "DECIMAL":                       # decimal_div UDF, div.rs:75-190
            try:
                out, ov = O.decimal_div(a, av, lt.scale, b, bv, rt.scale, self.dt.scale, False, self.mode)
            except O.OracleError:
                raise AnsiError(DIVIDE_BY_ZERO)
            return out, ov.astype(bool)
        valid = av & bv
        if lt.name in ("DOUBLE", "FLOAT"):             # Legacy: IEEE; TRY / ANSI: checked_div (zero divisor -> NULL / DIVIDE_BY_ZERO)
            with np.errstate(all="ignore"):
                out = a / b
            if self.mode != LEGACY:
                z = valid & (b == 0)
                if self.mode == ANSI and z.any():
                    raise AnsiError(DIVIDE_BY_ZERO)
                out = np.where(z, 0, out).astype(a.dtype)
                valid = valid & ~z
            return out, valid
        w = _int_width(lt)                             # integers: truncating division, zero divisor / MIN / -1 are errors
        mn = -(1 << (w - 1))
        bad = valid & ((b == 0) | ((a == mn) & (b == -1)))
        if bad.any():
            if self.mode == ANSI:
                raise AnsiError(*([DIVIDE_BY_ZERO] if (valid & (b == 0)).any() else []) + ([OVERFLOW] if (valid & (a == mn) & (b == -1)).any() else []))
            if self.mode == LEGACY:
                raise ArrowError()
        safe_b = np.where(bad | (b == 0), 1, b)
        q = np.abs(a.astype(object)) // np.abs(safe_b.astype(object))
        q = np.where((a < 0) != (safe_b < 0), -q, q).astype(np.int64)
        return np.where(bad, 0, q), valid & ~bad

    def eval(self, cols):
        (a, av), (b, bv) = self.l.eval(cols), self.r.eval(cols)
        if self.op == "divide":
            return self.eval_divide(a, av, b, bv)
        code = {"add": 0, "subtract": 1, "multiply": 2}[self.op]
        lt, rt = self.l.dt, self.r.dt
        if lt.name == "DECIMAL":
            try:
                if self.wide:
                    out, ov = O.wide_decimal(code, a, av, lt.scale, b, bv, rt.scale, self.dt.precision, self.dt.scale, self.mode)
                else:
                    out, ov, _, _ = O.plain_decimal(code, a, av, lt.precision, lt.scale, b, bv, rt.precision, rt.scale)
            except O.OracleError:
                raise AnsiError()
            return out, ov.astype(bool)
        if lt.name in ("DOUBLE", "FLOAT"):
            with np.errstate(all="ignore"):
                out = a + b if code == 0 else a - b if code == 1 else a * b
            return out, av & bv
        try:
            out, ov = O.int_arith(code, _int_width(lt), a, av, b, bv, self.mode)
        except O.OracleError:
            raise AnsiError()
        return out, ov.astype(bool)


def _total_key(x):
    """IEEE totalOrder as a signed integer key, in the value's own width (a float32 NaN widened to float64 loses its signalling bit)"""
    x = np.asarray(x)
    if x.dtype == np.float32:
        bits = np.ascontiguousarray(x).view(np.int32)
        return bits ^ ((bits >> 31) & np.int32(0x7FFFFFFF))
    bits = np.ascontiguousarray(x, dtype=np.float64).view(np.int64)
    return bits ^ ((bits >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))


class Cmp(Node):
    dt = P.BOOL

    def __init__(self, op, l, r):
        self.op, self.l, self.r = op, l, r

    def proto(self):
        return getattr(P, self.op)(self.l.proto(), self.r.proto())

    def eval(self, cols):
        (a, av), (b, bv) = self.l.eval(cols), self.r.eval(cols)
        if self.l.dt.name == "DECIMAL":
            x = np.array(O.dec_to_ints(a), dtype=object)
            y = np.array(O.dec_to_ints(b), dtype=object)
        elif self.l.dt.name in ("DOUBLE", "FLOAT"):
            x, y = _total_key(a), _total_key(b)  # arrow-ord compares floats by IEEE totalOrder
        else:
            x, y = a, b
        f = {"eq": lambda: x == y, "neq": lambda: x != y, "lt": lambda: x < y, "lt_eq": lambda: x <= y, "gt": lambda: x > y, "gt_eq": lambda: x >= y}[self.op]
        return np.asarray(f(), dtype=bool), av & bv


class Logic(Node):
    dt = P.BOOL

    def __init__(self, op, l, r):
        self.op, self.l, self.r = op, l, r

    def proto(self):
        return (P.and_ if self.op == "and" else P.or_)(self.l.proto(), self.r.proto())

    def eval(self, cols):  # Kleene
        (a, av), (b, bv) = self.l.eval(cols), self.r.eval(cols)
        at, af, bt, bf = av & a, av & ~a, bv & b, bv & ~b
        if self.op == "and":
            t, f = at & bt, af | bf
        else:
            t, f = at | bt, af & bf
        return t, t | f


class Not(Node):
    dt = P.BOOL

    def __init__(self, c):
        self.c = c

    def proto(self):
        return P.not_(self.c.proto())

    def eval(self, cols):
        a, av = self.c.eval(cols)
        return ~a, av


class IsNull(Node):
    dt = P.BOOL

    def __init__(self, c, negate=False):
        self.c, self.negate = c, negate

    def proto(self):
        return (P.is_not_null if self.negate else P.is_null)(self.c.proto())

    def eval(self, cols):
        _, av = self.c.eval(cols)
        return (av if self.negate else ~av), np.ones(len(av), dtype=bool)


class CheckOverflow(Node):
    def __init__(self, c, dt, fail=False):
        self.c, self.dt, self.fail = c, dt, fail

    def proto(self):
        return P.check_overflow(self.c.proto(), self.dt, self.fail)

    def eval(self, cols):
        c = self.c
        if isinstance(c, Arith) and c.l.dt.name == "DECIMAL" and c.wide and c.dt.precision == self.dt.precision and c.dt.scale == self.dt.scale:
            return c.eval(cols)  # planner.rs:606-613
        if isinstance(c, Cast) and c.c.dt.name == "DECIMAL" and c.dt.precision == self.dt.precision and c.dt.scale == self.dt.scale:
            a, av = c.c.eval(cols)  # planner.rs:617-637 DecimalRescaleCheckOverflow
            try:
                out, ov = O.decimal_rescale_check(a, av, c.c.dt.scale, self.dt.precision, self.dt.scale, self.fail)
            except O.OracleError:
                raise AnsiError()
            return out, ov.astype(bool)
        a, av = c.eval(cols)
        try:
            out, ov = O.check_overflow(a, av, self.dt.precision, self.fail)
        except O.OracleError:
            raise AnsiError()
        return out, ov.astype(bool)


class Cast(Node):
    def __init__(self, c, dt, mode=LEGACY):
        self.c, self.dt, self.mode = c, dt, mode

    def proto(self):
        return P.cast(self.c.proto(), self.dt, self.mode)

    def eval(self, cols):
        a, av = self.c.eval(cols)
        f, t = self.c.dt, self.dt
        if f == t:
            return a, av
        if f.name == "DECIMAL" and t.name == "DECIMAL":
            try:
                out, ov = O.decimal_rescale_check(a, av, f.scale, t.precision, t.scale, self.mode == ANSI)
            except O.OracleError:
                raise AnsiError()
            return out, ov.astype(bool)
        if t.name == "DECIMAL":  # int -> decimal
            try:
                out, ov = O.decimal_rescale_check(O.dec_from_i64(a), av, 0, t.precision, t.scale, self.mode == ANSI)
            except O.OracleError:
                raise AnsiError()
            return out, ov.astype(bool)
        if t.name == "DOUBLE":      # integers (held as int64) round once; float32 widens exactly, NaNs keep sign and payload
            with np.errstate(invalid="ignore"):         # a signalling NaN is made quiet
                return a.astype(np.float64), av
        if t.name == "FLOAT":       # integers only (the planner refuses double -> float)
            return a.astype(np.float32), av
        return a.astype(np.int64), av  # widening int casts


class If(Node):
    def __init__(self, c, a, b):
        self.c, self.a, self.b, self.dt = c, a, b, a.dt

    def proto(self):
        return P.if_(self.c.proto(), self.a.proto(), self.b.proto())

    def eval(self, cols):
        """each branch is evaluated on the rows that take it only (CaseExpr evaluates THEN under the selection), so an ANSI error
        of a row that does not take a branch is not raised"""
        c, cv = self.c.eval(cols)
        take = np.asarray(cv & c, dtype=bool)
        rows = lambda m: [(np.asarray(v)[m], np.asarray(ok)[m]) for v, ok in cols]
        (a, av), (b, bv) = self.a.eval(rows(take)), self.b.eval(rows(~take))
        a, b = np.asarray(a), np.asarray(b)
        out = np.zeros((len(take),) + a.shape[1:], dtype=np.result_type(a, b))
        out[take], out[~take] = a, b
        valid = np.zeros(len(take), dtype=bool)
        valid[take], valid[~take] = av, bv
        return out, valid


class In(Node):
    dt = P.BOOL

    def __init__(self, v, lits, negated=False):
        self.v, self.lits, self.negated = v, lits, negated

    def proto(self):
        return P.in_(self.v.proto(), [l.proto() for l in self.lits], self.negated)

    def eval(self, cols):
        a, av = self.v.eval(cols)
        name = self.v.dt.name
        vals = np.array(O.dec_to_ints(a), dtype=object) if name == "DECIMAL" else a
        fdt = {"FLOAT": (np.float32, np.uint32), "DOUBLE": (np.float64, np.uint64)}.get(name)
        if fdt:                      # floats match by their bits: IEEE totalOrder equality (NaN IN (NaN) is TRUE, 0.0 IN (-0.0) is not)
            vals = np.ascontiguousarray(a, dtype=fdt[0]).view(fdt[1])
        hit = np.zeros(len(av), dtype=bool)
        has_null = False
        for l in self.lits:
            if l.v is None:
                has_null = True
            else:
                hit |= np.asarray(vals == (np.array(l.v, dtype=fdt[0]).view(fdt[1]) if fdt else l.v), dtype=bool)
        out = ~hit if self.negated else hit
        valid = av & (hit | (not has_null))
        return out, valid


class Neg(Node):
    def __init__(self, c, fail=False):
        self.c, self.dt, self.fail = c, c.dt, fail

    def proto(self):
        return P.unary_minus(self.c.proto(), self.fail)

    def eval(self, cols):
        a, av = self.c.eval(cols)
        if self.dt.name == "DECIMAL":
            return O.dec_from_ints([-(x) for x in O.dec_to_ints(a)]), av
        if self.dt.name in ("DOUBLE", "FLOAT"):
            return -a, av
        w = _int_width(self.dt)
        out, _ = O.int_arith(1, w, np.zeros_like(a), None, a, None, LEGACY)
        if self.fail and (av & (a == -(1 << (w - 1)))).any():
            raise AnsiError()
        return out, av


class CaseWhen(Node):
    def __init__(self, whens, thens, els=None):
        self.whens, self.thens, self.els, self.dt = whens, thens, els, thens[0].dt

    def proto(self):
        return P.case_when([w.proto() for w in self.whens], [t.proto() for t in self.thens], None if self.els is None else self.els.proto())

    def eval(self, cols):
        tail = self.els if self.els is not None else Lit(None, self.dt)
        for w, t in reversed(list(zip(self.whens, self.thens))):
            tail = If(w, t, tail)
        return tail.eval(cols)
