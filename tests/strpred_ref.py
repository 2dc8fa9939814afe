"""CPU reference of the string predicates the planner lowers to StrPred, and interpreter nodes for them in the style of tests/exprs.py
(each node serialises to the reference's plan IR and evaluates column-at-a-time).

A string column is (values, valid): `values` a list of `str` (anything under a NULL slot), `valid` a numpy bool array.  The rules:

- Comparisons (=, !=, <, <=, >, >=) order by unsigned bytes of the UTF-8 encoding, a proper prefix first: arrow-ord `cmp` over Utf8
  (DataFusion's BinaryExpr, native/core/src/execution/planner.rs create_binary_expr) and Spark `UTF8String.compareTo`.
- IN: NULL value -> NULL; a match -> TRUE; otherwise NULL if the list holds a NULL, else FALSE; `negated` inverts (Spark In, DataFusion
  InListExpr).
- LIKE: the reference builds DataFusion's LikeExpr (native/core/src/execution/expressions/strings.rs:36-50).  `%` matches any run of
  characters and `_` exactly one character (one code point), both including '\\n'; `\\` escapes `%`, `_` and `\\`.  Any other use of
  `\\` is refused by the planner (the reference's handling of it is not pinned here).
- starts_with / ends_with / contains: byte prefix / suffix / substring (Comet's scalar-function bridge, serde/strings.scala:344-356); the
  empty literal is a prefix, suffix and substring of every value.
- A NULL value gives NULL; a NULL literal gives NULL for every row.
"""
import re

import numpy as np

from comet_b200 import proto as P

OPS = ("eq", "neq", "lt", "lt_eq", "gt", "gt_eq")
MIRROR = {"eq": "eq", "neq": "neq", "lt": "gt", "lt_eq": "gt_eq", "gt": "lt", "gt_eq": "lt_eq"}
# cb::StrOp (device/cb_strpred.h)
SP = dict(eq=0, neq=1, lt=2, lt_eq=3, gt=4, gt_eq=5, **{"in": 6}, like=7, starts_with=8, ends_with=9, contains=10)


class BadPattern(ValueError):
    pass


def cmp(op, a, b):
    """a <op> b over str values, by UTF-8 bytes"""
    x, y = a.encode(), b.encode()
    return {"eq": x == y, "neq": x != y, "lt": x < y, "lt_eq": x <= y, "gt": x > y, "gt_eq": x >= y}[op]


def like_regex(pattern):
    out, i = [], 0
    while i < len(pattern):
        c = pattern[i]
        if c == "\\":
            if i + 1 >= len(pattern) or pattern[i + 1] not in "%_\\":
                raise BadPattern(pattern)
            out.append(re.escape(pattern[i + 1]))
            i += 2
            continue
        out.append(".*" if c == "%" else "." if c == "_" else re.escape(c))
        i += 1
    return re.compile("".join(out), re.DOTALL)


def like(value, pattern):
    return like_regex(pattern).fullmatch(value) is not None


def func(name, value, lit):
    x, y = value.encode(), lit.encode()
    return {"starts_with": x.startswith(y), "ends_with": x.endswith(y), "contains": y in x}[name]


def in_list(value, lits):
    """(hit, list_has_null)"""
    return any(l is not None and l.encode() == value.encode() for l in lits), any(l is None for l in lits)


# ---- interpreter nodes (tests/exprs.py style) ------------------------------------------------------------------------------------
class StrCol:
    dt = P.STRING

    def __init__(self, i):
        self.i = i

    def proto(self):
        return P.bound(self.i, P.STRING)

    def eval(self, cols):
        return cols[self.i]


class StrLit:
    dt = P.STRING

    def __init__(self, v):
        self.v = v

    def proto(self):
        return P.literal(self.v, P.STRING)


def _map(col, cols, f):
    vals, valid = col.eval(cols)
    out = np.array([bool(f(v)) if ok else False for v, ok in zip(vals, valid)], dtype=bool)
    return out, np.asarray(valid, dtype=bool).copy()


class StrCmp:
    """column <op> literal, or literal <op> column with lit_left"""
    dt = P.BOOL

    def __init__(self, op, col, lit, lit_left=False):
        self.op, self.col, self.lit, self.lit_left = op, col, lit, lit_left

    def proto(self):
        l, r = (StrLit(self.lit), self.col) if self.lit_left else (self.col, StrLit(self.lit))
        return getattr(P, self.op)(l.proto(), r.proto())

    def eval(self, cols):
        if self.lit is None:
            n = len(cols[self.col.i][1])
            return np.zeros(n, dtype=bool), np.zeros(n, dtype=bool)
        op = MIRROR[self.op] if self.lit_left else self.op
        return _map(self.col, cols, lambda v: cmp(op, v, self.lit))


class StrIn:
    dt = P.BOOL

    def __init__(self, col, lits, negated=False):
        self.col, self.lits, self.negated = col, lits, negated

    def proto(self):
        return P.in_(self.col.proto(), [StrLit(l).proto() for l in self.lits], self.negated)

    def eval(self, cols):
        vals, valid = self.col.eval(cols)
        out = np.zeros(len(valid), dtype=bool)
        ok = np.asarray(valid, dtype=bool).copy()
        for i, (v, good) in enumerate(zip(vals, valid)):
            if not good:
                continue
            hit, has_null = in_list(v, self.lits)
            out[i] = hit != self.negated
            ok[i] = hit or not has_null
        return out, ok


class Like:
    dt = P.BOOL

    def __init__(self, col, pattern):
        self.col, self.pattern = col, pattern

    def proto(self):
        return P.like(self.col.proto(), StrLit(self.pattern).proto())

    def eval(self, cols):
        if self.pattern is None:
            n = len(cols[self.col.i][1])
            return np.zeros(n, dtype=bool), np.zeros(n, dtype=bool)
        rx = like_regex(self.pattern)
        return _map(self.col, cols, lambda v: rx.fullmatch(v) is not None)


class StrFunc:
    """starts_with / ends_with / contains (column, literal)"""
    dt = P.BOOL

    def __init__(self, name, col, lit):
        self.name, self.col, self.lit = name, col, lit

    def proto(self):
        return P.scalar_func(self.name, [self.col.proto(), StrLit(self.lit).proto()])

    def eval(self, cols):
        if self.lit is None:
            n = len(cols[self.col.i][1])
            return np.zeros(n, dtype=bool), np.zeros(n, dtype=bool)
        return _map(self.col, cols, lambda v: func(self.name, v, self.lit))
