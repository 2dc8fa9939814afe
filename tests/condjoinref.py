"""CPU reference for join conditions (HashJoinExec / SortMergeJoinExec with a JoinFilter, planner.rs:2462-2542), on top of the HashJoin
and SortMergeJoin references (tests/joinref.py, tests/smjref.py), whose key rules and row orders it keeps.  Each rule is the reference's:

- The condition is bound to the left columns followed by the right ones (operators.scala:2634-2640), whatever the build side and the
  join type: a semi / anti join's condition may read right columns although its output has none.
- A candidate is a (left row, right row) pair whose keys are equal (NullEqualsNothing: a NULL key matches nothing).  It passes when the
  condition is TRUE; FALSE and NULL fail.
- The condition is evaluated on candidates only -- never on a NULL-extended row -- so an ANSI error is raised only when a candidate
  raises it.
- "Match" in the join's rules now means "passing candidate":
  Inner: probe rows in input order, each one's passing candidates in build input order.
  LeftOuter: the same; a left row with no passing candidate (none at all, or all failed) once, in its place, with NULL right columns.
  RightOuter: the mirror.  FullOuter: LeftOuter's output, then every right row in no passing candidate, in right input order.
  LeftSemi: the left rows with a passing candidate; LeftAnti: every other left row (NULL keys included).

Conditions are tests/exprs.py / tests/strpred_ref.py nodes over columns (values, validity) of left ++ right; cond=None is no condition."""
from decimal import Decimal

import numpy as np
import pyarrow as pa

from joinref import INNER, LEFT_ANTI, LEFT_SEMI, _array, key_tuples, match_pairs
from smjref import FULL_OUTER, LEFT_OUTER, RIGHT_OUTER
from oracle import oracle as O


def _unscaled(v, scale):
    sign, digits, exp = v.as_tuple()
    n = int("".join(map(str, digits)) or "0") * 10 ** (exp + scale)
    return -n if sign else n


def node_columns(table):
    """the columns of a pa.Table as the expression nodes read them: (values, validity) per column"""
    out = []
    for i in range(table.num_columns):
        a = _array(table.column(i))
        valid = np.asarray(a.is_valid(), dtype=bool) if len(a) else np.zeros(0, bool)
        t = a.type
        if pa.types.is_decimal(t):
            out.append((O.dec_from_ints([_unscaled(v, t.scale) if isinstance(v, Decimal) else 0 for v in a.to_pylist()]), valid))
        elif pa.types.is_string(t) or pa.types.is_binary(t):
            out.append((np.array([v if v is not None else "" for v in a.to_pylist()], dtype=object), valid))
        elif pa.types.is_boolean(t):
            out.append((np.asarray(a.fill_null(False), dtype=bool), valid))
        elif pa.types.is_floating(t):
            out.append((np.asarray(a.fill_null(0)), valid))
        elif pa.types.is_date32(t):
            out.append((np.asarray(a.cast(pa.int32()).fill_null(0)).astype(np.int64), valid))
        elif pa.types.is_timestamp(t):
            out.append((np.asarray(a.cast(pa.int64()).fill_null(0)).astype(np.int64), valid))
        else:
            out.append((np.asarray(a.fill_null(0)).astype(np.int64), valid))
    return out


def pair_table(left, right, pairs):
    """left ++ right columns of (left row, right row) pairs, None = a NULL-extended side"""
    li = pa.array([p[0] for p in pairs], pa.int64())
    ri = pa.array([p[1] for p in pairs], pa.int64())
    cols = [_array(left.column(i)).take(li) for i in range(left.num_columns)]
    cols += [_array(right.column(i)).take(ri) for i in range(right.num_columns)]
    return pa.table(cols, names=[f"l{i}" for i in range(left.num_columns)] + [f"r{i}" for i in range(right.num_columns)])


def passes(left, right, pairs, cond):
    """the condition over candidate pairs: TRUE per pair (raises what the candidates raise)"""
    if cond is None:
        return [True] * len(pairs)
    if not pairs:
        return []
    v, valid = cond.eval(node_columns(pair_table(left, right, pairs)))
    return list(np.asarray(v, dtype=bool) & np.asarray(valid, dtype=bool))


def candidates(left, right, left_keys, right_keys, join_type, build_left=False):
    """the candidate pairs (left row, right row) in the operator's probe order"""
    lk, rk = key_tuples(left, left_keys), key_tuples(right, right_keys)
    if join_type == RIGHT_OUTER or (join_type == INNER and build_left):
        return [(l, r) for r, l in match_pairs(rk, lk)]     # probe = right: its rows in order
    return match_pairs(lk, rk)


def resolve(n_left, n_right, cands, ok, join_type, build_left=False):
    """the output rows from the candidates and their pass flags: (left row | None, right row | None) pairs, or left rows (semi / anti)"""
    passing = [c for c, p in zip(cands, ok) if p]
    if join_type == INNER:
        return passing
    if join_type in (LEFT_SEMI, LEFT_ANTI):
        hit = {l for l, _ in passing}
        return [i for i in range(n_left) if (i in hit) == (join_type == LEFT_SEMI)]
    if join_type == RIGHT_OUTER:
        by = {}
        for l, r in passing:
            by.setdefault(r, []).append(l)
        return [(l, r) for r in range(n_right) for l in by.get(r, [None])]
    by = {}
    for l, r in passing:
        by.setdefault(l, []).append(r)
    out = [(l, r) for l in range(n_left) for r in by.get(l, [None])]
    if join_type == FULL_OUTER:
        matched = {r for _, r in passing}
        out += [(None, r) for r in range(n_right) if r not in matched]
    return out


def output_rows(left, right, left_keys, right_keys, join_type, cond, build_left=False):
    """(output rows as resolve gives them, candidates the condition was evaluated on)"""
    if build_left and join_type != INNER:
        raise ValueError("only an inner hash join builds the left side")
    cands = candidates(left, right, left_keys, right_keys, join_type, build_left)
    return resolve(left.num_rows, right.num_rows, cands, passes(left, right, cands, cond), join_type, build_left), len(cands)


def to_table(left, right, rows, join_type):
    if join_type in (LEFT_SEMI, LEFT_ANTI):
        idx = pa.array(rows, pa.int64())
        return pa.table([_array(left.column(i)).take(idx) for i in range(left.num_columns)], names=[f"l{i}" for i in range(left.num_columns)])
    return pair_table(left, right, rows)


def cond_join_table(left, right, left_keys, right_keys, join_type, cond, build_left=False):
    """the operator's output over pa.Tables left and right"""
    rows, _ = output_rows(left, right, left_keys, right_keys, join_type, cond, build_left)
    return to_table(left, right, rows, join_type)


def candidate_count(left, right, left_keys, right_keys, join_type, build_left=False):
    """the candidates the condition is evaluated on (join_cond_pairs); none when a side is empty"""
    if left.num_rows == 0 or right.num_rows == 0:
        return 0
    return len(candidates(left, right, left_keys, right_keys, join_type, build_left))
