"""CPU reference for the SortMergeJoin operator (inner, left / right / full outer, left semi and left anti equi-joins), on top of the
HashJoin reference (tests/joinref.py), whose key rules it shares.  Each rule is the reference's or one of its valid answers:

- Plan shape (native/core/src/execution/planner.rs:2126-2190): SortMergeJoinExec over (left, right) with NullEqualsNothing.  The
  operator probes the side whose order its output keeps: the right one for RightOuter, the left one for every other type.
- Output schema: the left columns, then the right ones, for inner and the outer types; the left columns for LeftSemi / LeftAnti.
- Inner, LeftSemi, LeftAnti: joinref.join_table with BuildRight -- left rows in input order, an inner row's matches in right input order.
- LeftOuter: the same order; a left row without a match appears once, in its place, with NULL right columns.
- RightOuter: right rows in input order, each one's matches in left input order; an unmatched right row once, in its place, with NULL
  left columns.
- FullOuter: everything LeftOuter gives, then the right rows no left row matched (NULL keys included) in right input order, with NULL
  left columns.
On inputs sorted by the keys this is SortMergeJoinExec's own order for every type but FullOuter (whose order Spark leaves open), so
outputs compare bit-exact.  A key is a column index of its side; the output spells dictionaries out."""
import pyarrow as pa

from joinref import INNER, LEFT_ANTI, LEFT_SEMI, _array, join_table, key_tuples, match_pairs

LEFT_OUTER, RIGHT_OUTER, FULL_OUTER = "left_outer", "right_outer", "full_outer"


def _outer_pairs(probe_keys, build_keys):
    """match_pairs, plus (probe row, None) in its place for a probe row without a match"""
    by_probe = {}
    for i, j in match_pairs(probe_keys, build_keys):
        by_probe.setdefault(i, []).append(j)
    return [(i, j) for i in range(len(probe_keys)) for j in by_probe.get(i, [None])]


def sort_merge_join_table(left, right, left_keys, right_keys, join_type):
    """the operator's output over pa.Tables left and right"""
    if join_type in (INNER, LEFT_SEMI, LEFT_ANTI):
        return join_table(left, right, left_keys, right_keys, join_type)
    lk, rk = key_tuples(left, left_keys), key_tuples(right, right_keys)
    if join_type == RIGHT_OUTER:
        pairs = [(l, r) for r, l in _outer_pairs(rk, lk)]     # probe = right: its rows in order
    elif join_type in (LEFT_OUTER, FULL_OUTER):
        pairs = _outer_pairs(lk, rk)
    else:
        raise ValueError(join_type)
    if join_type == FULL_OUTER:
        matched = {r for _, r in pairs}
        pairs += [(None, j) for j in range(right.num_rows) if j not in matched]
    li = pa.array([p[0] for p in pairs], pa.int64())
    ri = pa.array([p[1] for p in pairs], pa.int64())
    cols = [_array(left.column(i)).take(li) for i in range(left.num_columns)]
    cols += [_array(right.column(i)).take(ri) for i in range(right.num_columns)]
    return pa.table(cols, names=[f"l{i}" for i in range(left.num_columns)] + [f"r{i}" for i in range(right.num_columns)])
