"""CPU reference for the HashJoin operator (inner, left semi and left anti equi-joins).  Each rule is the reference's:

- Plan shape (native/core/src/execution/planner.rs:2192-2266): HashJoinExec over (left, right) with the key pairs of
  left_join_keys / right_join_keys; BuildRight swaps the inputs so that the right child is the build side, BuildLeft keeps
  the left one.  The output schema does not depend on the build side: an inner join gives the left columns, then the right
  ones; LeftSemi / LeftAnti give the left columns (DataFusion's JoinType output schemas).
- Key equality (planner.rs:2227-2229): NullEquality::NullEqualsNothing -- a row with a NULL in any key equals no row, on
  either side, so it never matches.  An anti join therefore keeps a probe row with a NULL key, a semi or inner join drops it.
- Key values compare as values of their declared type, whatever the physical layout: integers, dates, timestamps and
  decimals (unscaled) numerically, booleans as booleans, strings by their bytes (never by dictionary code).
- Row order: the reference leaves it open.  This project defines it as probe rows in input order and, for an inner join,
  each probe row's matches in build input order -- one of the reference's valid answers, so outputs compare bit-exact.

A key is a column index of its side.  Tables may be dictionary-encoded; the output spells dictionaries out."""
import pyarrow as pa

INNER, LEFT_SEMI, LEFT_ANTI = "inner", "left_semi", "left_anti"


def _array(col):
    col = col.combine_chunks() if isinstance(col, pa.ChunkedArray) else col
    return col.dictionary_decode() if pa.types.is_dictionary(col.type) else col


def key_tuples(table, keys):
    """one tuple of key values per row, None where any key is NULL (NullEqualsNothing)"""
    cols = [_array(table.column(k)).to_pylist() for k in keys]
    out = []
    for vals in zip(*cols) if cols else []:
        out.append(None if any(v is None for v in vals) else tuple(vals))
    return out


def match_pairs(probe_keys, build_keys):
    """(probe row, build row) of every match: probe rows in order, each one's matches in build order"""
    index = {}
    for j, k in enumerate(build_keys):
        if k is not None:
            index.setdefault(k, []).append(j)
    return [(i, j) for i, k in enumerate(probe_keys) if k is not None for j in index.get(k, ())]


def join_table(left, right, left_keys, right_keys, join_type, build_left=False):
    """the operator's output over pa.Tables left and right"""
    if join_type != INNER and build_left:
        raise ValueError("semi / anti joins build the right side")
    lk, rk = key_tuples(left, left_keys), key_tuples(right, right_keys)
    if join_type == INNER:
        if build_left:
            pairs = [(l, r) for r, l in match_pairs(rk, lk)]     # probe = right: its rows in order
        else:
            pairs = match_pairs(lk, rk)
        li = pa.array([p[0] for p in pairs], pa.int64())
        ri = pa.array([p[1] for p in pairs], pa.int64())
        cols = [_array(left.column(i)).take(li) for i in range(left.num_columns)]
        cols += [_array(right.column(i)).take(ri) for i in range(right.num_columns)]
        return pa.table(cols, names=[f"l{i}" for i in range(left.num_columns)] + [f"r{i}" for i in range(right.num_columns)])
    matched = {i for i, _ in match_pairs(lk, rk)}
    keep = [i for i in range(left.num_rows) if (i in matched) == (join_type == LEFT_SEMI)]
    idx = pa.array(keep, pa.int64())
    return pa.table([_array(left.column(i)).take(idx) for i in range(left.num_columns)], names=[f"l{i}" for i in range(left.num_columns)])
