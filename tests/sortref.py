"""CPU reference for the Sort operator (ORDER BY and TopK).  Each rule is the reference's:

- Plan shape (native/core/src/execution/planner.rs:1488-1522): SortExec(LexOrdering(keys)).with_fetch(fetch), then
  GlobalLimitExec(skip) when skip > 0, so the output is sorted[skip : fetch] (sorted[skip:] without a fetch).  TopK
  (spark/.../CometExecUtils.scala:132-162 getTopKNativePlan) is the same message with fetch = limit, skip = offset.
- Keys (planner.rs:927-950 create_sort_expr): direction 1 is DESC, null_ordering 0 is NULLS FIRST, giving arrow
  SortOptions{descending, nulls_first}.  Null placement does not depend on the direction.
- Value order, arrow-rs arrow-ord (what DataFusion's SortExec uses): integers, dates and timestamps numerically; decimals by
  their signed unscaled value; booleans false < true; strings by unsigned bytes; floats by IEEE totalOrder
  (f32::total_cmp / f64::total_cmp: -NaN < -Inf < ... < -0.0 < +0.0 < ... < +Inf < +NaN, NaN sign and payload counted, nothing
  normalised -- docs/source/user-guide/latest/compatibility/floating-point.md; spark/.../serde/CometSortOrder.scala marks float keys
  incompatible for that reason).
- Ties: the reference leaves their order open; this project defines it as the input order (a stable sort), one of the reference's
  valid answers.

A key is (column, descending, nulls_first); column is a name or an index.  Each key becomes one int64 per row whose order is the key's
order (null rank, then the dense rank of the value, inverted for DESC); rows are ordered by stable sorts from the last key to the
first."""
import numpy as np
import pyarrow as pa


def _array(col):
    col = col.combine_chunks() if isinstance(col, pa.ChunkedArray) else col
    return col.dictionary_decode() if pa.types.is_dictionary(col.type) else col


def _fixed(arr, dtype, width=1):
    v = np.frombuffer(arr.buffers()[1], dtype=dtype)
    return v[arr.offset * width:(arr.offset + len(arr)) * width]


def value_order(arr):
    """an array whose numpy order is the reference's value order of arr's valid rows (NULL rows: anything)"""
    t = arr.type
    if pa.types.is_floating(t):
        u = _fixed(arr, np.uint32 if t == pa.float32() else np.uint64).astype(np.uint64)
        sign = np.uint64(1 << (t.bit_width - 1))
        mask = np.uint64((1 << t.bit_width) - 1)
        return np.where(u & sign, ~u & mask, u | sign)                         # totalOrder
    if pa.types.is_decimal(t):
        w = _fixed(arr, np.uint64, 2).reshape(-1, 2)
        lo = w[:, 0].view(np.int64)
        if (w[:, 1].view(np.int64) == lo >> 63).all():                         # every value fits i64
            return lo
        return np.array([(int(hi) << 64 | int(lo)) - ((int(hi) >> 63) << 128) for lo, hi in w], dtype=object)
    if pa.types.is_string(t) or pa.types.is_large_string(t) or pa.types.is_binary(t):
        return np.array([b"" if v is None else v for v in arr.cast(pa.binary()).to_pylist()], dtype=object)   # unsigned bytes
    if pa.types.is_boolean(t):
        return np.asarray(arr.fill_null(False), dtype=np.int64)
    if pa.types.is_date32(t) or pa.types.is_timestamp(t) or pa.types.is_integer(t):
        return _fixed(arr, {1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}[t.bit_width // 8]).astype(np.int64)
    raise TypeError(f"no sort order for {t}")


def key_ranks(arr, descending=False, nulls_first=True):
    """one int64 per row, ordered as the key orders rows; equal iff the rows tie on this key"""
    arr = _array(arr)
    valid = np.asarray(arr.is_valid())
    v = value_order(arr)
    ranks = np.zeros(len(arr), np.int64)
    if valid.any():
        _, inv = np.unique(v[valid], return_inverse=True)
        r = inv.astype(np.int64).reshape(-1)
        ranks[valid] = (r.max() - r if descending else r) + 1                 # 1 .. distinct values
    top = int(ranks.max()) + 1 if len(ranks) else 1
    ranks[~valid] = 0 if nulls_first else top
    return ranks


def _col(table, c):
    return table.column(c)


def order(table, keys):
    """the stable order of the rows: row indices"""
    idx = np.arange(table.num_rows)
    for c, desc, nf in reversed(keys):
        r = key_ranks(_col(table, c), desc, nf)
        idx = idx[np.argsort(r[idx], kind="stable")]
    return idx


def window(n, fetch=None, skip=None):
    """rows [lo, hi) of the sorted order the operator returns"""
    lo = min(skip or 0, n)
    hi = n if fetch is None else min(fetch, n)
    return lo, max(lo, hi)


def sort_table(table, keys, fetch=None, skip=None):
    """the operator's output: the rows of sorted[skip : fetch], dictionary columns spelled out"""
    idx = order(table, keys)
    lo, hi = window(len(idx), fetch, skip)
    take = pa.array(idx[lo:hi], pa.int64())
    return pa.table([_array(table.column(i)).take(take) for i in range(table.num_columns)], names=table.column_names)


def assert_sorted(table, keys):
    """the rows of `table` are in the keys' order (the comparator alone: no tie-break needed)"""
    if table.num_rows < 2:
        return
    cols = [key_ranks(_col(table, c), desc, nf) for c, desc, nf in keys]
    undecided = np.ones(table.num_rows - 1, bool)                             # adjacent pairs equal on all keys so far
    for r in cols:
        a, b = r[:-1], r[1:]
        bad = undecided & (a > b)
        assert not bad.any(), ("out of order at row", int(np.argmax(bad)))
        undecided &= a == b
