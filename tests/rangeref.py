"""CPU reference for range and round-robin repartitioning (ShuffleWriter with RangePartition / RoundRobinPartition).

Range (native/core/src/execution/planner.rs:3298-3358, native/shuffle/src/partitioners/multi_partition.rs:333-380): the sort orders
form a LexOrdering; each boundary row holds one literal per key; a row's partition id is `bounds.partition_point(|b| b <= row)`, the
number of boundary rows less than or equal to the row under the keys' SortOptions.  The value order of each key is sortref's
(tests/sortref.py: numeric, false < true, strings by unsigned bytes, floats by totalOrder, DESC inverts the value, NULLs placed by
nulls_first alone).  Rows keep their input order inside a partition.

Round-robin (planner.rs:3360-3370, multi_partition.rs:386-430): murmur3 (seed 42) chained over the first max_hash_columns columns
(all of them when it is <= 0), pmod num_partitions -- hash partitioning (tests/partref.py) over those columns.

Keys are (column, descending, nulls_first).  Boundary rows are given as a pyarrow table with one column per key, in key order, of the
key's type."""
import numpy as np
import pyarrow as pa

import partref
import sortref


def _plain(arr):
    arr = arr.combine_chunks() if isinstance(arr, pa.ChunkedArray) else arr
    return arr.dictionary_decode() if pa.types.is_dictionary(arr.type) else arr


def _values(table, keys, bounds):
    """per key: (valid, value order) of the table's rows followed by the boundary rows, comparable with each other"""
    out = []
    for j, (c, _, _) in enumerate(keys):
        col = _plain(table.column(c))
        b = _plain(bounds.column(j)).cast(col.type)
        both = pa.concat_arrays([col, b])
        out.append((np.asarray(both.is_valid()), sortref.value_order(both)))
    return out


def _cmp(vals, keys, i, j):
    """-1 / 0 / 1: entry i against entry j of the concatenation, key by key"""
    for (valid, v), (_, desc, nf) in zip(vals, keys):
        a, b = bool(valid[i]), bool(valid[j])
        if not a and not b:
            continue
        if a != b:                                      # the NULL one comes first iff nulls_first
            return (-1 if not a else 1) * (1 if nf else -1)
        x, y = v[i], v[j]
        if x == y:
            continue
        r = -1 if x < y else 1
        return -r if desc else r
    return 0


def brute_pids(table, keys, bounds):
    """partition_point spelled out: for each row, count the boundary rows b with b <= row by a pairwise comparison"""
    n, nb = table.num_rows, bounds.num_rows
    vals = _values(table, keys, bounds)
    return np.array([sum(1 for b in range(nb) if _cmp(vals, keys, n + b, i) <= 0) for i in range(n)], dtype=np.int64)


def _tuple_ranks(table, keys, bounds):
    """one int64 per row and per boundary row whose order is the lexicographic order of the keys (equal iff every key ties)"""
    n = table.num_rows
    cols = []
    for (valid, v), (_, desc, nf) in zip(_values(table, keys, bounds), keys):
        ranks = np.zeros(len(valid), np.int64)
        if valid.any():
            _, inv = np.unique(v[valid], return_inverse=True)
            r = inv.astype(np.int64).reshape(-1)
            ranks[valid] = (r.max() - r if desc else r) + 1
        ranks[~valid] = 0 if nf else int(ranks.max()) + 1
        cols.append(ranks)
    if not cols:
        return np.zeros(n, np.int64), np.zeros(bounds.num_rows, np.int64)
    stacked = np.stack(cols, axis=1)
    _, dense = np.unique(stacked, axis=0, return_inverse=True)      # np.unique over rows orders them lexicographically
    dense = dense.reshape(-1).astype(np.int64)
    return dense[:n], dense[n:]


def range_pids(table, keys, bounds):
    """partition ids: the number of boundary rows <= each row (vectorised: boundary rows must be in non-decreasing order)"""
    rows, bnd = _tuple_ranks(table, keys, bounds)
    assert (np.diff(bnd) >= 0).all(), "boundary rows out of order"
    return np.searchsorted(bnd, rows, side="right").astype(np.int64)


def place(pids, n_parts):
    """(starts, order) of the stable counting sort by partition id"""
    order = np.argsort(pids, kind="stable")
    counts = np.bincount(pids, minlength=n_parts)
    starts = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    return [int(s) for s in starts], order


def _take(table, order):
    idx = pa.array(order, pa.int64())
    return pa.table([_plain(table.column(i)).take(idx) for i in range(table.num_columns)], names=table.column_names)


def range_partition(table, keys, bounds, n_parts):
    """(starts, order, expected output): partition p is rows [starts[p], starts[p + 1]), dictionary columns spelled out"""
    pids = range_pids(table, keys, bounds)
    assert pids.max(initial=0) < n_parts
    starts, order = place(pids, n_parts)
    return starts, order, _take(table, order)


def round_robin_columns(n_cols, max_hash_columns):
    return n_cols if max_hash_columns <= 0 else min(max_hash_columns, n_cols)


def round_robin_partition(o, table, n_parts, max_hash_columns=0):
    k = round_robin_columns(table.num_columns, max_hash_columns)
    h = partref.key_hashes(o, table, list(range(k)))
    pids = pmod(h, n_parts)
    starts, order = place(pids, n_parts)
    return starts, order, _take(table, order)


def pmod(h, n):
    """Spark's pmod of the signed 32-bit hashes h (uint32)"""
    s = h.astype(np.uint32).view(np.int32).astype(np.int64)
    return np.mod(s, n)


def bound_literals(P, bounds, types):
    """the boundary rows as lists of proto literals (`types`: the proto type of each key); floats are sent by their bits"""
    rows = []
    for r in range(bounds.num_rows):
        row = []
        for j, t in enumerate(types):
            arr = _plain(bounds.column(j))
            v = arr[r]
            if not v.is_valid:
                row.append(P.literal(None, t))
            elif t.name in ("FLOAT", "DOUBLE"):
                bits = np.uint32 if t.name == "FLOAT" else np.uint64
                raw = np.frombuffer(arr.buffers()[1], dtype=bits)[arr.offset + r]
                row.append(P.literal_bits(int(raw), t))
            elif t.name == "DECIMAL":
                w = np.frombuffer(arr.buffers()[1], dtype=np.uint64)[(arr.offset + r) * 2:(arr.offset + r) * 2 + 2]
                unscaled = int(w[0]) | (int(w[1]) << 64)
                row.append(P.literal(unscaled - (1 << 128) if unscaled >> 127 else unscaled, t))
            elif t.name in ("DATE", "TIMESTAMP"):
                raw = np.frombuffer(arr.buffers()[1], dtype=np.int32 if t.name == "DATE" else np.int64)[arr.offset + r]
                row.append(P.literal(int(raw), t))
            else:
                row.append(P.literal(v.as_py(), t))
        rows.append(row)
    return rows
