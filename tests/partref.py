"""CPU reference for hash repartitioning (ShuffleWriter with HashPartitioning): Spark murmur3 (seed 42) chained over the key
columns, pmod, and a stable counting sort.  Every hash and the sort come from the oracle (murmur3_column / murmur3_strings /
partition_rows), which tests/test_oracle_kat.py pins to the reference's known-answer tests; this module only maps Arrow columns
onto the oracle's value kinds and spells the expected output out.

Key kinds by Arrow type (spark-expr/src/hash_funcs/utils.rs):
  bool -> bool, int8 -> i8, int16 -> i16, int32 -> i32, date32 -> date32, int64 -> i64, timestamp[us] -> timestamp,
  float32 -> f32, float64 -> f64, decimal p <= 18 -> dec_small, decimal p > 18 -> dec_large,
  string / dictionary<string> -> murmur3_strings over the spelled-out values.
A NULL leaves the running hash unchanged (utils.rs:38-42)."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc


def oracle_kind(t):
    """the oracle's murmur3 kind for Arrow type t, or "str" for strings hashed as their bytes"""
    if pa.types.is_dictionary(t):
        if not pa.types.is_string(t.value_type):
            raise TypeError(f"dictionary of {t.value_type}")
        return "str"
    if pa.types.is_string(t):
        return "str"
    if pa.types.is_decimal(t):
        return "dec_small" if t.precision <= 18 else "dec_large"
    if pa.types.is_timestamp(t):
        if t.unit != "us":
            raise TypeError(f"timestamp unit {t.unit}")
        return "timestamp"
    kinds = {pa.bool_(): "bool", pa.int8(): "i8", pa.int16(): "i16", pa.int32(): "i32", pa.date32(): "date32", pa.int64(): "i64",
             pa.float32(): "f32", pa.float64(): "f64"}
    if t not in kinds:
        raise TypeError(f"no hash kind for {t}")
    return kinds[t]


def _array(col):
    return col.combine_chunks() if isinstance(col, pa.ChunkedArray) else col


def plain(arr):
    """a dictionary-encoded string column spelled out as plain strings (what the hand-off exports); other columns as they are"""
    arr = _array(arr)
    return arr.dictionary_decode() if pa.types.is_dictionary(arr.type) else arr


def _fixed(arr, dtype, width=1):
    """the value buffer of a fixed-width array as numpy, `width` elements of dtype per row"""
    buf = arr.buffers()[1]
    v = np.frombuffer(buf, dtype=dtype)
    return v[arr.offset * width:(arr.offset + len(arr)) * width]


def hash_column(o, arr, hashes):
    """fold one key column into the running hashes (uint32, updated in place and returned)"""
    arr = plain(arr)
    kind = oracle_kind(arr.type)
    valid = np.asarray(arr.is_valid(), dtype=np.uint8)
    n = len(arr)
    if kind == "str":
        arr = arr.cast(pa.string())
        offs = np.frombuffer(arr.buffers()[1], dtype=np.int32)[arr.offset:arr.offset + n + 1].copy()
        data = np.frombuffer(arr.buffers()[2], dtype=np.uint8) if arr.buffers()[2] is not None else np.zeros(0, np.uint8)
        data = np.concatenate([data, np.zeros(1, np.uint8)])    # a non-NULL pointer for all-empty columns
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        o.lib().co_murmur3_strings(C.c_int64(n), p(offs), p(data), p(valid), p(hashes))
        return hashes
    if kind == "bool":
        values = np.asarray(arr.fill_null(False), dtype=np.uint8)
    elif kind in ("dec_small", "dec_large"):
        values = _fixed(arr, np.uint64, 2).reshape(-1, 2).copy()
        values[valid == 0] = 0                                  # garbage under a NULL is never hashed, but must fit i64 for dec_small
    elif kind == "date32":
        values = _fixed(arr, np.int32)
    elif kind == "timestamp":
        values = _fixed(arr, np.int64)
    else:
        values = _fixed(arr, np.dtype(arr.type.to_pandas_dtype()))
    return o.murmur3_column(kind, values, valid=valid, hashes=hashes)


def key_hashes(o, table, keys):
    """murmur3 (seed 42) of each row chained over the key columns, in order"""
    h = np.full(table.num_rows, 42, dtype=np.uint32)
    for k in keys:
        hash_column(o, table.column(k), h)
    return h


def partition(o, table, keys, n_parts):
    """(starts, row order, expected output table): partition p is rows [starts[p], starts[p + 1]) of the output, and the output is
    the input's rows in `order` -- partition by partition, input order inside each.  Dictionary columns come out spelled out."""
    h = key_hashes(o, table, keys)
    _, starts, order = o.partition_rows(h, n_parts)
    cols = [plain(table.column(i)).take(pa.array(order)) for i in range(table.num_columns)]
    return [int(s) for s in starts], order, pa.table(cols, names=table.column_names)


def assert_columns_equal(got, want, what=""):
    """every row of two columns equal: validity, values bit-exact (floats by their bits, so NaN payloads and -0.0 count), strings in
    full.  `want` may be dictionary-encoded (compared spelled out) and of a narrower timestamp zone / decimal view than `got`."""
    got, want = plain(got), plain(want)
    assert len(got) == len(want), (what, len(got), len(want))
    gnull, wnull = np.asarray(got.is_null()), np.asarray(want.is_null())
    assert (gnull == wnull).all(), (what, "validity", int(np.argmax(gnull != wnull)))
    ok = ~wnull
    if pa.types.is_floating(want.type):
        bits = np.uint32 if want.type == pa.float32() else np.uint64
        g, w = _fixed(got, bits), _fixed(want, bits)
        bad = (g != w) & ok
        assert not bad.any(), (what, "value", int(np.argmax(bad)), g[np.argmax(bad)], w[np.argmax(bad)])
    elif pa.types.is_string(want.type):
        eq = pc.equal(got.cast(pa.string()), want.cast(pa.string()))
        bad = ~np.asarray(eq.fill_null(True))
        assert not bad.any(), (what, "value", int(np.argmax(bad)))
    elif pa.types.is_boolean(want.type):
        g, w = np.asarray(got.fill_null(False)), np.asarray(want.fill_null(False))
        bad = (g != w) & ok
        assert not bad.any(), (what, "value", int(np.argmax(bad)))
    else:
        if pa.types.is_decimal(want.type):
            g, w = _fixed(got, np.uint64, 2).reshape(-1, 2), _fixed(want, np.uint64, 2).reshape(-1, 2)
            bad = (g != w).any(axis=1) & ok
        else:
            dt = {4: np.int32, 8: np.int64, 2: np.int16, 1: np.int8}[want.type.bit_width // 8]
            assert got.type.bit_width == want.type.bit_width, (what, got.type, want.type)
            g, w = _fixed(got, dt), _fixed(want, dt)
            bad = (g != w) & ok
        assert not bad.any(), (what, "value", int(np.argmax(bad)))


def assert_tables_equal(got, want):
    assert got.num_rows == want.num_rows, (got.num_rows, want.num_rows)
    assert got.num_columns == want.num_columns
    for j in range(want.num_columns):
        assert_columns_equal(got.column(j), want.column(j), want.column_names[j])
