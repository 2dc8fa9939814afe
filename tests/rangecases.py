"""Inputs of the range-partitioning tests: one column per sort-key type with type extremes, -0.0, NaNs of both signs and payloads and
NULLs, and boundary rows drawn from a table's own rows in the keys' order."""
import numpy as np
import pyarrow as pa

import rangeref as R
import sortref
from comet_b200 import proto as P

F64_SPECIAL = [0x8000000000000000, 0x0, 0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000000, 0xFFF0000000000000,
               0x7FF800000000BEEF, 0xFFF0000000000123, 0x7FEFFFFFFFFFFFFF, 0x0000000000000001]
F32_SPECIAL = [0x80000000, 0x0, 0x7FC00000, 0xFFC00000, 0x7F800000, 0xFF800000, 0x7FC0BEEF, 0xFF800123, 0x7F7FFFFF, 0x1]
WORDS = ["", "a", "ab", "b", "B", "é", "zz", "\U0001F601", "a\x00", "w1", "w2", "w10"]


def dec_array(unscaled, p, s, mask=None):
    w = np.zeros((len(unscaled), 2), np.uint64)
    for i, v in enumerate(unscaled):
        v = int(v) & ((1 << 128) - 1)
        w[i] = (v & ((1 << 64) - 1), v >> 64)
    valid = None if mask is None else pa.py_buffer(np.packbits(~np.asarray(mask), bitorder="little"))
    return pa.Array.from_buffers(pa.decimal128(p, s), len(unscaled), [valid, pa.py_buffer(w.tobytes())],
                                 null_count=-1 if mask is not None else 0)


def special_table(n, seed):
    """one column per key type, with type extremes, -0.0, NaNs of both signs and payloads, and about 20% NULLs"""
    rng = np.random.default_rng(seed)
    mask = lambda: rng.random(n) < 0.2
    ints = lambda dt, k: np.concatenate([np.array([np.iinfo(dt).min, np.iinfo(dt).max, 0, -1, 1], dt),
                                         rng.integers(-k, k, n - 5).astype(dt)])
    f64 = np.concatenate([np.array(F64_SPECIAL, np.uint64).view(np.float64), rng.integers(-4, 4, n - len(F64_SPECIAL)) / 2.0])
    f32 = np.concatenate([np.array(F32_SPECIAL, np.uint32).view(np.float32), (rng.integers(-4, 4, n - len(F32_SPECIAL)) / 2.0).astype(np.float32)])
    m38 = 10**38 - 1
    d38 = [m38, -m38, 0, -1, 1] + [int(x) * 10**20 for x in rng.integers(-5, 5, n - 5)]
    d18 = [10**18 - 1, -(10**18 - 1), 0, -1, 1] + [int(x) for x in rng.integers(-5, 5, n - 5)]
    return {
        "b": pa.array(rng.random(n) < 0.5, mask=mask()),
        "i8": pa.array(ints(np.int8, 5), mask=mask()), "i16": pa.array(ints(np.int16, 5), mask=mask()),
        "i32": pa.array(ints(np.int32, 5), mask=mask()), "i64": pa.array(ints(np.int64, 5), mask=mask()),
        "date": pa.array(ints(np.int32, 5), pa.date32(), mask=mask()),
        "ts": pa.array(ints(np.int64, 5), pa.timestamp("us"), mask=mask()),
        "f32": pa.array(f32, mask=mask()), "f64": pa.array(f64, mask=mask()),
        "d18": dec_array(d18, 18, 2, mask()), "d38": dec_array(d38, 38, 4, mask()),
        "s": pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, len(WORDS), n), pa.int32(), mask=mask()), pa.array(WORDS)),
    }


PTYPE = {"b": P.BOOL, "i8": P.INT8, "i16": P.INT16, "i32": P.INT32, "i64": P.INT64, "date": P.DATE, "ts": P.TIMESTAMP,
         "f32": P.FLOAT, "f64": P.DOUBLE, "d18": P.DECIMAL(18, 2), "d38": P.DECIMAL(38, 4), "s": P.STRING}


def pick_bounds(table, keys, nb, seed):
    """nb boundary rows drawn from the table's rows (NULLs, NaNs and extremes included), in the keys' order, duplicates kept"""
    rng = np.random.default_rng(seed)
    take = rng.integers(0, table.num_rows, nb)
    sub = pa.table([R._plain(table.column(c)).take(pa.array(take)) for c, _, _ in keys], names=[f"k{j}" for j in range(len(keys))])
    order = sortref.order(sub, [(f"k{j}", d, f) for j, (_, d, f) in enumerate(keys)])
    return sub.take(pa.array(order))
