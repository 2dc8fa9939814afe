"""GPU: hash repartitioning (ShuffleWriter with HashPartitioning) against the CPU reference (tests/partref.py) for every key type and
every physical layout a source hands the partitioner: Arrow streams (booleans as bitmaps, dictionaries with int8 / int16 / int32
indices, remapped or not), device tables (8-byte decimals), the Parquet scan (INT32-backed int8 / int16 / decimal(7, 2), INT64 and
FLBA decimals) and partial-aggregate state (booleans one byte per row).  Every case compares every output column -- values bit-exact,
floats by their bits, validity, strings in full -- and the partition starts."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import partref

pytestmark = pytest.mark.gpu

@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


WORDS = ["", "a", "ab", "abc", "abcd", "abcde", "abcdef", "abcdefg", "abcdefgh", "abcdefghi",   # every mm3_bytes tail length
         "é", "aé", "abcdé", "ÿ", "\U0001F601", "天地人", "x\u0080y", "zz\U0010FFFF"]          # tail bytes >= 0x80, multibyte UTF-8
WORDS += [f"w{i:03d}" for i in range(100 - len(WORDS))]                                        # 100 entries: fits int8 indices


def _dec(vals, p, s, mask=None):
    """a decimal128(p, s) array of the unscaled values: an int64 array, or (lo, hi) 64-bit words of each 128-bit value"""
    lo, hi = vals if isinstance(vals, tuple) else (vals, vals >> 63)
    words = np.empty((len(lo), 2), np.int64)
    words[:, 0], words[:, 1] = lo, hi
    nulls = 0 if mask is None else int(mask.sum())
    validity = pa.py_buffer(np.packbits(~mask, bitorder="little")) if nulls else None
    return pa.Array.from_buffers(pa.decimal128(p, s), len(lo), [validity, pa.py_buffer(words.tobytes())], null_count=nulls)


def _words(ints):
    """python ints -> (lo, hi) int64 words of their 128-bit two's complement"""
    u = [int(v) & ((1 << 128) - 1) for v in ints]
    return (np.array([x & ((1 << 64) - 1) for x in u], np.uint64).view(np.int64), np.array([x >> 64 for x in u], np.uint64).view(np.int64))


def _dec_values(rng, n, p):
    """unscaled decimal(p) values, random in range, with +-(10^p - 1), 0, -1 and 1 among them (p > 18: as (lo, hi) words)"""
    special = [10**p - 1, -(10**p - 1), 0, -1, 1]
    if p <= 18:
        return _specials(rng, n, rng.integers(-(10**p - 1), 10**p, n, dtype=np.int64), np.array(special, np.int64))
    lo = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64, endpoint=True)
    hi = rng.integers(-(10**(p - 20)), 10**(p - 20), n, dtype=np.int64)   # |hi * 2^64 + lo| < 10^p
    sl, sh = _words(special)
    k = min(n, len(special))
    lo[:k], hi[:k] = sl[:k], sh[:k]
    if n > 2 * len(special):
        at = rng.choice(n, len(special), replace=False)
        lo[at], hi[at] = sl, sh
    return lo, hi


def _specials(rng, n, base, specials):
    """base with the special values at the start (as many as fit) and again at random rows"""
    v = np.array(base)
    k = min(n, len(specials))
    v[:k] = specials[:k]
    if n > 2 * len(specials):
        v[rng.choice(n, len(specials), replace=False)] = specials
    return v


F64_SPECIAL = np.array([0x0000000000000000, 0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FF8000000000000,
                        0xFFF8000000000000, 0x7FF8DEADBEEF0001, 0xFFF0000000000123, 0x0000000000000001, 0x800FFFFFFFFFFFFF],
                       dtype=np.uint64).view(np.float64)   # +-0, +-Inf, NaNs with distinct payloads and signs, subnormals
F32_SPECIAL = np.array([0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7FC0BEEF, 0xFF800123, 0x00000001,
                        0x807FFFFF], dtype=np.uint32).view(np.float32)


def make_values(n, seed):
    """one column per key type (name -> (arrow array, proto type)), NULLs at different rows in each, MIN / MAX / +-0.0 / +-Inf / NaN
    payloads / subnormals / decimal +-(10^p - 1), 0, -1 / strings of every tail length among the values; plus "row" = the row number"""
    import comet_b200.proto as P
    rng = np.random.default_rng(seed)
    mask = lambda: rng.random(n) < 0.12
    ints = lambda dt: _specials(rng, n, rng.integers(np.iinfo(dt).min, np.iinfo(dt).max, n, dtype=dt, endpoint=True),
                                np.array([np.iinfo(dt).min, np.iinfo(dt).max, 0, -1, 1], dtype=dt))
    codes = lambda: rng.integers(0, len(WORDS), n)
    cols = {
        "b": (pa.array(rng.random(n) < 0.5, mask=mask()), P.BOOL),
        "i8": (pa.array(ints(np.int8), mask=mask()), P.INT8),
        "i16": (pa.array(ints(np.int16), mask=mask()), P.INT16),
        "i32": (pa.array(ints(np.int32), mask=mask()), P.INT32),
        "date": (pa.array(rng.integers(-30000, 30000, n).astype(np.int32), type=pa.date32(), mask=mask()), P.DATE),
        "i64": (pa.array(ints(np.int64), mask=mask()), P.INT64),
        "ts": (pa.array(ints(np.int64), type=pa.timestamp("us", tz="UTC"), mask=mask()), P.TIMESTAMP),
        "f32": (pa.array(_specials(rng, n, rng.standard_normal(n).astype(np.float32), F32_SPECIAL), mask=mask()), P.FLOAT),
        "f64": (pa.array(_specials(rng, n, rng.standard_normal(n), F64_SPECIAL), mask=mask()), P.DOUBLE),
        "d9": (_dec(_dec_values(rng, n, 9), 9, 2, mask()), P.DECIMAL(9, 2)),
        "d18": (_dec(_dec_values(rng, n, 18), 18, 0, mask()), P.DECIMAL(18, 0)),
        "d38": (_dec(_dec_values(rng, n, 38), 38, 4, mask()), P.DECIMAL(38, 4)),
        "s8": (pa.DictionaryArray.from_arrays(pa.array(codes(), pa.int8(), mask=mask()), pa.array(WORDS)), P.STRING),
        "s16": (pa.DictionaryArray.from_arrays(pa.array(codes(), pa.int16(), mask=mask()), pa.array(WORDS)), P.STRING),
        "s32": (pa.DictionaryArray.from_arrays(pa.array(codes(), pa.int32(), mask=mask()), pa.array(WORDS)), P.STRING),
        "row": (pa.array(np.arange(n, dtype=np.int64)), P.INT64),
    }
    return cols


def table_of(cols, names=None):
    names = names or list(cols)
    return pa.table({k: cols[k][0] for k in names}), [cols[k][1] for k in names]


def hash_plan(cb, child, types, names, keys, n_parts):
    P = cb.proto
    if n_parts is None:  # SinglePartition
        return P._op("shuffle_writer", P.f_len(1, P.f_len(2, b"")), (child,))
    return P.shuffle_writer(child, P.hash_partitioning([P.bound(names.index(k), types[names.index(k)]) for k in keys], n_parts))


def run(cb, plan, inputs, config=None):
    """every batch the plan returns, each with the partition starts that came with it"""
    out = []
    with cb.native.Plan(plan, inputs, config=config) as p:
        while True:
            b = p.execute()
            if b is None:
                break
            out.append((b, p.partition_starts()))
    return out


def check(oracle, got, tbl, keys, n_parts):
    """got: [(batch, starts)] of one plan over tbl -- each batch the partitioning of its own input rows, in input order"""
    n_eff = 1 if n_parts is None else n_parts
    row0 = 0
    for b, starts in got:
        part = tbl.slice(row0, b.num_rows)
        want_starts, _, want = partref.partition(oracle, part, keys, n_eff)
        assert starts == want_starts, (row0, b.num_rows)
        partref.assert_tables_equal(b, want)
        row0 += b.num_rows
    assert row0 == tbl.num_rows


def supports(cb, plan):
    from comet_b200 import native
    err = native._Error()
    ok = native.lib().cb200_supports(plan, len(plan), C.byref(err))
    return ok, err.code, err.message.decode(errors="replace")


def stream_case(cb, oracle, n, keys, n_parts, names=None, seed=1, chunk=8192, config=None):
    cols = make_values(n, seed)
    tbl, types = table_of(cols, names)
    plan = hash_plan(cb, cb.proto.scan(types), types, tbl.column_names, keys, n_parts)
    inputs = [tbl.to_batches(max_chunksize=chunk)] if n else [tbl]
    got = run(cb, plan, inputs, config)
    check(oracle, got, tbl, keys, n_parts)
    return got


ALL = ["b", "i8", "i16", "i32", "date", "i64", "ts", "f32", "f64", "d9", "d18", "d38", "s8", "s16", "s32"]


# ---- Arrow streams -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", ALL)
def test_stream_each_key_type(cb, oracle, key):
    stream_case(cb, oracle, 50_000, [key], 200, seed=ALL.index(key) + 10)


@pytest.mark.parametrize("keys,n_parts", [("i8+i16", 7), ("b+f32+s8", 2), ("d9+d38+ts+f64", 4096),
                                          ("s16+i32+date+b+d18", 6144),
                                          ("i8+i16+i32+i64+f32+f64+s32+d38", 200),
                                          ("b+i8+date+ts+d9+d18+s8+s16", 6145)])
def test_stream_key_combinations(cb, oracle, keys, n_parts):
    """up to 8 keys; every column has its own NULL rows, so rows have NULLs in different key positions"""
    keys = keys.split("+")
    stream_case(cb, oracle, 50_000, keys, n_parts, seed=len(keys) * 7 + n_parts)


@pytest.mark.parametrize("n", [1, 31, 1023, 1024, 1025, 50_000, 3 * 2**20 + 17])
def test_stream_sizes(cb, oracle, n):
    """row blocks of 1024 rows and chunks of 1024 blocks: 3 * 2^20 + 17 rows make four chunks, the last one partial"""
    n_parts = 6145 if n > 2**20 else 200
    stream_case(cb, oracle, n, ["i32", "s16", "f64", "b"], n_parts, names=["b", "i8", "i32", "f64", "d18", "d38", "s16", "row"], seed=n % 97,
                chunk=1 << 16)


@pytest.mark.parametrize("n_parts", [None, 1, 2, 7, 4096, 6144, 6145, 16384])
def test_partition_counts(cb, oracle, n_parts):
    """None = SinglePartition; above 6144 partitions the per-partition counters need more than the default 48 KB of shared memory"""
    got = stream_case(cb, oracle, 120_000, ["i64", "s32"], n_parts, names=["i64", "s32", "f64", "d9", "row"], seed=3)
    assert len(got[0][1]) == (1 if n_parts is None else n_parts) + 1


@pytest.mark.parametrize("n_parts", [16385, 20_000])
def test_too_many_partitions_refused(cb, n_parts):
    P = cb.proto
    plan = P.shuffle_writer(P.scan([P.INT64]), P.hash_partitioning([P.bound(0, P.INT64)], n_parts))
    ok, code, msg = supports(cb, plan)
    assert not ok and code == 1 and "partitions" in msg
    with pytest.raises(cb.native.Unsupported):
        run(cb, plan, [pa.table({"a": pa.array([1, 2, 3], pa.int64())})])


def test_nine_keys_refused(cb):
    P = cb.proto
    types = [P.INT32] * 9
    plan = P.shuffle_writer(P.scan(types), P.hash_partitioning([P.bound(i, P.INT32) for i in range(9)], 8))
    ok, code, msg = supports(cb, plan)
    assert not ok and code == 1 and "8 hash-partition keys" in msg
    eight = P.shuffle_writer(P.scan(types), P.hash_partitioning([P.bound(i, P.INT32) for i in range(8)], 8))
    assert supports(cb, eight)[0]


@pytest.mark.parametrize("index", [pa.int8(), pa.int16(), pa.int32()])
@pytest.mark.parametrize("remap", [False, True])
def test_dictionary_streams(cb, oracle, index, remap):
    """each record batch carries its own dictionary: the same one (codes pass through at their width) or a shuffled one (codes remapped
    to the plan's dictionary, int32)"""
    P = cb.proto
    rng = np.random.default_rng(5)
    n, per = 40_000, 5_000
    batches, plain = [], []
    for k in range(n // per):
        order = rng.permutation(len(WORDS)) if remap and k else np.arange(len(WORDS))
        d = pa.array([WORDS[i] for i in order])
        codes = rng.integers(0, len(WORDS), per)
        mask = rng.random(per) < 0.1
        s = pa.DictionaryArray.from_arrays(pa.array(codes, index, mask=mask), d)
        v = pa.array(rng.integers(-2**31, 2**31, per).astype(np.int32))
        batches.append(pa.record_batch([s, v], names=["s", "v"]))
        plain.append(pa.record_batch([s.dictionary_decode(), v], names=["s", "v"]))
    tbl = pa.Table.from_batches(plain)
    for keys in (["s"], ["v", "s"]):
        plan = hash_plan(cb, P.scan([P.STRING, P.INT32]), [P.STRING, P.INT32], ["s", "v"], keys, 200)
        check(oracle, run(cb, plan, [batches]), tbl, keys, 200)


# ---- empty input and several batches ---------------------------------------------------------------------------------------------------
def test_empty_input(cb, oracle):
    """an empty stream produces no batch (and no launch); a batch whose rows a filter removes produces a zero-row batch, all starts 0"""
    P = cb.proto
    cols = make_values(0, 1)
    tbl, types = table_of(cols, ["i32", "s16", "d9"])
    plan = hash_plan(cb, P.scan(types), types, tbl.column_names, ["i32"], 7)
    with cb.native.Plan(plan, [tbl]) as p:
        assert p.execute() is None
        assert p.partition_starts() == []
        assert p.kernel_launches == 0
    cols = make_values(1000, 1)
    tbl, types = table_of(cols, ["i32", "s16", "d9", "row"])
    never = P.filter_(P.scan(types), P.is_null(P.bound(3, P.INT64)))        # "row" has no NULLs
    got = run(cb, hash_plan(cb, never, types, tbl.column_names, ["i32"], 7), [tbl.to_batches(max_chunksize=256)])
    assert len(got) == 1
    b, starts = got[0]
    assert b.num_rows == 0 and b.num_columns == 4 and starts == [0] * 8


def test_chunks_smaller_than_the_input(cb, oracle):
    """spark.comet.b200.chunkRows below the input: each batch is the partitioning of its own rows, with its own starts"""
    got = stream_case(cb, oracle, 70_000, ["i16", "s8", "d38"], 13, names=["b", "i16", "s8", "d38", "f32", "row"], seed=9, chunk=3000,
                      config={"spark.comet.b200.chunkRows": "20000"})
    assert len(got) == 4


# ---- device tables ----------------------------------------------------------------------------------------------------------------------
def device_table(cb, tbl, types, dec8=()):
    """tbl's columns as caller-owned device buffers: booleans as bitmaps, dictionaries as their codes, decimals named in dec8 as 8 bytes"""
    import torch
    t = cb.native.DeviceTable(tbl.num_rows)
    for name, dt in zip(tbl.column_names, types):
        a = tbl.column(name).combine_chunks()
        valid = np.asarray(a.is_valid())
        vbits = np.packbits(valid, bitorder="little")
        vdev = torch.from_numpy(np.concatenate([vbits, np.zeros(16, np.uint8)])).cuda() if a.null_count else None
        dictionary = None
        if pa.types.is_boolean(a.type):
            raw, width = np.packbits(np.asarray(a.fill_null(False)), bitorder="little"), 0
        elif pa.types.is_dictionary(a.type):
            idx = a.indices
            width = idx.type.bit_width // 8
            raw = np.frombuffer(idx.buffers()[1], dtype=np.uint8)[idx.offset * width:(idx.offset + len(idx)) * width]
            dictionary = a.dictionary.to_pylist()
        elif pa.types.is_decimal(a.type):
            v = np.frombuffer(a.buffers()[1], dtype=np.int64)[2 * a.offset:2 * (a.offset + len(a))].reshape(-1, 2)
            if name in dec8:
                raw, width = v[:, 0].copy().view(np.uint8), 8
            else:
                raw, width = v.copy().view(np.uint8).reshape(-1), 16
        else:
            width = a.type.bit_width // 8
            raw = np.frombuffer(a.buffers()[1], dtype=np.uint8)[a.offset * width:(a.offset + len(a)) * width]
        vals = torch.from_numpy(np.concatenate([np.ascontiguousarray(raw).view(np.uint8).reshape(-1), np.zeros(16, np.uint8)])).cuda()
        t.add(dt, vals.data_ptr(), width, vdev.data_ptr() if vdev is not None else None, a.null_count, dictionary=dictionary, keep=(vals, vdev))
    return t


@pytest.mark.parametrize("keys,n_parts", [("b", 7), ("i8", 200), ("i16", 200), ("d9", 200), ("d18", 4096), ("d38", 7),
                                          ("s8+i32", 200), ("f32+s16+date+ts", 6145), ("d9+d18+i64+s32+f64", 2)])
def test_device_tables(cb, oracle, keys, n_parts):
    """device columns, decimal(9, 2) and decimal(18, 0) 8 bytes wide"""
    keys = keys.split("+")
    cols = make_values(50_000, 21 + n_parts)
    tbl, types = table_of(cols)
    t = device_table(cb, tbl, types, dec8=("d9", "d18"))
    plan = hash_plan(cb, cb.proto.scan(types), types, tbl.column_names, keys, n_parts)
    check(oracle, run(cb, plan, [t]), tbl, keys, n_parts)


def test_device_table_slices(cb, oracle):
    """a device table handed out in chunkRows slices: one batch per slice, each partitioned on its own"""
    cols = make_values(10_000, 4)
    tbl, types = table_of(cols, ["b", "i8", "d18", "s16", "f64", "row"])
    t = device_table(cb, tbl, types, dec8=("d18",))
    plan = hash_plan(cb, cb.proto.scan(types), types, tbl.column_names, ["d18", "b"], 31)
    got = run(cb, plan, [t], config={"spark.comet.b200.chunkRows": "3072"})
    assert [b.num_rows for b, _ in got] == [3072, 3072, 3072, 784]
    check(oracle, got, tbl, ["d18", "b"], 31)


# ---- Parquet scan -------------------------------------------------------------------------------------------------------------------------
def parquet_table(n, seed):
    """columns of every (physical, requested) pair the scan accepts: name -> (arrow array, requested proto type, stored pyarrow type)"""
    import comet_b200.proto as P
    cols = make_values(n, seed)
    rng = np.random.default_rng(seed + 1)
    mask = lambda: rng.random(n) < 0.15
    d7, d12, d28 = _dec_values(rng, n, 7), _dec_values(rng, n, 12), _dec_values(rng, n, 28)
    out = {
        "i8": (cols["i8"][0], P.INT8),                              # INT32 (INT_8) -> int8
        "i16": (cols["i16"][0], P.INT16),                           # INT32 (INT_16) -> int16
        "i32": (cols["i32"][0], P.INT32),
        "i32w": (cols["date"][0].cast(pa.int32()), P.INT64),        # INT32 -> int64
        "date": (cols["date"][0], P.DATE),
        "d7": (_dec(d7, 7, 2, mask()), P.DECIMAL(7, 2)),            # INT32 or FLBA(4)
        "i64": (cols["i64"][0], P.INT64),
        "ts": (cols["ts"][0].cast(pa.timestamp("us")), P.TIMESTAMP),
        "d12": (_dec(d12, 12, 2, mask()), P.DECIMAL(12, 2)),        # INT64 or FLBA(6)
        "d28": (_dec(d28, 28, 2, mask()), P.DECIMAL(28, 2)),        # FLBA(12)
        "f32": (cols["f32"][0], P.FLOAT),
        "f64": (cols["f64"][0], P.DOUBLE),
        "sd": (cols["s32"][0].dictionary_decode(), P.STRING),       # dictionary pages
        "sp": (cols["s16"][0].dictionary_decode(), P.STRING),       # PLAIN pages
        "row": (cols["row"][0], P.INT64),
    }
    return out


def write_parquet(path, cols, as_int):
    tbl = pa.table({k: cols[k][0] for k in cols})
    pq.write_table(tbl, path, row_group_size=40_000, data_page_size=1 << 16, use_dictionary=["sd"], store_decimal_as_integer=as_int,
                   compression="SNAPPY")
    return tbl


def scan_of(cb, cols, names, path):
    """NativeScan reading `names` as their requested types"""
    fields = [(k, cols[k][1], True) for k in names]
    return cb.proto.native_scan(fields, fields, [path]), [cols[k][1] for k in names]


def expected_table(cols, names):
    return pa.table({k: (cols[k][0].cast(pa.int64()) if k == "i32w" else cols[k][0]) for k in names})


@pytest.mark.parametrize("as_int", [True, False])
@pytest.mark.parametrize("keys,n_parts", [("i8", 200), ("i16", 200), ("d7", 200), ("d12", 4096), ("d28", 7),
                                          ("i32w+date", 7), ("i32", 2), ("ts+f32", 200), ("f64+i64", 6145),
                                          ("sd", 200), ("sp+d7+i8", 31),
                                          ("i8+i16+i32w+d7+d12+d28+sd+sp", 200)])
def test_native_scan(cb, oracle, tmp_path, as_int, keys, n_parts):
    """ShuffleWriter directly over NativeScan: decimals stored as INT32 / INT64 (store_decimal_as_integer) or FLBA, int8 / int16 as INT32"""
    keys = keys.split("+")
    n = 90_000
    cols = parquet_table(n, 31)
    path = str(tmp_path / "p.parquet")
    write_parquet(path, cols, as_int)
    names = ["i8", "i16", "i32", "i32w", "date", "d7", "i64", "ts", "d12", "d28", "f32", "f64", "sd", "sp", "row"]
    if keys in (["i8"], ["i16"]):  # integer and float columns only: the other cases carry the decimals and strings
        names = ["i8", "i16", "i32", "i32w", "date", "i64", "ts", "f32", "f64", "row"]
    scan, types = scan_of(cb, cols, names, path)
    plan = hash_plan(cb, scan, types, names, keys, n_parts)
    got = run(cb, plan, [], config={"spark.comet.b200.chunkRows": "50000"})
    assert len(got) >= 2
    check(oracle, got, expected_table(cols, names), keys, n_parts)


# ---- partial aggregate state ------------------------------------------------------------------------------------------------------------
def test_partial_aggregate_state(cb, oracle):
    """ShuffleWriter(HashAggregate(Partial)) keyed on a BOOLEAN group key and the SUM state's is_empty flag, both one byte per row"""
    P = cb.proto
    rng = np.random.default_rng(17)
    n = 60_000
    b = pa.array(rng.random(n) < 0.5, mask=rng.random(n) < 0.1)
    k = pa.array(rng.integers(0, 5000, n), pa.int64())
    v = _dec(rng.integers(-10**9, 10**9, n), 12, 2, mask=rng.random(n) < 0.3)
    tbl = pa.table({"b": b, "k": k, "v": v})
    agg = P.hash_agg(P.scan([P.BOOL, P.INT64, P.DECIMAL(12, 2)]), [P.bound(0, P.BOOL), P.bound(1, P.INT64)],
                     [P.agg_sum(P.bound(2, P.DECIMAL(12, 2)), P.DECIMAL(22, 2))], P.PARTIAL)
    state_types = [P.BOOL, P.INT64, P.DECIMAL(22, 2), P.BOOL]
    with cb.native.Plan(agg, [tbl.to_batches(max_chunksize=8192)]) as p:
        state = p.collect()
        assert p.stats()["agg_strategies"] & cb.native.AGG_TABLE      # device-resident state: booleans one byte per row
    names = state.column_names
    by_group = [("col_1", "ascending"), ("col_0", "ascending")]         # (b, k) is unique per state row
    for keys in (["col_0"], ["col_0", "col_3"], ["col_3", "col_1"]):
        got = run(cb, hash_plan(cb, agg, state_types, names, keys, 7), [tbl.to_batches(max_chunksize=8192)])
        assert len(got) == 1
        out, starts = got[0]
        out = pa.Table.from_batches([out])
        # the aggregate's row order is its own, so the rows are compared as a set; each row lies in its own partition and the
        # partition sizes are those of the reference
        partref.assert_tables_equal(out.sort_by(by_group), state.sort_by(by_group))
        want_starts, _, _ = partref.partition(oracle, state, keys, 7)
        assert starts == want_starts
        pids = np.array([oracle.pmod(int(h), 7) for h in partref.key_hashes(oracle, out, keys)])
        assert (pids == np.searchsorted(np.array(starts), np.arange(out.num_rows), side="right") - 1).all()
