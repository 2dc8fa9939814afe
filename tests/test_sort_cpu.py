"""CPU: the Sort reference (tests/sortref.py) against pyarrow's stable sort_indices where the two agree and against hand-worked cases
where they do not, the host compile of the row-key encoder (device/cb_sortkey.h) against the reference for every key type, layout,
direction and null placement, and which Sort plans the planner accepts.

pyarrow is Arrow C++, not the reference's arrow-rs.  It differs from it in three ways, each covered by hand-worked cases instead:
it treats -0.0 as equal to +0.0, it ignores the sign and payload of NaN, and it has one null placement for all keys."""
import ctypes as C
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import sortref as R

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "datafusion-comet_b200", "csrc")


def dec_array(unscaled, p, s, mask=None):
    """a decimal128(p, s) array of python-int unscaled values (NULL where mask)"""
    u = [int(v) & ((1 << 128) - 1) for v in unscaled]
    words = np.array([[x & ((1 << 64) - 1), x >> 64] for x in u], np.uint64).reshape(-1, 2)
    nulls = 0 if mask is None else int(mask.sum())
    validity = pa.py_buffer(np.packbits(~mask, bitorder="little")) if nulls else None
    return pa.Array.from_buffers(pa.decimal128(p, s), len(u), [validity, pa.py_buffer(words.tobytes())], null_count=nulls)


def _rng_table(n, seed):
    rng = np.random.default_rng(seed)
    mask = lambda: rng.random(n) < 0.15
    words = ["", "a", "ab", "b", "B", "é", "é", "zz", "\U0001F601", "a\x00", "ab\x00"]
    f64 = rng.choice([-2.5, -1.0, 0.5, 1.0, 3.0, np.inf, -np.inf], n)
    dec = rng.integers(-10**6, 10**6, n)
    cols = {
        "b": pa.array(rng.random(n) < 0.5, mask=mask()),
        "i8": pa.array(rng.integers(-128, 128, n).astype(np.int8), mask=mask()),
        "i16": pa.array(rng.integers(-5, 5, n).astype(np.int16), mask=mask()),
        "i32": pa.array(rng.integers(-2**31, 2**31, n).astype(np.int32), mask=mask()),
        "i64": pa.array(rng.integers(-3, 3, n), mask=mask()),
        "date": pa.array(rng.integers(-100, 100, n).astype(np.int32), pa.date32(), mask=mask()),
        "ts": pa.array(rng.integers(-10**12, 10**12, n), pa.timestamp("us", tz="UTC"), mask=mask()),
        "f64": pa.array(f64, mask=mask()),
        "f32": pa.array(f64.astype(np.float32), mask=mask()),
        "d9": dec_array(dec, 9, 2, mask()),
        "d38": dec_array([int(v) * 10**30 for v in dec], 38, 0, mask()),
        "s": pa.array([None if m else words[i] for i, m in zip(rng.integers(0, len(words), n), mask())]),
    }
    return pa.table(cols)


@pytest.mark.parametrize("nulls_first", [True, False])
@pytest.mark.parametrize("keys", [["b"], ["i8"], ["i16"], ["i32"], ["i64"], ["date"], ["ts"], ["f64"], ["f32"], ["d9"], ["d38"], ["s"],
                                  ["i16", "s"], ["b", "i64", "f64"], ["date", "d9", "s", "i8"]])
def test_reference_matches_pyarrow(keys, nulls_first):
    """no -0.0 and no NaN, one null placement for all keys: where pyarrow's stable sort_indices and the reference agree"""
    t = _rng_table(3000, len(keys) * 31 + nulls_first)
    for desc_mask in range(1 << len(keys)):
        desc = [(desc_mask >> k) & 1 == 1 for k in range(len(keys))]
        want = pc.sort_indices(t, sort_keys=[(k, "descending" if d else "ascending") for k, d in zip(keys, desc)],
                               null_placement="at_start" if nulls_first else "at_end").to_numpy()
        got = R.order(t, [(k, d, nulls_first) for k, d in zip(keys, desc)])
        assert (got == want).all(), (keys, desc)


F64_TOTAL = [0xFFF8000000000001, 0xFFF8000000000000, 0xFFF0000000000001, 0xFFF0000000000000, 0xC000000000000000, 0x8000000000000001,
             0x8000000000000000, 0x0000000000000000, 0x0000000000000001, 0x4000000000000000, 0x7FF0000000000000, 0x7FF0000000000001,
             0x7FF8000000000000, 0x7FF8000000000001]   # -NaN (payloads) < -Inf < -2 < -min subnormal < -0 < +0 < ... < +Inf < +NaN (payloads)


def _f64(bits):
    return pa.array(np.array(bits, np.uint64).view(np.float64))


def test_float_total_order():
    rng = np.random.default_rng(1)
    perm = rng.permutation(len(F64_TOTAL))
    t = pa.table({"f": _f64([F64_TOTAL[i] for i in perm])})
    got = np.array(t.column("f").to_numpy()).view(np.uint64)[R.order(t, [("f", False, True)])]
    assert [int(x) for x in got] == F64_TOTAL
    got = np.array(t.column("f").to_numpy()).view(np.uint64)[R.order(t, [("f", True, True)])]
    assert [int(x) for x in got] == F64_TOTAL[::-1]
    f32 = pa.array(np.array([0x80000000, 0x7FC00000, 0x00000000, 0xFFC00000, 0x7F800000, 0xFF800000], np.uint32).view(np.float32))
    got = np.array(f32.to_numpy()).view(np.uint32)[R.order(pa.table({"f": f32}), [("f", False, True)])]
    assert [hex(int(x)) for x in got] == ["0xffc00000", "0xff800000", "0x80000000", "0x0", "0x7f800000", "0x7fc00000"]


def test_integer_and_decimal_extremes():
    i64 = pa.array([0, 2**63 - 1, -1, -2**63, 1, None])
    assert R.order(pa.table({"v": i64}), [("v", False, False)]).tolist() == [3, 2, 0, 4, 1, 5]
    assert R.order(pa.table({"v": i64}), [("v", True, True)]).tolist() == [5, 1, 4, 0, 2, 3]
    m = 10**38 - 1
    d = pa.array([0, m, -m, -1, 1, None], pa.decimal128(38, 0))
    assert R.order(pa.table({"v": d}), [("v", False, True)]).tolist() == [5, 2, 3, 0, 4, 1]


def test_mixed_null_placement_and_ties():
    """each key places its own NULLs, whatever its direction; rows equal on every key keep their input order"""
    a = pa.array([1, None, 1, 2, None, 1, 2])
    b = pa.array(["x", "y", None, None, "x", "x", "y"])
    t = pa.table({"a": a, "b": b})
    # a ASC NULLS LAST, b DESC NULLS FIRST
    assert R.order(t, [("a", False, False), ("b", True, True)]).tolist() == [2, 0, 5, 3, 6, 1, 4]
    # a DESC NULLS FIRST, b ASC NULLS LAST
    assert R.order(t, [("a", True, True), ("b", False, False)]).tolist() == [4, 1, 6, 3, 0, 5, 2]


def test_window():
    assert R.window(10) == (0, 10)
    assert R.window(10, fetch=3) == (0, 3)
    assert R.window(10, fetch=3, skip=1) == (1, 3)
    assert R.window(10, skip=4) == (4, 10)
    assert R.window(10, fetch=20, skip=12) == (10, 10)
    assert R.window(10, fetch=0) == (0, 0)
    t = pa.table({"v": pa.array([3, 1, 2, 0])})
    assert R.sort_table(t, [("v", False, True)], fetch=3, skip=1).column("v").to_pylist() == [1, 2]


def test_assert_sorted_catches_disorder():
    t = pa.table({"a": pa.array([1, 1, 2]), "b": pa.array([2, 1, 0])})
    R.assert_sorted(t, [("a", False, True)])
    with pytest.raises(AssertionError):
        R.assert_sorted(t, [("a", False, True), ("b", False, True)])


# ---- the row-key encoder, compiled for the host --------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sk(tmp_path_factory):
    import subprocess
    so = str(tmp_path_factory.mktemp("cbsortkey") / "libcb200_sortkey.so")
    subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(CSRC, "sortkey_test.cpp")])
    lib = C.CDLL(so)
    lib.cb_sk_kind.argtypes = [C.c_char_p]
    lib.cb_sk_encode.restype = C.c_longlong
    return lib


def _layout(arr, kind):
    """(layout kind, value bits, value buffer, rank table) of arr stored as `kind`"""
    t = arr.type
    if pa.types.is_dictionary(t):
        d = arr.dictionary.to_pylist()
        enc = [v.encode() for v in d]
        srt = sorted(set(enc))
        rank = np.array([srt.index(v) for v in enc] + [0], np.uint32)
        return kind, 32, np.ascontiguousarray(R._fixed(arr.indices, {"dict8": np.int8, "dict16": np.int16, "dict32": np.int32}[kind])), rank
    if pa.types.is_boolean(t):
        vals = np.asarray(arr.fill_null(False))
        return kind, 1, (np.packbits(vals, bitorder="little") if kind == "bool" else vals.astype(np.uint8)), None
    if pa.types.is_decimal(t):
        w = R._fixed(arr, np.int64, 2).reshape(-1, 2)
        bits = 64 if t.precision <= 18 else 128
        data = {"dec_small_32": lambda: w[:, 0].astype(np.int32), "dec_small_64": lambda: w[:, 0].copy(), "dec_large_64": lambda: w[:, 0].copy(),
                "dec_small_128": lambda: w.copy(), "dec_large_128": lambda: w.copy()}[kind]()
        return kind, bits, np.ascontiguousarray(data), None
    bits = t.bit_width
    if pa.types.is_floating(t):
        v = R._fixed(arr, np.uint32 if bits == 32 else np.uint64)
    else:
        v = R._fixed(arr, {8: np.int8, 16: np.int16, 32: np.int32, 64: np.int64}[bits])
    if kind == "i32" and bits < 32:
        v = v.astype(np.int32)                                                 # INT32-backed int8 / int16 (the Parquet scan's layout)
    return kind, bits, np.ascontiguousarray(v), None


def encode(sk, cols, keys):
    """row keys of `cols` (list of (arrow array, layout kind)) as one python int per row"""
    n = len(cols[0][0])
    lay = [_layout(a, k) for a, k in cols]
    nk = len(cols)
    kinds = (C.c_int * nk)(*[sk.cb_sk_kind(k.encode()) for k, _, _, _ in lay])
    assert all(k >= 0 for k in kinds)
    bits = (C.c_int * nk)(*[b for _, b, _, _ in lay])
    desc = (C.c_int * nk)(*[int(d) for d, _ in keys])
    nf = (C.c_int * nk)(*[int(f) for _, f in keys])
    data = (C.c_void_p * nk)(*[v.ctypes.data for _, _, v, _ in lay])
    valids = [np.packbits(np.asarray(a.is_valid()), bitorder="little") if a.null_count else None for a, _ in cols]
    validity = (C.c_void_p * nk)(*[None if v is None else v.ctypes.data for v in valids])
    rank = (C.c_void_p * nk)(*[None if r is None else r.ctypes.data for _, _, _, r in lay])
    n_rank = (C.c_int * nk)(*[0 if r is None else len(r) - 1 for _, _, _, r in lay])
    total = sum(b + (1 if v is not None else 0) for (_, b, _, _), v in zip(lay, valids))
    words = max(1, (total + 63) // 64)
    out = np.zeros(n * words, np.uint64)
    bad = sk.cb_sk_encode(nk, kinds, bits, desc, nf, data, validity, rank, n_rank, C.c_longlong(n), words,
                          out.ctypes.data_as(C.POINTER(C.c_uint64)))
    assert bad == 0
    w = out.reshape(n, words)
    return [sum(int(w[i, j]) << (64 * (words - 1 - j)) for j in range(words)) for i in range(n)], total


def _special_table(n, seed):
    rng = np.random.default_rng(seed)
    mask = lambda: rng.random(n) < 0.2
    f64 = np.concatenate([np.array(F64_TOTAL, np.uint64).view(np.float64), rng.standard_normal(n - len(F64_TOTAL))])
    f32 = np.concatenate([np.array([0x80000000, 0x7FC00000, 0, 0xFFC00000, 0x7F800000, 0xFF800000, 0x7FC0BEEF, 0xFF800123, 1], np.uint32)
                          .view(np.float32), rng.standard_normal(n - 9).astype(np.float32)])
    ints = lambda dt: np.concatenate([np.array([np.iinfo(dt).min, np.iinfo(dt).max, 0, -1, 1], dt),
                                      rng.integers(np.iinfo(dt).min, np.iinfo(dt).max, n - 5, dtype=dt, endpoint=True)])
    m38 = 10**38 - 1
    d38 = [m38, -m38, 0, -1, 1] + [int(x) * 10**20 + int(y) for x, y in zip(rng.integers(-10**17, 10**17, n - 5), rng.integers(0, 10**18, n - 5))]
    d18 = np.concatenate([np.array([10**18 - 1, -(10**18 - 1), 0, -1, 1]), rng.integers(-10**18 + 1, 10**18, n - 5)])
    d9 = np.concatenate([np.array([10**9 - 1, -(10**9 - 1), 0, -1, 1]), rng.integers(-10**9 + 1, 10**9, n - 5)])
    words = ["", "a", "ab", "b", "B", "é", "zz", "\U0001F601", "a\x00", "w1", "w2"]
    dict_codes = rng.integers(0, len(words) + 1, n) % len(words)
    return {
        "b": pa.array(rng.random(n) < 0.5, mask=mask()),
        "i8": pa.array(ints(np.int8), mask=mask()), "i16": pa.array(ints(np.int16), mask=mask()),
        "i32": pa.array(ints(np.int32), mask=mask()), "i64": pa.array(ints(np.int64), mask=mask()),
        "date": pa.array(ints(np.int32), pa.date32(), mask=mask()),
        "ts": pa.array(ints(np.int64), pa.timestamp("us"), mask=mask()),
        "f32": pa.array(f32, mask=mask()), "f64": pa.array(f64, mask=mask()),
        "d9": dec_array(d9, 9, 2, mask()),
        "d18": dec_array(d18, 18, 0, mask()),
        "d38": dec_array(d38, 38, 4, mask()),
        "d38s": dec_array(d18, 38, 0, mask()),                                 # p > 18 values that fit 8 bytes
        "s": pa.DictionaryArray.from_arrays(pa.array(dict_codes, pa.int32(), mask=mask()), pa.array(words[::-1] + ["a"])),
    }


LAYOUTS = [("b", "bool"), ("b", "bool8"), ("i8", "i8"), ("i8", "i32"), ("i16", "i16"), ("i16", "i32"), ("i32", "i32"), ("date", "i32"),
           ("i64", "i64"), ("ts", "i64"), ("f32", "f32"), ("f64", "f64"), ("d9", "dec_small_32"), ("d9", "dec_small_64"),
           ("d18", "dec_small_64"), ("d18", "dec_small_128"), ("d38", "dec_large_128"), ("d38s", "dec_large_64"),
           ("s", "dict8"), ("s", "dict16"), ("s", "dict32")]


def _as_layout(arr, kind):
    if kind in ("dict8", "dict16"):
        return pa.DictionaryArray.from_arrays(arr.indices.cast(pa.int8() if kind == "dict8" else pa.int16()), arr.dictionary)
    return arr


@pytest.mark.parametrize("col,kind", LAYOUTS)
def test_header_orders_like_the_reference(sk, col, kind):
    """every type x layout x direction x null placement: the encoded keys order rows exactly as the reference does (stable)"""
    cols = _special_table(600, 7)
    arr = _as_layout(cols[col], kind)
    for desc in (False, True):
        for nf in (False, True):
            keys, _ = encode(sk, [(arr, kind)], [(desc, nf)])
            got = np.argsort(np.array(keys, dtype=object), kind="stable")
            want = R.order(pa.table({"c": arr}), [("c", desc, nf)])
            assert (got == want).all(), (col, kind, desc, nf)


@pytest.mark.parametrize("combo", [["i8", "s", "f64"], ["b", "d38", "i16", "date"], ["s", "b", "f32", "i64", "d9"],
                                   ["d38s", "i16", "s"]])
def test_header_multi_key(sk, combo):
    cols = _special_table(700, 11)
    kinds = dict(LAYOUTS[::-1])
    arrs = [(_as_layout(cols[c], kinds[c]), kinds[c]) for c in combo]
    rng = np.random.default_rng(len(combo))
    for _ in range(4):
        opts = [(bool(rng.integers(2)), bool(rng.integers(2))) for _ in combo]
        keys, total = encode(sk, arrs, opts)
        assert total <= 256
        got = np.argsort(np.array(keys, dtype=object), kind="stable")
        t = pa.table({f"c{i}": a for i, (a, _) in enumerate(arrs)})
        want = R.order(t, [(f"c{i}", d, f) for i, (d, f) in enumerate(opts)])
        assert (got == want).all(), (combo, opts)


# ---- planner --------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def native():
    import comet_b200
    from comet_b200 import native
    return native


def test_accepted_plans(native):
    from comet_b200 import proto as P
    types = [P.BOOL, P.INT8, P.INT16, P.INT32, P.INT64, P.DATE, P.TIMESTAMP, P.FLOAT, P.DOUBLE, P.DECIMAL(12, 2), P.DECIMAL(38, 4), P.STRING]
    scan = P.scan(types)
    for i, t in enumerate(types):
        for d in (False, True):
            for nf in (False, True):
                ok, why = native.supports(P.sort(scan, [P.sort_order(P.bound(i, t), d, nf)]))
                assert ok, (t, why)
    too_wide = P.sort(scan, [P.sort_order(P.bound(i, types[i])) for i in range(8)], fetch=10, skip=2)  # 1+8+16+32+64+32+64+32 + 8 = 257
    assert not native.supports(too_wide)[0]
    eight = P.sort(scan, [P.sort_order(P.bound(i, types[i])) for i in (0, 1, 2, 3, 5, 7, 11, 4)])      # 1+8+16+32+32+32+32+64 + 8 = 225
    assert native.supports(eight)[0]
    two_wide = P.sort(scan, [P.sort_order(P.bound(10, types[10])), P.sort_order(P.bound(4, P.INT64))])  # 129 + 65
    assert native.supports(two_wide)[0]
    topk = P.projection(P.sort(P.scan(types, source="TopKInput"), [P.sort_order(P.bound(8, P.DOUBLE), True)], fetch=100),
                        [P.bound(8, P.DOUBLE), P.bound(11, P.STRING)])
    assert native.supports(topk)[0]
    assert native.supports(P.sort(scan, [P.sort_order(P.bound(0, P.BOOL))], fetch=0, skip=0))[0]


def test_refused_plans(native):
    from comet_b200 import proto as P
    types = [P.INT32] * 9 + [P.DECIMAL(38, 0)] * 2 + [P.DOUBLE]
    scan = P.scan(types)
    ok, why = native.supports(P.sort(scan, [P.sort_order(P.add(P.bound(0, P.INT32), P.bound(1, P.INT32), P.INT32))]))
    assert not ok and "computed sort keys" in why
    ok, why = native.supports(P.sort(scan, [P.sort_order(P.bound(i, P.INT32)) for i in range(9)]))
    assert not ok and "8 sort keys" in why
    assert native.supports(P.sort(P.scan([P.INT16] * 8), [P.sort_order(P.bound(i, P.INT16)) for i in range(8)]))[0]   # 8 x 17 bits
    ok, why = native.supports(P.sort(scan, [P.sort_order(P.bound(i, P.INT32)) for i in range(8)]))                     # 8 x 33 bits
    assert not ok and "256 bits" in why
    ok, why = native.supports(P.sort(scan, [P.sort_order(P.bound(9, types[9])), P.sort_order(P.bound(10, types[10]))]))   # 2 x 129
    assert not ok and "256 bits" in why
    for field in ("fetch", "skip"):
        plan = P.sort(scan, [P.sort_order(P.bound(0, P.INT32))], **{field: -1})
        ok, why = native.supports(plan)
        assert not ok and "negative" in why
    ok, why = native.supports(P.sort(P.scan([P.DT("BYTES")]), [P.sort_order(P.bound(0, P.DT("BYTES")))]))
    assert not ok


def test_pipeline_below_a_sort_compiles(native):
    """cb200_compile_plan walks through the Sort to the filter / projection pipeline below it (NVRTC, no device)"""
    from comet_b200 import proto as P
    types = [P.INT64, P.DOUBLE, P.STRING]
    below = P.projection(P.filter_(P.scan(types), P.gt(P.bound(1, P.DOUBLE), P.literal(0.5, P.DOUBLE))), [P.bound(0, P.INT64), P.bound(2, P.STRING)])
    plan = P.sort(below, [P.sort_order(P.bound(1, P.STRING), True, False), P.sort_order(P.bound(0, P.INT64))], fetch=5)
    keys = native.compile_plan(plan)
    assert keys and keys == native.compile_plan(below)
    above = P.filter_(plan, P.is_not_null(P.bound(0, P.INT64)))
    assert native.compile_plan(above)
