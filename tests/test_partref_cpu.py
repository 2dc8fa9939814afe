"""CPU: tests/partref.py, the partitioning reference, pinned by cases worked by hand on top of the oracle's known-answer-tested murmur3."""
import decimal
import struct

import numpy as np
import pyarrow as pa
import pytest

import partref


def mm3(o, raw, seed=42):
    return o.murmur3_bytes(raw, seed)


def one(o, arr):
    return int(partref.key_hashes(o, pa.table({"k": arr}), ["k"])[0])


def test_kind_of_every_type():
    kinds = {pa.bool_(): "bool", pa.int8(): "i8", pa.int16(): "i16", pa.int32(): "i32", pa.date32(): "date32", pa.int64(): "i64",
             pa.timestamp("us"): "timestamp", pa.timestamp("us", tz="UTC"): "timestamp", pa.float32(): "f32", pa.float64(): "f64",
             pa.decimal128(9, 2): "dec_small", pa.decimal128(18, 0): "dec_small", pa.decimal128(19, 2): "dec_large",
             pa.decimal128(38, 10): "dec_large", pa.string(): "str", pa.dictionary(pa.int8(), pa.string()): "str"}
    for t, k in kinds.items():
        assert partref.oracle_kind(t) == k, t
    for t in (pa.timestamp("ms"), pa.uint32(), pa.binary(), pa.dictionary(pa.int32(), pa.int64())):
        with pytest.raises(TypeError):
            partref.oracle_kind(t)


def test_all_null_row_hashes_to_42(oracle):
    tbl = pa.table({
        "b": pa.array([None, True], pa.bool_()), "i8": pa.array([None, 1], pa.int8()), "f": pa.array([None, 1.0]),
        "d": pa.array([None, decimal.Decimal("1.00")], pa.decimal128(12, 2)), "D": pa.array([None, decimal.Decimal("1.00")], pa.decimal128(28, 2)),
        "s": pa.array([None, "x"]), "t": pa.array([None, 5], pa.timestamp("us")),
        "ds": pa.DictionaryArray.from_arrays(pa.array([None, 0], pa.int16()), pa.array(["x"])),
    })
    h = partref.key_hashes(oracle, tbl, list(range(tbl.num_columns)))
    assert h[0] == 42 and h[1] != 42
    # a NULL in the middle leaves the hash of the keys before it
    mid = pa.table({"a": pa.array([7], pa.int32()), "n": pa.array([None], pa.int64()), "c": pa.array([9], pa.int32())})
    want = mm3(oracle, struct.pack("<i", 9), mm3(oracle, struct.pack("<i", 7)))
    assert int(partref.key_hashes(oracle, mid, ["a", "n", "c"])[0]) == want


def test_signed_zero_hashes_alike(oracle):
    for t in (pa.float32(), pa.float64()):
        z = pa.array([0.0, -0.0], t)
        h = partref.key_hashes(oracle, pa.table({"z": z}), ["z"])
        assert h[0] == h[1], t
        assert h[0] == mm3(oracle, b"\0" * (4 if t == pa.float32() else 8))


def test_nans_hash_by_their_bits(oracle):
    bits64 = np.array([0x7FF8000000000000, 0x7FF8DEADBEEF0001, 0xFFF8000000000000, 0x7FF0000000000001], dtype=np.uint64)
    h = partref.key_hashes(oracle, pa.table({"f": pa.array(bits64.view(np.float64))}), ["f"])
    assert len(set(h.tolist())) == 4
    for b, x in zip(bits64, h):
        assert x == mm3(oracle, struct.pack("<Q", int(b)))
    bits32 = np.array([0x7FC00000, 0x7FC0BEEF, 0xFFC00000, 0x7F800001], dtype=np.uint32)
    h = partref.key_hashes(oracle, pa.table({"f": pa.array(bits32.view(np.float32))}), ["f"])
    assert len(set(h.tolist())) == 4
    for b, x in zip(bits32, h):
        assert x == mm3(oracle, struct.pack("<I", int(b)))


def test_small_ints_hash_as_i32(oracle):
    for v in (-1, 0, 1, -128, 127):
        want = mm3(oracle, struct.pack("<i", v))
        for t in (pa.int8(), pa.int16(), pa.int32(), pa.date32()):
            assert one(oracle, pa.array([v], pa.int32()).cast(t)) == want, (v, t)
    assert one(oracle, pa.array([-32768], pa.int16())) == mm3(oracle, struct.pack("<i", -32768))
    assert one(oracle, pa.array([True])) == mm3(oracle, struct.pack("<i", 1))
    assert one(oracle, pa.array([False])) == mm3(oracle, struct.pack("<i", 0))
    assert one(oracle, pa.array([-1], pa.int64())) == mm3(oracle, struct.pack("<q", -1))
    assert one(oracle, pa.array([-1], pa.timestamp("us"))) == mm3(oracle, struct.pack("<q", -1))


def test_decimals(oracle):
    # p <= 18: the unscaled value as an i64; p > 18: its 16 little-endian bytes
    for v in (0, -1, 1, 10**18 - 1, -(10**18 - 1)):
        d = decimal.Decimal(v).scaleb(-2)
        assert one(oracle, pa.array([d], pa.decimal128(18, 2))) == mm3(oracle, struct.pack("<q", v))
        if abs(v) < 10**7:
            assert one(oracle, pa.array([d], pa.decimal128(7, 2))) == mm3(oracle, struct.pack("<q", v))
    for v in (0, -1, 10**38 - 1, -(10**38 - 1), 2**64, -(2**64)):
        d = decimal.Decimal(v).scaleb(-2, context=decimal.Context(prec=60))
        assert one(oracle, pa.array([d], pa.decimal128(38, 2))) == mm3(oracle, (v & ((1 << 128) - 1)).to_bytes(16, "little"))


def test_strings_hash_their_bytes(oracle):
    vals = ["", "a", "ab", "abc", "abcd", "abcde", "ÿþ", "\U0001F601", "天地人", "x" * 9, "é", "aé", "abcdé"]
    h = partref.key_hashes(oracle, pa.table({"s": pa.array(vals)}), ["s"])
    for v, x in zip(vals, h):
        assert x == mm3(oracle, v.encode())
    # tail bytes >= 0x80 are sign-extended (murmur3.rs:131): "aé" ends in the tail bytes c3 a9
    def unsigned_tail(b):
        h1 = 42
        rot = lambda x, r: ((x << r) | (x >> (32 - r))) & 0xFFFFFFFF
        for byte in b:
            k1 = rot((byte * 0xcc9e2d51) & 0xFFFFFFFF, 15) * 0x1b873593 & 0xFFFFFFFF
            h1 = (rot(h1 ^ k1, 13) * 5 + 0xe6546b64) & 0xFFFFFFFF
        h1 ^= len(b)
        for s, m in ((16, 0x85ebca6b), (13, 0xc2b2ae35)):
            h1 = ((h1 ^ (h1 >> s)) * m) & 0xFFFFFFFF
        return h1 ^ (h1 >> 16)
    assert unsigned_tail(b"a") == mm3(oracle, b"a")
    assert int(h[vals.index("aé")]) != unsigned_tail("aé".encode())


@pytest.mark.parametrize("index", [pa.int8(), pa.int16(), pa.int32()])
def test_dictionary_hashes_like_its_plain_form(oracle, index):
    words = ["", "k", "été", "\U0001F601", "abcdefghi", None]
    rng = np.random.default_rng(3)
    codes = rng.integers(0, 5, 500)
    mask = rng.random(500) < 0.2
    d = pa.DictionaryArray.from_arrays(pa.array(codes, index, mask=mask), pa.array(words[:5]))
    p = pa.array([None if m else words[c] for c, m in zip(codes, mask)], pa.string())
    hd = partref.key_hashes(oracle, pa.table({"s": d}), ["s"])
    hp = partref.key_hashes(oracle, pa.table({"s": p}), ["s"])
    assert (hd == hp).all()
    # a slice (non-zero offset) reads its own rows
    hs = partref.key_hashes(oracle, pa.table({"s": d.slice(37, 100)}), ["s"])
    assert (hs == hp[37:137]).all()


def test_starts_are_the_cumulative_bincount(oracle):
    rng = np.random.default_rng(11)
    n = 5000
    tbl = pa.table({"a": pa.array(rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64), mask=rng.random(n) < 0.1),
                    "b": pa.array(rng.standard_normal(n).astype(np.float32)),
                    "row": pa.array(np.arange(n))})
    for n_parts in (1, 2, 7, 200, 6145):
        starts, order, out = partref.partition(oracle, tbl, ["a", "b"], n_parts)
        h = partref.key_hashes(oracle, tbl, ["a", "b"])
        pids = np.array([oracle.pmod(int(x), n_parts) for x in h])
        assert starts == [0] + np.cumsum(np.bincount(pids, minlength=n_parts)).tolist()
        # stable: inside a partition the rows keep their input order
        assert (np.asarray(out.column("row")) == order).all()
        for p in range(n_parts):
            seg = order[starts[p]:starts[p + 1]]
            assert (np.diff(seg) > 0).all() and (pids[seg] == p).all()
        partref.assert_tables_equal(out, tbl.take(pa.array(order)))


def test_compare_catches_differences():
    a = pa.array(np.array([0x7FF8000000000000, 0x7FF8000000000001], np.uint64).view(np.float64))
    with pytest.raises(AssertionError):
        partref.assert_columns_equal(a, a.take(pa.array([1, 0])))
    z = pa.array([0.0, -0.0])
    with pytest.raises(AssertionError):
        partref.assert_columns_equal(z, pa.array([0.0, 0.0]))
    with pytest.raises(AssertionError):
        partref.assert_columns_equal(pa.array([1, None]), pa.array([1, 2]))
    with pytest.raises(AssertionError):
        partref.assert_columns_equal(pa.array(["abc", "abd"]), pa.array(["abc", "abc"]))
    d = pa.array([decimal.Decimal("1.00"), decimal.Decimal("-1.00")], pa.decimal128(12, 2))
    with pytest.raises(AssertionError):
        partref.assert_columns_equal(d, d.take(pa.array([1, 0])))
    partref.assert_columns_equal(pa.array([1, None], pa.int8()), pa.array([1, None], pa.int8()))
