"""Range and round-robin repartitioning without a GPU: the CPU reference against a brute-force partition_point, the boundary search
header (device/cb_rangepart.h, built for the host with the row-key encoder) against the reference, the string rank against a direct
byte comparison, and the planner: what it accepts, refuses (code 1) and rejects as malformed (code 4)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pyarrow as pa
import pytest

import rangeref as R
import sortref
from comet_b200 import proto as P
from rangecases import PTYPE, pick_bounds, special_table

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "datafusion-comet_b200", "csrc")


# ---- the reference against partition_point spelled out ---------------------------------------------------------------------------
@pytest.mark.parametrize("cols", [["i32"], ["f64"], ["s"], ["d38"], ["b", "i8"], ["s", "f32", "date"], ["d18", "ts", "i16", "s"]])
def test_reference_matches_brute_force(cols):
    t = pa.table(special_table(300, len(cols)))
    rng = np.random.default_rng(7)
    for trial in range(4):
        keys = [(c, bool(rng.integers(2)), bool(rng.integers(2))) for c in cols]
        for nb in (0, 1, 7, 40):
            bounds = pick_bounds(t, keys, nb, trial * 100 + nb)
            want = R.brute_pids(t, keys, bounds)
            assert (R.range_pids(t, keys, bounds) == want).all(), (cols, keys, nb)


def test_reference_by_hand():
    t = pa.table({"x": pa.array([5, None, 1, 3, 3, 9], pa.int64())})
    b = pa.table({"k0": pa.array([3, 5], pa.int64())})
    assert R.range_pids(t, [("x", False, True)], b).tolist() == [2, 0, 0, 1, 1, 2]
    assert R.range_pids(t, [("x", False, False)], b).tolist() == [2, 2, 0, 1, 1, 2]     # NULLS LAST: after every value
    bd = pa.table({"k0": pa.array([5, 3], pa.int64())})
    assert R.range_pids(t, [("x", True, True)], bd).tolist() == [1, 0, 2, 2, 2, 0]      # DESC: 9 first, then 5, 3, 1
    starts, order = R.place(np.array([1, 0, 2, 0]), 4)
    assert starts == [0, 2, 3, 4, 4] and order.tolist() == [1, 3, 0, 2]


# ---- the boundary search header, compiled for the host ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def rp(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("cbrangepart") / "libcb200_rangepart.so")
    subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(CSRC, "sortkey_test.cpp"),
                           os.path.join(CSRC, "rangepart_test.cpp")])
    lib = C.CDLL(so)
    lib.cb_sk_kind.argtypes = [C.c_char_p]
    lib.cb_sk_encode.restype = C.c_longlong
    lib.cb_rp_encode.restype = C.c_longlong
    return lib


def _strings(vals):
    enc = [v.encode() for v in vals]
    off = np.concatenate([[0], np.cumsum([len(e) for e in enc])]).astype(np.int32)
    return off, np.frombuffer(b"".join(enc) + b"\0", np.uint8)


def string_ranks(rp, values, bound_strings):
    """rank of each dictionary entry against the distinct boundary strings, by the header"""
    b = sorted(set(s.encode() for s in bound_strings))
    off, chars = _strings(values)
    boff, bchars = _strings([s.decode() for s in b])
    out = np.zeros(len(values) + 1, np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rp.cb_rp_string_ranks(p(off), p(chars), C.c_longlong(len(values)), p(boff), p(bchars), C.c_longlong(len(b)), p(out))
    return out


def _field(rp, arr, strs):
    """(kind, bits, values, rank) of an array in the layout the device stores it in"""
    t = arr.type
    if pa.types.is_dictionary(t):
        return "dict32", 32, np.ascontiguousarray(arr.indices.fill_null(0).to_numpy().astype(np.int32)), string_ranks(rp, arr.dictionary.to_pylist(), strs)
    if pa.types.is_boolean(t):
        return "bool", 1, np.packbits(np.asarray(arr.fill_null(False)), bitorder="little"), None
    if pa.types.is_decimal(t):
        w = sortref._fixed(arr, np.int64, 2).reshape(-1, 2)
        return ("dec_small_128", 64, np.ascontiguousarray(w), None) if t.precision <= 18 else ("dec_large_128", 128, np.ascontiguousarray(w), None)
    bits = t.bit_width
    if pa.types.is_floating(t):
        return ("f32" if bits == 32 else "f64"), bits, np.ascontiguousarray(sortref._fixed(arr, np.uint32 if bits == 32 else np.uint64)), None
    return {8: "i8", 16: "i16", 32: "i32", 64: "i64"}[bits], bits, np.ascontiguousarray(sortref._fixed(arr, {8: np.int8, 16: np.int16, 32: np.int32, 64: np.int64}[bits])), None


def pack(rp, arrays, keys, strs):
    """row keys of the arrays (one per key), every field with a null bit, as uint64 words [n, W], packed as k_range_pids packs them
    (sk_row_reg); the same keys through sk_row must agree"""
    n = len(arrays[0])
    lay = [_field(rp, a, s) for a, s in zip(arrays, strs)]
    nk = len(arrays)
    total = sum(b + 1 for _, b, _, _ in lay)
    words = max(1, (total + 63) // 64)
    valids = [np.packbits(np.asarray(a.is_valid()), bitorder="little") for a in arrays]
    out = np.zeros(max(n, 1) * words, np.uint64)
    ints = lambda xs: (C.c_int * nk)(*xs)
    bad = rp.cb_rp_encode(nk, ints([rp.cb_sk_kind(k.encode()) for k, _, _, _ in lay]), ints([b for _, b, _, _ in lay]),
                          ints([int(d) for _, d, _ in keys]), ints([int(f) for _, _, f in keys]),
                          (C.c_void_p * nk)(*[v.ctypes.data for _, _, v, _ in lay]), (C.c_void_p * nk)(*[v.ctypes.data for v in valids]),
                          (C.c_void_p * nk)(*[None if r is None else r.ctypes.data for _, _, _, r in lay]),
                          ints([0 if r is None else len(r) - 1 for _, _, _, r in lay]), C.c_longlong(n), words,
                          out.ctypes.data_as(C.POINTER(C.c_uint64)))
    assert bad == 0
    ref = np.zeros_like(out)
    assert rp.cb_sk_encode(nk, ints([rp.cb_sk_kind(k.encode()) for k, _, _, _ in lay]), ints([b for _, b, _, _ in lay]),
                           ints([int(d) for _, d, _ in keys]), ints([int(f) for _, _, f in keys]),
                           (C.c_void_p * nk)(*[v.ctypes.data for _, _, v, _ in lay]), (C.c_void_p * nk)(*[v.ctypes.data for v in valids]),
                           (C.c_void_p * nk)(*[None if r is None else r.ctypes.data for _, _, _, r in lay]),
                           ints([0 if r is None else len(r) - 1 for _, _, _, r in lay]), C.c_longlong(n), words,
                           ref.ctypes.data_as(C.POINTER(C.c_uint64))) == 0
    assert (ref == out).all()
    return out[:n * words].reshape(n, words), words


def header_pids(rp, table, keys, bounds, budget):
    """partition ids by the header's search, the top level sized for `budget` bytes of shared memory"""
    strs = [bounds.column(j).drop_null().to_pylist() if pa.types.is_string(bounds.column(j).type) else None for j in range(len(keys))]
    rows, W = pack(rp, [table.column(c).combine_chunks() for c, _, _ in keys], keys, strs)
    bcols = [R._plain(bounds.column(j)) for j in range(len(keys))]
    bcols = [c.dictionary_encode() if pa.types.is_string(c.type) else c for c in bcols]
    bnd, _ = pack(rp, bcols, keys, strs) if bounds.num_rows else (np.zeros((0, W), np.uint64), W)
    nb = bounds.num_rows
    shift = rp.cb_rp_shift(nb, W, budget)
    out = np.zeros(max(table.num_rows, 1), np.uint32)
    bnd = np.ascontiguousarray(bnd)
    rows = np.ascontiguousarray(rows)
    assert rp.cb_rp_pids(bnd.ctypes.data_as(C.c_void_p), nb, W, shift, rows.ctypes.data_as(C.c_void_p), C.c_longlong(table.num_rows),
                         out.ctypes.data_as(C.c_void_p)) == 0
    return out[:table.num_rows].astype(np.int64), shift


@pytest.mark.parametrize("col", list(PTYPE))
def test_header_search_matches_reference(rp, col):
    """every key type x direction x NULL placement, bounds with NULL / NaN / -0.0 / extreme entries, all in shared memory or sampled"""
    t = pa.table(special_table(800, 3))
    for desc in (False, True):
        for nf in (False, True):
            keys = [(col, desc, nf)]
            for nb in (0, 1, 5, 64, 300):
                bounds = pick_bounds(t, keys, nb, nb)
                want = R.range_pids(t, keys, bounds)
                for budget in (1 << 20, 64):
                    got, shift = header_pids(rp, t, keys, bounds, budget)
                    assert (got == want).all(), (col, desc, nf, nb, budget, shift)
                    assert budget > 64 or nb < 16 or shift > 0


@pytest.mark.parametrize("cols", [["i8", "s", "f64"], ["b", "d38", "i16", "date"], ["s", "b", "f32", "i64", "d18"], ["d38", "i32", "d18"]])
def test_header_multi_key(rp, cols):
    """several keys, rows equal in a prefix: the later keys decide"""
    base = special_table(900, 5)
    t = pa.table({c: base[c] for c in cols})
    rng = np.random.default_rng(len(cols))
    for trial in range(4):
        keys = [(c, bool(rng.integers(2)), bool(rng.integers(2))) for c in cols]
        for nb in (3, 100, 700):
            bounds = pick_bounds(t, keys, nb, trial + nb)
            want = R.range_pids(t, keys, bounds)
            for budget in (1 << 20, 256):
                got, _ = header_pids(rp, t, keys, bounds, budget)
                assert (got == want).all(), (cols, keys, nb, budget)


def test_string_rank_against_byte_comparison(rp):
    rng = np.random.default_rng(3)
    alphabet = ["", "a", "b", "\xff", "é", "\x00", "zz"]
    for _ in range(30):
        vals = ["".join(rng.choice(alphabet, rng.integers(0, 4))) for _ in range(rng.integers(1, 40))]
        bnds = ["".join(rng.choice(alphabet, rng.integers(0, 4))) for _ in range(rng.integers(0, 10))]
        got = string_ranks(rp, vals, bnds)
        b = sorted(set(s.encode() for s in bnds))
        for i, v in enumerate(vals):
            e = v.encode()
            want = 2 * sum(1 for x in b if x < e) + (1 if e in b else 0)
            assert got[i] == want, (v, bnds)
        # the order of the ranks is the byte order of the strings up to the bounds
        for i, v in enumerate(vals):
            for j, bj in enumerate(b):
                assert (got[i] <= 2 * j + 1) == (v.encode() <= bj)


def test_shift_sizes_the_top_level(rp):
    assert rp.cb_rp_shift(0, 4, 48 * 1024) == 0
    assert rp.cb_rp_shift(1536, 4, 48 * 1024) == 0
    assert rp.cb_rp_shift(1537, 4, 48 * 1024) == 1
    assert rp.cb_rp_shift(16383, 4, 48 * 1024) == 4
    assert rp.cb_rp_shift(16383, 1, 48 * 1024) == 2


# ---- planner ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def native():
    import comet_b200
    from comet_b200 import native
    return native


def _why(native, plan):
    err = native._Error()
    ok = native.lib().cb200_supports(plan, len(plan), C.byref(err))
    return ok, err.code, err.message.decode(errors="replace")


TYPES = [P.BOOL, P.INT8, P.INT16, P.INT32, P.INT64, P.DATE, P.TIMESTAMP, P.FLOAT, P.DOUBLE, P.DECIMAL(12, 2), P.DECIMAL(38, 4), P.STRING,
         P.DT("BYTES")]
LIT = {"BOOL": True, "INT8": -3, "INT16": 300, "INT32": -70000, "INT64": 1 << 40, "DATE": 19000, "TIMESTAMP": 1 << 50, "FLOAT": 1.5,
       "DOUBLE": -2.25, "STRING": "m"}


def _lit(t, v=None):
    if v is None:
        v = LIT.get(t.name, 12345)
    return P.literal(v, t)


def _range(types, keys, n, rows):
    return P.shuffle_writer(P.scan(types), P.range_partitioning(keys, n, rows))


def test_accepted_range_plans(native):
    for i, t in enumerate(TYPES[:-1]):
        for d in (False, True):
            for nf in (False, True):
                key = P.sort_order(P.bound(i, t), d, nf)
                for rows in ([], [[_lit(t)]], [[P.literal(None, t)]], [[P.literal(None, t)], [_lit(t)]] if nf else [[_lit(t)], [P.literal(None, t)]]):
                    ok, code, why = _why(native, _range(TYPES, [key], 8, rows))
                    assert ok, (t, d, nf, code, why)
    # floats by their bits: NaNs with payloads, -0.0 < +0.0
    f = [P.literal_bits(b, P.DOUBLE) for b in (0xFFF8000000000001, 0x8000000000000000, 0x0, 0x7FF8000000000000, 0x7FF8000000000001)]
    assert _why(native, _range(TYPES, [P.sort_order(P.bound(8, P.DOUBLE))], 8, [[x] for x in f]))[0]
    assert not _why(native, _range(TYPES, [P.sort_order(P.bound(8, P.DOUBLE))], 8, [[x] for x in f[::-1]]))[0]
    assert _why(native, _range(TYPES, [P.sort_order(P.bound(8, P.DOUBLE), True)], 8, [[x] for x in f[::-1]]))[0]
    g = [P.literal_bits(b, P.FLOAT) for b in (0xFF800001, 0x80000000, 0x0, 0x7FC00000, 0x7FC00001)]
    assert _why(native, _range(TYPES, [P.sort_order(P.bound(7, P.FLOAT))], 8, [[x] for x in g]))[0]
    assert not _why(native, _range(TYPES, [P.sort_order(P.bound(7, P.FLOAT))], 8, [[g[4]], [g[3]]]))[0]
    # eight keys of 225 bits, several words; 1 partition with no bounds; 16 384 partitions
    eight = [P.sort_order(P.bound(i, TYPES[i])) for i in (0, 1, 2, 3, 5, 7, 11, 4)]
    row = [_lit(TYPES[i]) for i in (0, 1, 2, 3, 5, 7, 11, 4)]
    assert _why(native, _range(TYPES, eight, 200, [row, row]))[0]
    assert _why(native, _range(TYPES, [P.sort_order(P.bound(4, P.INT64))], 1, []))[0]
    big = [[_lit(P.INT64, v)] for v in range(16383)]
    assert _why(native, _range(TYPES, [P.sort_order(P.bound(4, P.INT64))], 16384, big))[0]
    # strings: equal bounds, the empty string
    s = [[_lit(P.STRING, v)] for v in ("", "a", "a", "b\xff")]
    assert _why(native, _range(TYPES, [P.sort_order(P.bound(11, P.STRING))], 8, s))[0]


def test_deduplicated_keys(native):
    """a repeated key column is dropped with its options; boundary rows hold the deduplicated keys, further entries ignored"""
    k0, k0_desc, k1 = P.sort_order(P.bound(4, P.INT64)), P.sort_order(P.bound(4, P.INT64), True), P.sort_order(P.bound(3, P.INT32))
    rows = [[_lit(P.INT64, 1), _lit(P.INT32, 9)], [_lit(P.INT64, 5), _lit(P.INT32, 0)]]
    assert _why(native, _range(TYPES, [k0, k0_desc, k1], 4, rows))[0]                 # ascending on col 4, the DESC repeat dropped
    ok, code, why = _why(native, _range(TYPES, [k0, k0_desc, k1], 4, rows[::-1]))
    assert not ok and code == 4 and "ascending" in why
    extra = [r + [_lit(P.STRING)] for r in rows]                                       # entries past the key count are not read
    assert _why(native, _range(TYPES, [k0, k1, k0], 4, extra))[0]
    ok, code, why = _why(native, _range(TYPES, [k0, k1, k0], 4, [[_lit(P.INT64, 1)]]))
    assert not ok and code == 4 and "1 entries for 2 keys" in why


def test_refused_range_plans(native):
    def refused(plan, words):
        ok, code, why = _why(native, plan)
        assert not ok and code == 1 and words in why, (code, why)
    types = [P.INT32] * 9 + [P.DECIMAL(38, 0)] * 2 + [P.DT("BYTES")]
    refused(_range(types, [P.sort_order(P.add(P.bound(0, P.INT32), P.bound(1, P.INT32), P.INT32))], 4, []), "put a Projection below")
    refused(_range(types, [P.sort_order(P.bound(11, P.DT("BYTES")))], 4, []), "binary")
    refused(_range(types, [P.sort_order(P.bound(i, P.INT32)) for i in range(9)], 4, []), "more than 8")
    refused(_range(types, [P.sort_order(P.bound(i, P.INT32)) for i in range(8)], 4, []), "256 bits")
    refused(_range(types, [P.sort_order(P.bound(9, types[9])), P.sort_order(P.bound(10, types[10]))], 4, []), "256 bits")
    refused(_range(types, [P.sort_order(P.bound(0, P.INT32))], 16385, []), "at most 16384")
    assert _why(native, _range([P.INT16] * 8, [P.sort_order(P.bound(i, P.INT16)) for i in range(8)], 4, []))[0]


def test_range_plan_errors(native):
    def malformed(plan, words):
        ok, code, why = _why(native, plan)
        assert not ok and code == 4 and words in why, (code, why)
    k = [P.sort_order(P.bound(4, P.INT64))]
    malformed(_range(TYPES, k, 0, []), "without partitions")
    malformed(_range(TYPES, k, -3, []), "without partitions")
    malformed(_range(TYPES, k, 4, [[P.bound(4, P.INT64)]]), "not a literal")
    malformed(_range(TYPES, k, 4, [[_lit(P.INT32, 1)]]), "is int32, its key int64")
    malformed(_range(TYPES, [P.sort_order(P.bound(9, TYPES[9]))], 4, [[P.literal(1, P.DECIMAL(12, 3))]]), "decimal128(12,3)")
    malformed(_range(TYPES, k, 4, [[]]), "0 entries for 1 keys")
    malformed(_range(TYPES, k, 3, [[_lit(P.INT64, v)] for v in (1, 2, 3)]), "3 range boundary rows for 3 partitions")
    malformed(_range(TYPES, k, 1, [[_lit(P.INT64, 1)]]), "for 1 partitions")
    malformed(_range(TYPES, k, 8, [[_lit(P.INT64, 2)], [_lit(P.INT64, 1)]]), "ascending")
    malformed(_range(TYPES, [P.sort_order(P.bound(4, P.INT64), nulls_first=False)], 8, [[P.literal(None, P.INT64)], [_lit(P.INT64, 1)]]), "ascending")
    malformed(_range(TYPES, [P.sort_order(P.bound(11, P.STRING))], 8, [[_lit(P.STRING, "b")], [_lit(P.STRING, "a")]]), "ascending")
    malformed(_range(TYPES, [], 4, []), "without sort orders")


def test_round_robin_plans(native):
    types = [P.INT32, P.STRING, P.DOUBLE, P.DECIMAL(38, 2), P.BOOL] * 3
    for m in (-5, -1, 0, 1, 3, len(types), len(types) + 4):
        ok, code, why = _why(native, P.shuffle_writer(P.scan(types), P.round_robin_partitioning(200, m)))
        assert ok, (m, code, why)
    assert _why(native, P.shuffle_writer(P.scan(types), P.round_robin_partitioning(16384)))[0]
    ok, code, why = _why(native, P.shuffle_writer(P.scan(types), P.round_robin_partitioning(16385)))
    assert not ok and code == 1 and "round-robin partitioning into 16385" in why
    ok, code, why = _why(native, P.shuffle_writer(P.scan(types), P.round_robin_partitioning(0)))
    assert not ok and code == 4
    nul = [P.INT32, P.DT("NULL")]
    ok, code, why = _why(native, P.shuffle_writer(P.scan(nul), P.round_robin_partitioning(8)))
    assert not ok and code == 1 and "round-robin partitioning on column 1" in why, why
    assert _why(native, P.shuffle_writer(P.scan(nul), P.round_robin_partitioning(8, 1)))[0]     # only column 0 is hashed


def test_hash_and_single_unchanged(native):
    types = [P.INT32] * 9
    assert _why(native, P.shuffle_writer(P.scan(types), P.hash_partitioning([P.bound(0, P.INT32)], 8)))[0]
    ok, code, why = _why(native, P.shuffle_writer(P.scan(types), P.hash_partitioning([P.bound(i, P.INT32) for i in range(9)], 8)))
    assert not ok and code == 1 and "more than 8 hash-partition keys" in why
    ok, code, why = _why(native, P.shuffle_writer(P.scan(types), P.hash_partitioning([P.bound(0, P.INT32)], 16385)))
    assert not ok and code == 1 and "hash partitioning into 16385" in why
    assert _why(native, P.shuffle_writer(P.scan(types), P.single_partitioning()))[0]
    ok, code, why = _why(native, P.shuffle_writer(P.scan(types), P.f_len(5, b"")))              # a partitioning this build does not know
    assert not ok and code == 1 and "partitioning field 5" in why, (code, why)


def test_round_robin_reference(oracle):
    """the round-robin reference is hash partitioning over the first columns, pmod by the oracle's rule"""
    import partref
    t = pa.table(special_table(400, 9))
    for m in (-1, 0, 1, 3, 12, 40):
        starts, order, _ = R.round_robin_partition(oracle, t, 7, m)
        k = R.round_robin_columns(t.num_columns, m)
        h = partref.key_hashes(oracle, t, list(range(k)))
        pids = np.array([oracle.pmod(int(x), 7) for x in h])
        _, want_starts, want_order = oracle.partition_rows(h, 7)
        assert starts == list(want_starts) and (order == want_order).all()
        assert (np.repeat(np.arange(7), np.diff(starts)) == pids[order]).all()


def test_partitioning_field_numbers():
    """partitioning.proto's oneof and message fields (tests/golden/reference_partitioning_fields.json)"""
    import json
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_partitioning_fields.json")) as f:
        ref = json.load(f)
    assert ref["Partitioning"] == P.PARTITIONING_FIELD
    assert ref["RangePartition"] == {"sort_orders": 1, "num_partitions": 2, "boundary_rows": 4}
    assert ref["BoundaryRow"] == {"partition_bounds": 1}
    assert ref["RoundRobinPartition"] == {"num_partitions": 1, "max_hash_columns": 2}
