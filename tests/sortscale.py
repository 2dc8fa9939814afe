"""Sort and TopK at scale: input generators whose packed row keys have a chosen digit shape, and a vectorised reference of the stable
order that keeps a 70 M-row sort to seconds.

The reference (`order`) is tests/sortref.py's rule -- a stable sort per key, last key first, each NULL placed by its own key -- with the
ranks taken straight from the values instead of from np.unique: one stable argsort of a uint64 order value per key, and one more of the
null flag when the key has NULLs.  Floats use the IEEE totalOrder bits of sortref.value_order, dictionary strings the byte-order rank of
their entry (one lookup table per distinct dictionary), decimals wider than 64 bits fall back to sortref.key_ranks.

Most generators describe the packed key itself: an (n, W) uint64 array of W words per row, word 0 the most significant, the layout of
device/cb_sortkey.h.  `words_table` turns it into key columns whose encoding is exactly those words: W INT64 keys without NULLs (64 bits
each; a DESC key stores the complement), or two INT32 keys per word (up to 7 keys).  The planner counts a NULL bit per key within its
256 bits, so a 4-word key keeps 224 value bits: word 0 holds only its low 32 (`fit`).  That the encoder really returns the
generator's words is checked through the host compile of the encoder (sortkey_test.cpp) in tests/test_sort_scale_cpu.py, so the digit
shape a test claims -- one digit varies, one row differs, a tile on one digit -- is the shape the radix sort sees.

Every table carries a `row` column, its input position, so the output's stability is compared bit for bit."""
import ctypes as C
import os
import subprocess
from dataclasses import dataclass, field

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc

import partref
import sortref as R

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "datafusion-comet_b200", "csrc")

TILE = 4096            # rows per tile of k_sort_hist / k_sort_scatter
SLICE = 512            # rows per warp of a tile in k_sort_scatter
BLOCK = 1024           # rows per block of k_sort_select_keep and the compaction plan
EDGE_SIZES = [1, 31, 32, 33, 511, 512, 513, 1023, 1024, 1025, 4095, 4096, 4097, 3 * TILE - 1, 3 * TILE + 1, 16 * TILE - 1, 16 * TILE + 1]
SIGN = np.uint64(1 << 63)


# ---- the reference ----------------------------------------------------------------------------------------------------------------------
_dict_cache = {}


def _dict_order(col):
    """uint64 byte-order rank of each row of a dictionary string column (chunks may carry different dictionaries)"""
    chunks = col.chunks if isinstance(col, pa.ChunkedArray) else [col]
    key = lambda d: (d.buffers()[1].address, d.offset, len(d))
    dicts = {key(c.dictionary): c.dictionary.cast(pa.binary()) for c in chunks}
    uniq = pc.unique(pa.concat_arrays(list(dicts.values())))
    uniq = uniq.take(pc.sort_indices(uniq))                                   # binary sorts by unsigned bytes
    _dict_cache.clear()
    parts = []
    for c in chunks:
        k = key(c.dictionary)
        if k not in _dict_cache:
            _dict_cache[k] = np.append(np.asarray(pc.index_in(dicts[k], value_set=uniq)).astype(np.uint64), np.uint64(0))
        parts.append(_dict_cache[k][np.asarray(c.indices.fill_null(0)).astype(np.int64)])
    return np.concatenate(parts) if parts else np.zeros(0, np.uint64)


def order_value(col, descending=False):
    """(uint64 order value, valid mask): rows are in the key's order for valid rows when sorted by the value ascending"""
    if pa.types.is_dictionary(col.type):
        u = _dict_order(col)
    else:
        arr = R._array(col)
        t = arr.type
        if pa.types.is_decimal(t) and t.precision > 18:
            u = R.key_ranks(arr, False, True).astype(np.uint64)   # NULL rows rank 0: overwritten below
        else:
            v = R.value_order(arr)
            u = v.view(np.uint64) ^ SIGN if v.dtype == np.int64 else v.astype(np.uint64)
    valid = np.asarray(col.is_valid()) if col.null_count else None
    if descending:
        u = ~u
    if valid is not None:
        u = np.where(valid, u, np.uint64(0))
    return u, valid


def order(table, keys):
    """the stable order of the rows (row indices), keys (column, descending, nulls_first) as in sortref"""
    idx = np.arange(table.num_rows)
    for c, desc, nf in reversed(keys):
        u, valid = order_value(table.column(c), desc)
        idx = idx[np.argsort(u[idx], kind="stable")]
        if valid is not None:
            flag = (valid if nf else ~valid).astype(np.uint8)                 # 0 first
            idx = idx[np.argsort(flag[idx], kind="stable")]
    return idx


def sort_table(table, keys, fetch=None, skip=None):
    """the operator's output, sorted[skip : fetch], dictionary columns spelled out (sortref.sort_table on the fast order)"""
    idx = order(table, keys)
    lo, hi = R.window(len(idx), fetch, skip)
    take = pa.array(idx[lo:hi], pa.int64())
    return pa.table([R._array(table.column(i)).take(take) for i in range(table.num_columns)], names=table.column_names)


def check(got, want, keys):
    """the device's output equals the reference's bit for bit, row column included, and is in the keys' order"""
    if want.num_rows == 0:
        assert got is None or got.num_rows == 0
        return
    assert got is not None, "no output"
    partref.assert_tables_equal(got, want)
    R.assert_sorted(got, keys)


# ---- packed keys -> key columns -----------------------------------------------------------------------------------------------------
def top_digit(W):
    """the highest digit of word 0 a key of W words can vary in here: the planner counts one NULL bit per key and allows 256 bits, so
    a 4-word key of NULL-free INT64 / INT32 keys holds at most 224 value bits -- word 0 keeps its low 32"""
    return 7 if W < 4 else 3


def fit(w):
    """the generator's words as a key of their width can hold them (top_digit): word 0 of a 4-word key cut to its low 32 bits"""
    if w.shape[1] == 4:
        w = w.copy()
        w[:, 0] &= np.uint64(0xFFFFFFFF)
    return w


def words_table(w, kind="i64", desc=None):
    """key columns whose packed row key is fit(w) ((n, W) uint64, word 0 most significant), then `row`.  kind "i64": one INT64 key per
    word (an INT32 for word 0 of 4), kind "i32": two INT32 keys per word (high half first; word 0 of 4 only its low half), so up to 7
    keys.  desc[k]: key k is DESC (its column holds the complement).  -> (table, keys)"""
    n, W = w.shape
    w = fit(w)
    halves = []                                                               # (word, shift, bits) of each key, first key first
    for j in range(W):
        if kind == "i64":
            halves.append((j, 0, 32 if W == 4 and j == 0 else 64))
        else:
            halves += [(j, 0, 32)] if W == 4 and j == 0 else [(j, 32, 32), (j, 0, 32)]
    desc = desc or [False] * len(halves)
    assert len(desc) == len(halves), (len(desc), len(halves))
    cols = []
    for (j, sh, bits), d in zip(halves, desc):
        if bits == 64:
            u = ~w[:, j] if d else w[:, j]
            cols.append(pa.array((u ^ SIGN).view(np.int64)))
        else:
            u = (w[:, j] >> np.uint64(sh)).astype(np.uint32)
            u = ~u if d else u
            cols.append(pa.array((u ^ np.uint32(1 << 31)).view(np.int32)))
    names = [f"k{i}" for i in range(len(halves))]
    cols.append(pa.array(np.arange(n, dtype=np.int64)))
    return pa.table(cols, names=names + ["row"]), [(i, bool(d), True) for i, d in enumerate(desc)]


def random_words(n, W, seed):
    return np.random.default_rng(seed).integers(0, 2**64, (n, W), dtype=np.uint64, endpoint=False)


def one_row_differs(n, W, at, word, digit, seed):
    """every row the same key but row `at`, which differs from it in digit `digit` (0 = lowest byte) of word `word` only"""
    rng = np.random.default_rng(seed)
    w = np.tile(rng.integers(0, 2**64, (1, W), dtype=np.uint64), (n, 1))
    w[at, word] ^= np.uint64(int(rng.integers(1, 256)) << (8 * digit))
    return w


def runs(n, W, length, seed):
    """the last word constant over runs of `length` rows (32: all lanes of a warp step on one digit, 512: a warp's slice, 4096: a tile);
    the words above it random per row"""
    rng = np.random.default_rng(seed)
    w = rng.integers(0, 2**64, (n, W), dtype=np.uint64)
    per = rng.integers(0, 2**64, (n + length - 1) // length, dtype=np.uint64)
    w[:, W - 1] = np.repeat(per, length)[:n]
    return w


def tile_on_one_digit(n, W, tile, seed):
    """random keys, except that every row of tile `tile` has the same last word: on one digit in every pass over that word"""
    w = random_words(n, W, seed)
    w[tile * TILE:(tile + 1) * TILE, W - 1] = w[tile * TILE, W - 1]
    return w


def pattern(n, W, kind, period=None, seed=0):
    """the last word: ascending (sorted), descending (reverse) or i mod period (sawtooth); the words above it one constant each"""
    i = np.arange(n, dtype=np.uint64)
    v = {"sorted": i, "reverse": np.uint64(n - 1) - i, "sawtooth": i % np.uint64(period or 1)}[kind]
    w = np.tile(np.random.default_rng(seed).integers(0, 2**64, (1, W), dtype=np.uint64), (n, 1))
    w[:, W - 1] = v
    return w


def one_digit_varies(n, W, where, seed, distinct=256):
    """only one digit varies, over `distinct` values (few distinct keys over many rows: stability): "low" the lowest digit of the
    last word, "top" the top digit of the first word (top_digit)"""
    rng = np.random.default_rng(seed)
    w = np.tile(rng.integers(0, 2**64, (1, W), dtype=np.uint64), (n, 1))
    word, sh = (W - 1, 0) if where == "low" else (0, 8 * top_digit(W))
    w[:, word] &= ~np.uint64(0xFF << sh)
    w[:, word] |= rng.integers(0, distinct, n).astype(np.uint64) << np.uint64(sh)
    return w


def decided_in_word(n, W, j, seed):
    """words above j take two values each (a row's prefix is shared by about n / 2^j rows), word j is random and the words below it
    too: the TopK select narrows through words 0 .. j - 1 and decides in word j"""
    rng = np.random.default_rng(seed)
    w = rng.integers(0, 2**64, (n, W), dtype=np.uint64)
    for k in range(j):
        two = rng.integers(0, 2**64, 2, dtype=np.uint64)
        w[:, k] = two[rng.integers(0, 2, n)]
    return w


def chunk_trend(n, chunk, improving, seed):
    """one key word: every chunk of `chunk` rows below all earlier ones (improving: each chunk replaces every TopK candidate) or above
    them (worsening: no chunk after the first replaces any)"""
    rng = np.random.default_rng(seed)
    c = (np.arange(n) // chunk).astype(np.uint64)
    n_chunks = int(c[-1]) + 1
    hi = (np.uint64(n_chunks) - c) if improving else c
    return ((hi << np.uint64(40)) | rng.integers(0, 2**40, n, dtype=np.uint64)).reshape(n, 1)


def tie_run_across_chunks(n, fetch, seed, below=None, run=None):
    """one key word: `below` rows (spread over the whole input) smaller than V, `run` rows equal to V spread over every chunk, the rest
    larger, so the TopK cut-off at `fetch` falls inside the run of V: the earliest V rows in input order must be kept"""
    rng = np.random.default_rng(seed)
    below = fetch // 2 if below is None else below
    run = 4 * fetch if run is None else run
    V = np.uint64(1 << 62)
    w = rng.integers(int(V) + 1, 2**64, n, dtype=np.uint64)
    pos = rng.permutation(n)
    w[pos[:below]] = rng.integers(0, int(V), below, dtype=np.uint64)
    w[pos[below:below + run]] = V
    return w.reshape(n, 1)


# ---- tables with NULLs, float specials, extremes and dictionaries -----------------------------------------------------------------------
F64_SPECIAL = [0xFFF8000000000001, 0xFFF8000000000000, 0xFFF0000000000000, 0x8000000000000000, 0x0000000000000000, 0x7FF0000000000000,
               0x7FF8000000000000, 0x7FF8000000000001]   # -NaN payload, -NaN, -Inf, -0.0, +0.0, +Inf, +NaN, +NaN payload


def cutoff_table(n, run, seed):
    """f64, i64 and f32 keys built of runs of `run` equal values -- NULL, -NaN payloads, -Inf, -0.0, +0.0, +Inf, NaNs, i64 MIN / MAX,
    f32 -0.0 / +0.0 -- scattered over the input; a fetch that is a multiple of `run` (+- 1) puts the TopK cut-off on a run edge.
    -> (table, class of each f64 row: 0 = NULL, 1 + index into F64_SPECIAL, 9 = an ordinary value)"""
    rng = np.random.default_rng(seed)
    cls = np.full(n, 9)
    pos = rng.permutation(n)
    for c in range(9):
        cls[pos[c * run:(c + 1) * run]] = c
    f64 = rng.standard_normal(n)
    bits = f64.view(np.uint64)
    for c, b in enumerate(F64_SPECIAL):
        bits[cls == c + 1] = np.uint64(b)
    i64 = rng.integers(-10, 10, n)
    ext = rng.integers(0, 4, n)
    i64 = np.where(ext == 0, np.iinfo(np.int64).min, np.where(ext == 1, np.iinfo(np.int64).max, i64))
    f32 = np.where(rng.integers(0, 2, n) == 0, np.float32(-0.0), np.float32(0.0)).astype(np.float32)
    i64_null = rng.random(n) < 0.01
    t = pa.table({"f64": pa.array(f64, mask=cls == 0), "i64": pa.array(i64, mask=i64_null), "f32": pa.array(f32),
                  "row": pa.array(np.arange(n, dtype=np.int64))})
    return t, cls


def dictionary_words(m, seed):
    """m distinct strings of 1 to 12 bytes, random order (some share long prefixes)"""
    rng = np.random.default_rng(seed)
    out, seen = [], set()
    alphabet = np.frombuffer(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_\xc3", np.uint8)
    while len(out) < m:
        ln = int(rng.integers(1, 13))
        s = bytes(alphabet[rng.integers(0, len(alphabet) - 1, ln)]).decode()
        if rng.random() < 0.2 and out:
            s = out[int(rng.integers(len(out)))] + s[:3]
        if s not in seen:
            seen.add(s)
            out.append(s)
    return out


def string_batches(n, batch, m, growing, seed, null_rate=0.05):
    """record batches of a dictionary string key `s` (int32 indices) over m entries and an INT32 key `v`, then `row`.  growing: batch
    b's dictionary is the first m * (b + 1) / batches entries (each batch a longer dictionary, codes within it); otherwise every batch
    carries the whole dictionary.  -> (batches, the same rows as one table)"""
    rng = np.random.default_rng(seed)
    words = dictionary_words(m, seed)
    nb = (n + batch - 1) // batch
    full = pa.array(words)
    out = []
    for b in range(nb):
        k = min(batch, n - b * batch)
        size = max(1, m * (b + 1) // nb) if growing else m
        d = full.slice(0, size) if growing else full
        codes = pa.array(rng.integers(0, size, k).astype(np.int32), mask=rng.random(k) < null_rate)
        s = pa.DictionaryArray.from_arrays(codes, d)
        v = pa.array(rng.integers(-3, 3, k).astype(np.int32))
        out.append(pa.record_batch([s, v, pa.array(np.arange(b * batch, b * batch + k, dtype=np.int64))], names=["s", "v", "row"]))
    return out, pa.Table.from_batches(out)


def scan_chunks(n):
    """4096-entry chunks of a pass's histogram (256 digits x tiles): k_scan_totals runs ceil(chunks / 1024) iterations"""
    return -(-256 * -(-n // TILE) // 4096)


def is_topk(fetch, chunk):
    """the operator keeps at most `fetch` candidates between chunks (SortNode::topk)"""
    return fetch is not None and fetch <= chunk


def selects(n, fetch, skip, chunk):
    """whether the radix select must run: some sort of the operator wants only the first rows of its input -- a TopK round whose
    merged candidates outnumber fetch (any input of more than one chunk), or a full sort with a fetch below n and no skip"""
    if fetch is None or fetch >= n:
        return False
    return is_topk(fetch, chunk) or not skip


# ---- plans ------------------------------------------------------------------------------------------------------------------------------
def types_of(P, table):
    m = {pa.int64(): P.INT64, pa.int32(): P.INT32, pa.float64(): P.DOUBLE, pa.float32(): P.FLOAT}
    return [P.STRING if pa.types.is_dictionary(f.type) else m[f.type] for f in table.schema]


def plan(P, table, keys, fetch=None, skip=None):
    types = types_of(P, table)
    return P.sort(P.scan(types), [P.sort_order(P.bound(i, types[i]), d, nf) for i, d, nf in keys], fetch=fetch, skip=skip)


# ---- the host encoder: the packed keys the device builds, and its digit passes --------------------------------------------------------
def sortkey_lib(directory):
    so = os.path.join(str(directory), "libcb200_sortkey_scale.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(CSRC, "sortkey_test.cpp")])
    lib = C.CDLL(so)
    lib.cb_sk_kind.argtypes = [C.c_char_p]
    lib.cb_sk_encode.restype = C.c_longlong
    return lib


def _field(col):
    """(layout name, value bits, values, rank table) of a column as the scan hands it to the sort"""
    arr = R._array(col) if not pa.types.is_dictionary(col.type) else (col.combine_chunks() if isinstance(col, pa.ChunkedArray) else col)
    t = arr.type
    if pa.types.is_dictionary(t):
        vals = arr.dictionary.cast(pa.binary()).to_pylist()
        srt = {v: i for i, v in enumerate(sorted(set(vals)))}
        rank = np.array([srt[v] for v in vals] + [0], np.uint32)
        return "dict32", 32, np.ascontiguousarray(R._fixed(arr.indices, np.int32)), rank
    if t in (pa.int64(), pa.float64()):
        return ("i64" if t == pa.int64() else "f64"), 64, np.ascontiguousarray(R._fixed(arr, np.uint64)), None
    if t in (pa.int32(), pa.float32()):
        return ("i32" if t == pa.int32() else "f32"), 32, np.ascontiguousarray(R._fixed(arr, np.uint32)), None
    raise TypeError(f"no scale layout for {t}")


def host_words(lib, table, keys):
    """the packed row keys of the sort of `table` by `keys`, (n, W) uint64, from the host compile of device/cb_sortkey.h.  A key has a
    NULL bit when its column has NULLs (the scan uploads a validity bitmap only then)."""
    n, nk = table.num_rows, len(keys)
    cols = [table.column(c) for c, _, _ in keys]
    lay = [_field(c) for c in cols]
    valids = [np.packbits(np.asarray(c.is_valid()), bitorder="little") if c.null_count else None for c in cols]
    total = sum(b + (v is not None) for (_, b, _, _), v in zip(lay, valids))
    W = max(1, (total + 63) // 64)
    ints = lambda xs: (C.c_int * nk)(*xs)
    out = np.zeros(n * W, np.uint64)
    bad = lib.cb_sk_encode(nk, ints([lib.cb_sk_kind(k.encode()) for k, _, _, _ in lay]), ints([b for _, b, _, _ in lay]),
                           ints([int(d) for _, d, _ in keys]), ints([int(f) for _, _, f in keys]),
                           (C.c_void_p * nk)(*[v.ctypes.data for _, _, v, _ in lay]),
                           (C.c_void_p * nk)(*[None if v is None else v.ctypes.data for v in valids]),
                           (C.c_void_p * nk)(*[None if r is None else r.ctypes.data for _, _, _, r in lay]),
                           ints([0 if r is None else len(r) - 1 for _, _, _, r in lay]), C.c_longlong(n), W,
                           out.ctypes.data_as(C.POINTER(C.c_uint64)))
    assert bad == 0
    return out.reshape(n, W)


def varying_digits(w):
    """the (word, digit) pairs, digit 0 the lowest byte of its word, that are not the same in every row of w"""
    if len(w) == 0:
        return []
    diff = np.bitwise_and.reduce(w, axis=0) ^ np.bitwise_or.reduce(w, axis=0)
    return [(j, d) for j in range(w.shape[1]) for d in range(8) if (int(diff[j]) >> (8 * d)) & 0xFF]


def digit_passes(w):
    """the radix passes a full sort of these keys runs: one per digit not constant over the rows"""
    return len(varying_digits(w))


# ---- the GPU file's cases ------------------------------------------------------------------------------------------------------------
def rounds(n, chunk, batch):
    """TopK rounds over n rows: the scan hands the sort record batches of `batch` rows gathered until they reach chunkRows"""
    return -(-n // (batch * -(-chunk // batch)))


@dataclass
class Case:
    """make(n) -> (table, keys, batches or None); the device sorts n rows through `windows` [(fetch, skip)] with chunkRows `chunk`"""
    make: object
    n: int
    windows: list = field(default_factory=lambda: [(None, None)])
    chunk: int = None
    batch: int = 1 << 20


def _words_case(gen, kind="i64", desc=None):
    def make(n):
        t, k = words_table(gen(n), kind, desc)
        return t, k, None
    return make


TOPK_CHUNK = 1 << 14
TOPK_ROWS = 101 * TOPK_CHUNK + 77                                            # 102 chunks of 2^14 rows, the last of 77
TOPK_FETCHES = [1, 1023, 1024, 1025, 4096, TOPK_CHUNK - 1, TOPK_CHUNK, TOPK_CHUNK + 1]
TOPK_WINDOWS = [(f, None) for f in TOPK_FETCHES] + [(None, 5000), (None, TOPK_ROWS - 1), (4096, 1000), (TOPK_CHUNK, TOPK_CHUNK - 1)]


def _cutoff_case(n):
    t, _ = cutoff_table(n, 2048, 41)
    return t, [(0, False, True), (1, True, False), (2, False, True)], None


def _cutoff_desc_case(n):
    t, _ = cutoff_table(n, 2048, 43)
    return t, [(0, True, False), (1, False, True), (2, True, True)], None


def _strings_case(m, growing, fetch_keys):
    def make(n):
        bs, t = string_batches(n, TOPK_CHUNK // 4, m, growing, 53 + growing)
        return t, fetch_keys, [bs]
    return make


CASES = {
    "topk-random-4w": Case(_words_case(lambda n: random_words(n, 4, 3)), TOPK_ROWS, TOPK_WINDOWS, TOPK_CHUNK, TOPK_CHUNK // 4),
    "topk-few-distinct": Case(_words_case(lambda n: one_digit_varies(n, 2, "low", 5, distinct=7)), TOPK_ROWS, TOPK_WINDOWS, TOPK_CHUNK,
                              TOPK_CHUNK // 4),
    "topk-tie-run": Case(_words_case(lambda n: tie_run_across_chunks(n, 4096, 7)), TOPK_ROWS, [(4096, None), (4095, None), (4096, 2000)],
                         TOPK_CHUNK, 3300),
    "topk-tie-run-small": Case(_words_case(lambda n: tie_run_across_chunks(n, 1024, 8, below=0, run=TOPK_ROWS // 3)), TOPK_ROWS,
                               [(1, None), (1024, None), (1025, 7)], TOPK_CHUNK, 3300),
    "topk-improving": Case(_words_case(lambda n: chunk_trend(n, TOPK_CHUNK, True, 9)), TOPK_ROWS,
                           [(1, None), (1024, None), (TOPK_CHUNK - 1, None), (TOPK_CHUNK, None)], TOPK_CHUNK, TOPK_CHUNK),
    "topk-worsening": Case(_words_case(lambda n: chunk_trend(n, TOPK_CHUNK, False, 10), desc=[True]), TOPK_ROWS,
                           [(1, None), (1024, None), (TOPK_CHUNK - 1, None), (TOPK_CHUNK, None)], TOPK_CHUNK, TOPK_CHUNK),
    **{f"topk-decided-word{j}": Case(_words_case(lambda n, j=j: decided_in_word(n, 4, j, 11 + j)), TOPK_ROWS,
                                     [(1, None), (1000, None), (4096, None), (TOPK_CHUNK, None)], TOPK_CHUNK, TOPK_CHUNK // 4)
       for j in range(4)},
    "topk-decided-3w": Case(_words_case(lambda n: decided_in_word(n, 3, 2, 17)), TOPK_ROWS, [(777, None), (TOPK_CHUNK - 1, None)],
                            TOPK_CHUNK, TOPK_CHUNK // 4),
    "topk-7-int32-keys": Case(_words_case(lambda n: decided_in_word(n, 4, 3, 19), "i32", desc=[False, True] * 3 + [False]), TOPK_ROWS,
                              [(1025, None), (4096, 3)], TOPK_CHUNK, TOPK_CHUNK // 4),
    "topk-cutoff-specials": Case(_cutoff_case, TOPK_ROWS, [(f, None) for f in (2047, 2048, 2049, 4096, 6143, 6144, 6145, 10240, 14336)]
                                 + [(8192, 4095)], TOPK_CHUNK, 3300),
    "topk-cutoff-specials-desc": Case(_cutoff_desc_case, TOPK_ROWS, [(f, None) for f in (1, 2047, 2048, 2049, 4095, 4096, 4097, 6144, 16384)],
                                      TOPK_CHUNK, 3300),
    "strings-large-dict": Case(_strings_case(120_000, False, [(0, False, True), (1, True, False)]), TOPK_ROWS,
                               [(None, None), (1000, None), (TOPK_CHUNK, 10)], TOPK_CHUNK, None),
    "strings-growing-dict": Case(_strings_case(120_000, True, [(0, True, False), (1, False, True)]), TOPK_ROWS,
                                 [(None, None), (None, 20), (1, None), (4097, None), (TOPK_CHUNK, None)], TOPK_CHUNK, None),
}
