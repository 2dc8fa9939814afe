"""The Parquet page matrix shared by tests/test_parquet_pages_cpu.py (which pins every file against pyarrow and the oracle) and
tests/test_gpu_parquet_pages.py (which decodes them on the device): hand-built files (tests/pqwrite.py) whose run shapes, bit widths,
level layouts, page shapes, codecs and Snappy element forms stock writers never produce.

A case is (files, column names, chunk_rows); a file is (columns, row groups of Chunks).  The expected output of a column is its chunks'
values / validity, concatenated in file and row-group order."""
import numpy as np

import pqwrite as W

# name -> (Column arguments, requested type name, DECIMAL (precision, scale) or None)
TYPES = {
    "i8": (dict(phys=W.INT32, converted=W.CT_INT_8), "INT8", None),
    "i16": (dict(phys=W.INT32, converted=W.CT_INT_16), "INT16", None),
    "i32": (dict(phys=W.INT32), "INT32", None),
    "date": (dict(phys=W.INT32, converted=W.CT_DATE), "DATE", None),
    "d9": (dict(phys=W.INT32, converted=W.CT_DECIMAL, precision=9, scale=2), "DECIMAL", (9, 2)),
    "i64": (dict(phys=W.INT64), "INT64", None),
    "d18": (dict(phys=W.INT64, converted=W.CT_DECIMAL, precision=18, scale=3), "DECIMAL", (18, 3)),
    "f32": (dict(phys=W.FLOAT), "FLOAT", None),
    "f64": (dict(phys=W.DOUBLE), "DOUBLE", None),
    "fl12": (dict(phys=W.FLBA, type_length=6, converted=W.CT_DECIMAL, precision=12, scale=2), "DECIMAL", (12, 2)),
    "fl30": (dict(phys=W.FLBA, type_length=13, converted=W.CT_DECIMAL, precision=30, scale=4), "DECIMAL", (30, 4)),
    "s": (dict(phys=W.BYTE_ARRAY, converted=0), "STRING", None),
}
FIXED = [t for t in TYPES if t != "s"]
SHAPES = ("packed", "rle", "rle1", "mixed", "long_tail", "packed_runs", "zero_runs")
ARROW_SHAPES = tuple(s for s in SHAPES if s != "zero_runs")   # Arrow's reader stops at a zero-length run


def column(kind, name=None, optional=True):
    return W.Column(name or kind, optional=optional, **TYPES[kind][0])


def gen(kind, n, rng):
    """n distinct-ish values of the type (ints; FLOAT / DOUBLE as bit patterns with NaN payloads, -0.0, infinities; strings as bytes)"""
    lim = {"i8": 7, "i16": 15, "d9": 29, "date": 20, "i32": 31, "i64": 63, "d18": 59, "fl12": 39, "fl30": 58}
    if kind in lim:
        b = lim[kind]
        v = [int(x) for x in rng.integers(-(2**b), 2**b, n, dtype=np.int64)] if b < 63 else [int(x) for x in rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)]
        if kind == "fl30":
            v = [x * 10**12 + int(y) for x, y in zip(v, rng.integers(0, 10**12, n))]
        return v
    if kind == "f32":
        sp = [0x7FC0BEEF, 0xFF800001, 0x80000000, 0x00000001, 0x7F800000, 0xFF800000]
        return (sp + [int(x) for x in rng.integers(0, 2**32, n, dtype=np.uint64)])[:n]
    if kind == "f64":
        sp = [0x7FF8DEADBEEF0001, 0xFFF0000000000001, 0x8000000000000000, 1, 0x7FF0000000000000, 0xFFF0000000000000]
        return (sp + [int(x) for x in rng.integers(0, 2**63, n, dtype=np.uint64)])[:n]
    return [f"w{int(x):05d}".encode() + (b"\xc3\xbc" if x % 7 == 0 else b"") for x in rng.integers(0, 10**5, n)]


def pick(dictionary, n, rng, null_frac=0.2):
    """n values drawn from the dictionary (every entry, including the last, appears when n allows), validity with null_frac NULLs"""
    idx = rng.integers(0, len(dictionary), n)
    idx[: min(n, 3)] = [len(dictionary) - 1, 0, len(dictionary) // 2][: min(n, 3)]
    valid = (rng.random(n) >= null_frac).tolist()
    return [dictionary[i] for i in idx], valid


# ---- dictionary indices ---------------------------------------------------------------------------------------------------------
def dict_case(kind, rows=240, seed=0):
    """One row group per (dictionary size, bit width): every width 0..32 (dictionaries of min(2^w, 257) entries: over-wide from 9 on),
    then 255 / 256 / 257 / 65 537 entries at their least width, one more, and 32; index and level shapes cycle through SHAPES."""
    rng = np.random.default_rng(seed)
    combos = [(1 if w == 0 else min(1 << w, 257), w) for w in range(33)]
    for d in (1, 2, 255, 256, 257, 65537):
        m = max(d - 1, 0).bit_length()
        combos += [(d, m), (d, m + 1), (d, 32)]
    col = column(kind)
    rgs = []
    for k, (d, w) in enumerate(combos):
        if d == 65537 and kind == "s":
            d = 4099                                                   # host dictionaries: kept small
        dictionary = list(dict.fromkeys(gen(kind, d + 64, rng)))[:d]
        vals, valid = pick(dictionary, rows, rng)
        if d > 256:
            vals[3:3 + min(d, 64)] = dictionary[-min(d, 64):]
        rgs.append([W.chunk(col, vals, valid, [61, 8, 100], dictionary=dictionary, bit_width=w, index_shape=SHAPES[k % len(SHAPES)],
                            level_shape=SHAPES[(k // 2) % len(SHAPES)], version=1 + k % 2, codec=(W.NONE, W.SNAPPY)[(k // 3) % 2],
                            encoding=(W.RLE_DICTIONARY, W.PLAIN_DICTIONARY)[(k // 5) % 2])])
    return ([((col,), rgs)], [kind], 2048)


# ---- definition levels ----------------------------------------------------------------------------------------------------------
LAYOUTS = ("none", "one", "alternating", "all", "stretch")


def layout(name, n, page):
    if name == "none":
        return [True] * n
    if name == "one":
        return [i != n // 2 for i in range(n)]
    if name == "alternating":
        return [i % 2 == 1 for i in range(n)]
    if name == "all":
        return [False] * n
    return [not (page - 9 <= i % (3 * page) <= 2 * page + 5) for i in range(n)]   # NULL stretches across page edges


def levels_case(null_count="exact", layouts=LAYOUTS, seed=1):
    """i64 PLAIN, optional: every level shape x page version x NULL layout, one row group each; the last row group of each layout ends
    in NULLs and the next starts with them (stretch)."""
    rng = np.random.default_rng(seed)
    col = column("i64")
    rgs = []
    for lay in layouts:
        for si, shape in enumerate(SHAPES):
            for ver in (1, 2):
                n, page = 150 + 7 * si, 40 + si
                valid = layout(lay, n, page)
                vals = gen("i64", n, rng)
                rgs.append([W.chunk(col, vals, valid, page, level_shape=shape, version=ver, null_count=null_count)])
    return ([((col,), rgs)], ["i64"], 1200)


# ---- page shapes ----------------------------------------------------------------------------------------------------------------
def tiny_pages_case(seed=2):
    """pages of 0, 1 and 7..9 values, then a chunk of thousands of 1..3-row pages"""
    rng = np.random.default_rng(seed)
    col = column("i32")
    v1, ok1 = gen("i32", 400, rng), (rng.random(400) > 0.3).tolist()
    v2, ok2 = gen("i32", 6000, rng), (rng.random(6000) > 0.3).tolist()
    rgs = [[W.chunk(col, v1, ok1, [0, 1, 7, 8, 9], version=1)], [W.chunk(col, v1, ok1, [1, 9, 8, 7], version=2, level_shape="packed")],
           [W.chunk(col, v2, ok2, [1, 2, 3], version=2, level_shape="rle1", codec=W.SNAPPY)]]
    return ([((col,), rgs)], ["i32"], 1 << 20)


def fallback_case(kind, seed=3):
    """a dictionary that falls back to PLAIN partway through the chunk, with both dictionary spellings across row groups"""
    rng = np.random.default_rng(seed)
    col = column(kind)
    rgs = []
    for k, enc in enumerate((W.RLE_DICTIONARY, W.PLAIN_DICTIONARY)):
        dictionary = list(dict.fromkeys(gen(kind, 40, rng)))
        vals, valid = pick(dictionary, 900, rng)
        vals[500:] = gen(kind, 400, rng)                              # values the dictionary does not hold: PLAIN from row 500 on
        rgs.append([W.chunk(col, vals, valid, 100, dictionary=dictionary, fallback_at=500, encoding=enc, version=1 + k, codec=W.SNAPPY)])
    return ([((col,), rgs)], [kind], 1 << 20)


def codecs_case(seed=4):
    """row groups of one column with NONE / SNAPPY / ZSTD codecs and their own dictionaries, v2 pages stored uncompressed inside
    SNAPPY chunks, and chunkRows so that one batch holds several row groups"""
    rng = np.random.default_rng(seed)
    cols = (column("i64"), column("fl30"), column("s"))
    rgs = []
    for k in range(9):
        codec = (W.NONE, W.SNAPPY, W.ZSTD)[k % 3]
        chunks = []
        for c in cols:
            dictionary = list(dict.fromkeys(gen(c.name, 30 + 20 * k, rng)))
            vals, valid = pick(dictionary, 700, rng)
            chunks.append(W.chunk(c, vals, valid, [150, 90], dictionary=dictionary, codec=codec, version=2 if k % 2 else 1,
                                  compressed=k % 4 != 1, index_shape=ARROW_SHAPES[k % len(ARROW_SHAPES)], level_shape=ARROW_SHAPES[(k + 2) % len(ARROW_SHAPES)]))
        rgs.append(chunks)
    return ([(cols, rgs)], [c.name for c in cols], 2500)


def required_optional_case(seed=5):
    """a required file and an optional one of the same column in one scan"""
    rng = np.random.default_rng(seed)
    req, opt = column("d18", optional=False), column("d18")
    v, ok = gen("d18", 500, rng), (rng.random(500) > 0.5).tolist()
    return ([((req,), [[W.chunk(req, v, [True] * 500, 64, level_shape="rle1")]]),
             ((opt,), [[W.chunk(opt, v, ok, 64, level_shape="rle1", null_count=None)]])], ["d18"], 1 << 20)


# ---- Snappy inside pages --------------------------------------------------------------------------------------------------------
def _snappy_page(col, vals, **el_kw):
    p = W.data_page(col, vals, [True] * len(vals))
    p.elements = W.snappy_elements(p.body, **el_kw)
    return p


def snappy_case(seed=6):
    """required i64 PLAIN v1 pages, each compressed by its own element list: every literal form, copy-1 / copy-2 / copy-4, overlapping
    copies of period 1..64, references past 8 KiB and 16 KiB, pages of exactly k x 64 KiB whose elements either end on every 64 KiB
    boundary or straddle it, references into an earlier 64 KiB segment, a 1 MiB page, and regular and irregular pages in one column."""
    rng = np.random.default_rng(seed)
    col = column("i64", optional=False)
    pages, values = [], []

    def add(vals, **kw):
        pages.append(_snappy_page(col, vals, **kw))
        values.extend(vals)
    rnd = lambda n: gen("i64", n, rng)
    for form, mx in ((0, 60), (1, 256), (2, 1000), (3, 5000), (4, 5000)):
        add(rnd(600), lit_form=form, max_lit=mx)                                   # every literal length form
    block = rnd(40)
    add(block * 30, copy_kind=1)                                                   # copy-1 (lengths 4..11, offsets < 2048)
    add(block * 30, copy_kind=2)
    add(block * 30, copy_kind=4)                                                   # 4-byte offsets below 64 KiB
    for period in (1, 2, 3, 7, 8, 13, 32, 63, 64):                                 # overlapping copies: byte patterns of period 1..64
        raw = bytes(rng.integers(0, 256, period, dtype=np.uint8)) * (4096 // period + 1)
        add([int.from_bytes(raw[i:i + 8], "little", signed=True) for i in range(0, 4096, 8)])
    for dist in (9 * 1024, 17 * 1024, 40 * 1024):                                  # references past the 8 KiB / 16 KiB rings
        a = rnd(dist // 8)
        add(a + a[:600] + rnd(100) + a[100:700])
    for k in (1, 2, 3):                                                            # k x 64 KiB, elements end on the boundaries ...
        add(rnd(8192 * k), max_lit=512)
        add(rnd(8192 * k), max_lit=1000)                                           # ... or straddle them (serial decoder)
    a = rnd(8192)
    add(a + a[-100:] + rnd(50), max_lit=512)                                       # the 2nd segment's copy reaches into the 1st
    add(rnd(65536) + rnd(65536)[:0] + [7] * 65536, max_lit=4096)                   # a 1 MiB page: random half, then one long run
    return ([((col,), [[W.Chunk(pages, values, [True] * len(values), W.SNAPPY, 0)]])], ["i64"], 1 << 20)


def snappy_dict_case(seed=7):
    """dictionary pages compressed with Snappy, an fl30 (16-byte) and a string dictionary, with long literals and copies"""
    rng = np.random.default_rng(seed)
    cols = (column("fl30"), column("s"))
    chunks = []
    for c in cols:
        dictionary = list(dict.fromkeys(gen(c.name, 3000, rng)))
        vals, valid = pick(dictionary, 4000, rng)
        chunks.append(W.chunk(c, vals, valid, 1000, dictionary=dictionary, codec=W.SNAPPY))
    return ([(cols, [chunks])], [c.name for c in cols], 1 << 20)


def cases():
    """name -> case"""
    out = {f"dict_{k}": (lambda k=k: dict_case(k, seed=i)) for i, k in enumerate(("i32", "i64", "fl30", "fl12", "f32", "s"))}
    out.update({f"fallback_{k}": (lambda k=k: fallback_case(k)) for k in FIXED})
    out.update({"levels": levels_case, "levels_no_stats": lambda: levels_case(None),
                "levels_fast_path": lambda: levels_case("exact", ("none",)), "tiny_pages": tiny_pages_case, "codecs": codecs_case,
                "required_optional": required_optional_case, "snappy": snappy_case, "snappy_dict": snappy_dict_case})
    return out


def expected(case):
    """column name -> (values, valid) concatenated over files and row groups"""
    files, names, _ = case
    out = {}
    for cols, rgs in files:
        for ci, c in enumerate(cols):
            v, ok = out.setdefault(c.name, ([], []))
            for chunks in rgs:
                v.extend(chunks[ci].values)
                ok.extend(chunks[ci].valid)
    return {n: out[n] for n in names}


def file_bytes(case):
    return [W.write_file(list(cols), rgs) for cols, rgs in case[0]]
