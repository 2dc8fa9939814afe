"""CPU-only: the hand-built page matrix (tests/pagecases.py, tests/pqwrite.py) pinned against pyarrow's reader and the oracle, the shared
hybrid decoder (csrc/device/cb_rle.h) on the host against the oracle's, and the scan planner's page tables for the new layouts."""
import ctypes as C
import decimal
import io
import os
import struct
import subprocess

import numpy as np
import pyarrow.parquet as pq
import pytest

import pagecases as PC
import pqwrite as W

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "datafusion-comet_b200", "csrc")
PHYS = {W.INT32: "INT32", W.INT64: "INT64", W.FLOAT: "FLOAT", W.DOUBLE: "DOUBLE", W.FLBA: "FIXED_LEN_BYTE_ARRAY", W.BYTE_ARRAY: "BYTE_ARRAY"}
CODEC = {W.NONE: "UNCOMPRESSED", W.SNAPPY: "SNAPPY", W.ZSTD: "ZSTD"}


def _arrow_values(arr, kind):
    """pyarrow's column as the writer's value convention (ints, float bit patterns, unscaled decimals, bytes); None at NULLs"""
    import pyarrow as pa
    if kind == "date":
        arr = arr.cast(pa.int32())
    if kind in ("f32", "f64"):
        bits = np.asarray(arr.fill_null(0)).view(np.uint32 if kind == "f32" else np.uint64)
        return [int(b) if ok else None for b, ok in zip(bits, arr.is_valid().to_pylist())]
    out = arr.to_pylist()
    if PC.TYPES[kind][2]:
        ctx = decimal.Context(prec=60)
        return [None if v is None else int(v.scaleb(PC.TYPES[kind][2][1], context=ctx)) for v in out]
    if kind == "s":
        return [None if v is None else v.encode() for v in out]
    return out


def _want(vals, valid):
    return [v if ok else None for v, ok in zip(vals, valid)]


def _kind(col):
    return next(k for k in PC.TYPES if col.name.startswith(k) and PC.TYPES[k][0]["phys"] == col.phys)


def _oracle_values(raw, col, rgs_meta):
    from oracle import parquet_oracle as po
    out, ok = [], []
    for c in rgs_meta:
        v, m = po.decode_chunk(raw, c["start"], c["size"], c["rows"], PHYS[col.phys], CODEC[c["codec"]], col.optional, col.type_length)
        if col.phys in (W.FLOAT, W.DOUBLE):
            v = v.view(np.uint32 if col.phys == W.FLOAT else np.uint64)     # by their bits: NaN payloads must survive
        out += [x if isinstance(x, bytes) else int(x) for x in v.tolist()]
        ok += m.tolist()
    return _want(out, ok)


def _chunks_meta(raw, ci):
    md = pq.ParquetFile(io.BytesIO(raw)).metadata
    out = []
    for g in range(md.num_row_groups):
        c = md.row_group(g).column(ci)
        start = c.dictionary_page_offset if c.has_dictionary_page and c.dictionary_page_offset else c.data_page_offset
        out.append({"start": start, "size": c.total_compressed_size, "rows": c.num_values, "codec": {"UNCOMPRESSED": 0, "SNAPPY": 1, "ZSTD": 6}[c.compression]})
    return out


@pytest.mark.parametrize("name", sorted(PC.cases()))
def test_writer_files_read_back_as_intended(name):
    """Every file of the device matrix holds what the writer says it does, read by pyarrow (Arrow C++) and by the oracle."""
    case = PC.cases()[name]()
    for (cols, rgs), raw in zip(case[0], PC.file_bytes(case)):
        # Arrow's reader takes a zero-length hybrid run (dict_*, levels*) and a page of 0 values (row group 0 of tiny_pages) for the end
        # of the stream / chunk: those files are pinned by the oracle alone
        arrow_rgs = [] if name.startswith(("dict_", "levels")) else [g for g in range(len(rgs)) if not (name == "tiny_pages" and g == 0)]
        tbl = pq.ParquetFile(io.BytesIO(raw)).read_row_groups(arrow_rgs) if arrow_rgs else None
        for ci, col in enumerate(cols):
            want = _want([v for rg in rgs for v in rg[ci].values], [v for rg in rgs for v in rg[ci].valid])
            if tbl is not None:
                want_a = _want([v for g in arrow_rgs for v in rgs[g][ci].values], [v for g in arrow_rgs for v in rgs[g][ci].valid])
                assert _arrow_values(tbl.column(ci).combine_chunks(), _kind(col)) == want_a, (name, col.name)
            assert _oracle_values(raw, col, _chunks_meta(raw, ci)) == want, (name, col.name)


@pytest.mark.parametrize("shape", PC.ARROW_SHAPES)
def test_writer_run_shapes_read_by_arrow(shape):
    """The shapes the matrix files mix, one at a time, for indices and levels of every width class, read by pyarrow."""
    rng = np.random.default_rng(20)
    for kind, d in (("i32", 3), ("i64", 300), ("fl30", 70000), ("s", 40)):
        col = PC.column(kind)
        dictionary = list(dict.fromkeys(PC.gen(kind, d + 50, rng)))[:d]
        vals, valid = PC.pick(dictionary, 500, rng)
        for ver in (1, 2):
            raw = W.write_file([col], [[W.chunk(col, vals, valid, 170, dictionary=dictionary, index_shape=shape, level_shape=shape, version=ver)]])
            assert _arrow_values(pq.read_table(io.BytesIO(raw)).column(0).combine_chunks(), kind) == _want(vals, valid), (kind, ver)


def test_writer_snappy_forms_decode():
    """Each literal form and copy kind the writer emits, through the oracle's decoder; and the writer's greedy element lists"""
    from oracle import parquet_oracle as po
    rng = np.random.default_rng(21)
    data = bytes(rng.integers(0, 256, 300, dtype=np.uint8))
    for form in range(5):
        stream, out = W.snappy([("lit", data[:50] if form == 0 else data[:200] if form == 1 else data, form)])
        assert po.snappy_decompress(stream) == out
    for kind in (1, 2, 4):
        stream, out = W.snappy([("lit", data), ("copy", 5, 11, kind), ("copy", 300, 4, kind)] + ([("copy", 1, 64, kind)] if kind != 1 else []))
        assert po.snappy_decompress(stream) == out
    body = data * 50
    for kw in (dict(copy_kind=1), dict(copy_kind=2), dict(copy_kind=4), dict(lit_form=3, max_lit=100)):
        stream, out = W.snappy(W.snappy_elements(body, **kw))
        assert out == body and po.snappy_decompress(stream) == body


# ---- device/cb_rle.h on the host --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def rle(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("cbrle") / "libcb200_rle.so")
    subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(CSRC, "rle_test.cpp")])
    f = C.CDLL(so).cb_rle_decode
    f.restype = C.c_longlong
    f.argtypes = [C.c_char_p, C.c_longlong, C.c_int, C.c_longlong, C.POINTER(C.c_uint)]

    def decode(stream, bw, want):
        out = (C.c_uint * max(want, 1))()
        k = f(bytes(stream), len(stream), bw, want, out)
        return k, list(out[:max(k, 0)])
    return decode


@pytest.mark.parametrize("bw", range(33))
def test_cb_rle_every_width_and_shape(rle, bw):
    """cb_rle.h's walk + unpack against the oracle's rle_hybrid: every shape at every bit width, values spanning the width"""
    from oracle import parquet_oracle as po
    rng = np.random.default_rng(bw)
    hi = 1 << bw
    for shape in PC.SHAPES:
        for n in (1, 7, 8, 9, 100, 517):
            vals = [int(x) for x in rng.integers(0, hi, n, dtype=np.uint64)] if bw else [0] * n
            if bw and n > 3:
                vals[:3] = [hi - 1, 0, hi >> 1]
            if shape in ("rle", "long_tail"):
                vals = sorted(vals)                                        # stretches of equal values
            stream = W.hybrid(W.runs_of(vals, shape), bw)
            k, got = rle(stream, bw, n)
            assert k == n and got == vals, (shape, n)
            assert po.rle_hybrid(stream, bw, n).tolist() == vals, (shape, n)


def test_cb_rle_long_headers_and_malformed(rle):
    vals = list(range(16))
    s = W.hybrid([("packed", 1, vals[:8], 3), ("rle", 8, 5, 5)], 4)            # non-minimal 3- and 5-byte headers
    assert rle(s, 4, 16) == (16, vals[:8] + [5] * 8)
    s = W.hybrid([("rle", 300, 9)], 4)                                        # a 2-byte header
    assert rle(s, 4, 300) == (300, [9] * 300)
    full = W.hybrid([("packed", 2, vals)], 5)
    assert rle(full, 5, 16)[0] == 16
    assert rle(full[:-3], 5, 16)[0] == -2                                     # packed run cut short: truncated
    assert rle(full[:-3], 5, 11)[0] == 11                                     # ... but only past the values wanted
    assert rle(W.hybrid([("rle", 5, 3)], 4), 4, 9)[0] == 5                     # stream ends early: fewer values than wanted
    assert rle(b"\x80\x80", 4, 9)[0] == -1                                    # header runs past the end
    assert rle(b"\x10", 17, 8)[0] == -1                                       # RLE value past the end
    assert rle(b"\xff\xff\xff\xff\x7f", 1, 9)[0] == -1                        # header wider than 32 bits
    assert rle(W.hybrid([("rle", 3, 1)], 1), 33, 3)[0] == -1                  # bit width 33
    assert rle(W.hybrid([("rle", 0, 1), ("packed", 0, []), ("rle", 3, 1)], 1), 1, 3) == (3, [1, 1, 1])   # zero-length runs


# ---- the planner --------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    import json
    cuda = os.environ.get("CUDA", "/usr/local/cuda")
    so = str(tmp_path_factory.mktemp("scanplan") / "libcb200_scanplan.so")
    srcs = [os.path.join(CSRC, f) for f in ("scan_plan_test.cpp", "scan_plan.cpp", "parquet.cpp", "host_codecs.cpp", "plan.cpp")]
    subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-fPIC", "-shared", f"-I{cuda}/include", "-o", so, *srcs, "-Wl,--no-undefined", "-lz", "-ldl"])
    lib = C.CDLL(so)
    lib.sp_plan.restype = C.c_char_p
    lib.sp_plan.argtypes = [C.c_char_p, C.c_size_t, C.c_longlong]

    def plan(scan_bytes, chunk_rows=1 << 26):
        out = json.loads(lib.sp_plan(scan_bytes, len(scan_bytes), chunk_rows))
        if "error" in out:
            return bytes.fromhex(out["error"]).decode()
        return out
    return plan


def _scan(cb, case, paths):
    P = cb.proto
    _, names, _ = case
    dt = lambda k: P.DECIMAL(*PC.TYPES[k][2]) if PC.TYPES[k][2] else getattr(P, PC.TYPES[k][1])
    fields = [(n, dt(n), True) for n in names]
    return P.native_scan(fields, fields, paths)


def _write(tmp_path, case):
    paths = []
    for i, raw in enumerate(PC.file_bytes(case)):
        p = str(tmp_path / f"f{i}.parquet")
        open(p, "wb").write(raw)
        paths.append(p)
    return paths


@pytest.mark.parametrize("name", ["tiny_pages", "codecs", "fallback_i64", "fallback_fl30", "snappy", "required_optional"])
def test_planner_tiles_new_layouts(planner, tmp_path, name):
    """Every data page of every row group, in order, tiles the batch's rows; v2 pages stored uncompressed in a SNAPPY chunk are read
    where they land; Snappy pages get one checkpoint per 64 KiB; dictionary pages come after the data pages."""
    import comet_b200 as cb
    case = PC.cases()[name]()
    out = planner(_scan(cb, case, _write(tmp_path, case)), case[2])
    assert not isinstance(out, str), out
    files = case[0]
    for b in out["batches"]:
        for ci, col in enumerate(b["columns"]):
            data = col["pages"][:col["n_data"]]
            row = 0
            for f, rg, rows, row0 in b["units"]:
                ch = files[f][1][rg][ci]
                mine, data = data[:sum(p.kind != W.DICTIONARY_PAGE for p in ch.pages)], data[sum(p.kind != W.DICTIONARY_PAGE for p in ch.pages):]
                for p, src in zip(mine, [p for p in ch.pages if p.kind != W.DICTIONARY_PAGE]):
                    assert p["dst_row"] == row and p["num_values"] == src.num_values
                    assert p["encoding"] == (8 if src.encoding in (W.RLE_DICTIONARY, W.PLAIN_DICTIONARY) else 0)
                    stored_raw = ch.codec == W.NONE or (src.kind == W.DATA_PAGE_V2 and not src.compressed)
                    assert (p["comp_bytes"] == 0) == (stored_raw or ch.codec != W.SNAPPY), (name, src.kind, ch.codec)
                    assert p["flags"] & 1 == (src.kind == W.DATA_PAGE and files[f][0][ci].optional)
                    if src.kind == W.DATA_PAGE_V2:
                        assert p["def_bytes"] == len(src.levels) and p["body_bytes"] == len(src.body)
                    row += src.num_values
                assert row == row0 + rows
            assert data == []


def test_planner_refuses_bit_packed_levels_and_missing_v2_levels(planner, tmp_path):
    """Deprecated BIT_PACKED definition levels (no length prefix, another bit order): refused at plan build, naming the column.  A v2
    page of an optional column without levels: refused, as Arrow does."""
    import comet_b200 as cb
    col = PC.column("i64", "bp")
    valid = [i % 3 != 0 for i in range(20)]
    bits = np.packbits(np.array(valid, dtype=np.uint8), bitorder="big").tobytes()
    page = W.Page(W.DATA_PAGE, 20, W.PLAIN, bits + W.plain(W.INT64, [i for i in range(20) if valid[i]]), def_encoding=W.BIT_PACKED)
    case = ([((col,), [[W.Chunk([page], list(range(20)), valid)]])], ["bp"], 1 << 20)
    p = str(tmp_path / "bp.parquet")
    open(p, "wb").write(PC.file_bytes(case)[0])
    P = cb.proto
    msg = planner(P.native_scan([("bp", P.INT64, True)], [("bp", P.INT64, True)], [p]))
    assert isinstance(msg, str) and "definition level encoding 4" in msg and "'bp'" in msg
    # the same page as a required column has no levels: the encoding field means nothing and is not checked
    req = W.Column("bp", W.INT64, optional=False)
    page = W.Page(W.DATA_PAGE, 20, W.PLAIN, W.plain(W.INT64, list(range(20))), def_encoding=W.BIT_PACKED)
    open(p, "wb").write(W.write_file([req], [[W.Chunk([page], list(range(20)), [True] * 20)]]))
    assert not isinstance(planner(P.native_scan([("bp", P.INT64, True)], [("bp", P.INT64, True)], [p])), str)
    # v2 without levels: Arrow refuses the page, and so does the planner
    pg = W.data_page(col, list(range(20)), [True] * 20, version=2)
    pg.levels = b""
    raw = W.write_file([col], [[W.Chunk([pg], list(range(20)), [True] * 20)]])
    with pytest.raises(OSError):
        pq.read_table(io.BytesIO(raw))
    open(p, "wb").write(raw)
    msg = planner(P.native_scan([("bp", P.INT64, True)], [("bp", P.INT64, True)], [p]))
    assert isinstance(msg, str) and "no definition levels" in msg and "'bp'" in msg


def test_v1_level_prefix_zero_is_refused_by_arrow():
    """The device's choice for a v1 level length of 0 on a page with values (an error) follows Arrow's"""
    col = PC.column("i64")
    pg = W.data_page(col, list(range(20)), [True] * 20)
    pg.body = struct.pack("<I", 0) + W.plain(W.INT64, list(range(20)))
    with pytest.raises(OSError):
        pq.read_table(io.BytesIO(W.write_file([col], [[W.Chunk([pg], list(range(20)), [True] * 20)]])))
