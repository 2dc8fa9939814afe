"""CPU-only: DELTA_BINARY_PACKED, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY and BYTE_STREAM_SPLIT pages.

The CPU restatement of these encodings (tests/parquet_encodings_ref.py) against pyarrow's reader, the shared DELTA_BINARY_PACKED walk (csrc/device/cb_delta.h)
on the host through a test-only driver, and the scan planner's page tables for files in these encodings."""
import ctypes as C
import decimal
import os
import struct
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "datafusion-comet_b200", "csrc")
ENC = {"PLAIN": 0, "DELTA_BINARY_PACKED": 5, "DELTA_LENGTH_BYTE_ARRAY": 6, "DELTA_BYTE_ARRAY": 7, "BYTE_STREAM_SPLIT": 9}


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def _table(n, seed, nullable=True):
    rng = np.random.default_rng(seed)
    ctx = decimal.Context(prec=60)
    mask = (lambda: rng.random(n) < 0.2) if nullable else (lambda: None)
    f64 = rng.standard_normal(n)
    f64[:8] = [np.nan, -0.0, 0.0, np.inf, -np.inf, 5e-324, -2.2250738585072014e-308, 1.0]
    d12 = rng.integers(-10**11, 10**11, n)
    d30 = [int(a) * 10**10 + int(b) for a, b in zip(rng.integers(-10**15, 10**15, n), rng.integers(0, 10**10, n))]
    words = np.array([f"prefix/{i:05d}" for i in range(700)] + ["", "ünï"])[rng.integers(0, 702, n)]
    m = [mask() for _ in range(8)]
    dec = lambda vals, p, s, mm: pa.array([decimal.Decimal(int(v)).scaleb(-s, context=ctx) for v in vals], type=pa.decimal128(p, s), mask=mm)
    return pa.table({
        "i32": pa.array(rng.integers(-2**31, 2**31, n).astype(np.int32), mask=m[0]),
        "i64": pa.array(np.cumsum(rng.integers(-1000, 5000, n)), mask=m[1]),
        "f32": pa.array(rng.standard_normal(n).astype(np.float32), mask=m[2]),
        "f64": pa.array(f64, mask=m[3]),
        "d12": dec(d12, 12, 2, m[4]),
        "d30": dec(d30, 30, 4, m[5]),
        "s_dlba": pa.array(words.tolist(), mask=m[6]).cast(pa.string()),
        "s_dba": pa.array(sorted(words.tolist()), mask=m[7]).cast(pa.string()),
    })


ENCODINGS = {"i32": "DELTA_BINARY_PACKED", "i64": "DELTA_BINARY_PACKED", "f32": "BYTE_STREAM_SPLIT", "f64": "BYTE_STREAM_SPLIT",
             "d12": "DELTA_BINARY_PACKED", "d30": "DELTA_BYTE_ARRAY", "s_dlba": "DELTA_LENGTH_BYTE_ARRAY", "s_dba": "DELTA_BYTE_ARRAY"}


def _write(tbl, path, encodings, compression="NONE", version="2.0", page_size=4096, row_group_size=5000):
    pq.write_table(tbl, path, row_group_size=row_group_size, compression=compression, use_dictionary=False, column_encoding=encodings,
                   data_page_version=version, data_page_size=page_size, store_decimal_as_integer=True)
    return path


@pytest.mark.parametrize("compression,version,nullable", [("NONE", "1.0", True), ("SNAPPY", "1.0", False), ("SNAPPY", "2.0", True), ("NONE", "2.0", False)])
def test_reference_delta_and_bss_match_pyarrow(tmp_path, compression, version, nullable):
    import parquet_encodings_ref as ref
    n = 12_000
    tbl = _table(n, 3, nullable)
    path = _write(tbl, str(tmp_path / "e.parquet"), ENCODINGS, compression, version)
    raw = open(path, "rb").read()
    md = pq.ParquetFile(path).metadata
    for ci, name in enumerate(tbl.column_names):
        assert ENCODINGS[name] in md.row_group(0).column(ci).encodings, name
        got_v, got_ok = [], []
        for rg in range(md.num_row_groups):
            c = md.row_group(rg).column(ci)
            tl = md.schema.column(ci).length if c.physical_type == "FIXED_LEN_BYTE_ARRAY" else 0
            v, ok = ref.decode_chunk(raw, c.data_page_offset, c.total_compressed_size, c.num_values, c.physical_type, c.compression, True, tl)
            got_v.append(v)
            got_ok.append(ok)
        v, ok = np.concatenate(got_v), np.concatenate(got_ok)
        want = tbl.column(name).to_pylist()
        assert [w is not None for w in want] == ok.tolist(), name
        for g, w in zip(v[ok].tolist(), [w for w in want if w is not None]):
            if name in ("d12", "d30"):
                assert g == int(w.scaleb(2 if name == "d12" else 4)), name
            elif name.startswith("s_"):
                assert g.decode() == w, name
            elif name == "f64":
                assert struct.pack("<d", g) == struct.pack("<d", w), name
            elif name == "f32":
                assert struct.pack("<f", g) == struct.pack("<f", w), name
            else:
                assert g == w, name


# ---- device/cb_delta.h on the host ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dbp(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("cbdelta") / "libcb200_delta.so")
    subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(CSRC, "delta_test.cpp")])
    lib = C.CDLL(so)
    f = lib.cb_dbp_decode
    f.restype = C.c_longlong
    f.argtypes = [C.c_char_p, C.c_longlong, C.c_int, C.c_longlong, C.POINTER(C.c_longlong), C.c_longlong, C.POINTER(C.c_longlong)]

    def decode(stream, bits, expect=-1):
        cap = max(expect, 0) + 4096
        out = (C.c_longlong * cap)()
        used = C.c_longlong(0)
        k = f(bytes(stream), len(stream), bits, expect, out, cap, C.byref(used))
        return (k, None, 0) if k < 0 else (k, list(out[:k]), used.value)
    return decode


def _dbp_pages(tmp_path, values, pa_type, page_size=1024):
    """the DELTA_BINARY_PACKED streams of a required column written with data page v2, uncompressed: (stream, its values)"""
    from oracle import parquet_oracle as po
    path = str(tmp_path / "dbp.parquet")
    tbl = pa.table({"v": pa.array(values, type=pa_type)}, schema=pa.schema([pa.field("v", pa_type, nullable=False)]))
    pq.write_table(tbl, path, compression="NONE", use_dictionary=False, data_page_version="2.0",
                   column_encoding={"v": "DELTA_BINARY_PACKED"}, data_page_size=page_size, write_statistics=False)
    raw = open(path, "rb").read()
    md = pq.ParquetFile(path).metadata
    out, row = [], 0
    for rg in range(md.num_row_groups):
        c = md.row_group(rg).column(0)
        pos, end = c.data_page_offset, c.data_page_offset + c.total_compressed_size
        while pos < end:
            h, body = po.page_header(raw, pos)
            pos = body + h["compressed"]
            if h["type"] != 3:
                continue
            assert h["encoding"] == 5 and h["def_bytes"] == 0
            out.append((raw[body:body + h["compressed"]], list(values[row:row + h["num_values"]])))
            row += h["num_values"]
    assert row == len(values)
    return out


def _blocks(stream):
    """(header total-count position and length, [(block width-byte position, used miniblocks, miniblocks)]) of a DBP stream"""
    from parquet_encodings_ref import uleb
    block, p = uleb(stream, 0)
    mbs, p = uleb(stream, p)
    tpos = p
    total, p = uleb(stream, p)
    tlen = p - tpos
    _, p = uleb(stream, p)
    per = block // mbs
    left, out = max(total - 1, 0), []
    while left > 0:
        _, p = uleb(stream, p)
        wpos = p
        p += mbs
        used = 0
        for m in range(mbs):
            if left <= 0:
                break
            p += per * stream[wpos + m] // 8
            left -= min(per, left)
            used += 1
        out.append((wpos, used, mbs))
    return (tpos, tlen), out


@pytest.mark.parametrize("shape", ["random", "monotone", "constant", "i64_extremes", "i32_extremes", "one", "odd_counts"])
def test_cb_delta_decodes_what_pyarrow_wrote(dbp, tmp_path, shape):
    rng = np.random.default_rng(11)
    bits = 64
    if shape == "random":
        v = rng.integers(-2**63, 2**63 - 1, 5000, dtype=np.int64)
    elif shape == "monotone":
        v = np.cumsum(rng.integers(0, 100, 5000)).astype(np.int64)
    elif shape == "constant":
        v = np.full(4000, -7, dtype=np.int64)                                           # width-0 miniblocks
    elif shape == "i64_extremes":
        v = np.array([-2**63, 2**63 - 1] * 1500, dtype=np.int64)                        # width 64, wrapping deltas
    elif shape == "i32_extremes":
        v, bits = np.array([-2**31, 2**31 - 1, 0, -1] * 800, dtype=np.int32), 32        # wraps at 32 bits
    elif shape == "one":
        v = np.array([123456789012], dtype=np.int64)
    else:
        v = rng.integers(-10**6, 10**6, 1001).astype(np.int64)                          # not a multiple of 32 or 128
    pages = _dbp_pages(tmp_path, v, pa.int32() if bits == 32 else pa.int64(), page_size=1024 if shape != "one" else 1 << 20)
    assert len(pages) >= 1
    for stream, want in pages:
        k, got, used = dbp(stream, bits, len(want))
        assert k == len(want) and got == [int(x) for x in want], shape
        assert used == len(stream)                                                      # the walk ends where the page ends


def test_cb_delta_same_length_patches(dbp, tmp_path):
    """Garbage bit widths in the unused miniblocks of the last block decode unchanged; a width of 65 or a count off by one is refused."""
    rng = np.random.default_rng(12)
    v = rng.integers(-10**9, 10**9, 1000).astype(np.int64)         # 999 deltas: the last block of 128 uses 4 of 4 miniblocks...
    v2 = rng.integers(-10**9, 10**9, 1000 - 64).astype(np.int64)   # ... this one: 935 deltas, 39 in the last block -> 2 used of 4
    checked_unused = False
    for vals in (v, v2):
        for stream, want in _dbp_pages(tmp_path, vals, pa.int64(), page_size=1 << 20):
            (tpos, tlen), blocks = _blocks(stream)
            wpos, used, mbs = blocks[-1]
            if used < mbs:
                s = bytearray(stream)
                for m in range(used, mbs):
                    s[wpos + m] = 0xEE                                                  # anything: those miniblocks have no bytes
                k, got, _ = dbp(bytes(s), 64, len(want))
                assert k == len(want) and got == [int(x) for x in want]
                checked_unused = True
            s = bytearray(stream)
            s[blocks[0][0]] = 65                                                        # wider than INT64
            assert dbp(bytes(s), 64, len(want))[0] == -1
            s = bytearray(stream)
            assert s[tpos] & 0x7F != 0x7F
            s[tpos] += 1                                                                # total value count + 1, same length
            assert dbp(bytes(s), 64, len(want))[0] < 0
    assert checked_unused


# ---- the scan planner -----------------------------------------------------------------------------------------------------------
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
        assert "error" not in out, bytes.fromhex(out["error"]).decode()
        out["dictionaries"] = [[bytes.fromhex(v).decode() for v in d] for d in out["dictionaries"]]
        return out
    return plan


def _fields(cb, names):
    P = cb.proto
    dts = {"i32": P.INT32, "i64": P.INT64, "f32": P.FLOAT, "f64": P.DOUBLE, "d12": P.DECIMAL(12, 2), "d30": P.DECIMAL(30, 4), "s_dlba": P.STRING, "s_dba": P.STRING}
    return [(name, dts[name], True) for name in names]


def _data_pages(raw, col):
    from oracle import parquet_oracle as po
    pos, end, out = col.data_page_offset, col.data_page_offset + col.total_compressed_size, []
    while pos < end:
        h, body = po.page_header(raw, pos)
        out.append((h, body))
        pos = body + h["compressed"]
    return [(h, b) for h, b in out if h["type"] in (0, 3)]


@pytest.mark.parametrize("compression,version", [("NONE", "1.0"), ("SNAPPY", "2.0"), ("ZSTD", "1.0"), ("ZSTD", "2.0")])
def test_planner_tiles_delta_and_bss_files(cb, planner, tmp_path, compression, version):
    """Every row group's data pages, in order, with the device encoding they decode by and a miniblock table of num_values / 32 + 2."""
    P = cb.proto
    n = 30_000
    tbl = _table(n, 6)
    path = _write(tbl, str(tmp_path / "t.parquet"), ENCODINGS, compression, version, row_group_size=7_000)
    fields = _fields(cb, tbl.column_names)
    out = planner(P.native_scan(fields, fields, [path]), chunk_rows=15_000)
    raw = open(path, "rb").read()
    md = pq.ParquetFile(path).metadata
    assert [u[1] for b in out["batches"] for u in b["units"]] == list(range(md.num_row_groups))
    for b in out["batches"]:
        for ci, col in enumerate(b["columns"]):
            name = tbl.column_names[ci]
            data, mb = col["pages"][:col["n_data"]], 0
            row = 0
            for _, rg, rows, row0 in b["units"]:
                pages = _data_pages(raw, md.row_group(rg).column(ci))
                mine, data = data[:len(pages)], data[len(pages):]
                assert len(mine) == len(pages)
                for p, (h, _) in zip(mine, pages):
                    assert h["encoding"] == ENC[ENCODINGS[name]]
                    assert p["dst_row"] == row and p["num_values"] == h["num_values"]
                    assert p["encoding"] == {5: 5, 9: 9, 6: 0, 7: 0}[h["encoding"]], name
                    if h["encoding"] == 5:
                        assert p["mb_base"] == mb and p["mb_cap"] == h["num_values"] // 32 + 2
                        mb += p["mb_cap"]
                    else:
                        assert "mb_cap" not in p
                    row += p["num_values"]
                assert row == row0 + rows
            assert data == [] and col["mb_entries"] == mb


@pytest.mark.parametrize("compression,version", [("NONE", "1.0"), ("SNAPPY", "2.0"), ("ZSTD", "2.0")])
def test_planner_codes_delta_strings_like_dictionary_and_plain(cb, planner, tmp_path, compression, version):
    """DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY, dictionary and PLAIN files of one string column in one scan: the same codes."""
    P = cb.proto
    rng = np.random.default_rng(8)
    n = 9_000
    words = np.array([f"w{i:04d}/tail" for i in range(500)] + ["", "ünï", "a" * 300])[rng.integers(0, 503, n)]
    tbl = pa.table({"word": pa.array(words.tolist(), mask=rng.random(n) < 0.1).cast(pa.string())})
    paths = []
    for i, enc in enumerate(("DELTA_LENGTH_BYTE_ARRAY", "DELTA_BYTE_ARRAY", None, "PLAIN")):
        p = str(tmp_path / f"w{i}.parquet")
        kw = {"use_dictionary": True} if enc is None else {"use_dictionary": False, "column_encoding": {"word": enc}}
        pq.write_table(tbl, p, row_group_size=4_000, compression=compression, data_page_version=version, data_page_size=2048, **kw)
        paths.append(p)
    fields = [("word", P.STRING, True)]
    out = planner(P.native_scan(fields, fields, paths), chunk_rows=4_000)      # one row group per batch
    dictionary = out["dictionaries"][0]
    want = [w for w in tbl.column("word").to_pylist() if w is not None]
    assert len(set(dictionary)) == len(dictionary) and set(dictionary) == set(want)
    per_file = {}
    for b in out["batches"]:
        col = b["columns"][0]
        f = b["units"][0][0]
        assert all(u[0] == f for u in b["units"])
        if f == 2:
            assert all(p["encoding"] == 8 for p in col["pages"])
        else:
            assert all(p["flags"] & 8 and p["encoding"] == 0 for p in col["pages"])
            per_file.setdefault(f, []).extend(c for p in col["pages"] for c in p["codes"])
    for f in (0, 1, 3):
        assert [dictionary[c] for c in per_file[f]] == want, f
    assert per_file[0] == per_file[1] == per_file[3]


@pytest.mark.parametrize("version", ["1.0", "2.0"])
def test_planner_reencodes_flba_delta_byte_array_as_plain(cb, planner, tmp_path, version):
    """DELTA_BYTE_ARRAY decimal pages come out of the host as PLAIN FIXED_LEN_BYTE_ARRAY: the original big-endian bytes."""
    P = cb.proto
    n = 6_000
    tbl = _table(n, 9, nullable=False).select(["d30"])
    path = _write(tbl, str(tmp_path / "d.parquet"), {"d30": "DELTA_BYTE_ARRAY"}, "NONE", version, row_group_size=2_500)
    fields = [("d30", P.DECIMAL(30, 4), True)]
    out = planner(P.native_scan(fields, fields, [path]))
    tl = pq.ParquetFile(path).metadata.schema.column(0).length
    body = b""
    for b in out["batches"]:
        for p in b["columns"][0]["pages"]:
            raw = bytes.fromhex(p["body"])
            body += raw[4 + struct.unpack_from("<I", raw)[0]:] if p["flags"] & 1 else raw  # v1: [u32 length][levels] stay in front
    want = [int(w.scaleb(4)) for w in tbl.column("d30").to_pylist()]
    assert len(body) >= n * tl
    assert [int.from_bytes(body[i * tl:(i + 1) * tl], "big", signed=True) for i in range(n)] == want
