"""CPU-only: the hand-written Parquet footer / page-header parser (Thrift compact) agrees with pyarrow's reader."""
import struct

import numpy as np
import pyarrow.parquet as pq
import pytest


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


@pytest.mark.parametrize("as_int", [True, False])
def test_footer_matches_pyarrow(cb, tmp_path, as_int):
    t = cb.tpch
    cols = t.gen_lineitem(50_000, seed=4)
    path = str(tmp_path / "li.parquet")
    t.write_lineitem_parquet(cols, path, "dec", row_group_size=16_384, decimal_as_int=as_int)
    mine = cb.native.parquet_describe(path)
    ref = pq.ParquetFile(path).metadata
    assert mine["num_rows"] == ref.num_rows == 50_000
    assert len(mine["row_groups"]) == ref.num_row_groups
    names = [c["name"] for c in mine["columns"]]
    assert names == t.Q1_COLUMNS
    phys = {"INT32": 1, "INT64": 2, "BYTE_ARRAY": 6, "FIXED_LEN_BYTE_ARRAY": 7, "DOUBLE": 5}
    for i, c in enumerate(mine["columns"]):
        rc = ref.schema.column(i)
        assert c["type"] == phys[rc.physical_type]
    assert mine["columns"][0]["type"] == (2 if as_int else 7) and mine["columns"][0]["precision"] == 12 and mine["columns"][0]["scale"] == 2
    for g in range(ref.num_row_groups):
        rg = ref.row_group(g)
        assert mine["row_groups"][g]["num_rows"] == rg.num_rows
        for c in range(rg.num_columns):
            a, b = mine["row_groups"][g]["columns"][c], rg.column(c)
            assert a["num_values"] == b.num_values and a["total_compressed"] == b.total_compressed_size
            assert a["data_page_offset"] == b.data_page_offset
            assert a["codec"] == 0
            if b.has_dictionary_page:
                assert a["dictionary_page_offset"] == b.dictionary_page_offset


def test_memory_file_registration(cb, tmp_path):
    t = cb.tpch
    path = str(tmp_path / "li.parquet")
    t.write_lineitem_parquet(t.gen_lineitem(1000, seed=1), path, "f64")
    image = np.fromfile(path, dtype=np.uint8)
    url = cb.native.register_memory_file("unit-test-file", image)
    assert url == "memory://unit-test-file"
    assert cb.native.parquet_describe(url) == cb.native.parquet_describe(path)
    cb.native.register_memory_file("unit-test-file", None)
    with pytest.raises(cb.native.CometB200Error):
        cb.native.parquet_describe(url)


def test_native_scan_plan_supported(cb):
    t = cb.tpch
    plan = t.q1_partial_plan("dec", scan=t.q1_native_scan("dec", ["file:///tmp/none.parquet"]))
    ok, why = cb.native.supports(plan)
    assert ok, why


@pytest.mark.parametrize("compression,version,dictionary", [("NONE", "1.0", False), ("SNAPPY", "1.0", True), ("SNAPPY", "2.0", False), ("NONE", "2.0", True)])
def test_parquet_oracle_matches_pyarrow(tmp_path, compression, version, dictionary):
    """oracle/parquet_oracle.py (page headers, Snappy, RLE hybrid levels, PLAIN / dictionary values) against pyarrow's reader."""
    import decimal
    import pyarrow as pa
    import pyarrow.parquet as pq
    from oracle import parquet_oracle as po
    rng = np.random.default_rng(3)
    n = 12_000
    ctx = decimal.Context(prec=60)
    m = [rng.random(n) < 0.2 for _ in range(5)]
    m[0][:700] = True
    i64 = rng.integers(-2**60, 2**60, n)
    low = rng.integers(0, 30, n).astype(np.int32)
    f64 = rng.standard_normal(n)
    d30 = [int(a) * 10**10 + int(b) for a, b in zip(rng.integers(-10**15, 10**15, n), rng.integers(0, 10**10, n))]
    words = np.array(["AIR", "MAIL", "SHIP", "", "TRUCK"])[rng.integers(0, 5, n)]
    tbl = pa.table({"i64": pa.array(i64, mask=m[0]), "low": pa.array(low, mask=m[1]), "f64": pa.array(f64, mask=m[2]),
                    "d30": pa.array([None if mm else decimal.Decimal(v).scaleb(-4, context=ctx) for v, mm in zip(d30, m[3])], type=pa.decimal128(30, 4)),
                    "word": pa.array(words.tolist(), mask=m[4]), "req": pa.array(i64)})
    path = str(tmp_path / "o.parquet")
    pq.write_table(tbl, path, row_group_size=5000, compression=compression, use_dictionary=True if dictionary else ["word"], data_page_version=version, data_page_size=4096)
    raw = open(path, "rb").read()
    md = pq.ParquetFile(path).metadata
    for ci, name in enumerate(tbl.column_names):
        got_v, got_ok = [], []
        for rg in range(md.num_row_groups):
            c = md.row_group(rg).column(ci)
            start = c.dictionary_page_offset if c.has_dictionary_page and c.dictionary_page_offset else c.data_page_offset
            start = min(start, c.data_page_offset)
            tl = md.schema.column(ci).length if c.physical_type == "FIXED_LEN_BYTE_ARRAY" else 0
            v, ok = po.decode_chunk(raw, start, c.total_compressed_size, c.num_values, c.physical_type, c.compression, True, tl)
            got_v.append(v)
            got_ok.append(ok)
        v, ok = np.concatenate(got_v), np.concatenate(got_ok)
        want = tbl.column(name).to_pylist()
        assert [w is not None for w in want] == ok.tolist(), name
        for g, w in zip(v[ok].tolist(), [w for w in want if w is not None]):
            if name == "d30":
                assert g == int(w.scaleb(4)), name
            elif name == "word":
                assert g.decode() == w, name
            elif name == "f64":
                assert struct.pack("<d", g) == struct.pack("<d", w), name
            else:
                assert g == w, name


def test_host_codecs_decompress_what_pyarrow_compressed():
    """ZSTD / LZ4_RAW / LZ4 (Hadoop framing) / GZIP pages are decompressed on the host (csrc/host_codecs.cpp: libzstd and liblz4 through
    dlopen, zlib linked) before the device decodes them; checked here against pyarrow's compressors without a GPU."""
    import ctypes as C
    import os
    import pyarrow as pa
    lib = C.CDLL(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "datafusion-comet_b200", "libcomet_b200.so"))
    f = getattr(lib, "_ZN5cb20015host_decompressEiPKhmPhm")       # cb200::host_decompress(int, const uint8_t*, size_t, uint8_t*, size_t)
    f.restype = None
    f.argtypes = [C.c_int, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]
    rng = np.random.default_rng(0)
    raw = rng.integers(0, 1000, 300_000).astype(np.int64).tobytes() + bytes(50_000) + rng.integers(0, 256, 70_000, dtype=np.uint8).tobytes()
    for codec_id, name in ((6, "zstd"), (7, "lz4_raw"), (5, "lz4_hadoop"), (5, "lz4_raw"), (2, "gzip")):
        if name == "lz4_hadoop":     # the deprecated LZ4 codec as Hadoop frames it: [u32 BE uncompressed][u32 BE compressed][raw block], here two blocks
            half = len(raw) // 2
            comp = b""
            for part in (raw[:half], raw[half:]):
                blk = pa.compress(part, codec="lz4_raw", asbytes=True)
                comp += len(part).to_bytes(4, "big") + len(blk).to_bytes(4, "big") + blk
        else:
            comp = pa.compress(raw, codec=name, asbytes=True)
        out = C.create_string_buffer(len(raw))
        f(codec_id, comp, len(comp), out, len(raw))
        assert out.raw == raw, name


# ---- the scan planner (csrc/scan_plan.cpp) without a GPU ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    """csrc/scan_plan_test.cpp linked with the planner and the host parsers only: -Wl,--no-undefined proves they need no CUDA runtime."""
    import ctypes as C
    import json
    import os
    import subprocess
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "datafusion-comet_b200", "csrc")
    cuda = os.environ.get("CUDA", "/usr/local/cuda")
    so = str(tmp_path_factory.mktemp("scanplan") / "libcb200_scanplan.so")
    srcs = [os.path.join(csrc, f) for f in ("scan_plan_test.cpp", "scan_plan.cpp", "parquet.cpp", "host_codecs.cpp", "plan.cpp")]
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


def _chunk_pages(raw, col):
    """(header, body offset) of every page of a column chunk, read by oracle/parquet_oracle.py"""
    from oracle import parquet_oracle as po
    pos = col.dictionary_page_offset if col.has_dictionary_page and col.dictionary_page_offset else col.data_page_offset
    pos, end = min(pos, col.data_page_offset), min(pos, col.data_page_offset) + col.total_compressed_size
    out = []
    while pos < end:
        h, body = po.page_header(raw, pos)
        out.append((h, body))
        pos = body + h["compressed"]
    return out


@pytest.mark.parametrize("compression,version,dictionary", [("NONE", "1.0", False), ("SNAPPY", "1.0", True), ("SNAPPY", "2.0", False), ("NONE", "2.0", True),
                                                            ("ZSTD", "1.0", True), ("ZSTD", "2.0", False)])
def test_planner_pages_tile_every_row_group(cb, planner, tmp_path, compression, version, dictionary):
    """Each column's data pages cover its row groups' rows exactly, in order, with the page headers' value counts and encodings."""
    import decimal
    import pyarrow as pa
    P = cb.proto
    rng = np.random.default_rng(6)
    n = 30_000
    mask = lambda: rng.random(n) < 0.15
    words = np.array(["AIR", "MAIL", "SHIP", "", "TRUCK", "ünï"])[rng.integers(0, 6, n)]
    tbl = pa.table({"i64": pa.array(rng.integers(-2**60, 2**60, n), mask=mask()), "low": pa.array(rng.integers(0, 30, n).astype(np.int32)),
                    "d12": pa.array([decimal.Decimal(int(v)).scaleb(-2) for v in rng.integers(-10**11, 10**11, n)], type=pa.decimal128(12, 2)),
                    "word": pa.array(words.tolist(), mask=mask()).cast(pa.string())})
    path = str(tmp_path / "p.parquet")
    pq.write_table(tbl, path, row_group_size=7_000, compression=compression, use_dictionary=dictionary, data_page_version=version, data_page_size=4096)
    fields = [("i64", P.INT64, True), ("low", P.INT32, True), ("d12", P.DECIMAL(12, 2), True), ("word", P.STRING, True)]
    out = planner(P.native_scan(fields, fields, [path]), chunk_rows=15_000)
    raw = open(path, "rb").read()
    md = pq.ParquetFile(path).metadata
    assert [u[1] for b in out["batches"] for u in b["units"]] == list(range(md.num_row_groups))
    for b in out["batches"]:
        for ci, col in enumerate(b["columns"]):
            data = col["pages"][:col["n_data"]]
            row = 0
            for _, rg, rows, row0 in b["units"]:
                assert row0 == row
                pages = [(h, off) for h, off in _chunk_pages(raw, md.row_group(rg).column(ci)) if h["type"] in (0, 3)]
                mine, data = data[:len(pages)], data[len(pages):]
                assert len(mine) == len(pages)
                for p, (h, _) in zip(mine, pages):
                    assert p["dst_row"] == row and p["num_values"] == h["num_values"]
                    assert p["encoding"] == (0 if h["encoding"] == 0 else 8)
                    lv = h["rep_bytes"] + h["def_bytes"] if h["type"] == 3 else 0
                    assert p["def_bytes"] == (h["def_bytes"] if h["type"] == 3 else 0)
                    if not p["flags"] & 8 or p["encoding"] != 0 or ci != 3:             # everything but host-encoded PLAIN strings: the page's own bytes
                        assert p["body_bytes"] == h["uncompressed"] - lv
                    row += p["num_values"]
                assert row == row0 + rows
            assert data == []


@pytest.mark.parametrize("compression,version", [("SNAPPY", "1.0"), ("NONE", "2.0")])
def test_planner_codes_plain_and_dictionary_strings_alike(cb, planner, tmp_path, compression, version):
    """A PLAIN file and a dictionary file of one string column: every value gets the same code, the dictionary holds it once."""
    import pyarrow as pa
    from oracle import parquet_oracle as po
    P = cb.proto
    rng = np.random.default_rng(4)
    n = 20_000
    words = np.array([f"w{i:04d}" for i in range(900)] + ["", "ünï", "a" * 300])[rng.integers(0, 903, n)]
    tbl = pa.table({"word": pa.array(words.tolist(), mask=rng.random(n) < 0.1).cast(pa.string())})
    p1, p2 = str(tmp_path / "plain.parquet"), str(tmp_path / "dict.parquet")
    pq.write_table(tbl, p1, row_group_size=8_000, compression=compression, use_dictionary=False, data_page_version=version, data_page_size=4096)
    pq.write_table(tbl, p2, row_group_size=8_000, compression=compression, use_dictionary=True, data_page_version=version)
    fields = [("word", P.STRING, True)]
    out = planner(P.native_scan(fields, fields, [p1, p2]), chunk_rows=n)
    dictionary = out["dictionaries"][0]
    want = [w for w in tbl.column("word").to_pylist() if w is not None]
    assert len(set(dictionary)) == len(dictionary) and set(dictionary) == set(want)
    code = {v: i for i, v in enumerate(dictionary)}
    plain_codes, remap = [], []
    for b in out["batches"]:
        col = b["columns"][0]
        if b["units"][0][0] == 0:
            assert col["remap"] == [] and all(p["flags"] & 8 and p["encoding"] == 0 for p in col["pages"])
            plain_codes += [c for p in col["pages"] for c in p["codes"]]
        else:
            assert all(p["encoding"] == 8 for p in col["pages"])
            remap += col["remap"]
    assert [dictionary[c] for c in plain_codes] == want
    raw = open(p2, "rb").read()
    md = pq.ParquetFile(p2).metadata
    dict_values = []
    for rg in range(md.num_row_groups):
        h, body = _chunk_pages(raw, md.row_group(rg).column(0))[0]
        data = raw[body:body + h["compressed"]]
        data = po.snappy_decompress(data) if compression == "SNAPPY" else data
        dict_values += [v.decode() for v in po.plain(data, "BYTE_ARRAY", h["num_values"])]
    assert remap == [code[v] for v in dict_values]


@pytest.mark.parametrize("variant", ["dec", "f64"])
def test_planner_prunes_q6_row_groups_by_min_max(cb, planner, tmp_path, variant):
    """The row groups the GPU test test_q6_row_groups_pruned_by_min_max expects to be read: those whose l_shipdate range meets 1994."""
    t = cb.tpch
    n = 400_000
    cols = t.gen_lineitem(n, seed=41)
    order = np.argsort(cols["l_shipdate"], kind="stable")
    cols = {k: v[order] for k, v in cols.items()}
    path = t.write_lineitem_parquet(cols, str(tmp_path / f"q6_{variant}.parquet"), variant, row_group_size=16_384, columns=t.Q6_COLUMNS)
    out = planner(t.q6_native_scan(variant, [path]), chunk_rows=60_000)
    ship = cols["l_shipdate"]
    groups = [(g, ship[g * 16_384:(g + 1) * 16_384]) for g in range((n + 16_383) // 16_384)]
    exp = [g for g, s in groups if s.max() >= t.DATE_1994_01_01 and s.min() < t.DATE_1995_01_01]
    assert [u[1] for b in out["batches"] for u in b["units"]] == exp
    assert out["pruned_row_groups"] == len(groups) - len(exp) >= len(groups) * 0.8
    assert out["pruned_rows"] == n - sum(len(s) for g, s in groups if g in exp)


def test_planner_file_splits_own_the_row_groups_that_start_inside_them(cb, planner, tmp_path):
    """Two splits of one file cut in the middle of a row group: each row group belongs to the split it starts in."""
    import os
    t = cb.tpch
    P = cb.proto
    path = t.write_lineitem_parquet(t.gen_lineitem(100_000, seed=45), str(tmp_path / "split.parquet"), "dec", row_group_size=10_000)
    size = os.path.getsize(path)
    md = pq.ParquetFile(path).metadata
    starts = [md.row_group(g).column(0).dictionary_page_offset or md.row_group(g).column(0).data_page_offset for g in range(md.num_row_groups)]
    cut = starts[4] + 1
    fields = list(zip(t.Q1_COLUMNS, t.q1_scan_fields("dec"), [True] * 7))
    got = []
    for lo, ln in ((0, cut), (cut, size - cut)):
        out = planner(P.native_scan(fields, fields, [(path, lo, ln, size)]))
        got.append([u[1] for b in out["batches"] for u in b["units"]])
    assert got == [[g for g in range(md.num_row_groups) if starts[g] < cut], [g for g in range(md.num_row_groups) if starts[g] >= cut]]
