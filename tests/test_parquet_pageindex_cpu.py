"""CPU-only: page-index pruning in the Parquet scan planner.

tests/page_index_ref.py reads ColumnIndex / OffsetIndex and restates the row selection from parquet.thrift; it is pinned here against
facts of the files themselves.  A test-only driver of the planner (csrc/page_index_test.cpp, linked without the CUDA runtime) must then
produce exactly the reference's selection, pages per column, segment tables, page tables and uploaded bytes."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "datafusion-comet_b200", "csrc")
OPS = {"eq": "eq", "lt": "lt", "le": "lt_eq", "gt": "gt", "ge": "gt_eq"}


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    cuda = os.environ.get("CUDA", "/usr/local/cuda")
    so = str(tmp_path_factory.mktemp("pageindex") / "libcb200_pageindex.so")
    srcs = [os.path.join(CSRC, f) for f in ("page_index_test.cpp", "scan_plan.cpp", "parquet.cpp", "host_codecs.cpp", "plan.cpp")]
    subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-fPIC", "-shared", f"-I{cuda}/include", "-o", so, *srcs, "-Wl,--no-undefined", "-lz", "-ldl"])
    lib = C.CDLL(so)
    lib.pi_plan.restype = C.c_char_p
    lib.pi_plan.argtypes = [C.c_char_p, C.c_size_t, C.c_longlong, C.c_int]

    def plan(scan_bytes, chunk_rows=1 << 26, no_prune=False, expect_error=False):
        out = json.loads(lib.pi_plan(scan_bytes, len(scan_bytes), chunk_rows, int(no_prune)))
        if expect_error:
            return bytes.fromhex(out["error"]).decode() if "error" in out else out
        assert "error" not in out, bytes.fromhex(out["error"]).decode()
        return out
    return plan


def lineitem(cb, n, path, seed=5, variant="dec", rg=100_000, page=16_384, version="1.0", compression="NONE", index=True, sort=True, encoding=None):
    """date-sorted (or not) lineitem, the Q1 columns; dictionary flag columns, `encoding` (None: PLAIN) for the others"""
    t = cb.tpch
    cols = t.gen_lineitem(n, seed=seed)
    if sort:
        order = np.argsort(cols["l_shipdate"], kind="stable")
        cols = {k: v[order] for k, v in cols.items()}
    tbl = t.lineitem_table(cols, variant, dictionary=True, columns=t.Q1_COLUMNS)
    kw = {"column_encoding": {k: encoding for k in t.Q1_COLUMNS if k not in ("l_returnflag", "l_linestatus")}} if encoding else {}
    pq.write_table(tbl, path, row_group_size=rg, compression=compression, use_dictionary=["l_returnflag", "l_linestatus"], data_page_version=version,
                   data_page_size=page, write_page_index=index, store_decimal_as_integer=True, **kw)
    return cols, path


def scan(cb, fields, paths, terms):
    """NativeScan over `paths`; terms: [(column position, op, literal)] pushed as one conjunction"""
    P = cb.proto
    preds = []
    for col, op, lit in terms:
        dt = fields[col][1]
        if op == "notnull":
            preds.append(P.is_not_null(P.bound(col, dt)))
        else:
            preds.append(getattr(P, OPS[op])(P.bound(col, dt), P.literal(lit, dt)))
    filt = []
    if preds:
        e = preds[0]
        for p in preds[1:]:
            e = P.and_(e, p)
        filt = [e]
    return P.native_scan(fields, fields, paths, data_filters=filt)


def _chunk_excludes(c, op, lit, phys):
    """the row-group rule over pyarrow's view of the chunk statistics (min_raw / max_raw are the physical values)"""
    import page_index_ref as ref
    st = c.statistics
    if st is None:
        return False
    if op == "notnull":
        return st.has_null_count and st.null_count == c.num_values and c.num_values > 0
    if not st.has_min_max:
        return False
    raw = lambda v: ref.stat_value(v, phys) if isinstance(v, bytes) else v
    return ref.excludes(op, lit, raw(st.min_raw), raw(st.max_raw), False)


def expected(paths, fields, terms):
    """units the planner must keep: [(file, rg, selected rows, ranges or None, [(pages, covered, segs)] or None, file start of each
    column chunk)] and the page counts / rows page pruning takes away"""
    import page_index_ref as ref
    units, pruned_pages, pruned_rows = [], 0, 0
    for fi, path in enumerate(paths):
        raw = open(path, "rb").read()
        md = pq.ParquetFile(path).metadata
        names = [md.schema.column(i).name for i in range(md.num_columns)]
        leaf = [names.index(f[0]) for f in fields]
        idx = ref.page_indexes(raw)
        for g in range(md.num_row_groups):
            rgm = md.row_group(g)
            n = rgm.num_rows
            phys = [rgm.column(leaf[k]).physical_type for k in range(len(fields))]
            if any(_chunk_excludes(rgm.column(leaf[col]), op, lit, phys[col]) for col, op, lit in terms):
                continue
            cols = [idx[g][leaf[k]] for k in range(len(fields))]
            usable = terms and all(oi is not None for oi, _ in cols) and all(cols[col][1] is not None for col, _, _ in terms)
            ranges = ref.selection([(col, op, lit, phys[col]) for col, op, lit in terms], cols, n) if usable else [(0, n)]
            rows = sum(b - a for a, b in ranges)
            starts = []
            for k in range(len(fields)):
                c = rgm.column(leaf[k])
                starts.append(c.dictionary_page_offset if c.has_dictionary_page and c.dictionary_page_offset < c.data_page_offset else c.data_page_offset)
            if rows == n:
                units.append((fi, g, n, None, None, starts))
                continue
            pruned_rows += n - rows
            windows = [ref.column_window(oi, n, ranges) for oi, _ in cols]
            pruned_pages += sum(len(oi) for oi, _ in cols) - sum(len(w[0]) for w in windows)
            if rows:
                units.append((fi, g, rows, ranges, windows, starts))
    return units, pruned_pages, pruned_rows


def check_plan(cb, planner, paths, fields, terms, chunk_rows=1 << 26):
    """the planner's selection, pages, segments, page tables and upload bytes against the reference; returns the plan"""
    import page_index_ref as ref
    out = planner(scan(cb, fields, paths, terms), chunk_rows)
    units, pruned_pages, pruned_rows = expected(paths, fields, terms)
    assert [(u["file"], u["rg"], u["rows"]) for u in out["units"]] == [u[:3] for u in units]
    assert out["pruned_pages"] == pruned_pages and out["page_pruned_rows"] == pruned_rows
    by_key = {(u[0], u[1]): u for u in units}
    for got in out["units"]:
        _, _, _, ranges, windows, _ = by_key[(got["file"], got["rg"])]
        assert got["ranges"] == (None if ranges is None else [list(r) for r in ranges])
        if windows is not None:
            assert [(c["pages"], c["covered"], [tuple(s) for s in c["segs"]]) for c in got["columns"]] == windows
    raws = [open(p, "rb").read() for p in paths]
    idxs = [ref.page_indexes(r) for r in raws]
    mds = [pq.ParquetFile(p).metadata for p in paths]
    for b in out["batches"]:
        upload = 0
        for f, g, rows, row0 in b["units"]:
            u = by_key[(f, g)]
            names = [mds[f].schema.column(i).name for i in range(mds[f].num_columns)]
            items = []
            for k, fd in enumerate(fields):
                c = mds[f].row_group(g).column(names.index(fd[0]))
                if u[4] is None:
                    items.append([u[5][k], u[5][k] + c.total_compressed_size])
                else:
                    items += ref.chunk_pieces(u[5][k], idxs[f][g][names.index(fd[0])][0], u[4][k][0])
            upload += ref.upload_bytes(items)
        assert b["upload_bytes"] == upload
        for k, fd in enumerate(fields):
            col = b["columns"][k]
            pages, segs, cov = [], [], 0
            for f, g, rows, row0 in b["units"]:
                u = by_key[(f, g)]
                names = [mds[f].schema.column(i).name for i in range(mds[f].num_columns)]
                oi = idxs[f][g][names.index(fd[0])][0]
                n = mds[f].row_group(g).num_rows
                if u[4] is None:
                    spans = ref.page_rows(oi, n) if oi else None
                    if spans:
                        pages += [[cov + a, b_ - a] for a, b_ in spans]
                    unit_segs, unit_cov = [(0, 0, rows)], n
                else:
                    sel, unit_cov, unit_segs = u[4][k]
                    spans = ref.page_rows(oi, n)
                    at = cov
                    for i in sel:
                        pages.append([at, spans[i][1] - spans[i][0]])
                        at += spans[i][1] - spans[i][0]
                for o, c, m in unit_segs:
                    s = [row0 + o, cov + c, m]
                    if segs and segs[-1][0] + segs[-1][2] == s[0] and segs[-1][1] + segs[-1][2] == s[1]:
                        segs[-1][2] += m
                    else:
                        segs.append(s)
                cov += unit_cov
            total = b["units"][-1][3] + b["units"][-1][2]
            assert col["covered"] == cov
            assert col["segs"] == ([] if cov == total else segs), fd[0]
            if all(idxs[f][g][names.index(fd[0])][0] for f, g, _, _ in b["units"]):
                assert col["pages"] == pages, fd[0]
    return out


def _fields(cb, variant="dec"):
    t = cb.tpch
    return list(zip(t.Q1_COLUMNS, t.q1_scan_fields(variant), [True] * 7))


# ---- the reference against the file -------------------------------------------------------------------------------------------------
def test_reference_reads_the_index_the_file_describes(cb, tmp_path):
    """page locations = the page headers the oracle walks; first_row_index = cumulative num_values; min / max = the page's own values.
    At data_page_size = 16384 the date, decimal and dictionary columns of one 100 k-row row group split into different page counts."""
    import page_index_ref as ref
    from oracle import parquet_oracle as po
    n = 100_000
    cols, path = lineitem(cb, n, str(tmp_path / "l.parquet"))
    raw = open(path, "rb").read()
    md = pq.ParquetFile(path).metadata
    tbl = pq.read_table(path)
    idx = ref.page_indexes(raw)
    counts = {}
    for ci in range(md.num_columns):
        c = md.row_group(0).column(ci)
        oi, cix = idx[0][ci]
        pos = min(c.data_page_offset, c.dictionary_page_offset) if c.has_dictionary_page else c.data_page_offset
        end, row, pages = pos + c.total_compressed_size, 0, []
        while pos < end:
            h, body = po.page_header(raw, pos)
            if h["type"] in (0, 3):
                pages.append((pos, body + h["compressed"] - pos, row))
                row += h["num_values"]
            pos = body + h["compressed"]
        assert oi == pages
        counts[md.schema.column(ci).name] = len(oi)
        vals = tbl.column(ci).combine_chunks()
        if pa.types.is_dictionary(vals.type):
            continue
        phys = c.physical_type
        for i, (a, b) in enumerate(ref.page_rows(oi, n)):
            page = vals.slice(a, b - a)
            assert not cix["null_pages"][i]
            if pa.types.is_date32(vals.type):
                lo, hi = page.cast(pa.int32()).to_numpy().min(), page.cast(pa.int32()).to_numpy().max()
            else:
                ints = [int(v.scaleb(2)) for v in page.to_pylist()]
                lo, hi = min(ints), max(ints)
            assert ref.stat_value(cix["min"][i], phys) == lo and ref.stat_value(cix["max"][i], phys) == hi
    assert counts["l_shipdate"] != counts["l_quantity"] != counts["l_returnflag"]


# ---- the planner against the reference ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("version,compression", [("1.0", "NONE"), ("2.0", "SNAPPY"), ("1.0", "ZSTD"), ("2.0", "ZSTD")])
def test_planner_selects_the_reference_rows(cb, planner, tmp_path, version, compression):
    """a date range inside a date-sorted file: the same rows, pages, segments, page tables and upload bytes as the reference"""
    t = cb.tpch
    _, path = lineitem(cb, 250_000, str(tmp_path / "l.parquet"), version=version, compression=compression)
    fields = _fields(cb)
    terms = [(6, "ge", t.DATE_1994_01_01), (6, "lt", t.DATE_1994_01_01 + 7)]
    out = check_plan(cb, planner, [path], fields, terms)
    assert out["pruned_pages"] > 0 and out["page_pruned_rows"] > 0
    assert any(u["ranges"] for u in out["units"])
    # chunkRows below the selection: the units still tile the batches
    check_plan(cb, planner, [path], fields, terms, chunk_rows=2_000)
    # pruning off: whole row groups, no selection
    off = planner(scan(cb, fields, [path], terms), no_prune=True)
    assert off["pruned_pages"] == 0 and all(u["ranges"] is None for u in off["units"])


@pytest.mark.parametrize("encoding", ["DELTA_BINARY_PACKED", "BYTE_STREAM_SPLIT", "PLAIN"])
def test_planner_over_delta_bss_and_plain_pages(cb, planner, tmp_path, encoding):
    t = cb.tpch
    _, path = lineitem(cb, 120_000, str(tmp_path / "e.parquet"), rg=60_000, version="2.0", compression="SNAPPY", encoding=encoding,
                       variant="dec" if encoding != "BYTE_STREAM_SPLIT" else "f64")
    fields = _fields(cb, "dec" if encoding != "BYTE_STREAM_SPLIT" else "f64")
    if encoding == "BYTE_STREAM_SPLIT":
        terms = [(2, "ge", 0.05), (2, "le", 0.07), (6, "gt", t.DATE_1995_06_17)]
    else:
        terms = [(6, "ge", t.DATE_1995_06_17), (6, "le", t.DATE_1995_06_17 + 30), (0, "lt", 2400)]
    check_plan(cb, planner, [path], fields, terms)


def _nullable_file(path, n=40_000, version="1.0"):
    """a sorted key with NULL stretches longer than a page (all-NULL pages; a page holds at most 500 rows) and a nullable value column
    whose pages end elsewhere"""
    rng = np.random.default_rng(3)
    key = np.sort(rng.integers(0, 10_000, n)).astype(np.int64)
    kmask = np.zeros(n, bool)
    kmask[5_000:11_000] = True
    kmask[30_000:30_500] = True
    vmask = rng.random(n) < 0.2
    vmask[20_000:26_000] = True
    tbl = pa.table({"k": pa.array(key, mask=kmask), "v": pa.array(rng.integers(-10**6, 10**6, n).astype(np.int32), mask=vmask),
                    "d": pa.array(rng.standard_normal(n))})
    pq.write_table(tbl, path, row_group_size=20_000, data_page_size=1024, write_batch_size=100, max_rows_per_page=500, write_page_index=True, data_page_version=version, compression="SNAPPY")
    return tbl, path


@pytest.mark.parametrize("version", ["1.0", "2.0"])
def test_planner_all_null_pages(cb, planner, tmp_path, version):
    """IsNotNull and comparisons drop all-NULL pages; a NULL-aware column is planned in covered rows"""
    P = cb.proto
    _, path = _nullable_file(str(tmp_path / "n.parquet"), version=version)
    fields = [("k", P.INT64, True), ("v", P.INT32, True), ("d", P.DOUBLE, True)]
    out = check_plan(cb, planner, [path], fields, [(0, "notnull", None)])
    assert out["pruned_pages"] > 0
    out = check_plan(cb, planner, [path], fields, [(1, "notnull", None), (0, "ge", 2_000)])
    assert out["pruned_pages"] > 0
    assert any(c["null_aware"] and c["segs"] for b in out["batches"] for c in b["columns"])


def test_eq_between_pages_drops_the_row_group(cb, planner, tmp_path):
    """an Eq literal inside the chunk's [min, max] that falls between two pages' ranges: every page goes, the row group with them"""
    import page_index_ref as ref
    P = cb.proto
    n = 50_000
    key = np.arange(n, dtype=np.int64) * 2                                            # even keys: an odd key lies between pages
    path = str(tmp_path / "eq.parquet")
    pq.write_table(pa.table({"k": key, "x": np.arange(n, dtype=np.int32)}), path, row_group_size=n, data_page_size=8192, write_page_index=True)
    oi, ci = ref.page_indexes(open(path, "rb").read())[0][0]
    hi0 = ref.stat_value(ci["max"][0], "INT64")
    fields = [("k", P.INT64, False), ("x", P.INT32, False)]
    out = check_plan(cb, planner, [path], fields, [(0, "eq", hi0 + 1)])
    assert out["units"] == [] and out["pruned_row_groups"] == 0 and out["dropped_row_groups"] == 1
    assert out["page_pruned_rows"] == n and out["pruned_pages"] == sum(len(ref.page_indexes(open(path, "rb").read())[0][c][0]) for c in range(2))


def test_page_spanning_two_selected_ranges(cb, planner, tmp_path):
    """two disjoint selected ranges inside one page of another column: that page is decoded once, two segments point into it"""
    P = cb.proto
    n = 40_000
    rng = np.random.default_rng(9)
    key = (np.arange(n, dtype=np.int64) // 500) % 4                                  # 0 1 2 3 0 1 2 3 ...: k in [1, 2] in disjoint ranges
    big = rng.integers(0, 4, n).astype(np.int32)                                   # 4 dictionary codes: ~2400 rows per 1 KB page
    path = str(tmp_path / "span.parquet")
    pq.write_table(pa.table({"k": key, "c": big}), path, row_group_size=n, data_page_size=1024, write_batch_size=100, write_page_index=True, use_dictionary=["c"])
    fields = [("k", P.INT64, False), ("c", P.INT32, False)]
    check_plan(cb, planner, [path], fields, [(0, "ge", 3)])
    u = check_plan(cb, planner, [path], fields, [(0, "ge", 1), (0, "le", 2)])["units"][0]
    # the selected rows of k come in disjoint ranges; some page of c covers two of them
    assert len(u["ranges"]) >= 2
    segs_c = u["columns"][1]["segs"]
    assert len(u["columns"][1]["pages"]) < len(segs_c)


def test_files_with_and_without_an_index_in_one_scan(cb, planner, tmp_path):
    t = cb.tpch
    _, a = lineitem(cb, 120_000, str(tmp_path / "a.parquet"), seed=1, rg=40_000)
    _, b = lineitem(cb, 120_000, str(tmp_path / "b.parquet"), seed=2, rg=40_000, index=False)
    fields = _fields(cb)
    terms = [(6, "ge", t.DATE_1995_06_17), (6, "lt", t.DATE_1995_06_17 + 10)]
    out = check_plan(cb, planner, [a, b, a], fields, terms, chunk_rows=50_000)
    files = {u["file"]: u["ranges"] is not None for u in out["units"]}
    assert files[0] and not files[1]


def test_contradicting_offset_index_never_changes_the_plan(cb, planner, tmp_path):
    """an OffsetIndex byte-patched to contradict its page headers is ignored or refused, never planned differently"""
    import page_index_ref as ref
    cols, path = lineitem(cb, 100_000, str(tmp_path / "l.parquet"))
    raw = bytearray(open(path, "rb").read())
    fields = _fields(cb)
    chunks = ref.footer_chunks(bytes(raw))[0]
    oi_pos = chunks[0]["oi"][0]                                                     # l_quantity's OffsetIndex
    oi = ref.offset_index(bytes(raw), oi_pos)
    ship = cols["l_shipdate"]
    terms = [(6, "ge", int(ship[oi[1][2]])), (6, "le", int(ship[oi[2][2] - 1]))]   # the dates of l_quantity's second page: it is selected
    good = check_plan(cb, planner, [path], fields, terms)
    assert 1 in good["units"][0]["columns"][0]["pages"]
    results = []
    # patch every varint of the second page location in place by +1 in its low bits (same length): offset, size or first row
    for field in range(3):
        bad = bytearray(raw)
        want = oi[1][field]
        enc = _zigzag_varint(want)
        at = bytes(bad).find(enc, oi_pos)
        assert 0 <= at < oi_pos + chunks[0]["oi"][1]
        bad[at] ^= 0x02                                                             # zigzag +-1, same byte count
        p = str(tmp_path / f"bad{field}.parquet")
        open(p, "wb").write(bad)
        got = planner(scan(cb, fields, [p], terms), expect_error=True)
        if isinstance(got, str):
            results.append("error")
            assert "offset index" in got or "page" in got, got
        else:                                                                       # ignored: the row group is read whole
            results.append("ignored")
            assert all(u["ranges"] is None for u in got["units"]) and got["pruned_pages"] == 0
    assert good["pruned_pages"] > 0 and len(results) == 3


def _zigzag_varint(v):
    z = (v << 1) ^ (v >> 63)
    out = bytearray()
    while True:
        b = z & 0x7F
        z >>= 7
        if z:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)
