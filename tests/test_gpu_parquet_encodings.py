"""GPU parity: DELTA_BINARY_PACKED and BYTE_STREAM_SPLIT pages decoded on the device, DELTA_LENGTH_BYTE_ARRAY / DELTA_BYTE_ARRAY
pages turned into PLAIN on the host, all through cb200_create_plan / cb200_execute against pyarrow's read of the same file."""
import decimal
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

RF = ["A", "N", "R"]
LS = ["F", "O"]


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def run(cb, plan, inputs=(), chunk_rows=None):
    cfg = {"spark.comet.b200.chunkRows": str(chunk_rows)} if chunk_rows else None
    with cb.native.Plan(plan, list(inputs), config=cfg) as p:
        t = p.collect()
        st = p.stats()
    return t, st


def unscaled(x):
    return None if x is None else int(x.scaleb(-x.as_tuple().exponent))


# column -> (pyarrow type, scan type, encoding)
def _columns(P):
    return {
        "i32": ("int32", P.INT32, "DELTA_BINARY_PACKED"),
        "i32w": ("int32", P.INT64, "DELTA_BINARY_PACKED"),        # INT32 page read as INT64: PQ_I32_TO_I64
        "i64": ("int64", P.INT64, "DELTA_BINARY_PACKED"),
        "date": ("date32", P.DATE, "DELTA_BINARY_PACKED"),
        "ts": ("timestamp_us", P.TIMESTAMP, "DELTA_BINARY_PACKED"),
        "d9": ("d9", P.DECIMAL(9, 2), "DELTA_BINARY_PACKED"),
        "d12": ("d12", P.DECIMAL(12, 2), "DELTA_BINARY_PACKED"),
        "f32": ("float32", P.FLOAT, "BYTE_STREAM_SPLIT"),
        "f64": ("float64", P.DOUBLE, "BYTE_STREAM_SPLIT"),
        "b32": ("int32", P.INT32, "BYTE_STREAM_SPLIT"),
        "b64": ("int64", P.INT64, "BYTE_STREAM_SPLIT"),
        "bd30": ("d30", P.DECIMAL(30, 4), "BYTE_STREAM_SPLIT"),    # FIXED_LEN_BYTE_ARRAY, 13 bytes
        "dd30": ("d30", P.DECIMAL(30, 4), "DELTA_BYTE_ARRAY"),     # on the host, then PLAIN FLBA on the device
        "s_dlba": ("string", P.STRING, "DELTA_LENGTH_BYTE_ARRAY"),
        "s_dba": ("string", P.STRING, "DELTA_BYTE_ARRAY"),
        "req": ("int64", P.INT64, "DELTA_BINARY_PACKED"),          # no NULLs: the null_count = 0 fast path in the same file
    }


def _table(cb, n, seed, null_frac=0.15):
    import pyarrow as pa
    rng = np.random.default_rng(seed)
    ctx = decimal.Context(prec=60)
    specials64 = np.array([0x7FF8DEADBEEF0001, 0xFFF0000000000001, 0x8000000000000000, 0x0000000000000001, 0x7FF0000000000000, 0xFFF0000000000000],
                          dtype=np.uint64).view(np.float64)          # NaN payloads, -0.0, subnormal, +-Inf
    specials32 = np.array([0x7FC0BEEF, 0xFF800001, 0x80000000, 0x00000001, 0x7F800000, 0xFF800000], dtype=np.uint32).view(np.float32)

    def mask():
        m = rng.random(n) < null_frac
        m[: n // 20] = True                      # a NULL stretch longer than a page: all-NULL pages
        m[n // 2: n // 2 + n // 40] = False
        return m
    f64 = rng.standard_normal(n) * 1e3
    f64[n // 3: n // 3 + 6] = specials64
    f32 = rng.standard_normal(n).astype(np.float32)
    f32[n // 3: n // 3 + 6] = specials32
    i64 = np.cumsum(rng.integers(-10**6, 10**9, n)).astype(np.int64)
    i64[n // 4: n // 4 + 100] = np.array([-2**63, 2**63 - 1] * 50)
    i32 = rng.integers(-2**31, 2**31, n).astype(np.int32)
    i32[n // 4: n // 4 + 100] = np.array([-2**31, 2**31 - 1] * 50)
    words = np.array([f"shipmode/{i:04d}" for i in range(900)] + ["", "ünï", "a" * 300])
    d30 = [int(a) * 10**12 + int(b) for a, b in zip(rng.integers(-10**17, 10**17, n), rng.integers(0, 10**12, n))]
    dec = lambda vals, p, s: pa.array([decimal.Decimal(int(v)).scaleb(-s, context=ctx) for v in vals], type=pa.decimal128(p, s), mask=mask())
    data = {
        "i32": pa.array(i32, mask=mask()),
        "i32w": pa.array(rng.integers(-2**31, 2**31, n).astype(np.int32), mask=mask()),
        "i64": pa.array(i64, mask=mask()),
        "date": pa.array(np.sort(rng.integers(8000, 10600, n)).astype(np.int32), type=pa.date32(), mask=mask()),
        "ts": pa.array(rng.integers(0, 2**60, n), type=pa.timestamp("us"), mask=mask()),
        "d9": dec(rng.integers(-10**9 + 1, 10**9, n), 9, 2),
        "d12": dec(rng.integers(-10**11, 10**11, n), 12, 2),
        "f32": pa.array(f32, mask=mask()),
        "f64": pa.array(f64, mask=mask()),
        "b32": pa.array(rng.integers(-2**31, 2**31, n).astype(np.int32), mask=mask()),
        "b64": pa.array(rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64), mask=mask()),
        "bd30": dec(d30, 30, 4),
        "dd30": dec(sorted(d30), 30, 4),
        "s_dlba": pa.array(words[rng.integers(0, len(words), n)].tolist(), mask=mask()).cast(pa.string()),
        "s_dba": pa.array(sorted(words[rng.integers(0, len(words), n)].tolist()), mask=mask()).cast(pa.string()),
        "req": pa.array(np.arange(n, dtype=np.int64) * 7 - 5),
    }
    return pa.table(data)


def _write(cb, tbl, path, compression, version, page_size=8192, row_group_size=20_000, encodings=None):
    import pyarrow.parquet as pq
    cols = _columns(cb.proto)
    enc = encodings or {k: v[2] for k, v in cols.items() if k in tbl.column_names}
    pq.write_table(tbl, path, row_group_size=row_group_size, compression=compression, use_dictionary=False, column_encoding=enc,
                   data_page_version=version, data_page_size=page_size, store_decimal_as_integer=True)
    return path


def _scan(cb, names, paths):
    P = cb.proto
    cols = _columns(P)
    fields = [(name, cols[name][1], True) for name in names]
    return P.projection(P.native_scan(fields, fields, paths), [P.bound(i, cols[name][1]) for i, name in enumerate(names)])


def _check(res, tbl, repeat=1):
    import pyarrow as pa
    for j, name in enumerate(tbl.column_names):
        got = res.column(j).combine_chunks()
        want = pa.concat_arrays([tbl.column(name).combine_chunks()] * repeat)
        assert got.null_count == want.null_count, name
        if name in ("f32", "f64"):
            bits = np.uint32 if name == "f32" else np.uint64
            ok = ~np.asarray(want.is_null())
            gv, wv = got.fill_null(0).to_numpy(), want.fill_null(0).to_numpy()
            assert (np.asarray(got.is_null()) == ~ok).all() and (gv[ok].view(bits) == wv[ok].view(bits)).all(), name
        elif name == "i32w":
            assert got.equals(want.cast(pa.int64())), name
        else:
            assert got.cast(want.type).equals(want), name


@pytest.mark.parametrize("compression,version", [("NONE", "1.0"), ("NONE", "2.0"), ("SNAPPY", "1.0"), ("SNAPPY", "2.0"), ("ZSTD", "1.0"), ("ZSTD", "2.0")])
def test_roundtrip_every_encoding_and_type(cb, tmp_path, compression, version):
    """Every (encoding, physical type, output type) pair, with NULL stretches, all-NULL pages and a NULL-free column in one file; small
    pages (many per batch) and batches that cut across row groups."""
    n = 60_000
    tbl = _table(cb, n, seed=5)
    path = _write(cb, tbl, str(tmp_path / "enc.parquet"), compression, version)
    for names in (tbl.column_names[:8], tbl.column_names[8:]):             # two scans of 8 columns: one projection kernel each
        res, st = run(cb, _scan(cb, names, [path]), chunk_rows=45_000)
        assert res.num_rows == n
        _check(res, tbl.select(names))


def test_mixed_encodings_in_one_batch(cb, tmp_path):
    """Dictionary, PLAIN, DELTA_BINARY_PACKED and BYTE_STREAM_SPLIT files of the same columns in ONE batch: each page decodes by its own
    encoding."""
    import pyarrow.parquet as pq
    n = 20_000
    tbl = _table(cb, n, seed=7).select(["i64", "d12", "i32", "req"])
    paths = []
    for i, enc in enumerate(("dict", "PLAIN", "DELTA_BINARY_PACKED", "BYTE_STREAM_SPLIT")):
        p = str(tmp_path / f"m{i}.parquet")
        if enc == "dict":
            pq.write_table(tbl, p, row_group_size=8_000, compression="SNAPPY", use_dictionary=True, data_page_size=4096, store_decimal_as_integer=True)
        else:
            pq.write_table(tbl, p, row_group_size=8_000, compression="SNAPPY", use_dictionary=False, data_page_size=4096, store_decimal_as_integer=True,
                           column_encoding={k: enc for k in tbl.column_names})
        paths.append(p)
    res, st = run(cb, _scan(cb, tbl.column_names, paths), chunk_rows=1 << 22)
    assert res.num_rows == 4 * n
    _check(res, tbl, repeat=4)


def _lineitem(cb, n, seed, variant, path, encodings, sort=False):
    import pyarrow.parquet as pq
    t = cb.tpch
    cols = t.gen_lineitem(n, seed=seed)
    if sort:
        order = np.argsort(cols["l_shipdate"], kind="stable")
        cols = {k: v[order] for k, v in cols.items()}
    names = t.Q6_COLUMNS if sort else t.Q1_COLUMNS
    tbl = t.lineitem_table(cols, variant, dictionary=True, columns=names)
    pq.write_table(tbl, path, row_group_size=16_384 if sort else 32_768, compression="NONE", use_dictionary=["l_returnflag", "l_linestatus"],
                   column_encoding={k: encodings for k in names if k not in ("l_returnflag", "l_linestatus") and (encodings != "BYTE_STREAM_SPLIT" or k != "l_shipdate")},
                   data_page_version="2.0", store_decimal_as_integer=True)
    return cols, path


def test_q1_dec_from_delta_parquet(cb, oracle, tmp_path):
    t = cb.tpch
    cols, path = _lineitem(cb, 300_000, 31, "dec", str(tmp_path / "q1d.parquet"), "DELTA_BINARY_PACKED")
    state, st = run(cb, t.q1_partial_plan("dec", scan=t.q1_native_scan("dec", [path])), chunk_rows=100_000)
    res, _ = run(cb, t.q1_final_plan("dec"), [state])
    d = oracle.dec_from_i64
    exp = oracle.q1_dec(d(cols["l_quantity"]), d(cols["l_extendedprice"]), d(cols["l_discount"]), d(cols["l_tax"]), cols["l_shipdate"],
                        cols["l_returnflag"], cols["l_linestatus"], 3, 2, t.Q1_CUTOFF, 1)
    got = {(r["col_0"], r["col_1"]): r for r in res.to_pylist()}
    for k, e in enumerate(exp):
        if e is None:
            continue
        g = got[(RF[k // 2], LS[k % 2])]
        for j, name in enumerate(["sum_qty", "sum_base", "sum_disc_price", "sum_charge", "avg_qty", "avg_price", "avg_disc"]):
            assert unscaled(g[f"col_{2 + j}"]) == e[name], (k, name)
        assert g["col_9"] == e["count"]


def test_q1_f64_from_bss_parquet(cb, tmp_path):
    t = cb.tpch
    cols, path = _lineitem(cb, 300_000, 11, "f64", str(tmp_path / "q1f.parquet"), "BYTE_STREAM_SPLIT")
    state, _ = run(cb, t.q1_partial_plan("f64", scan=t.q1_native_scan("f64", [path])), chunk_rows=100_000)
    res, _ = run(cb, t.q1_final_plan("f64"), [state])
    got = {(r["col_0"], r["col_1"]): r for r in res.to_pylist()}
    f = {k: (cols[k].astype(np.float64) / 100.0) for k in ("l_quantity", "l_extendedprice", "l_discount", "l_tax")}
    keep = cols["l_shipdate"] <= t.Q1_CUTOFF
    gid = cols["l_returnflag"].astype(np.int64) * 2 + cols["l_linestatus"]
    dp = f["l_extendedprice"] * (1.0 - f["l_discount"])
    ch = dp * (1.0 + f["l_tax"])
    for k in range(6):
        m = keep & (gid == k)
        if not m.any():
            assert (RF[k // 2], LS[k % 2]) not in got
            continue
        g = got[(RF[k // 2], LS[k % 2])]
        for j, v in enumerate([f["l_quantity"], f["l_extendedprice"], dp, ch]):
            exact = math.fsum(v[m])
            assert abs(g[f"col_{2 + j}"] - exact) <= math.ulp(exact), (k, j)
        assert g["col_9"] == int(m.sum())


def test_q6_prunes_delta_file(cb, oracle, tmp_path, monkeypatch):
    """Q6 over a date-clustered DELTA_BINARY_PACKED file: the statistics prune the same row groups, the result is the unpruned one."""
    t = cb.tpch
    n = 400_000
    cols, path = _lineitem(cb, n, 41, "dec", str(tmp_path / "q6.parquet"), "DELTA_BINARY_PACKED", sort=True)
    plan = t.q6_partial_plan("dec", scan=t.q6_native_scan("dec", [path]))
    state, st = run(cb, plan, chunk_rows=60_000)
    ship = cols["l_shipdate"]
    groups = [ship[g:g + 16_384] for g in range(0, n, 16_384)]
    exp_read = sum(1 for s in groups if s.max() >= t.DATE_1994_01_01 and s.min() < t.DATE_1995_01_01)
    assert st["scan_pruned_row_groups"] == len(groups) - exp_read
    monkeypatch.setenv("CB200_NO_PRUNE", "1")
    state_all, st_all = run(cb, plan, chunk_rows=60_000)
    assert st_all["scan_pruned_row_groups"] == 0 and state.equals(state_all)
    res, _ = run(cb, t.q6_final_plan("dec"), [state])
    d = oracle.dec_from_i64
    exp = oracle.q6_dec(d(cols["l_quantity"]), d(cols["l_extendedprice"]), d(cols["l_discount"]), ship, t.DATE_1994_01_01, t.DATE_1995_01_01, 5, 7, 2400, 1)
    assert unscaled(res.column(0)[0].as_py()) == exp


def test_delta_byte_array_strings_as_group_key(cb, tmp_path):
    P = cb.proto
    n = 50_000
    tbl = _table(cb, n, seed=13).select(["s_dba", "req"])
    path = _write(cb, tbl, str(tmp_path / "g.parquet"), "SNAPPY", "2.0")
    fields = [("s_dba", P.STRING, True), ("req", P.INT64, True)]
    out, _ = run(cb, P.hash_agg(P.native_scan(fields, fields, [path]), [P.bound(0, P.STRING)], [P.agg_count([P.literal(1, P.INT32)])], P.PARTIAL))
    exp = {}
    for w in tbl.column("s_dba").to_pylist():
        exp[w] = exp.get(w, 0) + 1
    got = {}
    for r in out.to_pylist():
        got[r["col_0"]] = got.get(r["col_0"], 0) + r["col_1"]
    assert got == exp


def test_malformed_delta_pages_raise(cb, tmp_path):
    """Same-length patches of an uncompressed DELTA_BINARY_PACKED page: a bit width of 65, a value count off by one.  Every read of the
    decoder is bounded by the page, so each comes back as an error, not as data."""
    import pyarrow as pa
    import pyarrow.parquet as pq
    from oracle import parquet_oracle as po
    from parquet_encodings_ref import uleb
    P = cb.proto
    n = 1000
    vals = np.random.default_rng(12).integers(-10**9, 10**9, n).astype(np.int64)
    path = str(tmp_path / "ok.parquet")
    pq.write_table(pa.table({"v": vals}, schema=pa.schema([pa.field("v", pa.int64(), nullable=False)])), path, compression="NONE", use_dictionary=False,
                   data_page_version="2.0", column_encoding={"v": "DELTA_BINARY_PACKED"}, write_statistics=False)
    raw = bytearray(open(path, "rb").read())
    c = pq.ParquetFile(path).metadata.row_group(0).column(0)
    h, body = po.page_header(raw, c.data_page_offset)
    assert h["type"] == 3 and h["encoding"] == 5 and h["num_values"] == n
    block, p = uleb(raw, body)
    mbs, p = uleb(raw, p)
    tpos = p
    _, p = uleb(raw, p)
    _, p = uleb(raw, p)
    _, p = uleb(raw, p)                                  # first block's min delta: p = its first bit-width byte
    fields = [("v", P.INT64, True)]
    res, _ = run(cb, P.projection(P.native_scan(fields, fields, [path]), [P.bound(0, P.INT64)]))
    assert res.column(0).to_numpy().tolist() == vals.tolist()
    for name, pos, byte in (("width65", p, 65), ("count", tpos, raw[tpos] + 1)):
        bad = bytearray(raw)
        bad[pos] = byte
        bp = str(tmp_path / f"{name}.parquet")
        open(bp, "wb").write(bytes(bad))
        with pytest.raises(cb.native.CometB200Error):
            run(cb, P.projection(P.native_scan(fields, fields, [bp]), [P.bound(0, P.INT64)]))


def test_scan_blocks_are_reused_across_delta_plans(cb, tmp_path):
    t = cb.tpch
    P = cb.proto
    n = 250_000
    cols, path = _lineitem(cb, n, 47, "dec", str(tmp_path / "reuse.parquet"), "DELTA_BINARY_PACKED")
    fields = list(zip(t.Q1_COLUMNS, t.q1_scan_fields("dec"), [True] * 7))
    sc = P.native_scan(fields, fields, [path])
    plan = P.hash_agg(sc, [], [P.agg_sum(P.bound(1, t.D12), P.DECIMAL(22, 2)), P.agg_sum(P.bound(3, t.D12), P.DECIMAL(22, 2)), P.agg_count([P.literal(1, P.INT32)])], P.PARTIAL)
    exp = (int(cols["l_extendedprice"].sum()), int(cols["l_tax"].sum()), n)
    for i in range(10):
        res, _ = run(cb, plan, chunk_rows=[20_000, 64_000, 250_000][i % 3])
        r = res.to_pylist()[0]
        assert (unscaled(r["col_0"]), unscaled(r["col_2"]), r["col_4"]) == exp, i

