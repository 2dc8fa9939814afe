"""GPU: scan-only plans handed to the caller -- a bare NativeScan, a bare Scan over an Arrow stream and a bare Scan over a device table --
through cb200_execute (spark.comet.batchSize slices included) and cb200_execute_device, against pyarrow's read of the same file or the
input table itself.  The sources keep some columns in a layout other than Arrow's: the Parquet scan stores INT32-backed int8 / int16 /
decimal(7, 2) 4 bytes per row and decimals with p <= 18 8 bytes per row, device tables may hold 8-byte decimals, streams keep booleans as
bitmaps.  The hand-off gives out the Arrow layout, and cb200_execute_device reports its width."""
import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import partref
from test_gpu_partition_layouts import device_table, expected_table, make_values, parquet_table, scan_of, table_of, write_parquet

pytestmark = pytest.mark.gpu

INTS = ["i8", "i16", "i32", "i32w", "date", "i64", "ts", "f32", "f64", "row"]
DECIMALS = ["d7", "d12", "d28", "row"]
STRINGS = ["sd", "sp", "row"]
ARROW_WIDTH = {pa.bool_(): 1, pa.int8(): 1, pa.int16(): 2, pa.int32(): 4, pa.date32(): 4, pa.int64(): 8, pa.float32(): 4, pa.float64(): 8}


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    """the same columns written with decimals as INT32 / INT64 (store_decimal_as_integer) and as FIXED_LEN_BYTE_ARRAY"""
    cols = parquet_table(70_000, 41)
    d = tmp_path_factory.mktemp("scan_export")
    paths = {}
    for as_int in (True, False):
        paths[as_int] = str(d / f"e{int(as_int)}.parquet")
        write_parquet(paths[as_int], cols, as_int)
    return cols, paths


def collect(cb, plan, inputs=(), batch_size=8192, config=None):
    with cb.native.Plan(plan, list(inputs), config=config, batch_size=batch_size) as p:
        batches = []
        while True:
            b = p.execute()
            if b is None:
                break
            assert b.num_rows <= batch_size
            batches.append(b)
    return pa.Table.from_batches(batches)


def device_batches(cb, plan, inputs=(), config=None):
    """every batch of cb200_execute_device read back through the reported layout: one pyarrow table per batch"""
    import torch
    from comet_b200.dist import device_bytes
    out = []
    with cb.native.Plan(plan, list(inputs), config=config) as p:
        while True:
            r = p.execute_device()
            if r is None:
                break
            rows, cols = r
            arrays = []
            for j in range(p.n_cols):
                c = cols[j]
                assert c.values and not c.host_values, j
                raw = device_bytes(torch, c.values, rows * c.value_width, "cuda").cpu().numpy()
                valid = None
                if c.validity:
                    bits = device_bytes(torch, c.validity, (rows + 7) // 8, "cuda").cpu().numpy()
                    valid = np.unpackbits(bits, bitorder="little")[:rows].astype(bool)
                arrays.append((c.type_id, c.precision, c.scale, c.value_width, c.n_dict, raw, valid,
                               p.dict_values(j, c.n_dict) if c.n_dict else None))
            out.append((rows, arrays))
    return out


def assert_device_matches(got, want):
    """got: device_batches(); want: the expected table (batches in order)"""
    row0 = 0
    for rows, arrays in got:
        part = want.slice(row0, rows)
        for j, (type_id, precision, scale, width, n_dict, raw, valid, dictionary) in enumerate(arrays):
            w = partref.plain(part.column(j))
            name = want.column_names[j]
            wvalid = np.asarray(w.is_valid())
            assert (np.ones(rows, bool) if valid is None else valid).tolist() == wvalid.tolist(), name
            if n_dict:
                codes = raw.view({1: np.int8, 2: np.int16, 4: np.int32}[width])
                spelled = [dictionary[int(c)] if ok else None for c, ok in zip(codes, wvalid)]
                assert spelled == w.to_pylist(), name
                continue
            if pa.types.is_decimal(w.type):
                assert width == 16 and (precision, scale) == (w.type.precision, w.type.scale), (name, width)
                got_arr = pa.Array.from_buffers(w.type, rows, [None, pa.py_buffer(raw)])
            elif pa.types.is_timestamp(w.type):
                assert width == 8, name
                got_arr = pa.Array.from_buffers(w.type, rows, [None, pa.py_buffer(raw)])
            else:
                assert width == ARROW_WIDTH[w.type], (name, width)
                if pa.types.is_boolean(w.type):
                    got_arr = pa.array(raw.astype(bool))
                else:
                    got_arr = pa.Array.from_buffers(w.type, rows, [None, pa.py_buffer(raw)])
            got_arr = pa.Array.from_buffers(got_arr.type, rows, [pa.py_buffer(np.packbits(wvalid, bitorder="little")), *got_arr.buffers()[1:]])
            partref.assert_columns_equal(got_arr, w, name)
        row0 += rows
    assert row0 == want.num_rows


# ---- bare NativeScan -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("as_int", [True, False])
@pytest.mark.parametrize("which", ["ints", "decimals", "strings"])
@pytest.mark.parametrize("batch_size", [8192, 7001])
def test_native_scan_export(cb, files, as_int, which, batch_size):
    """the scan's own batches (chunkRows 30 000 over 40 000-row row groups) cut into zero-offset slices of spark.comet.batchSize rows"""
    cols, paths = files
    names = {"ints": INTS, "decimals": DECIMALS, "strings": STRINGS}[which]
    scan, _ = scan_of(cb, cols, names, paths[as_int])
    got = collect(cb, scan, batch_size=batch_size, config={"spark.comet.b200.chunkRows": "30000", "spark.comet.batchSize": str(batch_size)})
    want = expected_table(cols, names)
    partref.assert_tables_equal(got, want)
    read = pq.read_table(paths[as_int], columns=[k for k in names if k != "i32w"])   # the file as pyarrow reads it
    for k in read.column_names:
        partref.assert_columns_equal(got.column(names.index(k)), read.column(k), k)


@pytest.mark.parametrize("as_int", [True, False])
@pytest.mark.parametrize("which", ["ints", "decimals", "strings"])
def test_native_scan_execute_device(cb, files, as_int, which):
    cols, paths = files
    names = {"ints": INTS, "decimals": DECIMALS, "strings": STRINGS}[which]
    scan, _ = scan_of(cb, cols, names, paths[as_int])
    got = device_batches(cb, scan, config={"spark.comet.b200.chunkRows": "30000"})
    assert len(got) >= 2
    assert_device_matches(got, expected_table(cols, names))


# ---- bare Scan over an Arrow stream / a device table ----------------------------------------------------------------------------------------
STREAM = ["b", "i8", "i16", "i32", "date", "i64", "ts", "f32", "f64", "d9", "d18", "d38", "s8", "s16", "s32", "row"]


@pytest.mark.parametrize("n,batch_size", [(1, 8192), (1025, 100), (50_000, 8192), (50_000, 4093)])
def test_stream_export(cb, n, batch_size):
    """booleans arrive as bitmaps, strings as dictionaries with int8 / int16 / int32 indices"""
    tbl, types = table_of(make_values(n, 7), STREAM)
    got = collect(cb, cb.proto.scan(types), [tbl.to_batches(max_chunksize=6000)], batch_size=batch_size,
                  config={"spark.comet.b200.chunkRows": "20000", "spark.comet.batchSize": str(batch_size)})
    partref.assert_tables_equal(got, tbl)


@pytest.mark.parametrize("partitioned", [False, True])
def test_stream_execute_device(cb, partitioned):
    """cb200_execute_device over a bare stream Scan and over ShuffleWriter(SinglePartition) of it (which keeps the row order)"""
    from test_gpu_partition_layouts import hash_plan
    tbl, types = table_of(make_values(30_000, 8), STREAM)
    plan = cb.proto.scan(types)
    if partitioned:
        plan = hash_plan(cb, plan, types, STREAM, [], None)
    got = device_batches(cb, plan, [tbl.to_batches(max_chunksize=7000)], config={"spark.comet.b200.chunkRows": "14000"})
    assert [r for r, _ in got] == [14_000, 14_000, 2_000]
    assert_device_matches(got, tbl)


def test_device_table_export(cb):
    """decimal(9, 2) and decimal(18, 0) handed in 8 bytes wide come out as Decimal128; bitmap booleans as one byte per row"""
    tbl, types = table_of(make_values(20_000, 9), STREAM)
    t = device_table(cb, tbl, types, dec8=("d9", "d18"))
    partref.assert_tables_equal(collect(cb, cb.proto.scan(types), [t], batch_size=5000, config={"spark.comet.batchSize": "5000"}), tbl)
    t = device_table(cb, tbl, types, dec8=("d9", "d18"))
    assert_device_matches(device_batches(cb, cb.proto.scan(types), [t], config={"spark.comet.b200.chunkRows": "8192"}), tbl)
