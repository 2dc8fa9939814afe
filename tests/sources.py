"""Sources in every physical layout the scan hands a pipeline, shared by the GPU suites: device tables (caller-owned device buffers,
booleans as bitmaps, decimals 8 or 16 bytes wide) and Parquet files read by NativeScan (decimals stored as INT32 / INT64 or as FLBA,
int8 / int16 stored as INT32)."""
import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq


def device_table(cb, tbl, types, dec8=()):
    """tbl's columns as caller-owned device buffers: booleans as bitmaps, dictionaries as their codes, decimals named in dec8 as 8 bytes"""
    import torch
    t = cb.native.DeviceTable(tbl.num_rows)
    for name, dt in zip(tbl.column_names, types):
        a = tbl.column(name).combine_chunks()
        valid = np.asarray(a.is_valid())
        vbits = np.packbits(valid, bitorder="little")
        vdev = torch.from_numpy(np.concatenate([vbits, np.zeros(16, np.uint8)])).cuda() if a.null_count else None
        dictionary = None
        if pa.types.is_boolean(a.type):
            raw, width = np.packbits(np.asarray(a.fill_null(False)), bitorder="little"), 0
        elif pa.types.is_dictionary(a.type):
            idx = a.indices
            width = idx.type.bit_width // 8
            raw = np.frombuffer(idx.buffers()[1], dtype=np.uint8)[idx.offset * width:(idx.offset + len(idx)) * width]
            dictionary = a.dictionary.to_pylist()
        elif pa.types.is_decimal(a.type):
            v = np.frombuffer(a.buffers()[1], dtype=np.int64)[2 * a.offset:2 * (a.offset + len(a))].reshape(-1, 2)
            if name in dec8:
                raw, width = v[:, 0].copy().view(np.uint8), 8
            else:
                raw, width = v.copy().view(np.uint8).reshape(-1), 16
        else:
            width = a.type.bit_width // 8
            raw = np.frombuffer(a.buffers()[1], dtype=np.uint8)[a.offset * width:(a.offset + len(a)) * width]
        vals = torch.from_numpy(np.concatenate([np.ascontiguousarray(raw).view(np.uint8).reshape(-1), np.zeros(16, np.uint8)])).cuda()
        t.add(dt, vals.data_ptr(), width, vdev.data_ptr() if vdev is not None else None, a.null_count, dictionary=dictionary, keep=(vals, vdev))
    return t


def write_parquet(path, cols, as_int):
    tbl = pa.table({k: cols[k][0] for k in cols})
    pq.write_table(tbl, path, row_group_size=40_000, data_page_size=1 << 16, use_dictionary=["sd"], store_decimal_as_integer=as_int,
                   compression="SNAPPY")
    return tbl


def scan_of(cb, cols, names, path):
    """NativeScan reading `names` as their requested types"""
    fields = [(k, cols[k][1], True) for k in names]
    return cb.proto.native_scan(fields, fields, [path]), [cols[k][1] for k in names]
