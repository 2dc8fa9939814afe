"""Arrow streams and Parquet files whose batches change physical layout from one device chunk to the next, for
tests/test_gpu_batch_layouts.py (runs them) and tests/test_batch_layouts_cpu.py (pins the builder against pyarrow).

The logical table stays the one the CPU references read; only how each chunk carries it changes.  `chunked` cuts a table into
chunks of exactly `chunk_rows` rows (the Arrow stream source takes whole batches until it holds at least chunkRows rows, so these
are the device chunks) and re-encodes every column of a chunk as its recipe entry says:

  validity   "none"     no validity buffer (the chunk must hold no NULL)
             "nulls"    a buffer with NULLs
             "zero"     a buffer, null_count 0 (the source drops it: no validity on the device)
             "unknown"  a buffer, null_count -1 (the source keeps it)
             "allnull"  every row NULL
  "_split"   sizes of the batches the chunk is cut into (default: one batch)
  "_offset"  every batch is a slice at this row offset of larger buffers (bitmaps at a bit offset)
  "_empty"   an empty batch before every batch of the chunk
  "_dict"    {column: "identity" | "remap"}: the batch dictionary as the plan-wide one (narrow codes stay) or reversed (codes are
             remapped to int32 on the device)

NativeScan files: `write_row_groups` writes one row group per `rows` rows, with or without statistics."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

VALIDITY = ("none", "nulls", "zero", "unknown", "allnull")
_OPTIONS = ("_split", "_offset", "_empty", "_dict")


def _ones(n):
    return pa.py_buffer(np.full((n + 7) // 8 + 8, 0xFF, dtype=np.uint8).tobytes())


def with_validity(arr, how, offset=0):
    """A non-dictionary array re-made with validity layout `how`, as a slice at row `offset` of larger buffers."""
    assert how in VALIDITY, how
    nulls = arr.null_count
    if how in ("none", "zero", "unknown"):
        assert nulls == 0, f"{how}: the chunk holds {nulls} NULLs"
    elif how == "nulls":
        assert 0 < nulls, "nulls: the chunk holds no NULL"
    else:
        assert nulls == len(arr), "allnull: the chunk holds a non-NULL value"
    offset = offset if len(arr) else 0
    pad = pa.concat_arrays([arr] * (offset // max(len(arr), 1) + 1)).slice(0, offset)
    full = pa.concat_arrays([pad, arr])   # offset 0, buffers of its own
    m = len(full)
    bufs = full.buffers()
    if how == "none":
        v, nc = None, 0
    elif how in ("zero", "unknown"):
        v, nc = _ones(m), 0 if how == "zero" else -1
    else:
        v, nc = bufs[0], full.null_count
    out = pa.Array.from_buffers(full.type, m, [v] + bufs[1:], null_count=nc)
    return out.slice(offset) if offset else out


def encode(arr, how, offset=0, dict_mode=None):
    """`arr` (one chunk's values of a column) in the layout of one recipe entry"""
    if pa.types.is_dictionary(arr.type):
        idx, dic = arr.indices, arr.dictionary
        if dic.null_count or len(set(dic.to_pylist())) != len(dic):
            raise ValueError("dictionaries here hold distinct non-NULL strings")
        if dict_mode == "remap":     # the same strings in reverse order: every batch code maps to another plan-wide code
            n = len(dic)
            dic = pa.array(dic.to_pylist()[::-1], type=dic.type)
            idx = pa.array([None if c is None else n - 1 - c for c in idx.to_pylist()], type=idx.type)
        idx = with_validity(idx, how, offset) if how else idx
        return pa.DictionaryArray.from_arrays(idx, dic)
    return with_validity(arr, how, offset) if how else arr


class Batches(list):
    """RecordBatches plus, per batch, the columns the stream must export with null_count -1 (`unknown`) or with an all-valid buffer
    and null_count 0 (`zero`): pyarrow's exporter counts the NULLs and drops a buffer without NULLs"""
    unknown = zero = ()


def chunked(table, chunk_rows, recipe):
    """-> a list of RecordBatches: chunk c is rows [c * chunk_rows, (c + 1) * chunk_rows) of `table`, encoded by recipe[c]
    ({column name: validity} plus the options above; a column it does not name keeps pyarrow's layout)."""
    names = table.column_names
    out, start, unknown, zero = Batches(), 0, [], []
    for spec in recipe:
        bad = set(spec) - set(names) - set(_OPTIONS)
        assert not bad, bad
        n = min(chunk_rows, table.num_rows - start)
        sizes = spec.get("_split", [n])
        assert sum(sizes) == n, (sizes, n)
        for sz in sizes:
            part = table.slice(start, sz)
            arrays = [encode(part.column(c).combine_chunks(), spec.get(c), spec.get("_offset", 0), spec.get("_dict", {}).get(c))
                      for c in names]
            if spec.get("_empty"):
                out.append(pa.RecordBatch.from_arrays([a.slice(0, 0) for a in arrays], names=names))
                unknown.append(frozenset())
                zero.append(frozenset())
            out.append(pa.RecordBatch.from_arrays(arrays, names=names))
            unknown.append(frozenset(i for i, c in enumerate(names) if spec.get(c) == "unknown"))
            zero.append(frozenset(i for i, c in enumerate(names) if spec.get(c) == "zero"))
            start += sz
    assert start == table.num_rows, (start, table.num_rows)
    out.unknown, out.zero = unknown, zero
    return out


def chunk_of(batches, chunk_rows):
    """chunk index of every batch, as the stream source groups them (whole batches until it holds chunk_rows rows)"""
    out, chunk, rows = [], 0, 0
    for b in batches:
        if rows >= chunk_rows:
            chunk, rows = chunk + 1, 0
        out.append(chunk)
        rows += b.num_rows
    return out


class _Array(C.Structure):
    pass


_Array._fields_ = [("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64), ("n_buffers", C.c_int64),
                   ("n_children", C.c_int64), ("buffers", C.POINTER(C.c_void_p)), ("children", C.POINTER(C.POINTER(_Array))),
                   ("dictionary", C.POINTER(_Array)), ("release", C.c_void_p), ("private_data", C.c_void_p)]


class _Schema(C.Structure):
    _fields_ = [("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64), ("n_children", C.c_int64),
                ("children", C.c_void_p), ("dictionary", C.c_void_p), ("release", C.c_void_p), ("private_data", C.c_void_p)]


def exported(batch):
    """What the C data interface hands the library for each column of `batch`: (length, null_count, offset, has validity buffer).
    For a dictionary column, its indices."""
    arr, sch = _Array(), _Schema()
    batch._export_to_c(C.addressof(arr), C.addressof(sch))
    try:
        out = []
        for i in range(arr.n_children):
            ch = arr.children[i].contents
            out.append((ch.length, ch.null_count, ch.offset, bool(ch.buffers[0])))
        return out
    finally:
        C.CFUNCTYPE(None, C.POINTER(_Array))(arr.release)(C.byref(arr))
        C.CFUNCTYPE(None, C.POINTER(_Schema))(sch.release)(C.byref(sch))


def device_validity(batch):
    """per column: whether the stream source gives it a validity buffer (null_count != 0 and a buffer)"""
    return [nc != 0 and has for _, nc, _, has in exported(batch)]


def write_row_groups(path, table, rows, statistics=True, dictionary_limit=None):
    """one row group per `rows` rows; string columns dictionary-encoded until a row group's dictionary outgrows `dictionary_limit`
    bytes (PLAIN from there on, in that row group only)"""
    kw = {} if dictionary_limit is None else {"dictionary_pagesize_limit": dictionary_limit}
    pq.write_table(table, path, row_group_size=rows, write_statistics=statistics, use_dictionary=True, data_page_size=1 << 14, **kw)
    return pq.ParquetFile(path).metadata


# ---- the C stream interface: null_count -1 ----------------------------------------------------------------------------------------
class _Stream(C.Structure):
    pass


_GET_SCHEMA = C.CFUNCTYPE(C.c_int, C.POINTER(_Stream), C.c_void_p)
_GET_NEXT = C.CFUNCTYPE(C.c_int, C.POINTER(_Stream), C.POINTER(_Array))
_LAST_ERROR = C.CFUNCTYPE(C.c_char_p, C.POINTER(_Stream))
_RELEASE = C.CFUNCTYPE(None, C.POINTER(_Stream))
_Stream._fields_ = [("get_schema", _GET_SCHEMA), ("get_next", _GET_NEXT), ("get_last_error", _LAST_ERROR), ("release", _RELEASE),
                    ("private_data", C.c_void_p)]
_LIVE = []   # streams the library may still call into
_ONES = np.full(1 << 17, 0xFF, dtype=np.uint8)   # an all-valid bitmap for up to 2^20 rows


class source:
    """A stream input for `native.Plan` that hands the library `batches` (a `Batches`) as the recipe says: null_count -1 on every
    column marked "unknown" (a producer that does not count NULLs), an all-valid buffer with null_count 0 on every one marked "zero"."""

    def __init__(self, batches):
        none = [frozenset()] * len(batches)
        self.batches = list(batches)
        self.unknown, self.zero = list(getattr(batches, "unknown", ())) or none, list(getattr(batches, "zero", ())) or none
        self.inner = _Stream()
        self.at = 0
        _LIVE.append(self)

    def _export_to_c(self, addr):
        reader = pa.RecordBatchReader.from_batches(self.batches[0].schema, self.batches)
        reader._export_to_c(C.addressof(self.inner))
        inner = self.inner

        def get_schema(_, out):
            return inner.get_schema(C.byref(inner), out)

        def get_next(_, out):
            rc = inner.get_next(C.byref(inner), out)
            if rc == 0 and out.contents.release and self.at < len(self.unknown):
                for c in self.unknown[self.at]:
                    out.contents.children[c].contents.null_count = -1
                for c in self.zero[self.at]:
                    ch = out.contents.children[c].contents
                    assert ch.offset + ch.length <= 8 * len(_ONES)
                    if ch.n_buffers and not ch.buffers[0]:
                        ch.buffers[0] = _ONES.ctypes.data
                self.at += 1
            return rc

        def last_error(_):
            return inner.get_last_error(C.byref(inner))

        def release(s):
            if inner.release:
                inner.release(C.byref(inner))
            s.contents.release = _RELEASE()

        self.callbacks = (_GET_SCHEMA(get_schema), _GET_NEXT(get_next), _LAST_ERROR(last_error), _RELEASE(release))
        outer = _Stream.from_address(addr)
        outer.get_schema, outer.get_next, outer.get_last_error, outer.release = self.callbacks
        outer.private_data = None
