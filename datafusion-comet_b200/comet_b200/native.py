"""ctypes binding of libcomet_b200.so -- the Python stand-in for the reference's JVM caller.

Mirrors `org.apache.comet.Native` (spark/src/main/scala/org/apache/comet/Native.scala:60-103):
createPlan / executePlan / releasePlan, driven the way `CometExecIterator`
(CometExecIterator.scala:109-210) drives them: serialized plan bytes in, Arrow C Data structs out.

The library is the product; this module only marshals.  It fails loudly if the shared library is
missing -- there is no CPU fallback.
"""
import ctypes as C
import os

import pyarrow as pa

_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB_PATH = os.path.join(_PKG, "libcomet_b200.so")
_lib = None


class CometB200Error(RuntimeError):
    def __init__(self, code, error_class, message):
        super().__init__(f"[{code}{' ' + error_class if error_class else ''}] {message}")
        self.code, self.error_class, self.message = code, error_class, message


class Unsupported(CometB200Error):
    """The plan is outside the GPU hot path; a caller keeps its CPU path (CB200_ERR_UNSUPPORTED)."""


class _Error(C.Structure):
    _fields_ = [("code", C.c_int32), ("error_class", C.c_char * 64), ("message", C.c_char * 952)]


class ArrowSchema(C.Structure):
    pass


class ArrowArray(C.Structure):
    pass


ArrowSchema._fields_ = [("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64),
                        ("n_children", C.c_int64), ("children", C.POINTER(C.POINTER(ArrowSchema))),
                        ("dictionary", C.POINTER(ArrowSchema)), ("release", C.c_void_p), ("private_data", C.c_void_p)]
ArrowArray._fields_ = [("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64), ("n_buffers", C.c_int64),
                       ("n_children", C.c_int64), ("buffers", C.POINTER(C.c_void_p)),
                       ("children", C.POINTER(C.POINTER(ArrowArray))), ("dictionary", C.POINTER(ArrowArray)),
                       ("release", C.c_void_p), ("private_data", C.c_void_p)]


class ArrowArrayStream(C.Structure):
    _fields_ = [("get_schema", C.c_void_p), ("get_next", C.c_void_p), ("get_last_error", C.c_void_p),
                ("release", C.c_void_p), ("private_data", C.c_void_p)]


class DeviceColumn(C.Structure):
    _fields_ = [("type_id", C.c_int32), ("precision", C.c_int32), ("scale", C.c_int32), ("value_width", C.c_int32),
                ("values", C.c_void_p), ("validity", C.c_void_p), ("host_values", C.c_void_p),
                ("host_validity_bytes", C.c_void_p), ("validity_bytes", C.c_void_p), ("bool_bytes", C.c_void_p),
                ("n_dict", C.c_int32), ("pad", C.c_int32)]


class Stats(C.Structure):
    _fields_ = [("kernel_launches", C.c_int64), ("pipeline_launches", C.c_int64), ("pipeline_ms", C.c_double),
                ("pipeline_rows", C.c_int64), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64),
                ("scan_pruned_row_groups", C.c_int64), ("scan_pruned_rows", C.c_int64), ("agg_strategies", C.c_int64),
                ("scan_pruned_pages", C.c_int64), ("scan_page_pruned_rows", C.c_int64), ("sort_rows", C.c_int64),
                ("sort_passes", C.c_int64), ("sort_pass_rows", C.c_int64), ("sort_select_rows", C.c_int64),
                ("join_build_rows", C.c_int64), ("join_probe_rows", C.c_int64), ("join_out_rows", C.c_int64),
                ("agg_range_levels", C.c_int64), ("agg_range_reruns", C.c_int64), ("join_cond_pairs", C.c_int64),
                ("partition_ids_ms", C.c_double), ("partition_place_ms", C.c_double), ("partition_gather_ms", C.c_double),
                ("agg_table_grows", C.c_int64), ("agg_stream_reruns", C.c_int64)]
AGG_DENSE, AGG_TABLE, AGG_STREAM, AGG_MIGRATED = 1, 2, 4, 8  # cb200_stats.agg_strategies bits (CB200_AGG_*)
RANGE_TIGHT, RANGE_TYPE, RANGE_SAFE = 1, 2, 4  # cb200_stats.agg_range_levels bits (CB200_RANGE_*)


EXPORTED = ["cb200_comm_unique_id", "cb200_comm_create", "cb200_comm_destroy", "cb200_comm_rank", "cb200_comm_world", "cb200_nccl_info", "cb200_exchange",
            "cb200_exchange_layout", "cb200_comm_allgather_small", "cb200_plan_stats", "cb200_register_memory_file", "cb200_parquet_describe", "cb200_table_add_column_bytes", "cb200_plan_dict_value", "cb200_plan_partition_starts", "cb200_compile_plan_assume", "cb200_reset_range_profiles", "cb200_version", "cb200_supports", "cb200_create_plan", "cb200_plan_num_columns", "cb200_execute",
            "cb200_release", "cb200_table_create", "cb200_table_add_column", "cb200_plan_bind_table",
            "cb200_table_release", "cb200_execute_device", "cb200_plan_kernel_launches", "cb200_compile_plan",
            "cb200_plan_kernel_source"]


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise ImportError(f"{_LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(make -C datafusion-comet_b200/csrc).  comet_b200 has no CPU fallback.")
        l = C.CDLL(_LIB_PATH)
        l.cb200_version.restype = C.c_char_p
        l.cb200_supports.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(_Error)]
        l.cb200_create_plan.restype = C.c_void_p
        l.cb200_create_plan.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.POINTER(C.c_void_p), C.c_int32,
                                        C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_Error)]
        l.cb200_plan_num_columns.argtypes = [C.c_void_p]
        l.cb200_execute.restype = C.c_int64
        l.cb200_execute.argtypes = [C.c_void_p, C.POINTER(ArrowArray), C.POINTER(ArrowSchema), C.c_int32, C.POINTER(_Error)]
        l.cb200_release.argtypes = [C.c_void_p]
        l.cb200_table_create.restype = C.c_void_p
        l.cb200_table_create.argtypes = [C.c_int64]
        l.cb200_table_add_column.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                             C.c_int64, C.POINTER(C.c_char_p), C.c_int32, C.POINTER(_Error)]
        l.cb200_plan_bind_table.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(_Error)]
        l.cb200_table_release.argtypes = [C.c_void_p]
        l.cb200_execute_device.restype = C.c_int64
        l.cb200_execute_device.argtypes = [C.c_void_p, C.POINTER(DeviceColumn), C.c_int32, C.POINTER(_Error)]
        l.cb200_plan_kernel_launches.restype = C.c_int64
        l.cb200_plan_kernel_launches.argtypes = [C.c_void_p]
        l.cb200_plan_stats.argtypes = [C.c_void_p, C.POINTER(Stats)]
        l.cb200_compile_plan.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.POINTER(_Error)]
        l.cb200_plan_kernel_source.argtypes = [C.c_char_p, C.c_size_t, C.c_int32, C.c_char_p, C.c_size_t, C.POINTER(_Error)]
        _lib = l
    return _lib


def _raise(err):
    cls = Unsupported if err.code == 1 else CometB200Error
    raise cls(err.code, err.error_class.decode(), err.message.decode(errors="replace"))


def version():
    return lib().cb200_version().decode()


def supports(op_bytes):
    err = _Error()
    ok = lib().cb200_supports(op_bytes, len(op_bytes), C.byref(err))
    return bool(ok), err.message.decode(errors="replace")


def compile_plan(op_bytes):
    """NVRTC-compile (no GPU needed) every pipeline kernel of the plan; returns the kernel keys."""
    err = _Error()
    buf = C.create_string_buffer(4096)
    n = lib().cb200_compile_plan(op_bytes, len(op_bytes), buf, 4096, C.byref(err))
    if n < 0:
        _raise(err)
    return [k for k in buf.value.decode().split(",") if k]


def compile_plan_assume(op_bytes, assume_bits, source_index=-1):
    """Pre-compile the range-specialised kernels for decimal columns assumed to satisfy |v| < 2^bits."""
    err = _Error()
    arr = (C.c_int32 * len(assume_bits))(*assume_bits)
    cap = 1 << 20
    buf = C.create_string_buffer(cap)
    lib().cb200_compile_plan_assume.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_char_p, C.c_size_t, C.POINTER(_Error)]
    n = lib().cb200_compile_plan_assume(op_bytes, len(op_bytes), arr, len(assume_bits), source_index, buf, cap, C.byref(err))
    if n < 0:
        _raise(err)
    return buf.value.decode()


_MEMFILES = {}


def register_memory_file(name, buf):
    """Expose a Parquet file image held in host memory as "memory://<name>" (buf: bytes-like / numpy / torch pinned tensor)."""
    import numpy as np
    if buf is None:
        lib().cb200_register_memory_file(name.encode(), None, 0)
        _MEMFILES.pop(name, None)
        return
    if hasattr(buf, "data_ptr"):  # torch tensor (pinned host memory)
        ptr, n = buf.data_ptr(), buf.numel() * buf.element_size()
    else:
        arr = np.frombuffer(buf, dtype=np.uint8) if not isinstance(buf, np.ndarray) else buf
        ptr, n = arr.ctypes.data, arr.nbytes
        buf = arr
    f = lib().cb200_register_memory_file
    f.argtypes = [C.c_char_p, C.c_void_p, C.c_size_t]
    f(name.encode(), ptr, n)
    _MEMFILES[name] = buf  # keep alive
    return "memory://" + name


def parquet_describe(path):
    import json
    err = _Error()
    cap = 1 << 22
    buf = C.create_string_buffer(cap)
    f = lib().cb200_parquet_describe
    f.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t, C.POINTER(_Error)]
    if f(path.encode(), buf, cap, C.byref(err)) < 0:
        _raise(err)
    return json.loads(buf.value.decode())


def reset_range_profiles():
    """Forget the value ranges earlier dense aggregates left for later plans with the same pipeline (cb200_reset_range_profiles)."""
    lib().cb200_reset_range_profiles()


def kernel_source(op_bytes, index=0):
    err = _Error()
    cap = 1 << 20
    buf = C.create_string_buffer(cap)
    n = lib().cb200_plan_kernel_source(op_bytes, len(op_bytes), index, buf, cap, C.byref(err))
    if n < 0:
        _raise(err)
    return buf.value.decode()


class ExchangeStats(C.Structure):
    _fields_ = [("rows_sent", C.c_int64), ("rows_received", C.c_int64), ("bytes_sent", C.c_int64), ("bytes_received", C.c_int64),
                ("payload_ms", C.c_double)]


def exchange_layout(counts, world, me):
    """(total, recv_counts, recv_offsets) of rank `me` from the row-major N x N count matrix (host arithmetic only)."""
    f = lib().cb200_exchange_layout
    f.restype = C.c_int64
    f.argtypes = [C.POINTER(C.c_int64), C.c_int32, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    m = (C.c_int64 * (world * world))(*[int(x) for x in counts])
    rc, ro = (C.c_int64 * world)(), (C.c_int64 * world)()
    total = f(m, world, me, rc, ro)
    return total, list(rc), list(ro)


class Comm:
    """One NCCL communicator per process / GPU, owned by the library (cb200_comm_*).  `bcast(bytes_or_None) -> bytes` is the
    caller's control channel for the 128-byte id (torch.distributed here; the Spark driver in the reference's world)."""

    def __init__(self, rank, world, device, bcast=None):
        l = lib()
        l.cb200_comm_create.restype = C.c_void_p
        l.cb200_comm_create.argtypes = [C.c_char_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_Error)]
        l.cb200_comm_unique_id.argtypes = [C.c_char_p, C.POINTER(_Error)]
        l.cb200_comm_destroy.argtypes = [C.c_void_p]
        err = _Error()
        idb = C.create_string_buffer(128)
        if world > 1:
            if rank == 0 and l.cb200_comm_unique_id(idb, C.byref(err)) != 0:
                _raise(err)
            got = bcast(bytes(idb.raw) if rank == 0 else None)
            idb = C.create_string_buffer(got, 128)
        self.rank, self.world, self.device = rank, world, device
        self.handle = l.cb200_comm_create(idb, rank, world, device, C.byref(err))
        if not self.handle:
            _raise(err)

    def exchange(self, map_plan):
        """Collective: partition r of every rank's last ShuffleWriter batch -> rank r.  Returns (DeviceTable, stats dict)."""
        l = lib()
        l.cb200_exchange.restype = C.c_void_p
        l.cb200_exchange.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(ExchangeStats), C.POINTER(_Error)]
        err, n, st = _Error(), C.c_int64(0), ExchangeStats()
        h = l.cb200_exchange(self.handle, map_plan.handle, C.byref(n), C.byref(st), C.byref(err))
        if not h:
            _raise(err)
        t = DeviceTable.__new__(DeviceTable)
        t.handle, t.n_rows, t._keep = h, n.value, []
        return t, {k: getattr(st, k) for k, _ in ExchangeStats._fields_}

    def allgather_small(self, payload, slot_bytes=1 << 16):
        """Every rank's small bytes payload on every rank (list of bytes, rank order).  slot_bytes must be the same on all ranks."""
        l = lib()
        l.cb200_comm_allgather_small.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.c_int64, C.c_char_p, C.POINTER(C.c_int64), C.POINTER(_Error)]
        if len(payload) + 8 > slot_bytes:
            raise ValueError(f"payload of {len(payload)} bytes does not fit the {slot_bytes}-byte slot (pass a larger slot_bytes on every rank)")
        out = C.create_string_buffer(slot_bytes * self.world)
        sizes = (C.c_int64 * self.world)()
        err = _Error()
        if l.cb200_comm_allgather_small(self.handle, payload, len(payload), slot_bytes, out, sizes, C.byref(err)) != 0:
            _raise(err)
        return [out.raw[r * slot_bytes: r * slot_bytes + sizes[r]] for r in range(self.world)]

    def destroy(self):
        if self.handle:
            lib().cb200_comm_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


def snappy_decompress(comp, uncompressed_len, device=0):
    """One raw Snappy buffer through the scan's device decompressor.  Returns (bytes, path): path 0 = segmented, 1 = serial fallback."""
    f = lib().cb200_snappy_decompress
    f.restype = C.c_int64
    f.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_int32, C.POINTER(C.c_int32), C.POINTER(_Error)]
    out = C.create_string_buffer(max(uncompressed_len, 1))
    path, err = C.c_int32(-1), _Error()
    n = f(bytes(comp), len(comp), out, uncompressed_len, device, C.byref(path), C.byref(err))
    if n < 0:
        _raise(err)
    return out.raw[:uncompressed_len], path.value


def nccl_info():
    f = lib().cb200_nccl_info
    f.restype = C.c_char_p
    return f().decode()


class DeviceTable:
    """Device-resident input columns (torch CUDA tensors or raw pointers) bound to a Scan."""

    def __init__(self, n_rows):
        self.handle = lib().cb200_table_create(n_rows)
        self.n_rows = n_rows
        self._keep = []

    def add(self, dt, values_ptr, value_width, validity_ptr=None, null_count=0, dictionary=None, keep=None):
        from . import proto
        err = _Error()
        if dictionary is not None:
            arr = (C.c_char_p * len(dictionary))(*[d.encode() if isinstance(d, str) else d for d in dictionary])
            nd = len(dictionary)
        else:
            arr, nd = None, 0
        rc = lib().cb200_table_add_column(self.handle, proto.DATA_TYPE_ID[dt.name], dt.precision, dt.scale, value_width,
                                          values_ptr, validity_ptr, null_count, arr, nd, C.byref(err))
        if rc != 0:
            _raise(err)
        self._keep.append(keep)
        return self

    def add_bytes(self, dt, values_ptr, value_width, validity_bytes_ptr=None, dictionary=None, keep=None):
        """Column in the exchange-friendly form: validity (and BOOL values) one byte per row."""
        from . import proto
        err = _Error()
        if dictionary is not None:
            arr = (C.c_char_p * len(dictionary))(*[d.encode() if isinstance(d, str) else d for d in dictionary])
            nd = len(dictionary)
        else:
            arr, nd = None, 0
        f = lib().cb200_table_add_column_bytes
        f.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(C.c_char_p), C.c_int32, C.POINTER(_Error)]
        if f(self.handle, proto.DATA_TYPE_ID[dt.name], dt.precision, dt.scale, value_width, values_ptr, validity_bytes_ptr, arr, nd, C.byref(err)) != 0:
            _raise(err)
        self._keep.append(keep)
        return self

    def release(self):
        if self.handle and lib is not None:
            lib().cb200_table_release(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class Plan:
    """One native plan handle = one Spark task's `CometExecIterator` (CometExecIterator.scala:64)."""

    def __init__(self, op_bytes, inputs=(), config=None, batch_size=8192, device=0, partition=0, partition_count=1):
        from . import proto
        self._lib = lib()
        self.handle = None
        cfg = proto.config_map(config) if config else b""
        n = len(inputs)
        self._streams = (ArrowArrayStream * max(n, 1))()
        ptrs = (C.c_void_p * max(n, 1))()
        self._tables = []
        for i, inp in enumerate(inputs):
            if isinstance(inp, DeviceTable):
                ptrs[i] = None
                self._tables.append((i, inp))
                continue
            if isinstance(inp, pa.Table):
                inp = inp.to_reader()
            elif isinstance(inp, (list, tuple)):
                inp = pa.RecordBatchReader.from_batches(inp[0].schema, inp)
            elif isinstance(inp, pa.RecordBatch):
                inp = pa.RecordBatchReader.from_batches(inp.schema, [inp])
            inp._export_to_c(C.addressof(self._streams[i]))  # ownership moves to native (ffi.md:60-150)
            ptrs[i] = C.addressof(self._streams[i])
        err = _Error()
        self.handle = self._lib.cb200_create_plan(op_bytes, len(op_bytes), cfg or None, len(cfg), ptrs, n, partition,
                                                  partition_count, batch_size, device, C.byref(err))
        if not self.handle:
            _raise(err)
        for i, t in self._tables:
            if self._lib.cb200_plan_bind_table(self.handle, i, t.handle, C.byref(err)) != 0:
                _raise(err)
        self.n_cols = self._lib.cb200_plan_num_columns(self.handle)

    def execute(self):
        """Next output batch as a pyarrow RecordBatch, or None at end of stream (executePlan == -1)."""
        arrays = (ArrowArray * self.n_cols)()
        schemas = (ArrowSchema * self.n_cols)()
        err = _Error()
        rows = self._lib.cb200_execute(self.handle, arrays, schemas, self.n_cols, C.byref(err))
        if rows == -1:
            return None
        if rows < 0:
            _raise(err)
        cols = [pa.Array._import_from_c(C.addressof(arrays[i]), C.addressof(schemas[i])) for i in range(self.n_cols)]
        return pa.RecordBatch.from_arrays(cols, names=[f"col_{i}" for i in range(self.n_cols)])

    def execute_device(self):
        """Next output batch left on the device: (rows, [DeviceColumn...]) or None."""
        cols = (DeviceColumn * self.n_cols)()
        err = _Error()
        rows = self._lib.cb200_execute_device(self.handle, cols, self.n_cols, C.byref(err))
        if rows == -1:
            return None
        if rows < 0:
            _raise(err)
        return rows, cols

    def collect(self):
        batches = []
        while True:
            b = self.execute()
            if b is None:
                break
            batches.append(b)
        if not batches:
            return None
        return pa.Table.from_batches(batches)

    def dict_values(self, col, n):
        f = self._lib.cb200_plan_dict_value
        f.restype = C.c_void_p
        f.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_int32)]
        out = []
        for i in range(n):
            ln = C.c_int32(0)
            ptr = f(self.handle, col, i, C.byref(ln))
            out.append(C.string_at(ptr, ln.value).decode())
        return out

    def partition_starts(self):
        f = self._lib.cb200_plan_partition_starts
        f.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.c_int32]
        n = f(self.handle, None, 0)  # the count first: N + 1 entries for N partitions
        buf = (C.c_int64 * max(n, 1))()
        n = f(self.handle, buf, n)
        return [buf[i] for i in range(n)]

    def stats(self):
        st = Stats()
        self._lib.cb200_plan_stats(self.handle, C.byref(st))
        return {k: getattr(st, k) for k, _ in Stats._fields_}

    @property
    def kernel_launches(self):
        return self._lib.cb200_plan_kernel_launches(self.handle)

    def release(self):
        if self.handle:
            self._lib.cb200_release(self.handle)
            self.handle = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.release()

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass
