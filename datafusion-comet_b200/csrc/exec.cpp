// exec.cpp -- executor: sources, fused pipelines, dense aggregation, Arrow export.
#include "exec.h"

#include "aot_kernels.h"
#include "device/cb_params.h"
#include "ranges.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <functional>
#include <map>
#include <mutex>
#include <set>
#include <sstream>

namespace cb200 {

// error bits raised by kernels (device/cb_kernels.cuh set_err)
enum { ERR_I128_OVERFLOW = 0, ERR_ANSI_OVERFLOW = 1, ERR_ORDER_DEPENDENT = 2, ERR_DIVIDE_BY_ZERO = 3, ERR_ARROW_DIVIDE_BY_ZERO = 4 };

bool trace_on() {
    static int on = -1;
    if (on < 0) { const char* e = getenv("CB200_TRACE"); on = (e && *e && *e != '0') ? 1 : 0; }
    return on == 1;
}
double now_ms() {
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
}
TraceSpan::TraceSpan(const char* n) : name(n), t0(trace_on() ? now_ms() : 0) {}
TraceSpan::~TraceSpan() {
    if (trace_on()) { static const double tz = now_ms(); const double t1 = now_ms(); fprintf(stderr, "[cb200 trace] %-28s %8.3f ms   (ends at +%.3f ms)\n", name, t1 - t0, t1 - tz); }
}

void cuda_check(cudaError_t e, const char* what) {
    if (e != cudaSuccess) throw ExecError(2, "", std::string("CUDA error in ") + what + ": " + cudaGetErrorString(e));
}

// Stream-ordered allocation from the device's default pool (kept warm: cudaFree on a process that holds
// tens of GB costs milliseconds and synchronises the device; cudaFreeAsync does neither).
static thread_local cudaStream_t tl_alloc_stream = nullptr;
void set_alloc_stream(cudaStream_t s) { tl_alloc_stream = s; }

// Large blocks are recycled by the library itself.  A query step allocates and frees the same multi-GB buffers over and over
// (state rows, partition outputs, exchange buffers); the driver's stream-ordered pool serves them from its free list most of the
// time, but when its best-fit search fails it maps fresh memory from the OS, and single cudaMallocAsync calls were measured at
// 400-530 ms (a 90 ms step became 650 ms).  Blocks >= 1 MiB are rounded up to a size class (1/8 octave, <= 12.5 % slack) and kept
// on a per-device free list keyed by class; a block freed on one stream and taken by another is ordered by an event.
namespace {
struct CachedBlock { void* ptr; cudaStream_t stream; cudaEvent_t ev; };
struct BlockCache {
    std::mutex mu;
    std::multimap<size_t, CachedBlock> free_blocks;
    size_t cached_bytes = 0;
};
BlockCache g_block_cache[64];
const size_t BLOCK_CACHE_MIN = 1 << 20;
size_t block_cache_limit() {
    static size_t lim = 0;
    if (!lim) { const char* e = getenv("CB200_BLOCK_CACHE_BYTES"); lim = e && *e ? (size_t)atoll(e) : (size_t)32 << 30; if (!lim) lim = 1; }
    return lim;
}
size_t size_class(size_t n) {
    size_t p2 = (size_t)1 << 20;
    while ((p2 << 1) <= n) p2 <<= 1;
    const size_t step = p2 >> 3;
    return (n + step - 1) / step * step;
}
int current_device() { int d = 0; cudaGetDevice(&d); return d >= 0 && d < 64 ? d : 0; }
// drop every cached block of a device (called when an allocation fails, and by cb200_release_cached_memory)
size_t block_cache_flush(int dev) {
    BlockCache& c = g_block_cache[dev];
    std::multimap<size_t, CachedBlock> take;
    size_t freed = 0;
    {
        std::lock_guard<std::mutex> lk(c.mu);
        take.swap(c.free_blocks);
        freed = c.cached_bytes;
        c.cached_bytes = 0;
    }
    for (auto& kv : take) { cudaEventSynchronize(kv.second.ev); cudaFreeAsync(kv.second.ptr, nullptr); cudaEventDestroy(kv.second.ev); } // the owner stream may be gone by now
    return freed;
}
} // namespace
size_t release_cached_device_memory() { return block_cache_flush(current_device()); }

DeviceBuf::DeviceBuf(size_t n) {
    bytes = (n + 255) / 256 * 256 + 256; // padded: TMA bulk copies round sizes up to 16 B
    stream = tl_alloc_stream;
    if (bytes >= BLOCK_CACHE_MIN) {
        bytes = size_class(bytes);
        BlockCache& c = g_block_cache[current_device()];
        CachedBlock blk{nullptr, nullptr, nullptr};
        {
            std::lock_guard<std::mutex> lk(c.mu);
            auto it = c.free_blocks.find(bytes);
            if (it != c.free_blocks.end()) { blk = it->second; c.free_blocks.erase(it); c.cached_bytes -= bytes; }
        }
        if (blk.ptr) {
            if (blk.stream != stream) cudaStreamWaitEvent(stream, blk.ev, 0); // the previous owner's work on this block is done before ours starts
            cudaEventDestroy(blk.ev);
            ptr = blk.ptr;
            return;
        }
    }
    cudaError_t e = cudaMallocAsync(&ptr, bytes, stream);
    if (e == cudaErrorMemoryAllocation) { // give the cached blocks back and try once more
        cudaGetLastError();
        block_cache_flush(current_device());
        cudaStreamSynchronize(stream);
        e = cudaMallocAsync(&ptr, bytes, stream);
    }
    cuda_check(e, "cudaMallocAsync");
}
DeviceBuf::~DeviceBuf() {
    if (!(owned && ptr)) return;
    if (bytes >= BLOCK_CACHE_MIN && bytes == size_class(bytes)) {
        BlockCache& c = g_block_cache[current_device()];
        cudaEvent_t ev = nullptr;
        if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) == cudaSuccess && cudaEventRecord(ev, stream) == cudaSuccess) {
            std::lock_guard<std::mutex> lk(c.mu);
            if (c.cached_bytes + bytes <= block_cache_limit()) {
                c.free_blocks.insert({bytes, CachedBlock{ptr, stream, ev}});
                c.cached_bytes += bytes;
                return;
            }
        }
        if (ev) cudaEventDestroy(ev);
    }
    cudaFreeAsync(ptr, stream);
}

void ExecContext::collect_timing() {
    if (!ev_pending) return;
    float ms = 0;
    if (cudaEventElapsedTime(&ms, ev0, ev1) == cudaSuccess) { pipeline_ms += ms; pipeline_launches++; }
    ev_pending = false;
}

void ExecContext::check_device_errors() {
    cuda_check(cudaMemcpyAsync(h_err, d_err, sizeof(int), cudaMemcpyDeviceToHost, stream), "error flag copy");
    cuda_check(cudaStreamSynchronize(stream), "stream sync");
    collect_timing();
    int e = *h_err;
    if (!e) return;
    cudaMemsetAsync(d_err, 0, sizeof(int), stream);
    if (e & (1 << ERR_ANSI_OVERFLOW))
        throw ExecError(10, "ARITHMETIC_OVERFLOW", "[ARITHMETIC_OVERFLOW] overflow in ANSI mode");
    if (e & (1 << ERR_DIVIDE_BY_ZERO)) // SparkError::DivideByZero (spark-expr/src/error.rs)
        throw ExecError(10, "DIVIDE_BY_ZERO", "[DIVIDE_BY_ZERO] Division by zero. Use `try_divide` to tolerate divisor being 0 and return NULL instead. "
                                              "If necessary set \"spark.sql.ansi.enabled\" to \"false\" to bypass this error.");
    if (e & (1 << ERR_ARROW_DIVIDE_BY_ZERO)) throw ExecError(11, "", "Arrow error: Divide by zero error"); // arrow-arith checked division in Legacy mode
    if (e & (1 << ERR_I128_OVERFLOW))
        throw ExecError(11, "", "Arrow error: Arithmetic overflow: Overflow happened on decimal arithmetic"); // arrow-arith checked ops
    if (e & (1 << ERR_ORDER_DEPENDENT))
        throw ExecError(12, "", "SUM/AVG overflow here depends on the row order (some orderings of these rows overflow, others do not); "
                                "the reference adds in row order -- the row-ordered fallback is not built yet, so the plan is refused rather than guessed");
    throw ExecError(13, "", "device error flags " + std::to_string(e));
}

// =================================================================================================
// expression helpers
// =================================================================================================
static ExprP clone_expr(const ExprP& e) {
    auto c = std::make_shared<Expr>(*e);
    for (auto& ch : c->children) ch = clone_expr(ch);
    return c;
}
// replace Bound(i) by cur[i]
static ExprP substitute(const ExprP& e, const std::vector<ExprP>& cur) {
    if (e->kind == ExprKind::Bound) {
        if (e->index < 0 || e->index >= (int)cur.size()) throw PlanError("bound reference out of range while fusing");
        return clone_expr(cur[e->index]);
    }
    auto c = std::make_shared<Expr>(*e);
    for (auto& ch : c->children) ch = substitute(ch, cur);
    return c;
}
static void collect_bound(const ExprP& e, std::vector<int>& order, std::set<int>& seen) {
    if (e->kind == ExprKind::Bound) {
        if (!seen.count(e->index)) { seen.insert(e->index); order.push_back(e->index); }
        return;
    }
    for (auto& c : e->children) collect_bound(c, order, seen);
}
static void rewrite_bound(const ExprP& e, const std::map<int, int>& slot_of) {
    if (e->kind == ExprKind::Bound) { e->index = slot_of.at(e->index); return; }
    for (auto& c : e->children) rewrite_bound(c, slot_of);
}

// =================================================================================================
// sources
// =================================================================================================
static Phys phys_of(const DType& t);
static Phys phys_of_type(const DType& t) { return phys_of(t); }
static Phys phys_of(const DType& t) {
    switch (t.id) {
    case TypeId::Bool: return Phys::Bitmap;
    case TypeId::Int8: return Phys::I8;
    case TypeId::Int16: return Phys::I16;
    case TypeId::Int32: case TypeId::Date: return Phys::I32;
    case TypeId::Int64: case TypeId::Timestamp: case TypeId::TimestampNtz: return Phys::I64;
    case TypeId::Float32: return Phys::F32;
    case TypeId::Float64: return Phys::F64;
    case TypeId::Decimal: return Phys::I128;
    default: return Phys::I32;
    }
}

static DType dtype_from_format(const char* f) {
    std::string s = f ? f : "";
    if (s == "b") return mk_type(TypeId::Bool);
    if (s == "c") return mk_type(TypeId::Int8);
    if (s == "s") return mk_type(TypeId::Int16);
    if (s == "i") return mk_type(TypeId::Int32);
    if (s == "l") return mk_type(TypeId::Int64);
    if (s == "f") return mk_type(TypeId::Float32);
    if (s == "g") return mk_type(TypeId::Float64);
    if (s == "u") return mk_type(TypeId::String);
    if (s == "z") return mk_type(TypeId::Binary);
    if (s == "tdD") return mk_type(TypeId::Date);
    if (s.rfind("tsu:", 0) == 0) return mk_type(s.size() > 4 ? TypeId::Timestamp : TypeId::TimestampNtz);
    if (s.rfind("d:", 0) == 0) {
        int p = 0, sc = 0, bits = 128;
        if (sscanf(s.c_str(), "d:%d,%d,%d", &p, &sc, &bits) < 2) throw PlanError("bad decimal format " + s);
        if (bits != 128) throw Unsupported("decimal bit width " + std::to_string(bits));
        return mk_decimal(p, sc);
    }
    throw Unsupported("Arrow format '" + s + "' is outside the GPU hot path");
}

struct SchemaOnlySource : ExecNode { // build-time stand-in: no data
    bool next(Batch&) override { return false; }
};

// ---- Arrow C stream -> device chunks (ScanExec: operators/scan.rs:46-170) -------------------------
struct StreamSource : ExecNode {
    ExecContext* ctx;
    ArrowArrayStream* stream;
    bool schema_checked = false, eof = false;
    std::vector<bool> col_is_dict;
    std::vector<int> dict_index_width;
    std::vector<DictionaryP> dicts; // plan-global dictionary per dict column

    StreamSource(ExecContext* c, ArrowArrayStream* s, const std::vector<DType>& fields) : ctx(c), stream(s) { schema = fields; }
    ~StreamSource() override {
        if (stream && stream->release) stream->release(stream); // ownership was transferred to native (planner.rs:1725-1737)
    }

    void check_schema() {
        ArrowSchema sc;
        memset(&sc, 0, sizeof(sc));
        if (stream->get_schema(stream, &sc) != 0) {
            const char* m = stream->get_last_error ? stream->get_last_error(stream) : nullptr;
            throw ExecError(3, "", std::string("Failed to import ArrowArrayStream schema: ") + (m ? m : "?"));
        }
        if (sc.n_children != (int64_t)schema.size()) {
            int64_t n = sc.n_children;
            if (sc.release) sc.release(&sc);
            throw PlanError("scan declares " + std::to_string(schema.size()) + " fields but the stream has " + std::to_string(n));
        }
        col_is_dict.assign(schema.size(), false);
        dict_index_width.assign(schema.size(), 4);
        dicts.assign(schema.size(), nullptr);
        for (size_t i = 0; i < schema.size(); i++) {
            ArrowSchema* ch = sc.children[i];
            if (ch->dictionary) {
                DType vt = dtype_from_format(ch->dictionary->format);
                DType it = dtype_from_format(ch->format);
                if (!vt.is_string() || !it.is_integer()) throw Unsupported("dictionary column that is not int -> utf8");
                if (!schema[i].is_string()) throw PlanError("scan field " + std::to_string(i) + " is " + schema[i].str() + " but the stream column is a string dictionary");
                col_is_dict[i] = true;
                dict_index_width[i] = it.arrow_width();
                if (it.arrow_width() == 8) throw Unsupported("int64 dictionary indices");
                dicts[i] = std::make_shared<Dictionary>();
            } else {
                DType t = dtype_from_format(ch->format);
                bool ok = t == schema[i] || (t.is_decimal() && schema[i].is_decimal() && t.scale == schema[i].scale) ||
                          (t.id == TypeId::Timestamp && schema[i].id == TypeId::TimestampNtz) || (t.id == TypeId::TimestampNtz && schema[i].id == TypeId::Timestamp);
                if (!ok) throw PlanError("scan field " + std::to_string(i) + " is " + schema[i].str() + " but the stream column is " + t.str());
            }
        }
        if (sc.release) sc.release(&sc);
        schema_checked = true;
    }

    bool next(Batch& out) override {
        if (!schema_checked) check_schema();
        if (eof) return false;
        std::vector<ArrowArray> arrs;
        int64_t total = 0;
        while (total < ctx->chunk_rows) {
            ArrowArray a;
            memset(&a, 0, sizeof(a));
            if (stream->get_next(stream, &a) != 0) {
                const char* m = stream->get_last_error ? stream->get_last_error(stream) : nullptr;
                for (auto& x : arrs) if (x.release) x.release(&x);
                throw ExecError(3, "", std::string("ArrowArrayStream get_next failed: ") + (m ? m : "?"));
            }
            if (!a.release) { eof = true; break; } // end of stream
            if (a.length > 0) { total += a.length; arrs.push_back(a); }
            else a.release(&a);
        }
        if (arrs.empty()) return false;
        try {
            upload(arrs, total, out);
        } catch (...) {
            for (auto& x : arrs) if (x.release) x.release(&x);
            throw;
        }
        cuda_check(cudaStreamSynchronize(ctx->stream), "H2D copies"); // host buffers are released right after
        for (auto& x : arrs) if (x.release) x.release(&x);
        return true;
    }

    // unify a batch dictionary with the plan-global one; returns remap table (empty = identity)
    std::vector<int32_t> unify_dict(size_t col, const ArrowArray* d) {
        Dictionary& g = *dicts[col];
        const int32_t* off = (const int32_t*)d->buffers[1] + d->offset;
        const char* chars = (const char*)d->buffers[2];
        std::vector<int32_t> remap((size_t)d->length);
        bool identity = true;
        for (int64_t k = 0; k < d->length; k++) {
            std::string v(chars + off[k], (size_t)(off[k + 1] - off[k]));
            auto it = std::find(g.values.begin(), g.values.end(), v);
            int32_t code;
            if (it == g.values.end()) { code = (int32_t)g.values.size(); g.values.push_back(v); }
            else code = (int32_t)(it - g.values.begin());
            remap[(size_t)k] = code;
            if (code != k) identity = false;
        }
        if (identity) remap.clear();
        return remap;
    }

    cudaError_t h2d(void* dst, const void* src, size_t n) {
        ctx->h2d_bytes += (int64_t)n;
        return cudaMemcpyAsync(dst, src, n, cudaMemcpyHostToDevice, ctx->stream);
    }

    void upload(std::vector<ArrowArray>& arrs, int64_t total, Batch& out) {
        TraceSpan ts("source.upload");
        out.n_rows = total;
        out.cols.clear();
        out.cols.resize(schema.size());
        cudaStream_t st = ctx->stream;
        for (size_t c = 0; c < schema.size(); c++) {
            Column& col = out.cols[c];
            col.type = schema[c];
            bool any_nulls = false;
            for (auto& a : arrs) {
                ArrowArray* ch = a.children[c];
                if (ch->null_count != 0 && ch->buffers[0]) any_nulls = true;
            }
            if (any_nulls) {
                col.validity = std::make_shared<DeviceBuf>((size_t)(total + 7) / 8 + 8);
                cuda_check(cudaMemsetAsync(col.validity->ptr, 0, col.validity->bytes, st), "memset validity");
            }
            std::vector<DeviceBufP> temps;
            if (col_is_dict[c]) {
                col.is_dict = true;
                col.dict = dicts[c];
                int w = dict_index_width[c];
                bool need_remap = false;
                std::vector<std::vector<int32_t>> remaps;
                for (auto& a : arrs) {
                    remaps.push_back(unify_dict(c, a.children[c]->dictionary));
                    if (!remaps.back().empty()) need_remap = true;
                }
                if (!need_remap) {
                    col.phys = w == 1 ? Phys::I8 : w == 2 ? Phys::I16 : Phys::I32;
                    col.data = std::make_shared<DeviceBuf>((size_t)total * w);
                } else {
                    col.phys = Phys::I32;
                    col.data = std::make_shared<DeviceBuf>((size_t)total * 4);
                }
                int64_t row = 0;
                for (size_t k = 0; k < arrs.size(); k++) {
                    ArrowArray* ch = arrs[k].children[c];
                    const char* src = (const char*)ch->buffers[1] + ch->offset * w;
                    if (!need_remap) {
                        cuda_check(h2d((char*)col.data->ptr + row * w, src, (size_t)ch->length * w), "H2D dict codes");
                    } else {
                        auto tmp = std::make_shared<DeviceBuf>((size_t)ch->length * w);
                        temps.push_back(tmp);
                        cuda_check(h2d(tmp->ptr, src, (size_t)ch->length * w), "H2D dict codes");
                        std::vector<int32_t> table = remaps[k];
                        if (table.empty()) { table.resize((size_t)ch->dictionary->length); for (size_t i = 0; i < table.size(); i++) table[i] = (int32_t)i; }
                        auto dt = std::make_shared<DeviceBuf>(table.size() * 4 + 4);
                        temps.push_back(dt);
                        cuda_check(h2d(dt->ptr, table.data(), table.size() * 4), "H2D remap table");
                        cuda_check(cudaStreamSynchronize(st), "remap table copy"); // table is a stack temporary
                        launch_remap_codes(tmp->ptr, w, ch->length, (const int*)dt->ptr, (int)table.size(), (int*)col.data->ptr + row, st);
                    }
                    row += ch->length;
                }
            } else if (schema[c].is_string()) {
                // plain Utf8: ship offsets + chars; key columns are dictionary-encoded on the device
                int64_t total_chars = 0;
                for (auto& a : arrs) {
                    ArrowArray* ch = a.children[c];
                    const int32_t* off = (const int32_t*)ch->buffers[1] + ch->offset;
                    total_chars += off[ch->length] - off[0];
                }
                if (total_chars > INT32_MAX) throw Unsupported("more than 2 GiB of string data in one chunk");
                col.offsets = std::make_shared<DeviceBuf>((size_t)(total + 1) * 4);
                col.chars = std::make_shared<DeviceBuf>((size_t)total_chars + 16);
                std::vector<int32_t> offs((size_t)total + 1);
                int64_t row = 0;
                int32_t base = 0;
                for (auto& a : arrs) {
                    ArrowArray* ch = a.children[c];
                    const int32_t* off = (const int32_t*)ch->buffers[1] + ch->offset;
                    for (int64_t i = 0; i < ch->length; i++) offs[(size_t)(row + i)] = base + (off[i] - off[0]);
                    int32_t nchars = off[ch->length] - off[0];
                    if (nchars) cuda_check(h2d((char*)col.chars->ptr + base, (const char*)ch->buffers[2] + off[0], (size_t)nchars), "H2D chars");
                    base += nchars;
                    row += ch->length;
                }
                offs[(size_t)total] = base;
                cuda_check(h2d(col.offsets->ptr, offs.data(), offs.size() * 4), "H2D offsets");
                cuda_check(cudaStreamSynchronize(st), "offsets copy");
                col.phys = Phys::I32;
            } else {
                col.phys = phys_of(schema[c]);
                int w = schema[c].arrow_width();
                if (w == 0) { // boolean values: bitmap
                    col.data = std::make_shared<DeviceBuf>((size_t)(total + 7) / 8 + 8);
                    cuda_check(cudaMemsetAsync(col.data->ptr, 0, col.data->bytes, st), "memset bool");
                    int64_t row = 0;
                    for (auto& a : arrs) {
                        ArrowArray* ch = a.children[c];
                        append_bits((uint32_t*)col.data->ptr, row, (const uint8_t*)ch->buffers[1], ch->offset, ch->length, temps);
                        row += ch->length;
                    }
                } else {
                    col.data = std::make_shared<DeviceBuf>((size_t)total * w);
                    int64_t row = 0;
                    for (auto& a : arrs) {
                        ArrowArray* ch = a.children[c];
                        cuda_check(h2d((char*)col.data->ptr + row * w, (const char*)ch->buffers[1] + ch->offset * w, (size_t)ch->length * w), "H2D column");
                        row += ch->length;
                    }
                }
            }
            if (any_nulls) {
                int64_t row = 0, nulls = 0;
                for (auto& a : arrs) {
                    ArrowArray* ch = a.children[c];
                    bool has = ch->null_count != 0 && ch->buffers[0];
                    append_bits((uint32_t*)col.validity->ptr, row, has ? (const uint8_t*)ch->buffers[0] : nullptr, ch->offset, ch->length, temps);
                    nulls += has ? (ch->null_count < 0 ? 1 : ch->null_count) : 0;
                    row += ch->length;
                }
                col.null_count = nulls;
            }
            if (!temps.empty()) cuda_check(cudaStreamSynchronize(st), "temp buffers");
        }
    }

    // append n bits of a host bitmap (nullptr = ones) at dst bit offset `row`
    void append_bits(uint32_t* dst, int64_t row, const uint8_t* src, int64_t src_off, int64_t n, std::vector<DeviceBufP>& temps) {
        if (n <= 0) return;
        if (src && (row & 7) == 0 && (src_off & 7) == 0 && ((n & 7) == 0)) {
            cuda_check(h2d((char*)dst + (row >> 3), src + (src_off >> 3), (size_t)(n >> 3)), "H2D bitmap");
            return;
        }
        const uint8_t* dsrc = nullptr;
        int64_t doff = 0;
        if (src) {
            int64_t b0 = src_off >> 3, b1 = (src_off + n + 7) >> 3;
            auto tmp = std::make_shared<DeviceBuf>((size_t)(b1 - b0) + 8);
            temps.push_back(tmp);
            cuda_check(h2d(tmp->ptr, src + b0, (size_t)(b1 - b0)), "H2D bitmap");
            dsrc = (const uint8_t*)tmp->ptr;
            doff = src_off & 7;
        }
        launch_bitmap_append(dst, row, dsrc, doff, n, ctx->stream);
    }
};

// ---- caller-owned device-resident table -------------------------------------------------------------
struct TableSource : ExecNode {
    std::shared_ptr<DeviceTable> table;
    ExecContext* ctx = nullptr;
    bool done = false;
    TableSource(std::shared_ptr<DeviceTable> t, const std::vector<DType>& fields, ExecContext* c) : table(std::move(t)), ctx(c) {
        schema = fields;
        if (table->cols.size() != fields.size()) throw PlanError("bound device table has " + std::to_string(table->cols.size()) + " columns, scan declares " + std::to_string(fields.size()));
    }
    // The table is handed out in slices of spark.comet.b200.chunkRows rows (a multiple of 1024, so every slice starts on the byte /
    // tile boundaries the kernels assume): a consumer's per-batch state -- hash-table headroom for "every row a new group" -- is
    // bounded by the chunk, not by the table.
    int64_t pos = 0;
    bool packed = false;
    int64_t rows_hint() const override { return table->n_rows - pos; }
    bool next(Batch& out) override {
        if (done) return false;
        if (table->needs_packing && !packed) { // byte-per-row validity / booleans (received from an exchange) -> Arrow bitmaps, once
            size_t n = (size_t)table->n_rows;
            for (auto& c : table->cols) {
                if (c.valid_bytes && !c.validity) {
                    c.validity = std::make_shared<DeviceBuf>((n + 31) / 32 * 4 + 8);
                    launch_bytes_to_bitmap((const unsigned char*)c.valid_bytes->ptr, table->n_rows, (uint32_t*)c.validity->ptr, ctx->stream);
                    ctx->kernel_launches++;
                }
                if (c.bool_bytes && !c.data) {
                    c.data = std::make_shared<DeviceBuf>((n + 31) / 32 * 4 + 8);
                    launch_bytes_to_bitmap((const unsigned char*)c.bool_bytes->ptr, table->n_rows, (uint32_t*)c.data->ptr, ctx->stream);
                    ctx->kernel_launches++;
                }
            }
            packed = true;
        }
        const int64_t chunk = std::max<int64_t>(1024, ctx->chunk_rows / 1024 * 1024);
        const int64_t r0 = pos, r1 = std::min(table->n_rows, pos + chunk);
        pos = r1;
        if (pos >= table->n_rows) done = true;
        out.n_rows = r1 - r0;
        out.cols = table->cols;
        if (r0 > 0 || r1 < table->n_rows) {
            for (auto& c : out.cols) {
                auto slice = [&](DeviceBufP& b, size_t num, size_t den) { // element = num / den bytes
                    if (!b) return;
                    auto v = std::make_shared<DeviceBuf>((char*)b->ptr + (size_t)r0 * num / den, (size_t)(r1 - r0) * num / den + 1);
                    v->owner = b;
                    b = v;
                };
                const int w = phys_bytes(c.is_dict && c.phys == Phys::I32 ? Phys::Dict32 : c.phys);
                if (w == 0) slice(c.data, 1, 8);
                else slice(c.data, (size_t)w, 1);
                slice(c.validity, 1, 8);
                slice(c.valid_bytes, 1, 1);
                slice(c.bool_bytes, 1, 1);
                if (c.null_count > 0) c.null_count = -1;
            }
        }
        return out.n_rows > 0;
    }
};


// =================================================================================================
// fused pipeline nodes
// =================================================================================================
struct FusedBase : ExecNode {
    ExecContext* ctx;
    ExecNodeP child;
    std::vector<ExprP> predicates;   // over child columns (Bound.index = child column)
    std::vector<int> used_cols;      // child columns staged, in slot order
    std::map<int, int> slot_of;

    // build the staged-column list for one batch signature
    std::vector<SourceCol> stage_cols(const Batch* b) const { return stage_cols_of(b, used_cols); }
    std::vector<SourceCol> stage_cols_of(const Batch* b, const std::vector<int>& which) const {
        std::vector<SourceCol> cols;
        for (int ci : which) {
            SourceCol sc;
            sc.src_index = ci;
            sc.type = child->schema[ci];
            if (b) {
                const Column& c = b->cols[ci];
                sc.phys = c.phys;
                sc.has_validity = c.validity != nullptr;
                if (c.is_dict) sc.phys = c.phys == Phys::I8 ? Phys::I8 : c.phys == Phys::I16 ? Phys::I16 : Phys::Dict32;
            } else {
                sc.phys = sc.type.is_string() ? Phys::Dict32 : phys_of(sc.type);
                sc.has_validity = false;
            }
            cols.push_back(sc);
        }
        return cols;
    }
    void assign_slots(const std::vector<ExprP>& roots) {
        std::set<int> seen;
        for (auto& e : roots) collect_bound(e, used_cols, seen);
        for (size_t i = 0; i < used_cols.size(); i++) slot_of[used_cols[i]] = (int)i;
    }
    static std::vector<ExprP> to_slots(const std::vector<ExprP>& es, const std::map<int, int>& slot_of) {
        std::vector<ExprP> out;
        for (auto& e : es) {
            ExprP c = clone_expr(e);
            rewrite_bound(c, slot_of);
            out.push_back(c);
        }
        return out;
    }
    void fill_inputs(cb::PipeParams& p, const Batch& b, int tile, int64_t row0 = 0, int64_t row1 = -1) const { fill_inputs_of(p, b, used_cols, tile, row0, row1); }
    void fill_inputs_of(cb::PipeParams& p, const Batch& b, const std::vector<int>& which, int tile, int64_t row0 = 0, int64_t row1 = -1) const {
        memset(&p, 0, sizeof(p));
        if (row1 < 0) row1 = b.n_rows;
        if (row0 & 1023) throw ExecError(15, "", "internal: launch range must start on a 1024-row boundary");
        for (size_t i = 0; i < which.size(); i++) {
            const Column& c = b.cols[which[i]];
            if (!c.data) throw Unsupported("column " + std::to_string(which[i]) + " (" + c.type.str() + ") has no fixed-width device representation");
            int w = phys_bytes(c.is_dict && c.phys == Phys::I32 ? Phys::Dict32 : c.phys);
            p.col[i] = (const cb::u8*)c.data->ptr + (w == 0 ? row0 / 8 : row0 * w);
            p.val[i] = c.validity ? (const cb::u8*)c.validity->ptr + row0 / 8 : nullptr;
        }
        p.n_rows = row1 - row0;
        p.n_tiles = (int)((p.n_rows + tile - 1) / tile);
        p.err = ctx->d_err;
    }
    void launch(cudaKernel_t k, dim3 grid, dim3 block, size_t smem, void* params) {
        cuda_check(cudaFuncSetAttribute((const void*)k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute(smem)");
        void* args[] = {params};
        if (ctx->ev_pending) { cuda_check(cudaStreamSynchronize(ctx->stream), "stream sync"); ctx->collect_timing(); }
        cuda_check(cudaEventRecord(ctx->ev0, ctx->stream), "event record");
        cuda_check(cudaLaunchKernel((const void*)k, grid, block, args, smem, ctx->stream), "kernel launch");
        cuda_check(cudaEventRecord(ctx->ev1, ctx->stream), "event record");
        ctx->ev_pending = true;
        ctx->kernel_launches++;
    }
};

static const size_t SMEM_BUDGET = 220 * 1024;

// ---- filter + project -> compacted batch ----------------------------------------------------------------
struct SelectNode : FusedBase {
    std::vector<ExprP> outputs;
    DeviceBufP sel_off, sel_chunk, counters; // reused across batches
    std::vector<int> pred_cols;              // child columns the predicates read (pass 1 stages only these)
    std::map<int, int> pred_slot_of;
    std::vector<int> out_cols_used;          // child columns the projections read (all a masked pass 2 stages)
    std::map<int, int> out_slot_of;
    DeviceBufP sel_mask;                     // keep bit per row, pass 1 -> pass 2

    void assign_pred_slots() {
        std::set<int> seen;
        for (auto& e : predicates) collect_bound(e, pred_cols, seen);
        for (size_t i = 0; i < pred_cols.size(); i++) pred_slot_of[pred_cols[i]] = (int)i;
        std::set<int> seen2;
        for (auto& e : outputs) collect_bound(e, out_cols_used, seen2);
        for (size_t i = 0; i < out_cols_used.size(); i++) out_slot_of[out_cols_used[i]] = (int)i;
    }
    // With predicates, pass 2 takes pass 1's keep bits instead of staging and evaluating the predicate columns a second time
    // (Config 1: 4 of 27.7 bytes per row).  Needs at least one projected column to stage.
    bool masked() const { return !predicates.empty() && !out_cols_used.empty(); }
    static int stage_bytes_for(const PipelineSpec& s) {
        int sb = 0;
        for (auto& c : s.cols) {
            int w = phys_bytes(c.phys);
            sb += ((w == 0 ? s.tile / 8 : s.tile * w) + 127) / 128 * 128;
            if (c.has_validity) sb += (s.tile / 8 + 127) / 128 * 128;
        }
        return sb;
    }
    static int stages_for(const PipelineSpec& s) {
        const int sb = stage_bytes_for(s);
        return (int)std::max<size_t>(2, std::min<size_t>(16, (SMEM_BUDGET - 1024) / (size_t)std::max(sb, 1)));
    }
    PipelineSpec make_spec(const Batch* b) const {
        PipelineSpec s;
        if (masked()) {
            s.cols = stage_cols_of(b, out_cols_used);
            s.outputs = to_slots(outputs, out_slot_of);
            s.masked = true;
        } else {
            s.cols = stage_cols(b);
            s.predicates = to_slots(predicates, slot_of);
            s.outputs = to_slots(outputs, slot_of);
        }
        s.sink = SinkKind::Select;
        s.threads = 512; // 16 consumer warps: with 8 both passes were issue / latency bound (ncu: 14 % achieved occupancy, pass 1 at 3.5 TB/s)
        s.tile = 1024;
        s.stages = stages_for(s);
        return s;
    }
    // pass 1: the predicates alone over the columns they read; same tile / warp geometry as pass 2
    PipelineSpec make_count_spec(const Batch* b) const {
        PipelineSpec s;
        s.cols = stage_cols_of(b, pred_cols);
        s.predicates = to_slots(predicates, pred_slot_of);
        s.sink = SinkKind::Count;
        s.threads = 512;
        s.ltile = 1024;
        for (int tile : {4096, 2048, 1024}) { // the widest stage that still leaves a 3-deep ring (wide predicate columns: decimals)
            s.tile = tile;
            if (stage_bytes_for(s) * 3 + 1024 <= (int)SMEM_BUDGET) break;
        }
        s.stages = stages_for(s);
        return s;
    }

    bool next(Batch& out) override {
        Batch in;
        while (child->next(in)) {
            if (in.n_rows == 0) continue;
            run(in, out);
            return true; // a batch with zero kept rows is still a (possibly empty) batch
        }
        return false;
    }

    void run(const Batch& in, Batch& out) {
        if (in.n_rows >= ((int64_t)1 << 32) - 8192) throw Unsupported("filter/projection over more than 2^32 rows per batch (lower spark.comet.b200.chunkRows)");
        PipelineSpec spec = make_spec(&in);
        GeneratedKernel g = generate_pipeline(spec);
        auto mod = jit_get(g, true);
        ctx->last_kernel_key = g.key;
        cb::PipeParams p;
        if (masked()) fill_inputs_of(p, in, out_cols_used, g.tile);
        else fill_inputs(p, in, g.tile);
        out.cols.clear();
        out.cols.resize(g.out_cols.size());
        cudaStream_t st = ctx->stream;
        for (size_t i = 0; i < g.out_cols.size(); i++) {
            Column& c = out.cols[i];
            c.type = g.out_cols[i].type;
            c.phys = c.type.id == TypeId::Bool ? Phys::I8 : phys_of(c.type);
            if (c.type.is_string()) { // dictionary codes pass through; the dictionary is the source column's
                const Column& src = in.cols.at((size_t)outputs[i]->index);
                if (!src.is_dict) throw Unsupported("plain Utf8 columns through a fused filter/projection (dictionary-encoded strings only)");
                c.phys = Phys::I32;
                c.is_dict = true;
                c.dict = src.dict;
            }
            c.data = std::make_shared<DeviceBuf>((size_t)in.n_rows * g.out_bytes[i]);
            p.out[i] = (cb::u8*)c.data->ptr;
            if (g.out_cols[i].nullable) {
                c.validity = std::make_shared<DeviceBuf>((size_t)(in.n_rows + 31) / 32 * 4 + 8);
                cuda_check(cudaMemsetAsync(c.validity->ptr, 0, c.validity->bytes, st), "memset out validity");
                p.out_valid[i] = (cb::u32*)c.validity->ptr;
                c.null_count = -1;
            }
        }
        const int grid = std::min(ctx->num_sms, p.n_tiles);
        int64_t kept = in.n_rows;
        int64_t* h_kept = nullptr;
        if (!predicates.empty()) {
            // pass 1: kept rows per (tile, warp), then their exclusive prefix sum = where pass 2 writes
            GeneratedKernel cg = generate_pipeline(make_count_spec(&in));
            auto cmod = jit_get(cg, true);
            cb::PipeParams cp;
            fill_inputs_of(cp, in, pred_cols, cg.tile);
            const size_t m = (size_t)p.n_tiles * (size_t)(g.threads / 32);
            const size_t n_chunks = (m + CB_SCAN_CHUNK - 1) / CB_SCAN_CHUNK;
            if (!sel_off || sel_off->bytes < m * 4) sel_off = std::make_shared<DeviceBuf>(m * 4 + m / 2);
            if (!sel_chunk || sel_chunk->bytes < (n_chunks + 1) * 4) sel_chunk = std::make_shared<DeviceBuf>((n_chunks + 1) * 4 + n_chunks * 2);
            if (!counters) counters = std::make_shared<DeviceBuf>(64);
            cp.sel_off = (cb::u32*)sel_off->ptr;
            if (masked()) {
                const size_t words = (size_t)p.n_tiles * (size_t)g.tile / 32 + 64;
                if (!sel_mask || sel_mask->bytes < words * 4) sel_mask = std::make_shared<DeviceBuf>(words * 4 + words);
                cp.sel_mask = (cb::u32*)sel_mask->ptr;
                p.sel_mask = cp.sel_mask;
            }
            launch(cmod->kernel(cg.entry), dim3(std::min(ctx->num_sms, cp.n_tiles)), dim3(cg.threads + 32), cg.dyn_smem(0), &cp);
            launch_scan_u32((unsigned*)sel_off->ptr, (long long)m, CB_SCAN_CHUNK, (unsigned*)sel_chunk->ptr, (long long*)counters->ptr, st);
            ctx->kernel_launches += 2;
            p.sel_off = (cb::u32*)sel_off->ptr;
            p.sel_chunk = (cb::u32*)sel_chunk->ptr;
            h_kept = (int64_t*)ctx->h_err + 1; // pinned scratch next to the error flag
            cuda_check(cudaMemcpyAsync(h_kept, counters->ptr, 8, cudaMemcpyDeviceToHost, st), "read kept count"); ctx->d2h_bytes += (int64_t)(8);
        }
        launch(mod->kernel(g.entry), dim3(grid), dim3(g.threads + 32), g.dyn_smem(0), &p);
        ctx->pipeline_rows += in.n_rows;
        ctx->check_device_errors(); // also synchronises
        if (h_kept) kept = *h_kept;
        out.n_rows = kept;
        // boolean outputs were written one byte per row; repack lazily at export
    }
};

// build-time only (cb200_compile_plan_assume): value-range assumptions per source column, so the specialised
// kernels of known workloads can be compiled ahead of time
std::vector<int> g_build_assume;

// value ranges seen by earlier plans, per pipeline signature (see AggNode::consume)
static std::mutex g_profile_mu;
static std::map<std::string, std::vector<int>> g_range_profile;

// ---- dense / ungrouped aggregation --------------------------------------------------------------------
struct AggNode : FusedBase {
    std::vector<ExprP> keys;          // over child columns; each must be a plain column reference
    std::vector<AggExpr> aggs;        // children/filter over child columns (Partial)
    std::vector<std::vector<int>> state_cols; // Final: child column index of each state column
    AggMode mode = AggMode::Partial;
    bool ungrouped = false;
    bool emitted = false;
    std::vector<Batch> outq;          // output batches (more than one only after a dense -> hash migration)
    size_t outq_pos = 0;

    // running state
    std::vector<int> cards;                       // current cardinality per key (incl. null slot)
    std::vector<bool> key_has_null;
    std::vector<DictionaryP> key_dicts;           // strings per key (dict columns); empty for bool keys
    DeviceBufP totals, spill, partials;
    int totals_groups = 0, n_words = 0;
    std::vector<int> word_kinds;
    bool have_totals = false;
    GeneratedKernel last_gen;
    std::shared_ptr<CompiledModule> last_mod;
    // device string dictionaries for plain Utf8 keys
    struct DevDict { StringDictDev d; std::vector<DeviceBufP> bufs; DeviceBufP row_slot; int host_known = 0; };
    std::vector<std::shared_ptr<DevDict>> dev_dicts;

    // ---- hash aggregation state ---------------------------------------------------------------------------
    bool hash_mode = false, strategy_decided = false;
    // Partial + hash over clustered keys: one state row per run of equal adjacent keys, no key table (device/cb_kernels.cuh CB_STREAM)
    bool stream_mode = false, stream_decided = false;
    double stream_ratio = 1.0;         // state rows per input row seen so far in stream mode
    DeviceBufP hkeys, hkey_of_gid, htotals, hflags;
    int64_t hcap = 0, max_groups = 0;
    int key_words = 1;                 // 64-bit words per packed group key (hkey_of_gid stride)
    int hash_threads = 512;            // consumer threads of the hash-aggregate kernel (spark.comet.b200.hashThreads)
    static constexpr int DENSE_MAX_GROUPS = 64;

    // ---- range assumptions (see ranges.h) ----------------------------------------------------------------
    enum Level { SAFE = 0, TYPE = 1, TIGHT = 2 };
    std::vector<int> observed_bits; // per child column: max bit length of (v ^ sign) over every valid row scanned so far (-1: none)
    int64_t rows_scanned = 0;
    DeviceBufP vmask;

    static int type_bits(const DType& t) { return r_bitlen(r_prec_max(t.precision)); }
    int assume_for(int child_col, Level lv) const {
        const DType& t = child->schema[(size_t)child_col];
        if (!t.is_decimal() || lv == SAFE || mode != AggMode::Partial) return 0;
        int k = type_bits(t);
        if (!ctx && (size_t)child_col < g_build_assume.size() && g_build_assume[(size_t)child_col] > 0) k = std::min(k, g_build_assume[(size_t)child_col]);
        if (lv == TIGHT && !observed_bits.empty() && observed_bits[(size_t)child_col] >= 0) k = std::min(k, observed_bits[(size_t)child_col] + 2);
        return std::min(k, 126);
    }

    PipelineSpec make_spec(const Batch* b, int n_groups, Level lv = TYPE) const {
        PipelineSpec s;
        s.cols = stage_cols(b);
        for (auto& c : s.cols) c.assume_bits = assume_for(c.src_index, lv);
        s.predicates = to_slots(predicates, slot_of);
        s.sink = SinkKind::Agg;
        s.mode = mode;
        s.ungrouped = ungrouped;
        s.hash = hash_mode;
        s.keys = to_slots(keys, slot_of);
        for (size_t k = 0; k < keys.size(); k++) s.key_nullable.push_back(b ? key_has_null[k] : false);
        for (auto& a : aggs) {
            AggExpr c = a;
            if (mode == AggMode::Partial) {
                c.children = to_slots(a.children, slot_of);
                if (a.filter) c.filter = to_slots({a.filter}, slot_of)[0];
            }
            s.aggs.push_back(c);
        }
        for (auto& sc : state_cols) {
            std::vector<int> v;
            for (int ci : sc) v.push_back(slot_of.at(ci));
            s.state_slots.push_back(v);
        }
        s.threads = 256;
        s.tile = 512;
        s.stages = 3;
        if (hash_mode) {
            // every row is a chain of dependent L2/HBM round trips (slot probe, then atomics that return a value): the kernel is
            // latency-bound and wants rows in flight, not registers -- 16+ consumer warps per SM instead of 8 (measured on Config 4:
            // 21.8 ms at 256 threads, 15.6 ms at 512)
            const int ht = ctx ? ctx->hash_threads : hash_threads;
            s.threads = ht;
            s.tile = 2 * ht;
            s.stream = stream_mode;
        }
        // first pass to learn the accumulator footprint, then size the ring to the remaining smem
        GeneratedKernel probe = generate_pipeline(s);
        size_t acc = (!ungrouped && !hash_mode) ? (size_t)std::max(n_groups, 1) * probe.n_words * s.threads * 8 : 0;
        while (acc + 2 * (size_t)probe.stage_bytes + 1024 > SMEM_BUDGET && s.threads > 32) {
            s.threads /= 2; // shrink the thread-private accumulator file (wide Final-mode merges are tiny inputs)
            acc /= 2;
        }
        if (acc + 2 * (size_t)probe.stage_bytes + 1024 > SMEM_BUDGET)
            throw Unsupported("too many groups x aggregates for the thread-private accumulators of the dense path");
        s.stages = (int)std::max<size_t>(2, std::min<size_t>(6, (SMEM_BUDGET - 1024 - acc) / (size_t)probe.stage_bytes));
        return s;
    }

    // make key column k of batch `b` a code column; returns cardinality (without null slot)
    int prepare_key(Batch& b, size_t k) {
        int ci = keys[k]->index;
        Column& c = b.cols[ci];
        if (c.type.id == TypeId::Bool) return 2;
        if (!c.type.is_string()) return -1; // integer / date / decimal keys: hash aggregation
        if (c.is_dict) {
            key_dicts[k] = c.dict;
            return (int)c.dict->values.size();
        }
        // plain Utf8 -> device dictionary builder
        if (!dev_dicts[k]) {
            auto dd = std::make_shared<DevDict>();
            const int64_t cap = 1 << 16;
            const int max_codes = 4096;
            const int64_t bytes_cap = 1 << 20;
            auto alloc = [&](size_t n) { auto bfr = std::make_shared<DeviceBuf>(n); cuda_check(cudaMemsetAsync(bfr->ptr, 0, bfr->bytes, ctx->stream), "memset dict"); dd->bufs.push_back(bfr); return bfr->ptr; };
            dd->d.tags = (unsigned long long*)alloc((size_t)cap * 8);
            dd->d.slot_code = (int*)alloc((size_t)cap * 4);
            dd->d.capacity = cap;
            dd->d.n_codes = (int*)alloc(64);
            dd->d.bytes_used = (unsigned long long*)((char*)dd->d.n_codes + 16);
            dd->d.err = (int*)((char*)dd->d.n_codes + 32);
            dd->d.max_codes = max_codes;
            dd->d.code_off = (long long*)alloc((size_t)max_codes * 8);
            dd->d.code_len = (int*)alloc((size_t)max_codes * 4);
            dd->d.bytes = (unsigned char*)alloc((size_t)bytes_cap);
            dd->d.bytes_cap = bytes_cap;
            dev_dicts[k] = dd;
            key_dicts[k] = std::make_shared<Dictionary>();
        }
        DevDict& dd = *dev_dicts[k];
        if (!c.offsets || !c.chars) throw Unsupported("string key column without offsets/chars buffers");
        auto row_slot = std::make_shared<DeviceBuf>((size_t)b.n_rows * 4);
        auto codes = std::make_shared<DeviceBuf>((size_t)b.n_rows * 4);
        launch_dict_encode(dd.d, (const int*)c.offsets->ptr, (const unsigned char*)c.chars->ptr, c.validity ? (const unsigned char*)c.validity->ptr : nullptr,
                           b.n_rows, (int*)row_slot->ptr, (int*)codes->ptr, ctx->stream);
        ctx->kernel_launches += 2;
        int hdr[12];
        cuda_check(cudaMemcpyAsync(hdr, dd.d.n_codes, sizeof(hdr), cudaMemcpyDeviceToHost, ctx->stream), "dict header");
        cuda_check(cudaStreamSynchronize(ctx->stream), "dict encode");
        int n_codes = hdr[0], derr = hdr[8];
        if (derr & CB_DICT_FULL) throw Unsupported("plain Utf8 group key with more distinct values than the device dictionary holds (dictionary-encode the column)");
        if (derr & CB_DICT_COLLISION) throw ExecError(14, "", "64-bit hash collision between distinct group key strings");
        // fetch newly added dictionary strings (metadata-sized)
        if (n_codes > dd.host_known) {
            std::vector<long long> off((size_t)n_codes);
            std::vector<int> len((size_t)n_codes);
            cuda_check(cudaMemcpy(off.data(), dd.d.code_off, (size_t)n_codes * 8, cudaMemcpyDeviceToHost), "dict offsets");
            cuda_check(cudaMemcpy(len.data(), dd.d.code_len, (size_t)n_codes * 4, cudaMemcpyDeviceToHost), "dict lengths");
            for (int i = dd.host_known; i < n_codes; i++) {
                std::string s((size_t)len[(size_t)i], '\0');
                if (len[(size_t)i]) cuda_check(cudaMemcpy(&s[0], dd.d.bytes + off[(size_t)i], (size_t)len[(size_t)i], cudaMemcpyDeviceToHost), "dict bytes");
                key_dicts[k]->values.push_back(s);
            }
            dd.host_known = n_codes;
        }
        c.data = codes;
        c.phys = Phys::I32;
        c.is_dict = true;
        c.dict = key_dicts[k];
        return n_codes;
    }

    void regroup(const std::vector<int>& new_cards) { // cardinalities grew: move totals to the new mixed-radix layout
        int old_groups = totals_groups, new_groups = 1;
        for (int c : new_cards) new_groups *= c;
        std::vector<uint64_t> oldt((size_t)old_groups * n_words * 2), newt((size_t)new_groups * n_words * 2);
        cuda_check(cudaMemcpy(oldt.data(), totals->ptr, oldt.size() * 8, cudaMemcpyDeviceToHost), "regroup D2H");
        for (int g = 0; g < new_groups; g++)
            for (int w = 0; w < n_words; w++) {
                uint64_t id = word_kinds[(size_t)w] == W_MIN ? 0x7fffffffffffffffull : word_kinds[(size_t)w] == W_MAX ? 0x8000000000000000ull : 0;
                newt[((size_t)g * n_words + w) * 2] = id;
                newt[((size_t)g * n_words + w) * 2 + 1] = 0;
            }
        for (int g = 0; g < old_groups; g++) {
            int rem = g, ng = 0, mul = 1;
            std::vector<int> code(cards.size());
            for (int k = (int)cards.size() - 1; k >= 0; k--) { code[(size_t)k] = rem % cards[(size_t)k]; rem /= cards[(size_t)k]; }
            for (int k = (int)cards.size() - 1; k >= 0; k--) {
                int cd = code[(size_t)k];
                // the null slot is always the last one of its key
                if (key_has_null_prev[(size_t)k] && cd == cards[(size_t)k] - 1) cd = new_cards[(size_t)k] - 1;
                ng += cd * mul;
                mul *= new_cards[(size_t)k];
            }
            memcpy(&newt[(size_t)ng * n_words * 2], &oldt[(size_t)g * n_words * 2], (size_t)n_words * 16);
        }
        totals = std::make_shared<DeviceBuf>(newt.size() * 8);
        cuda_check(cudaMemcpyAsync(totals->ptr, newt.data(), newt.size() * 8, cudaMemcpyHostToDevice, ctx->stream), "regroup H2D");
        cuda_check(cudaStreamSynchronize(ctx->stream), "regroup sync");
        totals_groups = new_groups;
    }
    std::vector<bool> key_has_null_prev;

    void consume(Batch& b) {
        std::vector<int> nc(keys.size());
        std::vector<bool> hn(keys.size());
        for (size_t k = 0; k < keys.size(); k++) {
            int card = prepare_key(b, k);
            const Column& c = b.cols[keys[k]->index];
            hn[k] = key_has_null[k] || c.validity != nullptr;
            nc[k] = card < 0 ? -1 : std::max(card, 1) + (hn[k] ? 1 : 0);
            if (!cards.empty() && nc[k] >= 0) nc[k] = std::max(nc[k], cards[k]);
        }
        bool densifiable = true;
        for (int c : nc) if (c < 0) densifiable = false;
        int n_groups = 1;
        if (densifiable) for (int c : nc) { n_groups *= c; if (n_groups > 1 << 20) break; }
        if (!strategy_decided) {
            hash_mode = !ungrouped && (!densifiable || n_groups > DENSE_MAX_GROUPS);
            strategy_decided = true;
        } else if (!hash_mode && (!densifiable || n_groups > DENSE_MAX_GROUPS)) {
            // The key cardinality outgrew the dense layout mid-stream.  A Partial / PartialMerge aggregate may emit a group more
            // than once (the Final stage merges state rows, exactly as it does for Spark's own spilling partial aggregates): flush
            // what the dense path has accumulated as one state batch and carry on with the hash table.
            if (mode == AggMode::Final) throw Unsupported("group cardinality grew past the dense path mid-stream in a Final aggregate");
            if (have_totals) {
                Batch early;
                finalize(early);
                if (early.n_rows > 0) outq.push_back(std::move(early));
            }
            have_totals = false;
            totals.reset(); spill.reset(); partials.reset();
            totals_groups = 0; n_words = 0; word_kinds.clear(); cards.clear(); rows_scanned = 0;
            hash_mode = true;
        }
        if (hash_mode) {
            key_has_null_prev = key_has_null;
            key_has_null = hn;
            consume_hash(b);
            return;
        }
        key_has_null_prev = key_has_null;
        key_has_null = hn;
        if (have_totals && nc != cards) {
            if (n_words == 0) throw ExecError(15, "", "internal: regroup before layout");
            regroup(nc);
        }
        cards = nc;
        if (observed_bits.empty()) observed_bits.assign(child->schema.size(), -1);
        const int64_t SAMPLE = 1 << 20;
        bool have_obs = false;
        for (int ci : used_cols) if (child->schema[(size_t)ci].is_decimal() && observed_bits[(size_t)ci] >= 0) have_obs = true;
        if (mode == AggMode::Partial && !have_obs && b.n_rows > 2 * SAMPLE) {
            // Range profile of the last plan with this very pipeline (the previous task of the same stage reads the same table):
            // start at its ranges instead of sampling again.  A profile is only a guess -- every launch validates it.
            profile_key = pipeline_signature(make_spec(&b, n_groups, SAFE));
            std::lock_guard<std::mutex> lk(g_profile_mu);
            auto it = g_range_profile.find(profile_key);
            if (it != g_range_profile.end() && it->second.size() == observed_bits.size()) {
                observed_bits = it->second;
                for (int ci : used_cols) if (child->schema[(size_t)ci].is_decimal() && observed_bits[(size_t)ci] >= 0) have_obs = true;
            }
        }
        if (mode != AggMode::Partial) {
            run_range(b, 0, b.n_rows, n_groups, SAFE);
        } else if (!have_obs && b.n_rows > 2 * SAMPLE) {
            // sample-then-specialise: a short launch measures the value ranges, the bulk launch runs the kernel
            // specialised to them (64-bit arithmetic, unconditional accumulation); every launch validates its
            // assumptions through the value masks, so a violated guess only costs a re-run.
            run_range(b, 0, SAMPLE, n_groups, TYPE);
            run_range(b, SAMPLE, b.n_rows, n_groups, TIGHT);
        } else {
            run_range(b, 0, b.n_rows, n_groups, have_obs ? TIGHT : TYPE);
        }
        if (!profile_key.empty()) {
            std::lock_guard<std::mutex> lk(g_profile_mu);
            if (g_range_profile.size() > 256) g_range_profile.clear();
            g_range_profile[profile_key] = observed_bits;
        }
    }
    std::string profile_key;

    // ---- hash aggregation: table sizing, launch, flags ------------------------------------------------------------
    void launch_named(const std::shared_ptr<CompiledModule>& mod, const char* name, dim3 grid, dim3 block, void** args) {
        cuda_check(cudaLaunchKernel((const void*)mod->kernel(name), grid, block, args, 0, ctx->stream), name);
        ctx->kernel_launches++;
    }
    void hash_params(cb::PipeParams& p) const {
        p.hkeys = (cb::u64*)hkeys->ptr;
        p.hkey_of_gid = (cb::u64*)hkey_of_gid->ptr;
        p.htotals = (cb::u64*)htotals->ptr;
        p.hmask = (cb::u32)(hcap - 1);
        p.max_groups = (cb::i32)max_groups;
        p.hflags = (cb::i32*)hflags->ptr;
    }
    bool zero_identity() const {
        for (int k : word_kinds) if (k == W_MIN || k == W_MAX) return false;
        return true;
    }
    void init_totals(const std::shared_ptr<CompiledModule>& mod, cb::u64* totals, int64_t first, int64_t n) {
        if (n <= 0) return;
        if (zero_identity()) {
            cuda_check(cudaMemsetAsync(totals + first * n_words * 2, 0, (size_t)n * n_words * 16, ctx->stream), "memset totals");
        } else {
            long long f = first, nn = n;
            void* a1[] = {&totals, &f, &nn};
            launch_named(mod, "cb_hash_init", dim3((unsigned)((n + 255) / 256)), dim3(256), a1);
        }
    }
    // ---- group ids: CB_GID_RANGES counters (device/cb_params.h); the host sees per-range counts ------------------------------------
    static constexpr int GK = CB_GID_RANGES;
    struct HashFlags { int w[CB_HFLAG_WORDS]; };
    void ensure_flags() {
        if (hflags) return;
        hflags = std::make_shared<DeviceBuf>(sizeof(HashFlags));
        cuda_check(cudaMemsetAsync(hflags->ptr, 0, sizeof(HashFlags), ctx->stream), "memset hash flags");
    }
    // device -> host (synchronises); cnt[r] = ids handed out in range r (a counter that ran past its range is clamped); returns their sum
    int64_t read_flags(HashFlags& hf, int64_t cnt[GK]) {
        memset(&hf, 0, sizeof(hf));
        if (hflags) {
            cuda_check(cudaMemcpyAsync(&hf, hflags->ptr, sizeof(hf), cudaMemcpyDeviceToHost, ctx->stream), "read hash flags"); ctx->d2h_bytes += (int64_t)sizeof(hf);
            cuda_check(cudaStreamSynchronize(ctx->stream), "hash flags sync");
        }
        const int64_t R = max_groups / GK;
        int64_t total = 0;
        bool overshoot = false;
        for (int r = 0; r < GK; r++) {
            if (hf.w[CB_HFLAG_CTR + r] > R || hf.w[CB_HFLAG_CTR + r] < 0) overshoot = true;
            cnt[r] = std::min<int64_t>(std::max(hf.w[CB_HFLAG_CTR + r], 0), R);
            if (hf.w[CB_HFLAG_CTR + r] < 0) cnt[r] = R; // wrapped: it was full long ago
            total += cnt[r];
        }
        if (overshoot && hflags) { // warps that found a range full still bumped its counter: put it back to "full" so it can never wrap
            for (int r = 0; r < GK; r++) hf.w[CB_HFLAG_CTR + r] = (int)cnt[r];
            write_flags(hf);
        }
        return total;
    }
    void write_flags(const HashFlags& hf) {
        cuda_check(cudaMemcpyAsync(hflags->ptr, &hf, sizeof(hf), cudaMemcpyHostToDevice, ctx->stream), "write hash flags");
        cuda_check(cudaStreamSynchronize(ctx->stream), "flags sync");
    }
    // new accumulator / key arrays for nm ids (a multiple of GK): range r's rows move from r * R_old to r * R_new, the two reserved
    // groups to the new tail.  zero_fill: every other word gets its identity (the key table path updates with atomics).
    void grow_rows(const std::shared_ptr<CompiledModule>& mod, const int64_t cnt[GK], int64_t nm, bool zero_fill) {
        cudaStream_t st = ctx->stream;
        if (nm + 2 >= INT32_MAX) throw ExecError(16, "", "more than 2^31 groups in one partition; lower spark.comet.b200.chunkRows");
        const int64_t Ro = max_groups / GK, Rn = nm / GK;
        auto ntot = std::make_shared<DeviceBuf>((size_t)(nm + 2) * n_words * 16);
        auto nkog = std::make_shared<DeviceBuf>((size_t)nm * 8 * key_words + 16);
        cb::u64* tp = (cb::u64*)ntot->ptr;
        if (zero_fill) init_totals(mod, tp, 0, nm + 2);
        else if (!htotals) init_totals(mod, tp, nm, 2);
        if (htotals) {
            for (int r = 0; r < GK; r++) {
                if (cnt[r] <= 0) continue;
                cuda_check(cudaMemcpyAsync(tp + (size_t)r * Rn * n_words * 2, (cb::u64*)htotals->ptr + (size_t)r * Ro * n_words * 2, (size_t)cnt[r] * n_words * 16,
                                           cudaMemcpyDeviceToDevice, st), "copy totals");
                cuda_check(cudaMemcpyAsync((cb::u64*)nkog->ptr + (size_t)r * Rn * key_words, (cb::u64*)hkey_of_gid->ptr + (size_t)r * Ro * key_words,
                                           (size_t)cnt[r] * 8 * key_words, cudaMemcpyDeviceToDevice, st), "copy group keys");
            }
            cuda_check(cudaMemcpyAsync(tp + (size_t)nm * n_words * 2, (cb::u64*)htotals->ptr + (size_t)max_groups * n_words * 2, (size_t)2 * n_words * 16,
                                       cudaMemcpyDeviceToDevice, st), "copy reserved groups");
        }
        cuda_check(cudaStreamSynchronize(st), "table growth"); // old buffers die below
        htotals = ntot; hkey_of_gid = nkog; max_groups = nm;
    }
    static int64_t round_ids(int64_t n) { return (n + GK - 1) / GK * GK; }

    // make sure `incoming` more rows (each possibly a new group) fit: dense accumulators by group id, key table at load <= 0.5
    void ensure_table(const std::shared_ptr<CompiledModule>& mod, int64_t incoming) {
        cudaStream_t st = ctx->stream;
        ensure_flags();
        HashFlags hf;
        int64_t cnt[GK];
        const int64_t cur = read_flags(hf, cnt);
        const int64_t need = cur + incoming;
        if (need + 2 >= INT32_MAX) throw ExecError(16, "", "more than 2^31 groups in one partition; lower spark.comet.b200.chunkRows");
        bool relocated = false;
        if (need > max_groups) {
            int64_t nm = std::max<int64_t>(need, max_groups + max_groups / 4);
            // When the source knows how many rows are still to come, size for them at the distinct ratio seen so far (+30 %) in ONE
            // step: growing means copying the totals and re-inserting every key.
            const int64_t remaining = child->rows_hint();
            if (remaining > 0 && rows_scanned == 0 && mode != AggMode::Partial) {
                // merging state rows (Final / PartialMerge): most keys are new -- size for everything that is still to come at once
                nm = std::max(nm, need + remaining);
            }
            if (remaining > 0 && rows_scanned > 0 && cur > 0) {
                const double ratio = std::min(1.0, 1.3 * (double)cur / (double)rows_scanned);
                const int64_t est = cur + incoming + (int64_t)(ratio * (double)remaining);
                nm = std::max(nm, std::min<int64_t>(est, cur + incoming + remaining));
            }
            if (nm + 2 + GK >= INT32_MAX) nm = INT32_MAX - 3 - GK;
            relocated = cur > 0;
            grow_rows(mod, cnt, round_ids(nm), true);
        }
        int64_t cap = std::max<int64_t>(hcap, 1 << 16);
        while (cap < 2 * std::max(need, max_groups)) cap <<= 1; // load <= 0.5 even when every reserved group id gets used
        if (cap != hcap || relocated) { // a relocation changes the ids: the slots must be rebuilt even at the same capacity
            auto nkeys = cap != hcap ? std::make_shared<DeviceBuf>((size_t)cap * 16) : hkeys;
            cuda_check(cudaMemsetAsync(nkeys->ptr, 0xff, (size_t)cap * 16, st), "memset key slots");
            if (cur > 0) {
                const cb::u64* kog = (const cb::u64*)hkey_of_gid->ptr;
                int rr = (int)(max_groups / GK);
                const int* ctr = (const int*)hflags->ptr + CB_HFLAG_CTR;
                cb::u64* kp = (cb::u64*)nkeys->ptr;
                cb::u32 mask = (cb::u32)(cap - 1);
                void* a2[] = {&kog, &rr, &ctr, &kp, &mask};
                launch_named(mod, "cb_hash_rehash", dim3((unsigned)((max_groups + 255) / 256)), dim3(256), a2);
                cuda_check(cudaStreamSynchronize(st), "rehash");
            }
            hkeys = nkeys; hcap = cap;
        }
    }

    // ---- stream mode: state-row arrays only (no key table).  ids max_groups / max_groups + 1 stay reserved (the NULL-key group is
    //      shared by all its runs and updated with atomics: zero / identity filled) -----------------------------------------------
    int64_t stream_groups = 0;         // state rows handed out so far
    DeviceBufP reserved_snap;          // totals of the two reserved groups before a launch (restored when the launch is repeated)
    void ensure_stream_rows(const std::shared_ptr<CompiledModule>& mod, const int64_t cnt[GK], int64_t want_groups) {
        ensure_flags();
        if (htotals && want_groups <= max_groups) return;
        grow_rows(mod, cnt, round_ids(std::max<int64_t>(want_groups, max_groups + max_groups / 2)), false);
    }
    // one CB_STREAM launch over rows [r0, r1) of b; returns the state rows handed out so far (and the flags / per-range counts after it)
    int64_t stream_launch(Batch& b, int64_t r0, int64_t r1, const PipelineSpec& spec, const GeneratedKernel& g, const std::shared_ptr<CompiledModule>& mod,
                          HashFlags& hf, int64_t cnt[GK]) {
        if (!vmask) vmask = std::make_shared<DeviceBuf>(CB_MAX_COLS * 16);
        cuda_check(cudaMemsetAsync(vmask->ptr, 0, CB_MAX_COLS * 16, ctx->stream), "memset vmask");
        cb::PipeParams p;
        fill_inputs(p, b, g.tile, r0, r1);
        p.hkeys = nullptr;
        p.hkey_of_gid = (cb::u64*)hkey_of_gid->ptr;
        p.htotals = (cb::u64*)htotals->ptr;
        p.hmask = 0;
        p.max_groups = (cb::i32)max_groups;
        p.hflags = (cb::i32*)hflags->ptr;
        p.vmask = (cb::u64*)vmask->ptr;
        p.n_groups = 2;
        int grid = std::max(1, std::min(ctx->num_sms, p.n_tiles));
        launch(mod->kernel(g.entry), dim3(grid), dim3(g.threads + 32), g.dyn_smem(0), &p);
        uint64_t masks[CB_MAX_COLS * 2];
        cuda_check(cudaMemcpyAsync(masks, vmask->ptr, sizeof(masks), cudaMemcpyDeviceToHost, ctx->stream), "read value masks"); ctx->d2h_bytes += (int64_t)(sizeof(masks));
        ctx->check_device_errors();
        const int64_t total = read_flags(hf, cnt);
        if (hf.w[0] & 4) throw Unsupported("decimal(p > 18) group key whose value does not fit 64 bits");
        if (!(hf.w[0] & 2))
            for (size_t i = 0; i < spec.cols.size(); i++) {
                if (!spec.cols[i].type.is_decimal()) continue;
                uint64_t lo = masks[2 * i], hi = masks[2 * i + 1];
                int bl = hi ? 64 + r_bitlen(hi) : r_bitlen(lo);
                observed_bits[(size_t)used_cols[i]] = std::max(observed_bits[(size_t)used_cols[i]], bl);
            }
        return total;
    }
    void snapshot_reserved(bool restore) {
        const size_t bytes = (size_t)2 * n_words * 16;
        if (!reserved_snap || reserved_snap->bytes < bytes) reserved_snap = std::make_shared<DeviceBuf>(bytes);
        cb::u64* tail = (cb::u64*)htotals->ptr + (size_t)max_groups * n_words * 2;
        if (restore) cuda_check(cudaMemcpyAsync(tail, reserved_snap->ptr, bytes, cudaMemcpyDeviceToDevice, ctx->stream), "restore reserved groups");
        else cuda_check(cudaMemcpyAsync(reserved_snap->ptr, tail, bytes, cudaMemcpyDeviceToDevice, ctx->stream), "snapshot reserved groups");
    }
    // Are equal keys adjacent?  Run the stream kernel over the first rows of the first batch and look at state rows per input row.
    void decide_stream(Batch& b) {
        stream_decided = true;
        stream_mode = false;
        if (mode != AggMode::Partial || !ctx || ctx->stream_agg_min_rows < 0) return;
        const int64_t hint = child->rows_hint();
        if (b.n_rows + std::max<int64_t>(hint, 0) < ctx->stream_agg_min_rows || b.n_rows == 0) return;
        stream_mode = true;
        PipelineSpec spec = make_spec(&b, 2, SAFE);
        GeneratedKernel g = generate_pipeline(spec);
        auto mod = jit_get(g, true);
        n_words = g.n_words; word_kinds = g.word_kinds; key_words = g.key_words;
        const int64_t sample = std::min<int64_t>(b.n_rows, 1 << 20);
        HashFlags hf;
        int64_t cnt[GK] = {0};
        ensure_stream_rows(mod, cnt, 2 * sample + 4096); // room for every row being its own run, in whichever ranges the warps draw from
        const int64_t runs = stream_launch(b, 0, sample, spec, g, mod, hf, cnt);
        stream_ratio = (hf.w[0] & 2) ? 1.0 : (double)runs / (double)sample;
        // the sample's rows are scanned again with the rest: forget its state rows (and whatever it added to the shared NULL-key group)
        memset(&hf, 0, sizeof(hf));
        write_flags(hf);
        init_totals(mod, (cb::u64*)htotals->ptr, max_groups, 2);
        if (stream_ratio > ctx->stream_agg_max_ratio) {
            stream_mode = false;
            htotals.reset(); hkey_of_gid.reset(); hflags.reset(); max_groups = 0; n_words = 0; word_kinds.clear();
        }
    }
    void consume_stream(Batch& b) {
        PipelineSpec spec = make_spec(&b, 2, SAFE);
        GeneratedKernel g = generate_pipeline(spec);
        auto mod = jit_get(g, true);
        ctx->last_kernel_key = g.key;
        if (have_totals && (g.n_words != n_words || g.word_kinds != word_kinds || g.key_words != key_words))
            throw ExecError(15, "", "internal: accumulator layout changed between launches");
        n_words = g.n_words; word_kinds = g.word_kinds; key_words = g.key_words;
        HashFlags before, hf;
        int64_t cnt0[GK], cnt[GK];
        const int64_t cur = read_flags(before, cnt0);
        // state rows this batch (and, when the source says how much is still to come, the rest) will need at the ratio seen so far
        const int64_t remaining = std::max<int64_t>(child->rows_hint(), 0);
        int64_t want = cur + std::min<int64_t>(b.n_rows, (int64_t)(1.25 * stream_ratio * (double)b.n_rows) + 65536);
        if (!htotals || want > max_groups) want += std::min<int64_t>(remaining, (int64_t)(1.25 * stream_ratio * (double)remaining));
        while (true) {
            {
                TraceSpan ts("stream.ensure_rows");
                ensure_stream_rows(mod, cnt0, want);
            }
            snapshot_reserved(false);
            stream_groups = stream_launch(b, 0, b.n_rows, spec, g, mod, hf, cnt);
            if (!(hf.w[0] & 2)) break;
            // more runs than state rows: nothing of this launch is kept (its rows only touched ids past the old counts and the shared group)
            snapshot_reserved(true);
            for (int r = 0; r < GK; r++) before.w[CB_HFLAG_CTR + r] = (int)cnt0[r];
            write_flags(before);
            want = cur + b.n_rows + GK; // every row its own run
        }
        ctx->pipeline_rows += b.n_rows;
        if (b.n_rows > 0) stream_ratio = std::max(stream_ratio, (double)(stream_groups - cur) / (double)b.n_rows);
        rows_scanned += b.n_rows;
        have_totals = true;
        last_gen = g;
        last_mod = mod;
    }

    void consume_hash(Batch& b) {
        if (keys.size() > CB_MAX_KEYS) throw Unsupported("more than 4 group keys");
        if (observed_bits.empty()) observed_bits.assign(child->schema.size(), -1);
        if (!stream_decided) decide_stream(b);
        if (stream_mode) { consume_stream(b); return; }
        // updates go straight into the table, so a launch cannot be discarded: no speculative assumptions here
        PipelineSpec spec = make_spec(&b, 2, SAFE);
        GeneratedKernel g = generate_pipeline(spec);
        auto mod = jit_get(g, true);
        ctx->last_kernel_key = g.key;
        if (have_totals && (g.n_words != n_words || g.word_kinds != word_kinds)) throw ExecError(15, "", "internal: accumulator layout changed between launches");
        n_words = g.n_words;
        word_kinds = g.word_kinds;
        if (have_totals && g.key_words != key_words) throw ExecError(15, "", "internal: group key packing changed between launches");
        key_words = g.key_words;
        {
            TraceSpan ts("hash.ensure_table");
            ensure_table(mod, b.n_rows);
        }
        if (!vmask) vmask = std::make_shared<DeviceBuf>(CB_MAX_COLS * 16);
        cuda_check(cudaMemsetAsync(vmask->ptr, 0, CB_MAX_COLS * 16, ctx->stream), "memset vmask");
        cb::PipeParams p;
        fill_inputs(p, b, g.tile);
        hash_params(p);
        p.vmask = (cb::u64*)vmask->ptr;
        p.n_groups = 2;
        int grid = std::max(1, std::min(ctx->num_sms, p.n_tiles));
        launch(mod->kernel(g.entry), dim3(grid), dim3(g.threads + 32), g.dyn_smem(0), &p);
        ctx->pipeline_rows += b.n_rows;
        uint64_t masks[CB_MAX_COLS * 2];
        int flags[8];
        cuda_check(cudaMemcpyAsync(masks, vmask->ptr, sizeof(masks), cudaMemcpyDeviceToHost, ctx->stream), "read value masks"); ctx->d2h_bytes += (int64_t)(sizeof(masks));
        cuda_check(cudaMemcpyAsync(flags, hflags->ptr, sizeof(flags), cudaMemcpyDeviceToHost, ctx->stream), "read hash flags"); ctx->d2h_bytes += (int64_t)(sizeof(flags));
        ctx->check_device_errors();
        if (flags[0] & 2) throw ExecError(15, "", "internal: hash table full");
        if (flags[0] & 4) throw Unsupported("decimal(p > 18) group key whose value does not fit 64 bits");
        for (size_t i = 0; i < spec.cols.size(); i++) {
            if (!spec.cols[i].type.is_decimal()) continue;
            uint64_t lo = masks[2 * i], hi = masks[2 * i + 1];
            int bl = hi ? 64 + r_bitlen(hi) : r_bitlen(lo);
            observed_bits[(size_t)used_cols[i]] = std::max(observed_bits[(size_t)used_cols[i]], bl);
        }
        rows_scanned += b.n_rows;
        have_totals = true;
        last_gen = g;
        last_mod = mod;
    }

    // hash results: groups are dense by id, so finalize writes the output columns directly (no compaction)
    void finalize_hash(Batch& out) {
        TraceSpan ts("agg.finalize_hash");
        const GeneratedKernel& g = last_gen;
        cudaStream_t st = ctx->stream;
        HashFlags hfl;
        int64_t cnt[GK];
        const int64_t ng = read_flags(hfl, cnt);
        const int* flags = hfl.w;
        const int64_t n_out = ng + ((flags[0] & 1) ? 1 : 0) + ((flags[0] & 8) ? 1 : 0);
        cb::FinParams fp;
        memset(&fp, 0, sizeof(fp));
        fp.totals = (cb::u64*)htotals->ptr;
        fp.hkeys = (const cb::u64*)hkey_of_gid->ptr;
        fp.sentinel_used = flags[0] & 1;
        fp.null_group_used = (flags[0] & 8) ? 1 : 0;
        fp.n_hash_groups = (int)ng;
        fp.max_groups = (int)max_groups;
        fp.gid_range = (int)(max_groups / GK);
        {
            int64_t run = 0;
            for (int r = 0; r < GK; r++) { fp.gid_prefix[r] = (int)run; run += cnt[r]; }
            fp.gid_prefix[GK] = (int)run;
        }
        fp.n_groups = (int)n_out;
        fp.err = ctx->d_err;
        fill_certificates(fp);
        if (g.out_cols.size() > CB_MAX_OUT) throw Unsupported("too many output columns");
        out.n_rows = n_out;
        out.cols.clear();
        std::vector<DeviceBufP> vbytes;
        size_t rows_alloc = (size_t)std::max<int64_t>(n_out, 1);
        for (size_t i = 0; i < g.out_cols.size(); i++) {
            Column c;
            c.type = g.out_cols[i].type;
            c.phys = c.type.id == TypeId::Bool ? Phys::I8 : (c.type.is_string() ? Phys::I32 : phys_of_type(c.type));
            c.data = std::make_shared<DeviceBuf>(rows_alloc * g.out_bytes[i]);
            vbytes.push_back(std::make_shared<DeviceBuf>(rows_alloc));
            fp.out[i] = (cb::u8*)c.data->ptr;
            fp.outv[i] = (cb::u8*)vbytes.back()->ptr;
            if ((int)i < g.n_key_cols && c.type.is_string()) { c.is_dict = true; c.dict = key_dicts[i]; }
            out.cols.push_back(c);
        }
        auto present = std::make_shared<DeviceBuf>(rows_alloc);
        fp.present = (cb::u8*)present->ptr;
        if (n_out > 0) {
            void* args[] = {&fp};
            launch_named(last_mod, g.finalize_entry.c_str(), dim3((unsigned)((n_out + 127) / 128)), dim3(128), args);
            for (size_t i = 0; i < out.cols.size(); i++) {
                Column& c = out.cols[i];
                c.valid_bytes = vbytes[i];
                c.validity = std::make_shared<DeviceBuf>((size_t)(n_out + 31) / 32 * 4 + 8);
                launch_bytes_to_bitmap((const unsigned char*)vbytes[i]->ptr, n_out, (uint32_t*)c.validity->ptr, st);
                ctx->kernel_launches++;
                c.null_count = -1;
                if (c.type.id == TypeId::Bool) c.bool_bytes = c.data;
            }
        }
        ctx->check_device_errors();
    }

    // one (possibly split) launch over rows [row0,row1) at assumption level lv, escalating on violated assumptions
    void run_range(Batch& b, int64_t row0, int64_t row1, int n_groups, Level lv) {
        TraceSpan tsr("agg.run_range");
        while (true) {
            PipelineSpec spec;
            GeneratedKernel g;
            std::shared_ptr<CompiledModule> mod;
            {
                TraceSpan ts("agg.codegen+jit");
                spec = make_spec(&b, n_groups, lv);
                g = generate_pipeline(spec);
                mod = jit_get(g, true);
            }
            ctx->last_kernel_key = g.key;
            if (have_totals && (g.n_words != n_words || g.word_kinds != word_kinds))
                throw ExecError(15, "", "internal: accumulator layout changed between launches");
            n_words = g.n_words;
            word_kinds = g.word_kinds;
            const int64_t max_rows = (int64_t)ctx->num_sms * g.threads * (1ll << CB_RPT_LOG2) / 1024 * 1024;
            bool ok = true;
            for (int64_t r0 = row0; r0 < row1 && ok; r0 += max_rows) ok = launch_one(b, r0, std::min(row1, r0 + max_rows), n_groups, spec, g, mod);
            if (ok) return;
            if (lv == SAFE) throw ExecError(15, "", "internal: value-mask validation failed without assumptions");
            lv = lv == TIGHT ? TYPE : SAFE; // widen: observed ranges -> declared precision -> no assumption (fully checked code)
            // partial sub-launches of the failed attempt were already folded only if they validated; restart the remainder
            row0 = failed_from;
        }
    }
    int64_t failed_from = 0;

    bool launch_one(Batch& b, int64_t r0, int64_t r1, int n_groups, const PipelineSpec& spec, const GeneratedKernel& g,
                    const std::shared_ptr<CompiledModule>& mod) {
        cudaStream_t st = ctx->stream;
        size_t tot_bytes = (size_t)n_groups * n_words * 16;
        if (!have_totals) {
            totals = std::make_shared<DeviceBuf>(tot_bytes);
            totals_groups = n_groups;
        }
        if (!spill || spill->bytes < tot_bytes) {
            spill = std::make_shared<DeviceBuf>(tot_bytes);
            cuda_check(cudaMemsetAsync(spill->ptr, 0, spill->bytes, st), "memset spill");
        }
        if (!vmask) vmask = std::make_shared<DeviceBuf>(CB_MAX_COLS * 16);
        cuda_check(cudaMemsetAsync(vmask->ptr, 0, CB_MAX_COLS * 16, st), "memset vmask");
        cb::PipeParams p;
        fill_inputs(p, b, g.tile, r0, r1);
        int grid = std::max(1, std::min(ctx->num_sms, p.n_tiles));
        size_t part_bytes = (size_t)grid * tot_bytes;
        if (!partials || partials->bytes < part_bytes) partials = std::make_shared<DeviceBuf>(part_bytes);
        p.n_groups = n_groups;
        for (size_t k = 0; k < cards.size() && k < CB_MAX_KEYS; k++) p.key_card[k] = cards[k];
        p.partials = (cb::u8*)partials->ptr;
        p.spill = (cb::u64*)spill->ptr;
        p.vmask = (cb::u64*)vmask->ptr;
        launch(mod->kernel(g.entry), dim3(grid), dim3(g.threads + 32), g.dyn_smem(n_groups), &p); // + producer warp
        ctx->pipeline_rows += r1 - r0;
        uint64_t masks[CB_MAX_COLS * 2];
        cuda_check(cudaMemcpyAsync(masks, vmask->ptr, sizeof(masks), cudaMemcpyDeviceToHost, st), "read value masks"); ctx->d2h_bytes += (int64_t)(sizeof(masks));
        ctx->check_device_errors(); // synchronises
        // validate the assumptions this kernel was specialised for
        std::vector<int> seen(spec.cols.size(), -1);
        bool ok = true;
        for (size_t i = 0; i < spec.cols.size(); i++) {
            if (!spec.cols[i].type.is_decimal()) continue;
            uint64_t lo = masks[2 * i], hi = masks[2 * i + 1];
            int bl = hi ? 64 + r_bitlen(hi) : r_bitlen(lo);
            seen[i] = bl;
            if (spec.cols[i].assume_bits > 0 && bl > spec.cols[i].assume_bits) ok = false;
        }
        if (!ok) {
            // discard this launch: partials are simply not folded; the exact-escape accumulators must be cleared
            cuda_check(cudaMemsetAsync(spill->ptr, 0, spill->bytes, st), "memset spill");
            // remember what we saw so the retry is specialised correctly
            for (size_t i = 0; i < spec.cols.size(); i++)
                if (seen[i] >= 0) observed_bits[(size_t)used_cols[i]] = std::max(observed_bits[(size_t)used_cols[i]], seen[i]);
            failed_from = r0;
            return false;
        }
        for (size_t i = 0; i < spec.cols.size(); i++)
            if (seen[i] >= 0) observed_bits[(size_t)used_cols[i]] = std::max(observed_bits[(size_t)used_cols[i]], seen[i]);
        rows_scanned += r1 - r0;
        cb::FinParams fp;
        memset(&fp, 0, sizeof(fp));
        fp.partials = (const cb::u64*)partials->ptr;
        fp.spill = (cb::u64*)spill->ptr;
        fp.totals = (cb::u64*)totals->ptr;
        fp.n_ctas = grid;
        fp.n_groups = n_groups;
        fp.first = have_totals ? 0 : 1;
        fp.err = ctx->d_err;
        int total_words = n_groups * n_words;
        void* args[] = {&fp};
        cuda_check(cudaLaunchKernel((const void*)mod->kernel("cb_fold"), dim3((total_words + 127) / 128), dim3(128), args, 0, st), "fold launch");
        ctx->kernel_launches++;
        have_totals = true;
        last_gen = g;
        last_mod = mod;
        return true;
    }

    // Host side of the overflow certificate: a bound on the magnitude of any single addend of decimal SUM / AVG `ai`, from the value
    // masks observed on its input columns pushed through the same range propagation the code generator uses.  finalize multiplies
    // it by the group's own addend count (cb::cert_level): n * B <= 10^p - 1 means no row order can overflow.
    u128r certificate(size_t ai) const {
        const AggExpr& a = aggs[ai];
        if (!(a.kind == AggKind::Sum || a.kind == AggKind::Avg) || !a.datatype.is_decimal()) return 0;
        std::vector<u128r> bounds(child->schema.size(), RSAT);
        for (size_t c = 0; c < bounds.size(); c++)
            if (child->schema[c].is_decimal() && !observed_bits.empty())
                bounds[c] = observed_bits[c] < 0 ? 0 : (observed_bits[c] >= 127 ? RSAT : (u128r)1 << observed_bits[c]);
        if (mode == AggMode::Partial) return expr_maxabs(*a.children[0], bounds);
        return bounds[(size_t)state_cols[ai][0]];
    }
    void fill_certificates(cb::FinParams& fp) const {
        for (size_t ai = 0; ai < aggs.size() && ai < CB_MAX_OUT; ai++) {
            const u128r b = certificate(ai);
            fp.cert_b[ai][0] = b >= RSAT ? ~0ull : (uint64_t)b;
            fp.cert_b[ai][1] = b >= RSAT ? ~0ull : (uint64_t)(b >> 64);
            // bit 63 of the high word (free: B < 2^127): B is the bound 2^bits of a value mask, i.e. addends lie in [-B, B - 1]
            const bool direct = mode != AggMode::Partial || aggs[ai].children[0]->kind == ExprKind::Bound;
            if (b < RSAT && b != 0 && direct) fp.cert_b[ai][1] |= 1ull << 63;
        }
    }

    bool next(Batch& out) override {
        if (emitted) {
            if (outq_pos >= outq.size()) return false;
            out = std::move(outq[outq_pos++]);
            return true;
        }
        if (keys.size() > CB_MAX_KEYS) throw Unsupported("more than 4 group keys");
        key_has_null.assign(keys.size(), false);
        key_dicts.assign(keys.size(), nullptr);
        dev_dicts.assign(keys.size(), nullptr);
        Batch in;
        while (child->next(in)) {
            if (in.n_rows == 0) continue;
            consume(in);
            ctx->check_device_errors();
        }
        emitted = true;
        if (!have_totals) {
            if (!ungrouped) { // grouped aggregate over no (further) rows
                if (outq_pos >= outq.size()) return false;
                out = std::move(outq[outq_pos++]);
                return true;
            }
            // ungrouped aggregate over an empty input still emits one row: run finalize over identities
            PipelineSpec spec = make_spec(nullptr, 1);
            last_gen = generate_pipeline(spec);
            last_mod = jit_get(last_gen, true);
            n_words = last_gen.n_words;
            word_kinds = last_gen.word_kinds;
            std::vector<uint64_t> id((size_t)n_words * 2, 0);
            for (int w = 0; w < n_words; w++) id[(size_t)w * 2] = word_kinds[(size_t)w] == W_MIN ? 0x7fffffffffffffffull : word_kinds[(size_t)w] == W_MAX ? 0x8000000000000000ull : 0;
            totals = std::make_shared<DeviceBuf>(id.size() * 8);
            cuda_check(cudaMemcpyAsync(totals->ptr, id.data(), id.size() * 8, cudaMemcpyHostToDevice, ctx->stream), "identity totals");
            cuda_check(cudaStreamSynchronize(ctx->stream), "identity totals sync");
            totals_groups = 1;
        }
        Batch last;
        if (hash_mode) finalize_hash(last);
        else finalize(last);
        outq.push_back(std::move(last));
        out = std::move(outq[outq_pos++]);
        return true;
    }

    void finalize(Batch& out) {
        TraceSpan ts("agg.finalize");
        const GeneratedKernel& g = last_gen;
        int ng = totals_groups;
        cb::FinParams fp;
        memset(&fp, 0, sizeof(fp));
        fp.totals = (cb::u64*)totals->ptr;
        fp.n_groups = ng;
        fp.err = ctx->d_err;
        fill_certificates(fp);
        // all finalize outputs live in ONE device buffer so the (tiny) result comes back in a single copy
        std::vector<size_t> off_v, off_n;
        size_t total_bytes = 0;
        auto take = [&](size_t n) { size_t o = total_bytes; total_bytes += (n + 15) / 16 * 16; return o; };
        for (size_t i = 0; i < g.out_cols.size(); i++) { off_v.push_back(take((size_t)ng * g.out_bytes[i])); off_n.push_back(take((size_t)ng)); }
        size_t off_present = take((size_t)ng);
        auto dbuf = std::make_shared<DeviceBuf>(total_bytes);
        for (size_t i = 0; i < g.out_cols.size(); i++) {
            fp.out[i] = (cb::u8*)dbuf->ptr + off_v[i];
            fp.outv[i] = (cb::u8*)dbuf->ptr + off_n[i];
        }
        fp.present = (cb::u8*)dbuf->ptr + off_present;
        void* args[] = {&fp};
        cuda_check(cudaLaunchKernel((const void*)last_mod->kernel(g.finalize_entry), dim3((ng + 127) / 128), dim3(128), args, 0, ctx->stream), "finalize launch");
        ctx->kernel_launches++;
        std::vector<uint8_t> hbuf(total_bytes);
        cuda_check(cudaMemcpyAsync(hbuf.data(), dbuf->ptr, total_bytes, cudaMemcpyDeviceToHost, ctx->stream), "agg results D2H"); ctx->d2h_bytes += (int64_t)(total_bytes);
        ctx->check_device_errors(); // synchronises
        const uint8_t* pres = hbuf.data() + off_present;
        std::vector<int> rows;
        for (int gi = 0; gi < ng; gi++) if (ungrouped || pres[(size_t)gi]) rows.push_back(gi);
        out.n_rows = (int64_t)rows.size();
        out.cols.clear();
        // key columns
        for (size_t k = 0; k < keys.size(); k++) {
            Column c;
            c.type = schema[k];
            c.on_host = true;
            bool any_null = false;
            std::vector<int> codes;
            for (int gi : rows) {
                int rem = gi;
                std::vector<int> code(cards.size());
                for (int kk = (int)cards.size() - 1; kk >= 0; kk--) { code[(size_t)kk] = rem % cards[(size_t)kk]; rem /= cards[(size_t)kk]; }
                codes.push_back(code[k]);
            }
            c.h_valid.assign(rows.size(), 1);
            if (c.type.id == TypeId::Bool) {
                c.h_data.resize(rows.size());
                for (size_t r = 0; r < rows.size(); r++) {
                    bool isnull = key_has_null[k] && codes[r] == cards[k] - 1;
                    c.h_data[r] = isnull ? 0 : (uint8_t)codes[r];
                    if (isnull) { c.h_valid[r] = 0; any_null = true; }
                }
            } else {
                c.h_offsets.push_back(0);
                for (size_t r = 0; r < rows.size(); r++) {
                    bool isnull = key_has_null[k] && codes[r] == cards[k] - 1;
                    if (isnull) { c.h_valid[r] = 0; any_null = true; }
                    else {
                        const std::string& s = key_dicts[k]->values.at((size_t)codes[r]);
                        c.h_data.insert(c.h_data.end(), s.begin(), s.end());
                    }
                    c.h_offsets.push_back((int32_t)c.h_data.size());
                }
            }
            if (!any_null) c.h_valid.clear();
            out.cols.push_back(c);
        }
        for (size_t i = 0; i < g.out_cols.size(); i++) {
            Column c;
            c.type = g.out_cols[i].type;
            c.on_host = true;
            int w = g.out_bytes[i];
            const uint8_t* all = hbuf.data() + off_v[i];
            const uint8_t* allv = hbuf.data() + off_n[i];
            c.h_data.resize(rows.size() * w);
            c.h_valid.resize(rows.size());
            bool any_null = false;
            for (size_t r = 0; r < rows.size(); r++) {
                memcpy(&c.h_data[r * w], &all[(size_t)rows[r] * w], (size_t)w);
                c.h_valid[r] = allv[(size_t)rows[r]];
                if (!c.h_valid[r]) any_null = true;
            }
            if (!any_null) c.h_valid.clear();
            out.cols.push_back(c);
        }
    }
};


// =================================================================================================
// hash repartitioning (ShuffleWriterExec with HashPartition, native/shuffle/src/partitioners/multi_partition.rs)
// =================================================================================================
// Output: the child's rows reordered so that partition p occupies rows [starts[p], starts[p+1]) -- what the
// reference writes as per-partition IPC blocks, kept on the device for the NVLink exchange.
struct PartitionNode : ExecNode {
    ExecContext* ctx;
    ExecNodeP child;
    std::vector<int> key_cols;
    int n_parts = 1;

    bool next(Batch& out) override {
        Batch in;
        if (!child->next(in)) return false;
        TraceSpan ts("partition");
        to_device(in);
        int64_t n = in.n_rows;
        cudaStream_t st = ctx->stream;
        HashKeyCols kc;
        memset(&kc, 0, sizeof(kc));
        if (key_cols.size() > 8) throw Unsupported("more than 8 hash-partition keys");
        std::vector<DeviceBufP> keep;
        for (int ci : key_cols) {
            const Column& c = in.cols[(size_t)ci];
            HashKeyCol& k = kc.col[kc.n++];
            k.data = c.data ? c.data->ptr : nullptr;
            k.validity = c.validity ? (const unsigned char*)c.validity->ptr : nullptr;
            switch (c.type.id) {
            case TypeId::Bool: k.kind = HK_BOOL; break;
            case TypeId::Int8: k.kind = HK_I8; break;
            case TypeId::Int16: k.kind = HK_I16; break;
            case TypeId::Int32: case TypeId::Date: k.kind = HK_I32; break;
            case TypeId::Int64: case TypeId::Timestamp: case TypeId::TimestampNtz: k.kind = HK_I64; break;
            case TypeId::Float32: k.kind = HK_F32; break;
            case TypeId::Float64: k.kind = HK_F64; break;
            case TypeId::Decimal:
                if (c.phys == Phys::I64) k.kind = c.type.precision <= 18 ? HK_DEC_SMALL_64 : HK_DEC_LARGE_64;
                else k.kind = c.type.precision <= 18 ? HK_DEC_SMALL_128 : HK_DEC_LARGE_128;
                break;
            case TypeId::String: case TypeId::Binary:
                if (c.is_dict) {
                    k.kind = c.phys == Phys::I8 ? HK_DICT8 : c.phys == Phys::I16 ? HK_DICT16 : HK_DICT32;
                    std::vector<int32_t> off{0};
                    std::string chars;
                    for (auto& v : c.dict->values) { chars += v; off.push_back((int32_t)chars.size()); }
                    auto doff = std::make_shared<DeviceBuf>(off.size() * 4), dch = std::make_shared<DeviceBuf>(chars.size() + 16);
                    cuda_check(cudaMemcpyAsync(doff->ptr, off.data(), off.size() * 4, cudaMemcpyHostToDevice, st), "dict offsets");
                    if (!chars.empty()) cuda_check(cudaMemcpyAsync(dch->ptr, chars.data(), chars.size(), cudaMemcpyHostToDevice, st), "dict chars");
                    cuda_check(cudaStreamSynchronize(st), "dict upload");
                    keep.push_back(doff); keep.push_back(dch);
                    k.dict_offsets = (const int*)doff->ptr;
                    k.dict_chars = (const unsigned char*)dch->ptr;
                } else {
                    if (!c.offsets || !c.chars) throw Unsupported("string partition key without offsets/chars");
                    k.kind = HK_UTF8;
                    k.dict_offsets = (const int*)c.offsets->ptr;
                    k.dict_chars = (const unsigned char*)c.chars->ptr;
                }
                break;
            default: throw Unsupported("hash partitioning on " + c.type.str());
            }
        }
        size_t nb = (size_t)(n + 1023) / 1024 + 1;
        auto pids = std::make_shared<DeviceBuf>((size_t)n * 4 + 16);
        auto hist = std::make_shared<DeviceBuf>(nb * n_parts * 4);
        auto base = std::make_shared<DeviceBuf>(nb * n_parts * 8);
        auto starts = std::make_shared<DeviceBuf>((size_t)(n_parts + 1) * 8);
        auto row_idx = std::make_shared<DeviceBuf>((size_t)n * 8 + 16);
        cuda_check(cudaMemsetAsync(starts->ptr, 0, (size_t)(n_parts + 1) * 8, st), "memset starts");
        auto chunk_tmp = std::make_shared<DeviceBuf>((size_t)(partition_chunks(n) + 1) * n_parts * 8);
        launch_partition(kc, n, (unsigned)n_parts, nullptr, (unsigned*)pids->ptr, (int*)hist->ptr, (long long*)base->ptr, (long long*)chunk_tmp->ptr,
                         (long long*)starts->ptr, (long long*)row_idx->ptr, st);
        ctx->kernel_launches += 6;
        out.n_rows = n;
        out.cols.clear();
        for (auto& c : in.cols) {
            Column o = c;
            if (c.offsets) throw Unsupported("repartitioning plain string columns (dictionary-encode them first)");
            int w = phys_bytes(c.is_dict && c.phys == Phys::I32 ? Phys::Dict32 : c.phys);
            if (w == 0) { // bit-packed booleans: gather to bytes, repack
                auto bytes = std::make_shared<DeviceBuf>((size_t)n + 16);
                launch_gather_bits(c.data->ptr, (const long long*)row_idx->ptr, n, bytes->ptr, st);
                o.data = std::make_shared<DeviceBuf>((size_t)(n + 31) / 32 * 4 + 8);
                launch_bytes_to_bitmap((const unsigned char*)bytes->ptr, n, (uint32_t*)o.data->ptr, st);
                o.bool_bytes = bytes;
                ctx->kernel_launches += 2;
            } else {
                o.data = std::make_shared<DeviceBuf>((size_t)std::max<int64_t>(n, 1) * w);
                launch_gather(c.data->ptr, w, (const long long*)row_idx->ptr, n, o.data->ptr, st);
                ctx->kernel_launches++;
                if (c.type.id == TypeId::Bool) o.bool_bytes = o.data; // aggregate outputs keep booleans one byte per row
            }
            if (c.validity) {
                auto bytes = std::make_shared<DeviceBuf>((size_t)n + 16);
                launch_gather_bits(c.validity->ptr, (const long long*)row_idx->ptr, n, bytes->ptr, st);
                o.validity = std::make_shared<DeviceBuf>((size_t)(n + 31) / 32 * 4 + 8);
                launch_bytes_to_bitmap((const unsigned char*)bytes->ptr, n, (uint32_t*)o.validity->ptr, st);
                o.valid_bytes = bytes;
                ctx->kernel_launches += 2;
            }
            out.cols.push_back(o);
        }
        ctx->partition_starts.assign((size_t)n_parts + 1, 0);
        cuda_check(cudaMemcpyAsync(ctx->partition_starts.data(), starts->ptr, (size_t)(n_parts + 1) * 8, cudaMemcpyDeviceToHost, st), "starts D2H"); ctx->d2h_bytes += (int64_t)((size_t)(n_parts + 1) * 8);
        ctx->check_device_errors();
        return true;
    }

    // small host-resident aggregate results -> device columns
    void to_device(Batch& b) {
        for (auto& c : b.cols) {
            if (!c.on_host) continue;
            size_t n = (size_t)b.n_rows;
            if (c.type.is_string()) { // dictionary-encode on the host: these are group keys of a dense aggregate (a handful of rows)
                auto d = std::make_shared<Dictionary>();
                std::vector<int32_t> codes(n);
                for (size_t r = 0; r < n; r++) {
                    std::string v((const char*)c.h_data.data() + c.h_offsets[r], (size_t)(c.h_offsets[r + 1] - c.h_offsets[r]));
                    auto it = std::find(d->values.begin(), d->values.end(), v);
                    if (it == d->values.end()) { codes[r] = (int32_t)d->values.size(); d->values.push_back(v); }
                    else codes[r] = (int32_t)(it - d->values.begin());
                }
                c.data = std::make_shared<DeviceBuf>(n * 4 + 16);
                if (n) cuda_check(cudaMemcpyAsync(c.data->ptr, codes.data(), n * 4, cudaMemcpyHostToDevice, ctx->stream), "keys H2D");
                cuda_check(cudaStreamSynchronize(ctx->stream), "keys H2D sync");
                c.is_dict = true; c.dict = d; c.phys = Phys::I32;
            } else if (c.type.id == TypeId::Bool) {
                std::vector<uint8_t> bits((n + 7) / 8 + 8, 0);
                for (size_t r = 0; r < n; r++) if (c.h_data[r]) bits[r >> 3] |= (uint8_t)(1u << (r & 7));
                c.data = std::make_shared<DeviceBuf>(bits.size());
                cuda_check(cudaMemcpyAsync(c.data->ptr, bits.data(), bits.size(), cudaMemcpyHostToDevice, ctx->stream), "bool H2D");
                cuda_check(cudaStreamSynchronize(ctx->stream), "bool H2D sync");
                c.phys = Phys::Bitmap;
            } else {
                c.data = std::make_shared<DeviceBuf>(c.h_data.size() + 16);
                if (!c.h_data.empty()) cuda_check(cudaMemcpyAsync(c.data->ptr, c.h_data.data(), c.h_data.size(), cudaMemcpyHostToDevice, ctx->stream), "col H2D");
                cuda_check(cudaStreamSynchronize(ctx->stream), "col H2D sync");
                c.phys = phys_of(c.type);
            }
            if (!c.h_valid.empty()) {
                std::vector<uint8_t> bits((n + 7) / 8 + 8, 0);
                for (size_t r = 0; r < n; r++) if (c.h_valid[r]) bits[r >> 3] |= (uint8_t)(1u << (r & 7));
                c.validity = std::make_shared<DeviceBuf>(bits.size());
                cuda_check(cudaMemcpyAsync(c.validity->ptr, bits.data(), bits.size(), cudaMemcpyHostToDevice, ctx->stream), "validity H2D");
                cuda_check(cudaStreamSynchronize(ctx->stream), "validity H2D sync");
            }
            c.on_host = false;
        }
    }
};

// =================================================================================================
// plan -> executor tree
// =================================================================================================
static ExprP bound_ref(int i, const DType& t) {
    auto e = std::make_shared<Expr>();
    e->kind = ExprKind::Bound;
    e->index = i;
    e->type = t;
    return e;
}

static ExecNodeP build_node(const OperatorP& op, ExecContext* ctx, PlanInputs* inputs, bool build_only);

static ExecNodeP build_source(const OperatorP& op, ExecContext* ctx, PlanInputs* inputs, bool build_only) {
    if (op->kind == OpKind::Scan || op->kind == OpKind::ShuffleScan) {
        if (build_only) {
            auto s = std::make_shared<SchemaOnlySource>();
            s->schema = op->schema;
            return s;
        }
        if (inputs->streams.empty() && inputs->tables.empty()) throw PlanError("No input for scan");
        ArrowArrayStream* st = inputs->streams.empty() ? nullptr : inputs->streams.front();
        std::shared_ptr<DeviceTable> tb = inputs->tables.empty() ? nullptr : inputs->tables.front();
        if (!inputs->streams.empty()) inputs->streams.erase(inputs->streams.begin());
        if (!inputs->tables.empty()) inputs->tables.erase(inputs->tables.begin());
        if (tb) return std::make_shared<TableSource>(tb, op->schema, ctx);
        if (!st) throw PlanError("No input for scan");
        return std::make_shared<StreamSource>(ctx, st, op->schema);
    }
    if (op->kind == OpKind::NativeScan) {
        if (build_only) {
            auto s = std::make_shared<SchemaOnlySource>();
            s->schema = op->schema;
            return s;
        }
        return make_native_scan(op, ctx);
    }
    return build_node(op, ctx, inputs, build_only);
}

static ExecNodeP build_node(const OperatorP& op, ExecContext* ctx, PlanInputs* inputs, bool build_only) {
    OperatorP cur = op;
    OperatorP agg_op;
    if (cur->kind == OpKind::ShuffleWriter) {
        auto n = std::make_shared<PartitionNode>();
        n->ctx = ctx;
        n->child = build_node(cur->children[0], ctx, inputs, build_only);
        n->schema = cur->schema;
        n->n_parts = cur->num_partitions;
        for (auto& e : cur->hash_exprs) {
            if (e->kind != ExprKind::Bound) throw Unsupported("computed hash-partition keys (only plain column keys)");
            n->key_cols.push_back(e->index);
        }
        return n;
    }
    if (cur->kind == OpKind::HashAgg) { agg_op = cur; cur = cur->children[0]; }
    std::vector<OperatorP> chain; // top-down
    while (cur->kind == OpKind::Filter || cur->kind == OpKind::Projection) { chain.push_back(cur); cur = cur->children[0]; }
    if (!agg_op && chain.empty()) return build_source(cur, ctx, inputs, build_only);
    ExecNodeP src = build_source(cur, ctx, inputs, build_only);
    // compose bottom-up
    std::vector<ExprP> cols;
    for (size_t i = 0; i < src->schema.size(); i++) cols.push_back(bound_ref((int)i, src->schema[i]));
    std::vector<ExprP> preds;
    for (auto it = chain.rbegin(); it != chain.rend(); ++it) {
        const OperatorP& o = *it;
        if (o->kind == OpKind::Filter) preds.push_back(substitute(o->predicate, cols));
        else {
            std::vector<ExprP> nc;
            for (auto& e : o->project_list) nc.push_back(substitute(e, cols));
            cols = nc;
        }
    }
    if (!preds.empty()) src->push_filters(preds); // the fused filter still runs on every row; the source may prune with it
    if (agg_op) {
        auto n = std::make_shared<AggNode>();
        n->ctx = ctx;
        n->child = src;
        n->schema = agg_op->schema;
        n->predicates = preds;
        n->mode = agg_op->mode;
        n->ungrouped = agg_op->grouping.empty();
        std::vector<ExprP> roots = preds;
        for (auto& gexp : agg_op->grouping) {
            ExprP k = substitute(gexp, cols);
            if (k->kind != ExprKind::Bound) throw Unsupported("computed group keys (only plain column keys are fused)");
            n->keys.push_back(k);
            roots.push_back(k);
        }
        size_t state_at = agg_op->grouping.size();
        for (auto& a : agg_op->aggs) {
            AggExpr c = a;
            if (agg_op->mode == AggMode::Partial) {
                for (auto& ch : c.children) { ch = substitute(ch, cols); roots.push_back(ch); }
                if (c.filter) { c.filter = substitute(c.filter, cols); roots.push_back(c.filter); }
            } else {
                std::vector<int> sc;
                for (size_t k = 0; k < agg_state_types(a).size(); k++) {
                    ExprP e = cols.at(state_at++);
                    if (e->kind != ExprKind::Bound) throw Unsupported("final aggregate over computed state columns");
                    sc.push_back(e->index);
                    roots.push_back(e);
                }
                n->state_cols.push_back(sc);
            }
            n->aggs.push_back(c);
        }
        n->assign_slots(roots);
        if (n->used_cols.empty()) {
            // COUNT(*) / COUNT(1) alone reads no column: stage the narrowest fixed-width one just to drive the row loop
            int best = -1, best_w = 1 << 30;
            for (size_t c = 0; c < src->schema.size(); c++) {
                const DType& t = src->schema[c];
                if (t.is_string()) continue;
                int w = std::max(1, phys_bytes(phys_of(t)));
                if (w < best_w) { best = (int)c; best_w = w; }
            }
            if (best < 0) throw Unsupported("COUNT(*) over a child with only string columns");
            n->used_cols.push_back(best);
            n->slot_of[best] = 0;
        }
        return n;
    }
    auto n = std::make_shared<SelectNode>();
    n->ctx = ctx;
    n->child = src;
    n->schema = op->schema;
    n->predicates = preds;
    n->outputs = cols;
    for (auto& e : cols)
        if (e->type.is_string() && e->kind != ExprKind::Bound) throw Unsupported("string expressions through a fused filter/projection (only column references)");
    std::vector<ExprP> roots = preds;
    for (auto& e : cols) roots.push_back(e);
    n->assign_slots(roots);
    n->assign_pred_slots();
    if (n->used_cols.empty()) throw Unsupported("projection of constants only");
    return n;
}

ExecNodeP build_exec(const OperatorP& op, ExecContext* ctx, PlanInputs* inputs) { return build_node(op, ctx, inputs, false); }

std::vector<GeneratedKernel> plan_kernels_for_build(const OperatorP& op, const std::vector<int>& assume) {
    g_build_assume = assume;
    std::vector<GeneratedKernel> out;
    ExecNodeP root = build_node(op, nullptr, nullptr, true);
    std::function<void(const ExecNodeP&)> walk = [&](const ExecNodeP& n) {
        if (auto s = std::dynamic_pointer_cast<SelectNode>(n)) {
            out.push_back(generate_pipeline(s->make_spec(nullptr)));
            if (!s->predicates.empty()) out.push_back(generate_pipeline(s->make_count_spec(nullptr)));
            walk(s->child);
        } else if (auto pn = std::dynamic_pointer_cast<PartitionNode>(n)) {
            walk(pn->child);
        } else if (auto a = std::dynamic_pointer_cast<AggNode>(n)) {
            a->key_has_null.assign(a->keys.size(), false);
            for (auto& k : a->keys) if (!k->type.is_string() && k->type.id != TypeId::Bool) a->hash_mode = true;
            out.push_back(generate_pipeline(a->make_spec(nullptr, a->ungrouped ? 1 : 6)));
            if (a->hash_mode && a->mode == AggMode::Partial) { // the run-combining variant the sampled decision may pick at run time
                a->stream_mode = true;
                out.push_back(generate_pipeline(a->make_spec(nullptr, 6)));
                a->stream_mode = false;
            }
            walk(a->child);
        }
    };
    walk(root);
    return out;
}

// =================================================================================================
// Arrow C Data export (prepare_output jni_api.rs:674-742, move_to_spark execution/utils.rs:32-62)
// =================================================================================================
namespace {
struct ArrayHolder {
    std::vector<std::vector<uint8_t>> bufs;
    const void* ptrs[3] = {nullptr, nullptr, nullptr};
};
void release_array(ArrowArray* a) {
    delete (ArrayHolder*)a->private_data;
    a->release = nullptr;
}
struct SchemaHolder {
    std::string format, name;
};
void release_schema(ArrowSchema* s) {
    delete (SchemaHolder*)s->private_data;
    s->release = nullptr;
}
std::string arrow_format(const DType& t) {
    switch (t.id) {
    case TypeId::Bool: return "b";
    case TypeId::Int8: return "c";
    case TypeId::Int16: return "s";
    case TypeId::Int32: return "i";
    case TypeId::Int64: return "l";
    case TypeId::Float32: return "f";
    case TypeId::Float64: return "g";
    case TypeId::String: return "u";
    case TypeId::Binary: return "z";
    case TypeId::Date: return "tdD";
    case TypeId::Timestamp: return "tsu:UTC";
    case TypeId::TimestampNtz: return "tsu:";
    case TypeId::Decimal: return "d:" + std::to_string(t.precision) + "," + std::to_string(t.scale);
    default: throw Unsupported("export of " + t.str());
    }
}
std::vector<uint8_t> pack_bits(const uint8_t* bytes, size_t n) {
    std::vector<uint8_t> out((n + 7) / 8 + 8, 0);
    for (size_t i = 0; i < n; i++) if (bytes[i]) out[i >> 3] |= (uint8_t)(1u << (i & 7));
    return out;
}
} // namespace

// bits [row0, row0 + n) of a device bitmap as a host bitmap that starts at bit 0 (Arrow export is zero-offset only, jni_api.rs:716-732)
static std::vector<uint8_t> fetch_bits(ExecContext* ctx, const void* dev_bitmap, int64_t row0, size_t n) {
    const size_t first = (size_t)row0 >> 3, shift = (size_t)row0 & 7, nbytes = (shift + n + 7) / 8;
    std::vector<uint8_t> raw(nbytes + 9, 0);
    if (n) {
        cuda_check(cudaMemcpyAsync(raw.data(), (const uint8_t*)dev_bitmap + first, nbytes, cudaMemcpyDeviceToHost, ctx->stream), "D2H validity");
        cuda_check(cudaStreamSynchronize(ctx->stream), "D2H sync");
        ctx->d2h_bytes += (int64_t)nbytes;
    }
    if (shift == 0) { raw.resize((n + 7) / 8 + 8); return raw; }
    std::vector<uint8_t> out((n + 7) / 8 + 8, 0);
    for (size_t i = 0; i < (n + 7) / 8; i++) out[i] = (uint8_t)((raw[i] >> shift) | (raw[i + 1] << (8 - shift)));
    return out;
}

// rows [row0, row0 + n_rows) of batch b as Arrow C Data arrays (the caller's spark.comet.batchSize slices a large batch, CometConf.scala:539-544)
void export_batch(Batch& b, ExecContext* ctx, ArrowArray* out_arrays, ArrowSchema* out_schemas, int n_cols, int64_t row0, int64_t n_rows) {
    TraceSpan ts("export_batch");
    if ((int)b.cols.size() != n_cols) throw PlanError("executePlan: caller passed " + std::to_string(n_cols) + " output slots, plan produces " + std::to_string(b.cols.size()) + " columns");
    if (row0 < 0 || n_rows < 0 || row0 + n_rows > b.n_rows) throw PlanError("export_batch: slice out of range");
    const size_t n = (size_t)n_rows, r0 = (size_t)row0;
    for (int i = 0; i < n_cols; i++) {
        Column& c = b.cols[(size_t)i];
        auto* h = new ArrayHolder();
        int64_t null_count = 0;
        std::vector<uint8_t> validity, data, offs;
        if (c.on_host) {
            if (!c.h_valid.empty()) {
                validity = pack_bits(c.h_valid.data() + r0, n);
                for (size_t r = 0; r < n; r++) null_count += c.h_valid[r0 + r] ? 0 : 1;
            }
            if (c.type.is_string()) {
                offs.resize((n + 1) * 4);
                const int32_t* ho = (const int32_t*)c.h_offsets.data();
                int32_t* o = (int32_t*)offs.data();
                for (size_t r = 0; r <= n; r++) o[r] = ho[r0 + r] - ho[r0];
                data.assign(c.h_data.begin() + ho[r0], c.h_data.begin() + ho[r0 + n]);
                data.resize(data.size() + 8);
            } else if (c.type.id == TypeId::Bool) data = pack_bits(c.h_data.data() + r0, n);
            else {
                const size_t w = (size_t)c.type.arrow_width();
                data.assign(c.h_data.begin() + (ptrdiff_t)(r0 * w), c.h_data.begin() + (ptrdiff_t)((r0 + n) * w));
                data.resize(data.size() + 8);
            }
        } else if (c.is_dict) {
            // dictionary-coded string keys of a hash aggregate: fetch the codes, spell the strings out on the host
            std::vector<int32_t> codes(n + 1);
            if (n) cuda_check(cudaMemcpyAsync(codes.data(), (const uint8_t*)c.data->ptr + r0 * 4, n * 4, cudaMemcpyDeviceToHost, ctx->stream), "D2H key codes");
            cuda_check(cudaStreamSynchronize(ctx->stream), "D2H sync");
            ctx->d2h_bytes += (int64_t)n * 4;
            std::vector<uint8_t> vb = c.validity && n ? fetch_bits(ctx, c.validity->ptr, row0, n) : std::vector<uint8_t>((n + 7) / 8 + 8, 0xff);
            offs.resize((n + 1) * 4);
            int32_t* o = (int32_t*)offs.data();
            o[0] = 0;
            for (size_t r = 0; r < n; r++) {
                bool valid = (vb[r >> 3] >> (r & 7)) & 1;
                if (valid) { const std::string& sv = c.dict->values.at((size_t)codes[r]); data.insert(data.end(), sv.begin(), sv.end()); }
                else null_count++;
                o[r + 1] = (int32_t)data.size();
            }
            data.resize(data.size() + 8);
            if (null_count) validity = vb;
        } else {
            if (c.type.is_string()) throw Unsupported("export of device string columns");
            int w = c.type.id == TypeId::Bool ? 1 : c.type.arrow_width();
            std::vector<uint8_t> raw(n * (size_t)w + 8);
            if (n) cuda_check(cudaMemcpyAsync(raw.data(), (const uint8_t*)c.data->ptr + r0 * (size_t)w, n * (size_t)w, cudaMemcpyDeviceToHost, ctx->stream), "D2H output");
            ctx->d2h_bytes += (int64_t)(n * (size_t)w);
            cuda_check(cudaStreamSynchronize(ctx->stream), "D2H sync");
            if (c.validity) {
                validity = fetch_bits(ctx, c.validity->ptr, row0, n);
                for (size_t r = 0; r < n; r++) null_count += ((validity[r >> 3] >> (r & 7)) & 1) ? 0 : 1;
                if (null_count == 0) validity.clear();
            }
            if (c.type.id == TypeId::Bool) data = pack_bits(raw.data(), n);
            else data = std::move(raw);
        }
        bool is_str = c.type.is_string();
        h->bufs.push_back(std::move(validity));
        if (is_str) h->bufs.push_back(std::move(offs));
        h->bufs.push_back(std::move(data));
        h->ptrs[0] = h->bufs[0].empty() ? nullptr : h->bufs[0].data();
        h->ptrs[1] = h->bufs[1].data();
        if (is_str) h->ptrs[2] = h->bufs[2].data();
        ArrowArray& a = out_arrays[i];
        memset(&a, 0, sizeof(a));
        a.length = (int64_t)n;
        a.null_count = null_count;
        a.offset = 0; // zero offset only (jni_api.rs:716-732)
        a.n_buffers = is_str ? 3 : 2;
        a.buffers = h->ptrs;
        a.release = release_array;
        a.private_data = h;
        auto* sh = new SchemaHolder();
        sh->format = arrow_format(c.type);
        sh->name = "col_" + std::to_string(i); // projection.rs:60
        ArrowSchema& s = out_schemas[i];
        memset(&s, 0, sizeof(s));
        s.format = sh->format.c_str();
        s.name = sh->name.c_str();
        s.flags = ARROW_FLAG_NULLABLE;
        s.release = release_schema;
        s.private_data = sh;
    }
}

} // namespace cb200
