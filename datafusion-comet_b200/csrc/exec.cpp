// exec.cpp -- executor: sources, filter / projection pipelines, hash repartitioning, plan building, Arrow export.
// Aggregation is in agg.cpp.
#include "exec_internal.h"

#include "aot_kernels.h"

#include <algorithm>
#include <cstdlib>
#include <ctime>
#include <mutex>

namespace cb200 {

// error bits raised by kernels (device/cb_kernels.cuh set_err)
enum { ERR_I128_OVERFLOW = 0, ERR_ANSI_OVERFLOW = 1, ERR_ORDER_DEPENDENT = 2, ERR_DIVIDE_BY_ZERO = 3, ERR_ARROW_DIVIDE_BY_ZERO = 4, ERR_DICT_CODE = 5 };

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
    if (e & (1 << ERR_DICT_CODE)) // a valid row's dictionary code outside its dictionary: the input batch is malformed
        throw ExecError(3, "", "dictionary code out of range: a non-NULL row of a dictionary-encoded string column has a code outside its dictionary");
    if (e & (1 << ERR_ORDER_DEPENDENT))
        throw ExecError(12, "", "SUM/AVG overflow here depends on the row order (some orderings of these rows overflow, others do not); "
                                "the reference adds in row order -- the row-ordered fallback is not built yet, so the plan is refused rather than guessed");
    throw ExecError(13, "", "device error flags " + std::to_string(e));
}

// =================================================================================================
// string predicate masks (exec_internal.h)
// =================================================================================================
void StrMasks::bind(cb::PipeParams& p, const PipelineSpec& spec, const Batch& b, ExecContext* ctx) {
    const std::vector<ExprP> preds = str_preds_of(spec);
    cudaStream_t st = ctx->stream;
    for (size_t j = 0; j < preds.size(); j++) {
        const Expr& e = *preds[j];
        const int src = spec.cols.at((size_t)e.children[0]->index).src_index;
        const Column& c = b.cols.at((size_t)src);
        if (!c.is_dict || !c.dict) throw Unsupported("string predicate over a plain (non-dictionary) Utf8 column");
        StrMask& m = by_key[std::to_string(src) + "@" + str_pred_key(e)];
        if (!m.payload) { // [lit_off: n_lits + 1 x i32][LIKE items: u16][literal bytes]
            std::vector<uint8_t> blob;
            std::vector<int32_t> off{0};
            std::string bytes;
            for (auto& l : e.str_lits) { bytes += l; off.push_back((int32_t)bytes.size()); }
            auto put = [&](const void* q, size_t n) { size_t at = (blob.size() + 15) / 16 * 16; blob.resize(at + n); if (n) memcpy(blob.data() + at, q, n); return at; };
            const size_t o_off = put(off.data(), off.size() * 4), o_pat = put(e.like_items.data(), e.like_items.size() * 2), o_lit = put(bytes.data(), bytes.size());
            m.payload = std::make_shared<DeviceBuf>(blob.size() + 16);
            cuda_check(cudaMemcpyAsync(m.payload->ptr, blob.data(), blob.size(), cudaMemcpyHostToDevice, st), "H2D string predicate");
            ctx->h2d_bytes += (int64_t)blob.size();
            const uint8_t* base = (const uint8_t*)m.payload->ptr;
            m.dev.op = (int)e.str_op;
            m.dev.n_lits = (int)e.str_lits.size();
            m.dev.lit_off = (const int*)(base + o_off);
            m.dev.pat = (const uint16_t*)(base + o_pat);
            m.dev.pat_len = (int)e.like_items.size();
            m.dev.lit = base + o_lit;
        }
        if (m.dict != c.dict) { m.dict = c.dict; m.done = 0; }
        const std::vector<std::string>& vals = c.dict->values();
        const int64_t n = (int64_t)vals.size();
        if (n > INT32_MAX) throw Unsupported("string predicate over a dictionary of more than 2^31 entries");
        const size_t words = (size_t)(n + 31) / 32;
        if (!m.bits || m.bits->bytes < words * 4) {
            const size_t cap = std::max<size_t>({words, m.bits ? m.bits->bytes / 2 : 0, 64}); // bytes / 2 = twice the words
            auto nb = std::make_shared<DeviceBuf>(cap * 4);
            if (m.bits && m.done > 0) cuda_check(cudaMemcpyAsync(nb->ptr, m.bits->ptr, (size_t)(m.done + 31) / 32 * 4, cudaMemcpyDeviceToDevice, st), "grow mask");
            m.bits = nb;
        }
        if (m.done < n) {
            // the tail [first, n), first on a word boundary: the partial last word of the previous update is evaluated again
            const int64_t first = m.done & ~(int64_t)31;
            std::vector<int32_t>& off = m.h_off;
            std::string& chars = m.h_chars;
            off.assign((size_t)(n - first) + 1, 0);
            size_t total = 0;
            for (int64_t i = first; i < n; i++) total += vals[(size_t)i].size();
            if (total > INT32_MAX) throw Unsupported("string predicate over more than 2 GiB of new dictionary bytes");
            chars.clear();
            chars.reserve(total);
            for (int64_t i = first; i < n; i++) { chars += vals[(size_t)i]; off[(size_t)(i - first + 1)] = (int32_t)chars.size(); }
            if (!m.off || m.off->bytes < off.size() * 4) m.off = std::make_shared<DeviceBuf>(off.size() * 4 * 2);
            if (!m.chars || m.chars->bytes < chars.size() + 16) m.chars = std::make_shared<DeviceBuf>(chars.size() * 2 + 16);
            cuda_check(cudaMemcpyAsync(m.off->ptr, off.data(), off.size() * 4, cudaMemcpyHostToDevice, st), "H2D dictionary offsets");
            if (!chars.empty()) cuda_check(cudaMemcpyAsync(m.chars->ptr, chars.data(), chars.size(), cudaMemcpyHostToDevice, st), "H2D dictionary chars");
            ctx->h2d_bytes += (int64_t)(off.size() * 4 + chars.size());
            launch_str_pred(m.dev, (const int*)m.off->ptr, (const unsigned char*)m.chars->ptr, first, n, (unsigned*)m.bits->ptr, st);
            cuda_check(cudaGetLastError(), "k_str_pred launch");
            ctx->kernel_launches++;
            m.done = n;
        }
        p.smask[j].bits = (const cb::u32*)m.bits->ptr;
        p.smask[j].n_entries = (cb::i32)n;
    }
}

// =================================================================================================
// bitmaps
// =================================================================================================
DeviceBufP bytes_to_bitmap(const DeviceBufP& bytes, int64_t n, ExecContext* ctx) {
    auto bits = std::make_shared<DeviceBuf>(bitmap_bytes(n));
    launch_bytes_to_bitmap((const unsigned char*)bytes->ptr, n, (uint32_t*)bits->ptr, ctx->stream);
    ctx->kernel_launches++;
    return bits;
}

// n bytes (nonzero = set) as a host bitmap, 8 bytes of slack behind it
static std::vector<uint8_t> pack_bits(const uint8_t* bytes, size_t n) {
    std::vector<uint8_t> out((n + 7) / 8 + 8, 0);
    for (size_t i = 0; i < n; i++) if (bytes[i]) out[i >> 3] |= (uint8_t)(1u << (i & 7));
    return out;
}

// =================================================================================================
// sources
// =================================================================================================
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
            const int32_t code = g.intern(std::string(chars + off[k], (size_t)(off[k + 1] - off[k])));
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
            for (auto& c : table->cols) {
                if (c.valid_bytes && !c.validity) c.validity = bytes_to_bitmap(c.valid_bytes, table->n_rows, ctx);
                if (c.bool_bytes && !c.data) c.data = bytes_to_bitmap(c.bool_bytes, table->n_rows, ctx);
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
                const int w = phys_bytes(c.phys);
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
    std::vector<PipelineSpec> build_specs() const override {
        std::vector<PipelineSpec> out{make_spec(nullptr)};
        if (!predicates.empty()) out.push_back(make_count_spec(nullptr));
        return out;
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
        cb::PipeParams p;
        if (masked()) fill_inputs_of(p, in, out_cols_used, g.tile);
        else fill_inputs(p, in, g.tile);
        bind_str_masks(p, spec, in);
        out.cols.clear();
        out.cols.resize(g.out_cols.size());
        cudaStream_t st = ctx->stream;
        for (size_t i = 0; i < g.out_cols.size(); i++) {
            Column& c = out.cols[i];
            c.type = g.out_cols[i].type;
            c.phys = kernel_out_phys(c.type);
            if (c.type.is_string()) { // dictionary codes pass through; the dictionary is the source column's
                const Column& src = in.cols.at((size_t)outputs[i]->index);
                if (!src.is_dict) throw Unsupported("plain Utf8 columns through a fused filter/projection (dictionary-encoded strings only)");
                c.is_dict = true;
                c.dict = src.dict;
            }
            c.data = std::make_shared<DeviceBuf>((size_t)in.n_rows * g.out_bytes[i]);
            p.out[i] = (cb::u8*)c.data->ptr;
            if (g.out_cols[i].nullable) {
                c.validity = std::make_shared<DeviceBuf>(bitmap_bytes(in.n_rows));
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
            const PipelineSpec cspec = make_count_spec(&in);
            GeneratedKernel cg = generate_pipeline(cspec);
            auto cmod = jit_get(cg, true);
            cb::PipeParams cp;
            fill_inputs_of(cp, in, pred_cols, cg.tile);
            bind_str_masks(cp, cspec, in);
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


// =================================================================================================
// hash repartitioning (ShuffleWriterExec with HashPartition, native/shuffle/src/partitioners/multi_partition.rs)
// =================================================================================================
// The HK_* kind of a key column (device/cb_sortkey.h), for hash partitioning and the sort.  The logical type decides how Spark hashes
// a value (utils.rs: i8 / i16 / i32 / date as i32, decimal(p <= 18) as i64, wider decimals as 16 bytes) and how many bits its sort key
// takes; the stored layout (DESIGN.md, "Data layout in HBM") decides how it is read.
static int key_kind(const Column& c) {
    const Phys ph = c.phys;
    switch (c.type.id) {
    case TypeId::Bool: return ph == Phys::Bitmap ? HK_BOOL : HK_BOOL8;
    case TypeId::Int8: return ph == Phys::I32 ? HK_I32 : HK_I8; // sign-extended to i32 either way
    case TypeId::Int16: return ph == Phys::I32 ? HK_I32 : HK_I16;
    case TypeId::Int32: case TypeId::Date: return HK_I32;
    case TypeId::Int64: case TypeId::Timestamp: case TypeId::TimestampNtz: return HK_I64;
    case TypeId::Float32: return HK_F32;
    case TypeId::Float64: return HK_F64;
    case TypeId::Decimal:
        if (ph == Phys::I32) return HK_DEC_SMALL_32;
        if (ph == Phys::I64) return c.type.precision <= 18 ? HK_DEC_SMALL_64 : HK_DEC_LARGE_64;
        return c.type.precision <= 18 ? HK_DEC_SMALL_128 : HK_DEC_LARGE_128;
    case TypeId::String: case TypeId::Binary:
        if (!c.is_dict) return HK_UTF8;
        return ph == Phys::I8 ? HK_DICT8 : ph == Phys::I16 ? HK_DICT16 : HK_DICT32;
    default: throw Unsupported("hash partitioning on " + c.type.str());
    }
}

// small host-resident aggregate results -> device columns
static void columns_to_device(Batch& b, ExecContext* ctx) {
    for (auto& c : b.cols) {
        if (!c.on_host) continue;
        size_t n = (size_t)b.n_rows;
        if (c.type.is_string()) { // dictionary-encode on the host: these are group keys of a dense aggregate (a handful of rows)
            auto d = std::make_shared<Dictionary>();
            std::vector<int32_t> codes(n);
            for (size_t r = 0; r < n; r++)
                codes[r] = d->intern(std::string((const char*)c.h_data.data() + c.h_offsets[r], (size_t)(c.h_offsets[r + 1] - c.h_offsets[r])));
            c.data = std::make_shared<DeviceBuf>(n * 4 + 16);
            if (n) cuda_check(cudaMemcpyAsync(c.data->ptr, codes.data(), n * 4, cudaMemcpyHostToDevice, ctx->stream), "keys H2D");
            cuda_check(cudaStreamSynchronize(ctx->stream), "keys H2D sync");
            c.is_dict = true; c.dict = d; c.phys = Phys::I32;
        } else if (c.type.id == TypeId::Bool) {
            std::vector<uint8_t> bits = pack_bits(c.h_data.data(), n);
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
            std::vector<uint8_t> bits = pack_bits(c.h_valid.data(), n);
            c.validity = std::make_shared<DeviceBuf>(bits.size());
            cuda_check(cudaMemcpyAsync(c.validity->ptr, bits.data(), bits.size(), cudaMemcpyHostToDevice, ctx->stream), "validity H2D");
            cuda_check(cudaStreamSynchronize(ctx->stream), "validity H2D sync");
        }
        c.on_host = false;
    }
}

// out's columns = in's rows row_idx[0, n), in that order.  Bit-packed booleans and validity are gathered one byte per row and repacked
// (the byte forms are kept: the exchange sends them).  `op` names the operator in the refusal of plain Utf8 columns.
template <typename I> static void gather_columns(const Batch& in, const I* row_idx, int64_t n, Batch& out, ExecContext* ctx, const char* op) {
    cudaStream_t st = ctx->stream;
    out.n_rows = n;
    out.cols.clear();
    for (auto& c : in.cols) {
        Column o = c;
        if (c.offsets) throw Unsupported(std::string(op) + " plain string columns (dictionary-encode them first)");
        int w = phys_bytes(c.phys);
        if (w == 0) { // bit-packed booleans: gather to bytes, repack
            auto bytes = std::make_shared<DeviceBuf>((size_t)n + 16);
            launch_gather_bits(c.data->ptr, row_idx, n, bytes->ptr, st);
            ctx->kernel_launches++;
            o.data = bytes_to_bitmap(bytes, n, ctx);
            o.bool_bytes = bytes;
        } else {
            o.data = std::make_shared<DeviceBuf>((size_t)std::max<int64_t>(n, 1) * w);
            launch_gather(c.data->ptr, w, row_idx, n, o.data->ptr, st);
            ctx->kernel_launches++;
            if (c.type.id == TypeId::Bool) o.bool_bytes = o.data; // aggregate outputs keep booleans one byte per row
        }
        if (c.validity) {
            auto bytes = std::make_shared<DeviceBuf>((size_t)n + 16);
            launch_gather_bits(c.validity->ptr, row_idx, n, bytes->ptr, st);
            ctx->kernel_launches++;
            o.validity = bytes_to_bitmap(bytes, n, ctx);
            o.valid_bytes = bytes;
        }
        out.cols.push_back(o);
    }
    cuda_check(cudaGetLastError(), "gathers");
}

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
        columns_to_device(in, ctx);
        int64_t n = in.n_rows;
        cudaStream_t st = ctx->stream;
        HashKeyCols kc;
        memset(&kc, 0, sizeof(kc));
        std::vector<DeviceBufP> keep;
        for (int ci : key_cols) {
            const Column& c = in.cols[(size_t)ci];
            HashKeyCol& k = kc.col[kc.n++];
            k.data = c.data ? c.data->ptr : nullptr;
            k.validity = c.validity ? (const unsigned char*)c.validity->ptr : nullptr;
            k.kind = key_kind(c);
            switch (k.kind) {
            case HK_DICT8: case HK_DICT16: case HK_DICT32: {
                std::vector<int32_t> off{0};
                std::string chars;
                for (auto& v : c.dict->values()) { chars += v; off.push_back((int32_t)chars.size()); }
                auto doff = std::make_shared<DeviceBuf>(off.size() * 4), dch = std::make_shared<DeviceBuf>(chars.size() + 16);
                cuda_check(cudaMemcpyAsync(doff->ptr, off.data(), off.size() * 4, cudaMemcpyHostToDevice, st), "dict offsets");
                if (!chars.empty()) cuda_check(cudaMemcpyAsync(dch->ptr, chars.data(), chars.size(), cudaMemcpyHostToDevice, st), "dict chars");
                cuda_check(cudaStreamSynchronize(st), "dict upload");
                keep.push_back(doff); keep.push_back(dch);
                k.dict_offsets = (const int*)doff->ptr;
                k.dict_chars = (const unsigned char*)dch->ptr;
                break;
            }
            case HK_UTF8:
                if (!c.offsets || !c.chars) throw Unsupported("string partition key without offsets/chars");
                k.dict_offsets = (const int*)c.offsets->ptr;
                k.dict_chars = (const unsigned char*)c.chars->ptr;
                break;
            default: break;
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
        cuda_check(launch_partition(kc, n, (unsigned)n_parts, nullptr, (unsigned*)pids->ptr, (int*)hist->ptr, (long long*)base->ptr, (long long*)chunk_tmp->ptr,
                                    (long long*)starts->ptr, (long long*)row_idx->ptr, st), "partition launches");
        ctx->kernel_launches += 6;
        gather_columns(in, (const long long*)row_idx->ptr, n, out, ctx, "repartitioning");
        ctx->partition_starts.assign((size_t)n_parts + 1, 0);
        cuda_check(cudaMemcpyAsync(ctx->partition_starts.data(), starts->ptr, (size_t)(n_parts + 1) * 8, cudaMemcpyDeviceToHost, st), "starts D2H"); ctx->d2h_bytes += (int64_t)((size_t)(n_parts + 1) * 8);
        ctx->check_device_errors();
        return true;
    }
};

// ---- shared by Sort and HashJoin -------------------------------------------------------------------------------------------------
// the rows of bs in one batch (`bs` non-empty, every batch on the device): values and validity appended in order; dictionary-coded strings
// that carry different Dictionary objects are recoded into one (the first batch's entries, then the others' new entries)
static Batch concat_batches(const std::vector<Batch>& bs, ExecContext* ctx, const char* op) {
    cudaStream_t st = ctx->stream;
    Batch out;
    for (auto& b : bs) out.n_rows += b.n_rows;
    const size_t n = (size_t)out.n_rows;
    std::vector<DeviceBufP> temps;
    for (size_t j = 0; j < bs[0].cols.size(); j++) {
        const Column& c0 = bs[0].cols[j];
        Column o;
        o.type = c0.type;
        o.phys = c0.phys;
        o.is_dict = c0.is_dict;
        o.dict = c0.dict;
        bool same = true, nulls = false;
        for (auto& b : bs) {
            const Column& c = b.cols[j];
            if (c.phys != c0.phys || c.dict != c0.dict || c.is_dict != c0.is_dict) same = false;
            if (c.validity) nulls = true;
        }
        if (!same && !c0.is_dict) throw Unsupported(std::string(op) + " input whose batches store column " + std::to_string(j) + " in different layouts");
        if (same) {
            const int w = phys_bytes(c0.phys);
            o.data = std::make_shared<DeviceBuf>(w == 0 ? bitmap_bytes((int64_t)n) : std::max<size_t>(n, 1) * (size_t)w);
            if (w == 0) cuda_check(cudaMemsetAsync(o.data->ptr, 0, o.data->bytes, st), "memset bools");
            int64_t row = 0;
            for (auto& b : bs) {
                const Column& c = b.cols[j];
                if (w == 0) { launch_bitmap_append((uint32_t*)o.data->ptr, row, (const uint8_t*)c.data->ptr, 0, b.n_rows, st); ctx->kernel_launches++; }
                else cuda_check(cudaMemcpyAsync((char*)o.data->ptr + (size_t)row * w, c.data->ptr, (size_t)b.n_rows * w, cudaMemcpyDeviceToDevice, st), "concat column");
                row += b.n_rows;
            }
        } else { // dictionary codes -> int32 codes of one dictionary
            auto d = std::make_shared<Dictionary>(*c0.dict);
            o.phys = Phys::I32;
            o.dict = d;
            o.data = std::make_shared<DeviceBuf>(std::max<size_t>(n, 1) * 4);
            int64_t row = 0;
            for (auto& b : bs) {
                const Column& c = b.cols[j];
                const std::vector<std::string>& vals = c.dict->values();
                std::vector<int32_t> table(vals.size());
                for (size_t k = 0; k < table.size(); k++) table[k] = c.dict == c0.dict ? (int32_t)k : d->intern(vals[k]);
                auto dt = std::make_shared<DeviceBuf>(table.size() * 4 + 4);
                temps.push_back(dt);
                if (!table.empty()) cuda_check(cudaMemcpyAsync(dt->ptr, table.data(), table.size() * 4, cudaMemcpyHostToDevice, st), "H2D remap table");
                cuda_check(cudaStreamSynchronize(st), "remap table copy"); // table is a loop temporary
                launch_remap_codes(c.data->ptr, phys_bytes(c.phys), b.n_rows, (const int*)dt->ptr, (int)table.size(), (int*)o.data->ptr + row, st);
                ctx->kernel_launches++;
                row += b.n_rows;
            }
        }
        if (nulls) {
            o.validity = std::make_shared<DeviceBuf>(bitmap_bytes((int64_t)n));
            cuda_check(cudaMemsetAsync(o.validity->ptr, 0, o.validity->bytes, st), "memset validity");
            int64_t row = 0;
            for (auto& b : bs) {
                const Column& c = b.cols[j];
                launch_bitmap_append((uint32_t*)o.validity->ptr, row, c.validity ? (const uint8_t*)c.validity->ptr : nullptr, 0, b.n_rows, st);
                ctx->kernel_launches++;
                row += b.n_rows;
            }
            o.null_count = -1;
        }
        out.cols.push_back(o);
    }
    cuda_check(cudaGetLastError(), "concat launches");
    return out;
}

// the stable order of m rows whose keys (`words` words each) are in keys0, by the given digits: row indices [0, m); `sorted_keys`, if
// given, receives the keys in that order
static DeviceBufP radix_order(ExecContext* ctx, DeviceBufP keys0, int words, int64_t m, const std::vector<int>& digits, DeviceBufP* sorted_keys = nullptr) {
    cudaStream_t st = ctx->stream;
    const int64_t nt = sort_tiles(m);
    auto keys1 = std::make_shared<DeviceBuf>((size_t)m * words * 8);
    auto idx0 = std::make_shared<DeviceBuf>((size_t)m * 4), idx1 = std::make_shared<DeviceBuf>((size_t)m * 4);
    auto hist = std::make_shared<DeviceBuf>((size_t)nt * 256 * 4), chunk_off = std::make_shared<DeviceBuf>((size_t)(nt * 256 / 4096 + 2) * 4);
    auto total = std::make_shared<DeviceBuf>(8);
    RadixScratch s{{(unsigned long long*)keys0->ptr, (unsigned long long*)keys1->ptr}, {(unsigned*)idx0->ptr, (unsigned*)idx1->ptr},
                   (unsigned*)hist->ptr, (unsigned*)chunk_off->ptr, (long long*)total->ptr};
    int r = 0;
    cuda_check(launch_sort_passes(s, words, m, digits.data(), (int)digits.size(), &r, st), "sort passes");
    ctx->kernel_launches += digits.empty() ? 1 : 4 * (int64_t)digits.size();
    if (sorted_keys) *sorted_keys = r ? keys1 : keys0;
    return r ? idx1 : idx0; // the other buffers go back to the stream-ordered pool
}

// the row keys of kc (kc.words words each) for n rows.  h_and_or[0, W) receives their AND and [W, 2W) their OR, `digits` the 8-bit
// digits of the `bits`-bit key that are not the same in every row, least significant first.  Synchronises: a dictionary code outside its
// dictionary fails here.
static DeviceBufP pack_row_keys(const cb::SortKeyCols& kc, int64_t n, int bits, ExecContext* ctx, uint64_t* h_and_or, std::vector<int>& digits) {
    cudaStream_t st = ctx->stream;
    const int W = kc.words;
    auto keys0 = std::make_shared<DeviceBuf>((size_t)n * W * 8);
    auto and_or = std::make_shared<DeviceBuf>(2 * cb::SK_MAX_WORDS * 8);
    cuda_check(cudaMemsetAsync(and_or->ptr, 0xff, (size_t)W * 8, st), "memset key and");
    cuda_check(cudaMemsetAsync((char*)and_or->ptr + W * 8, 0, (size_t)W * 8, st), "memset key or");
    launch_sort_keys(kc, n, (unsigned long long*)keys0->ptr, (unsigned long long*)and_or->ptr, st);
    cuda_check(cudaGetLastError(), "k_sort_keys launch");
    ctx->kernel_launches++;
    cuda_check(cudaMemcpyAsync(h_and_or, and_or->ptr, (size_t)W * 16, cudaMemcpyDeviceToHost, st), "D2H key and / or");
    ctx->check_device_errors(); // also synchronises
    digits.clear();
    for (int d = 0; d < (bits + 7) / 8; d++) {
        const int w = W - 1 - d / 8, sh = (d % 8) * 8;
        if (((h_and_or[w] ^ h_and_or[W + w]) >> sh) & 0xff) digits.push_back(d);
    }
    return keys0;
}

// =================================================================================================
// sort (SortExec(LexOrdering).with_fetch(fetch) then GlobalLimitExec(skip), planner.rs:1488-1522)
// =================================================================================================
// The output is the child's rows in a stable order of the keys (ties keep the input order: batches as they arrive, rows in order
// within a batch), rows [skip, fetch).  Without a fetch, or with one above spark.comet.b200.chunkRows, the child is drained and its
// batches concatenated on the device, sorted once and emitted as one batch.  With a smaller fetch (TopK) at most `fetch` candidate rows
// are kept between chunks: each chunk is sorted, its first `fetch` rows are sorted together with the candidates (which come first, being
// earlier input) and the first `fetch` of those become the next candidates, so device memory is bounded by fetch + one chunk.  Keys are
// built again every round from the columns: a string's rank changes as its dictionary grows.
struct SortNode : ExecNode {
    ExecContext* ctx;
    ExecNodeP child;
    std::vector<SortKey> keys; // expr: Bound child column
    int64_t fetch = -1, skip = 0;
    bool done = false;
    struct Rank { const Dictionary* dict = nullptr; size_t n = 0; DeviceBufP table; };
    std::vector<Rank> ranks; // per key: code -> byte-order rank of the dictionary it was built for

    bool topk() const { return fetch >= 0 && fetch <= ctx->chunk_rows; }
    void count_passes(int64_t m, const std::vector<int>& digits) {
        ctx->sort_passes += (int64_t)digits.size();
        ctx->sort_pass_rows += m * (int64_t)digits.size();
    }

    bool next(Batch& out) override {
        if (done) return false;
        done = true;
        if (fetch == 0) return false;
        TraceSpan ts("sort");
        Batch all, in;
        bool any = false;
        if (topk()) {
            while (child->next(in)) {
                arrive(in);
                if (in.n_rows == 0) continue;
                // the chunk's own first `fetch` rows, then those merged behind the candidates (earlier input: first among equal keys)
                Batch top;
                sort_rows(in, 0, std::min<int64_t>(fetch, in.n_rows), top);
                in = Batch();
                if (any) {
                    Batch u = concat_batches({all, top}, ctx, "sort");
                    sort_rows(u, 0, std::min<int64_t>(fetch, u.n_rows), all);
                } else all = std::move(top);
                any = true;
            }
        } else {
            std::vector<Batch> batches;
            while (child->next(in)) {
                arrive(in);
                if (in.n_rows > 0) batches.push_back(std::move(in));
                in = Batch();
            }
            any = !batches.empty();
            if (any) all = batches.size() == 1 ? std::move(batches[0]) : concat_batches(batches, ctx, "sort");
        }
        if (!any) return false;
        const int64_t lo = std::min(skip, all.n_rows), hi = fetch >= 0 ? std::min(fetch, all.n_rows) : all.n_rows;
        if (hi <= lo) return false;
        if (topk() && lo == 0) { out = std::move(all); return true; } // the candidates are already in order
        sort_rows(all, lo, hi, out);
        return true;
    }

    void arrive(Batch& b) {
        columns_to_device(b, ctx);
        for (auto& c : b.cols)
            if (c.offsets) throw Unsupported("sorting plain string columns (dictionary-encode them first)");
    }

    // the code -> rank table of dictionary d: equal strings get equal ranks, ranks follow unsigned byte order.  Rebuilt when the
    // column carries another dictionary or its dictionary has grown.
    const uint32_t* rank_table(size_t key, const DictionaryP& d) {
        Rank& r = ranks[key];
        const std::vector<std::string>& v = d->values();
        if (r.table && r.dict == d.get() && r.n == v.size()) return (const uint32_t*)r.table->ptr;
        std::vector<uint32_t> order(v.size()), rank(v.size() + 1, 0);
        for (size_t i = 0; i < v.size(); i++) order[i] = (uint32_t)i;
        std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return v[a] < v[b]; }); // char_traits<char>: unsigned bytes
        uint32_t next = 0;
        for (size_t i = 0; i < order.size(); i++) {
            if (i > 0 && v[order[i]] != v[order[i - 1]]) next++;
            rank[order[i]] = next;
        }
        r.table = std::make_shared<DeviceBuf>(rank.size() * 4);
        cuda_check(cudaMemcpyAsync(r.table->ptr, rank.data(), rank.size() * 4, cudaMemcpyHostToDevice, ctx->stream), "H2D sort ranks");
        cuda_check(cudaStreamSynchronize(ctx->stream), "sort ranks copy");
        ctx->h2d_bytes += (int64_t)(rank.size() * 4);
        r.dict = d.get();
        r.n = v.size();
        return (const uint32_t*)r.table->ptr;
    }

    // out = b's rows [lo, hi) of the stable order of the keys.  When only the first rows are wanted (lo = 0, hi < n: TopK), an MSD radix
    // select finds the key of row hi - 1 of that order, the rows up to it are compacted (the smaller keys, then the equal ones in input
    // order) and only those are sorted.
    void sort_rows(const Batch& b, int64_t lo, int64_t hi, Batch& out) {
        const int64_t n = b.n_rows;
        if (n >= ((int64_t)1 << 32)) throw Unsupported("sorting 2^32 rows or more");
        cudaStream_t st = ctx->stream;
        cb::SortKeyCols kc;
        memset(&kc, 0, sizeof(kc));
        kc.n = (int)keys.size();
        kc.err = ctx->d_err;
        ranks.resize(keys.size());
        int bits = 0;
        for (size_t k = keys.size(); k-- > 0;) { // the last key is the least significant field
            const Column& c = b.cols.at((size_t)keys[k].expr->index);
            cb::SortKeyCol& f = kc.col[k];
            f.kind = key_kind(c);
            f.bits = sort_key_bits(c.type);
            f.desc = keys[k].descending;
            f.nulls_first = keys[k].nulls_first;
            f.has_null = c.validity != nullptr;
            f.data = c.data ? c.data->ptr : nullptr;
            f.validity = c.validity ? (const uint8_t*)c.validity->ptr : nullptr;
            if (c.is_dict) {
                f.rank = rank_table(k, c.dict);
                f.n_rank = (int)c.dict->values().size();
            }
            f.off = bits;
            bits += f.bits + f.has_null;
        }
        const int W = kc.words = std::max(1, (bits + 63) / 64);
        uint64_t h_and_or[2 * cb::SK_MAX_WORDS];
        std::vector<int> digits;
        DeviceBufP keys0 = pack_row_keys(kc, n, bits, ctx, h_and_or, digits);
        ctx->sort_rows += n;
        if (lo > 0 || hi >= n) {
            DeviceBufP idx = radix_order(ctx, keys0, W, n, digits);
            count_passes(n, digits);
            keys0.reset();
            gather_columns(b, (const unsigned*)idx->ptr + lo, hi - lo, out, ctx, "sorting");
            ctx->check_device_errors();
            return;
        }
        // select: bits equal in every row are decided already; then one histogram per differing digit, most significant first
        SortSelectKey p;
        for (int j = 0; j < W; j++) { p.mask[j] = ~(h_and_or[j] ^ h_and_or[W + j]); p.want[j] = h_and_or[j] & p.mask[j]; }
        int64_t r = hi; // the selected key's rank among the rows that match p
        auto hist = std::make_shared<DeviceBuf>(256 * 4);
        std::vector<uint32_t> hh(256);
        for (size_t q = digits.size(); q-- > 0;) {
            const int d = digits[q], w = W - 1 - d / 8, sh = (d % 8) * 8;
            cuda_check(cudaMemsetAsync(hist->ptr, 0, 256 * 4, st), "memset select histogram");
            cuda_check(launch_sort_select_hist((const unsigned long long*)keys0->ptr, W, n, p, d, (unsigned*)hist->ptr, st), "select histogram");
            ctx->kernel_launches++;
            ctx->sort_select_rows += n;
            cuda_check(cudaMemcpyAsync(hh.data(), hist->ptr, 256 * 4, cudaMemcpyDeviceToHost, st), "D2H select histogram");
            cuda_check(cudaStreamSynchronize(st), "select histogram sync");
            int v = 0;
            for (; v < 255 && r > (int64_t)hh[(size_t)v]; v++) r -= hh[(size_t)v];
            p.mask[w] |= (uint64_t)0xff << sh;
            p.want[w] |= (uint64_t)v << sh;
        }
        const size_t nb = (size_t)(n + 1023) / 1024;
        auto eq = std::make_shared<DeviceBuf>((size_t)n + 16), keep = std::make_shared<DeviceBuf>((size_t)n + 16);
        auto counts = std::make_shared<DeviceBuf>(nb * 4 + 4), offsets = std::make_shared<DeviceBuf>(nb * 8 + 8), kept = std::make_shared<DeviceBuf>(8);
        cuda_check(launch_sort_select_keep((const unsigned long long*)keys0->ptr, W, n, p, r, (unsigned char*)eq->ptr, (int*)counts->ptr,
                                           (long long*)offsets->ptr, (long long*)kept->ptr, (unsigned char*)keep->ptr, st), "select keep");
        launch_compact_plan((const unsigned char*)keep->ptr, n, (int*)counts->ptr, (long long*)offsets->ptr, (long long*)kept->ptr, st);
        auto rows = std::make_shared<DeviceBuf>((size_t)n * 4);
        launch_sort_iota((unsigned*)rows->ptr, n, st);
        auto ckeys = std::make_shared<DeviceBuf>((size_t)hi * W * 8), crows = std::make_shared<DeviceBuf>((size_t)hi * 4);
        launch_compact_scatter((const unsigned char*)keep->ptr, n, (const long long*)offsets->ptr, keys0->ptr, W * 8, ckeys->ptr, st);
        launch_compact_scatter((const unsigned char*)keep->ptr, n, (const long long*)offsets->ptr, rows->ptr, 4, crows->ptr, st);
        cuda_check(cudaGetLastError(), "select compaction");
        ctx->kernel_launches += 9;
        int64_t m = 0;
        cuda_check(cudaMemcpyAsync(&m, kept->ptr, 8, cudaMemcpyDeviceToHost, st), "D2H kept rows");
        cuda_check(cudaStreamSynchronize(st), "select sync");
        if (m != hi) throw ExecError(15, "", "internal: TopK selection kept " + std::to_string(m) + " rows for a fetch of " + std::to_string(hi));
        keys0.reset(); rows.reset(); eq.reset(); keep.reset();
        DeviceBufP order = radix_order(ctx, ckeys, W, m, digits);
        count_passes(m, digits);
        auto idx = std::make_shared<DeviceBuf>((size_t)m * 4);
        launch_gather(crows->ptr, 4, (const unsigned*)order->ptr, m, idx->ptr, st); // compacted position -> row of b
        ctx->kernel_launches++;
        gather_columns(b, (const unsigned*)idx->ptr, m, out, ctx, "sorting");
        ctx->check_device_errors();
    }
};

// =================================================================================================
// hash join (HashJoinExec with NullEquality::NullEqualsNothing, planner.rs:2192-2266): inner, left semi and left anti
// =================================================================================================
// The build side is drained before the first probe batch and concatenated on the device.  Its row keys (the sort's encoding,
// device/cb_sortkey.h) are radix-sorted, so equal keys form runs in build input order, and every run without a NULL key gets one slot of
// an open-addressing table.  A probe batch then costs one key pass and one lookup per row; an inner join scans the match counts, writes
// the (probe row, build row) pairs and gathers both sides, a semi / anti join compacts the probe rows it keeps.  Output order: probe rows
// in input order, an inner-join row's matches in build input order; an inner join's output above spark.comet.b200.chunkRows rows leaves
// in several batches.
//
// Equal key tuples give equal words on both sides because the field layout is fixed by the declared key types (every field has a null
// bit, whatever a batch's validity) and a string field holds a canonical code rather than the dictionary code: the code of the first
// equal entry of the build side's dictionary, or that dictionary's size (which no build key has) for a probe string it lacks.
struct JoinNode : ExecNode {
    ExecContext* ctx;
    ExecNodeP build_child, probe_child;
    std::vector<int> build_keys, probe_keys; // key columns of each side, in key order
    JoinType type = JoinType::Inner;
    bool build_left = false;
    int bits = 0, W = 1;                     // packed key bits (fixed per plan) and words
    cb::u64 nullmask[cb::SK_MAX_WORDS] = {0, 0, 0, 0};

    bool built = false;
    Batch build;                             // the build side's rows, concatenated
    DeviceBufP keys, rows, run_start, slots; // sorted build keys and their rows, run starts (+ the end), the table
    JoinTable table{};
    uint32_t h_build_rows = 0;
    std::vector<DeviceBufP> build_canon;     // per key: build dictionary code -> canonical code
    struct Canon { DictionaryP dict; size_t n = 0; DeviceBufP table; };
    std::vector<Canon> probe_canon;          // per key: the probe dictionary it was built for, code -> canonical code

    Batch probe;                             // the probe batch being emitted ...
    DeviceBufP run_of, offs, chunk_off, kept_rows;
    int64_t total = 0, pos = 0;              // ... its output rows, and those emitted

    // the key layout from the declared key types: the last key is the least significant field, each with a null bit above its value
    void set_layout(const std::vector<DType>& key_types) {
        bits = 0;
        for (size_t k = key_types.size(); k-- > 0;) bits += sort_key_bits(key_types[k]) + 1;
        W = std::max(1, (bits + 63) / 64);
        int off = 0;
        for (size_t k = key_types.size(); k-- > 0;) {
            off += sort_key_bits(key_types[k]);
            cb::sk_put(nullmask, W, off, 1, 1);
            off++;
        }
    }

    void arrive(Batch& b) {
        columns_to_device(b, ctx);
        for (auto& c : b.cols)
            if (c.offsets) throw Unsupported("joining plain string columns (dictionary-encode them first)");
    }

    DeviceBufP upload_codes(const std::vector<uint32_t>& v) {
        auto t = std::make_shared<DeviceBuf>(v.size() * 4 + 4);
        if (!v.empty()) cuda_check(cudaMemcpyAsync(t->ptr, v.data(), v.size() * 4, cudaMemcpyHostToDevice, ctx->stream), "H2D join codes");
        cuda_check(cudaStreamSynchronize(ctx->stream), "join codes copy"); // v is the caller's temporary
        ctx->h2d_bytes += (int64_t)(v.size() * 4);
        return t;
    }
    // canonical codes of key k's dictionary d on the build side: the first equal entry (a caller's dictionary may repeat values)
    const uint32_t* build_codes(size_t k, const DictionaryP& d) {
        const std::vector<std::string>& v = d->values();
        std::vector<uint32_t> c(v.size());
        for (size_t i = 0; i < v.size(); i++) c[i] = (uint32_t)d->find(v[i]);
        build_canon[k] = upload_codes(c);
        return (const uint32_t*)build_canon[k]->ptr;
    }
    // ... and on the probe side: rebuilt when the column carries another dictionary or its dictionary has grown
    const uint32_t* probe_codes(size_t k, const DictionaryP& d) {
        Canon& p = probe_canon[k];
        const std::vector<std::string>& v = d->values();
        if (p.table && p.dict == d && p.n == v.size()) return (const uint32_t*)p.table->ptr;
        const DictionaryP& bd = build.cols[(size_t)build_keys[k]].dict;
        const uint32_t absent = (uint32_t)bd->values().size();
        std::vector<uint32_t> c(v.size());
        for (size_t i = 0; i < v.size(); i++) {
            const int32_t code = bd->find(v[i]);
            c[i] = code < 0 ? absent : (uint32_t)code;
        }
        p.table = upload_codes(c);
        p.dict = d;
        p.n = v.size();
        return (const uint32_t*)p.table->ptr;
    }
    cb::SortKeyCols key_cols(const Batch& b, const std::vector<int>& cols, bool build_side) {
        cb::SortKeyCols kc;
        memset(&kc, 0, sizeof(kc));
        kc.n = (int)cols.size();
        kc.words = W;
        kc.err = ctx->d_err;
        int off = 0;
        for (size_t k = cols.size(); k-- > 0;) {
            const Column& c = b.cols.at((size_t)cols[k]);
            cb::SortKeyCol& f = kc.col[k];
            f.kind = key_kind(c);
            f.bits = sort_key_bits(c.type);
            f.nulls_first = 1; // null bit set on a valid value
            f.has_null = 1;
            f.data = c.data ? c.data->ptr : nullptr;
            f.validity = c.validity ? (const uint8_t*)c.validity->ptr : nullptr;
            if (c.is_dict) {
                f.rank = build_side ? build_codes(k, c.dict) : probe_codes(k, c.dict);
                f.n_rank = (int)c.dict->values().size();
            }
            f.off = off;
            off += f.bits + 1;
        }
        return kc;
    }

    void build_table() {
        built = true;
        std::vector<Batch> bs;
        Batch in;
        while (build_child->next(in)) {
            arrive(in);
            ctx->join_build_rows += in.n_rows;
            if (in.n_rows > 0) bs.push_back(std::move(in));
            in = Batch();
        }
        if (bs.empty()) return;
        TraceSpan ts("join.build");
        build = bs.size() == 1 ? std::move(bs[0]) : concat_batches(bs, ctx, "hash join build");
        bs.clear();
        const int64_t n = build.n_rows;
        if (n >= ((int64_t)1 << 32)) throw Unsupported("a hash join build side of 2^32 rows or more");
        cudaStream_t st = ctx->stream;
        build_canon.assign(build_keys.size(), nullptr);
        probe_canon.assign(build_keys.size(), Canon());
        uint64_t h_and_or[2 * cb::SK_MAX_WORDS];
        std::vector<int> digits;
        DeviceBufP k0 = pack_row_keys(key_cols(build, build_keys, true), n, bits, ctx, h_and_or, digits);
        rows = radix_order(ctx, k0, W, n, digits, &keys);
        k0.reset();
        const size_t nb = (size_t)(n + 1023) / 1024;
        auto head = std::make_shared<DeviceBuf>((size_t)n + 16), iota = std::make_shared<DeviceBuf>((size_t)n * 4);
        auto counts = std::make_shared<DeviceBuf>(nb * 4 + 4), offsets = std::make_shared<DeviceBuf>(nb * 8 + 8), d_runs = std::make_shared<DeviceBuf>(8);
        run_start = std::make_shared<DeviceBuf>((size_t)(n + 1) * 4);
        launch_join_heads((const unsigned long long*)keys->ptr, W, n, (unsigned char*)head->ptr, st);
        launch_compact_plan((const unsigned char*)head->ptr, n, (int*)counts->ptr, (long long*)offsets->ptr, (long long*)d_runs->ptr, st);
        launch_sort_iota((unsigned*)iota->ptr, n, st);
        launch_compact_scatter((const unsigned char*)head->ptr, n, (const long long*)offsets->ptr, iota->ptr, 4, run_start->ptr, st);
        cuda_check(cudaGetLastError(), "join run heads");
        ctx->kernel_launches += 5;
        int64_t n_runs = 0;
        cuda_check(cudaMemcpyAsync(&n_runs, d_runs->ptr, 8, cudaMemcpyDeviceToHost, st), "D2H join runs");
        cuda_check(cudaStreamSynchronize(st), "join runs sync");
        h_build_rows = (uint32_t)n;
        cuda_check(cudaMemcpyAsync((uint32_t*)run_start->ptr + n_runs, &h_build_rows, 4, cudaMemcpyHostToDevice, st), "H2D run end");
        size_t cap = 1024;
        while (cap < (size_t)n_runs * 2) cap <<= 1;
        slots = std::make_shared<DeviceBuf>(cap * 8);
        cuda_check(cudaMemsetAsync(slots->ptr, 0, cap * 8, st), "memset join table");
        table.keys = (const unsigned long long*)keys->ptr;
        table.rows = (const unsigned*)rows->ptr;
        table.run_start = (const unsigned*)run_start->ptr;
        table.slots = (unsigned long long*)slots->ptr;
        table.mask = cap - 1;
        table.words = W;
        for (int j = 0; j < cb::SK_MAX_WORDS; j++) table.nullmask[j] = nullmask[j];
        launch_join_insert(table, n_runs, st);
        cuda_check(cudaGetLastError(), "k_join_insert launch");
        ctx->kernel_launches++;
        ctx->check_device_errors();
    }

    // the lookups of probe batch `in`: `total` output rows to emit from it
    void probe_batch(Batch& in) {
        TraceSpan ts("join.probe");
        const int64_t n = in.n_rows;
        if (n >= ((int64_t)1 << 32)) throw Unsupported("a hash join probe batch of 2^32 rows or more");
        cudaStream_t st = ctx->stream;
        uint64_t h_and_or[2 * cb::SK_MAX_WORDS];
        std::vector<int> digits;
        DeviceBufP pk = pack_row_keys(key_cols(in, probe_keys, false), n, bits, ctx, h_and_or, digits);
        probe = std::move(in);
        pos = 0;
        if (type == JoinType::Inner) {
            const size_t n_chunks = (size_t)(n + CB_SCAN_CHUNK - 1) / CB_SCAN_CHUNK;
            run_of = std::make_shared<DeviceBuf>((size_t)n * 4);
            offs = std::make_shared<DeviceBuf>((size_t)n * 4);
            chunk_off = std::make_shared<DeviceBuf>((n_chunks + 1) * 4);
            auto tot = std::make_shared<DeviceBuf>(16);
            cuda_check(cudaMemsetAsync(tot->ptr, 0, 16, st), "memset join total");
            launch_join_probe(table, (const unsigned long long*)pk->ptr, n, CB_JOIN_COUNT, (unsigned*)offs->ptr, (unsigned*)run_of->ptr,
                              (unsigned long long*)tot->ptr, nullptr, st);
            launch_scan_u32((unsigned*)offs->ptr, n, CB_SCAN_CHUNK, (unsigned*)chunk_off->ptr, (long long*)tot->ptr + 1, st);
            cuda_check(cudaGetLastError(), "join probe");
            ctx->kernel_launches += 3;
            cuda_check(cudaMemcpyAsync(&total, tot->ptr, 8, cudaMemcpyDeviceToHost, st), "D2H join total");
            ctx->check_device_errors();
            // the scan's offsets are 32-bit
            if (total >= ((int64_t)1 << 32)) throw Unsupported("a probe batch whose inner join output has 2^32 rows or more (lower spark.comet.b200.chunkRows)");
        } else {
            const size_t nb = (size_t)(n + 1023) / 1024;
            auto keep = std::make_shared<DeviceBuf>((size_t)n + 16), iota = std::make_shared<DeviceBuf>((size_t)n * 4);
            auto counts = std::make_shared<DeviceBuf>(nb * 4 + 4), offsets = std::make_shared<DeviceBuf>(nb * 8 + 8), kept = std::make_shared<DeviceBuf>(8);
            kept_rows = std::make_shared<DeviceBuf>((size_t)n * 4);
            launch_join_probe(table, (const unsigned long long*)pk->ptr, n, type == JoinType::LeftSemi ? CB_JOIN_SEMI : CB_JOIN_ANTI, nullptr, nullptr, nullptr,
                              (unsigned char*)keep->ptr, st);
            launch_compact_plan((const unsigned char*)keep->ptr, n, (int*)counts->ptr, (long long*)offsets->ptr, (long long*)kept->ptr, st);
            launch_sort_iota((unsigned*)iota->ptr, n, st);
            launch_compact_scatter((const unsigned char*)keep->ptr, n, (const long long*)offsets->ptr, iota->ptr, 4, kept_rows->ptr, st);
            cuda_check(cudaGetLastError(), "join probe");
            ctx->kernel_launches += 5;
            cuda_check(cudaMemcpyAsync(&total, kept->ptr, 8, cudaMemcpyDeviceToHost, st), "D2H join kept rows");
            ctx->check_device_errors();
        }
    }

    // the next at most chunkRows output rows of the probe batch
    void emit(Batch& out) {
        const int64_t k = std::min<int64_t>(total - pos, std::max<int64_t>(ctx->chunk_rows, 1));
        if (type == JoinType::Inner) {
            auto pidx = std::make_shared<DeviceBuf>((size_t)k * 4), bidx = std::make_shared<DeviceBuf>((size_t)k * 4);
            launch_join_emit(table, (const unsigned*)run_of->ptr, (const unsigned*)offs->ptr, (const unsigned*)chunk_off->ptr, probe.n_rows, pos, pos + k,
                             (unsigned*)pidx->ptr, (unsigned*)bidx->ptr, ctx->stream);
            cuda_check(cudaGetLastError(), "k_join_emit launch");
            ctx->kernel_launches++;
            Batch pb, bb;
            gather_columns(probe, (const unsigned*)pidx->ptr, k, pb, ctx, "joining");
            gather_columns(build, (const unsigned*)bidx->ptr, k, bb, ctx, "joining");
            Batch& l = build_left ? bb : pb;
            Batch& r = build_left ? pb : bb;
            out.n_rows = k;
            out.cols = std::move(l.cols);
            for (auto& c : r.cols) out.cols.push_back(std::move(c));
        } else {
            gather_columns(probe, (const unsigned*)kept_rows->ptr + pos, k, out, ctx, "joining");
        }
        pos += k;
        ctx->join_out_rows += k;
        ctx->check_device_errors();
        if (pos >= total) { probe = Batch(); run_of.reset(); offs.reset(); chunk_off.reset(); kept_rows.reset(); }
    }

    bool next(Batch& out) override {
        if (!built) build_table();
        const bool empty_build = build.n_rows == 0;
        if (empty_build && type != JoinType::LeftAnti) return false; // nothing matches
        for (;;) {
            if (pos < total) { emit(out); return true; }
            Batch in;
            if (!probe_child->next(in)) return false;
            arrive(in);
            ctx->join_probe_rows += in.n_rows;
            if (in.n_rows == 0) continue;
            if (empty_build) { // anti: every probe row
                ctx->join_out_rows += in.n_rows;
                out = std::move(in);
                return true;
            }
            probe_batch(in);
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

// build_only: schema-only sources; `assume`: build-time value-range assumptions per source column (see make_agg_node)
static ExecNodeP build_node(const OperatorP& op, ExecContext* ctx, PlanInputs* inputs, bool build_only, const std::vector<int>& assume);

static ExecNodeP build_source(const OperatorP& op, ExecContext* ctx, PlanInputs* inputs, bool build_only, const std::vector<int>& assume) {
    const bool scan = op->kind == OpKind::Scan || op->kind == OpKind::ShuffleScan;
    if (build_only && (scan || op->kind == OpKind::NativeScan)) {
        auto s = std::make_shared<SchemaOnlySource>();
        s->schema = op->schema;
        return s;
    }
    if (scan) {
        if (inputs->streams.empty() && inputs->tables.empty()) throw PlanError("No input for scan");
        ArrowArrayStream* st = inputs->streams.empty() ? nullptr : inputs->streams.front();
        std::shared_ptr<DeviceTable> tb = inputs->tables.empty() ? nullptr : inputs->tables.front();
        if (!inputs->streams.empty()) inputs->streams.erase(inputs->streams.begin());
        if (!inputs->tables.empty()) inputs->tables.erase(inputs->tables.begin());
        if (tb) return std::make_shared<TableSource>(tb, op->schema, ctx);
        if (!st) throw PlanError("No input for scan");
        return std::make_shared<StreamSource>(ctx, st, op->schema);
    }
    if (op->kind == OpKind::NativeScan) return make_native_scan(op, ctx);
    return build_node(op, ctx, inputs, build_only, assume);
}

static ExecNodeP build_node(const OperatorP& op, ExecContext* ctx, PlanInputs* inputs, bool build_only, const std::vector<int>& assume) {
    OperatorP cur = op;
    OperatorP agg_op;
    if (cur->kind == OpKind::ShuffleWriter) {
        auto n = std::make_shared<PartitionNode>();
        n->ctx = ctx;
        n->child = build_node(cur->children[0], ctx, inputs, build_only, assume);
        n->schema = cur->schema;
        n->n_parts = cur->num_partitions;
        for (auto& e : cur->hash_exprs) {
            if (e->kind != ExprKind::Bound) throw Unsupported("computed hash-partition keys (only plain column keys)");
            n->key_cols.push_back(e->index);
        }
        if (n->key_cols.size() > 8) throw Unsupported("more than 8 hash-partition keys");
        if (n->n_parts > CB_MAX_HASH_PARTITIONS)
            throw Unsupported("hash partitioning into " + std::to_string(n->n_parts) + " partitions (at most " + std::to_string((int)CB_MAX_HASH_PARTITIONS) + ")");
        for (int ci : n->key_cols) { // refuses key types murmur3 has no rule for
            if (ci < 0 || ci >= (int)cur->schema.size()) throw PlanError("hash-partition key out of range");
            Column c;
            c.type = cur->schema[(size_t)ci];
            key_kind(c);
        }
        return n;
    }
    if (cur->kind == OpKind::Sort) {
        auto n = std::make_shared<SortNode>();
        n->ctx = ctx;
        n->child = build_node(cur->children[0], ctx, inputs, build_only, assume);
        n->schema = cur->schema;
        n->keys = cur->sort_keys;
        n->fetch = cur->fetch;
        n->skip = std::max<int64_t>(cur->skip, 0);
        for (auto& k : n->keys)
            if (k.expr->index < 0 || k.expr->index >= (int)cur->schema.size()) throw PlanError("sort key out of range");
        return n;
    }
    if (cur->kind == OpKind::HashJoin) {
        auto n = std::make_shared<JoinNode>();
        n->ctx = ctx;
        ExecNodeP left = build_node(cur->children[0], ctx, inputs, build_only, assume); // inputs are taken in Scan order: left first
        ExecNodeP right = build_node(cur->children[1], ctx, inputs, build_only, assume);
        n->schema = cur->schema;
        n->type = cur->join_type;
        n->build_left = cur->build_left;
        std::vector<int> lk, rk;
        std::vector<DType> key_types;
        for (size_t i = 0; i < cur->left_keys.size(); i++) {
            lk.push_back(cur->left_keys[i]->index);
            rk.push_back(cur->right_keys[i]->index);
            key_types.push_back(cur->left_keys[i]->type);
        }
        n->build_child = cur->build_left ? left : right;
        n->probe_child = cur->build_left ? right : left;
        n->build_keys = cur->build_left ? lk : rk;
        n->probe_keys = cur->build_left ? rk : lk;
        n->set_layout(key_types);
        return n;
    }
    if (cur->kind == OpKind::HashAgg) { agg_op = cur; cur = cur->children[0]; }
    std::vector<OperatorP> chain; // top-down
    while (cur->kind == OpKind::Filter || cur->kind == OpKind::Projection) { chain.push_back(cur); cur = cur->children[0]; }
    if (!agg_op && chain.empty()) return build_source(cur, ctx, inputs, build_only, assume);
    ExecNodeP src = build_source(cur, ctx, inputs, build_only, assume);
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
    if (agg_op) return make_agg_node(agg_op, src, preds, cols, ctx, assume);
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

ExecNodeP build_exec(const OperatorP& op, ExecContext* ctx, PlanInputs* inputs) { return build_node(op, ctx, inputs, false, {}); }

// the pipeline kernels of the tree under n, top-down; a join's left child before its right one
static void collect_kernels(ExecNodeP n, std::vector<GeneratedKernel>& out) {
    while (n) {
        if (auto f = std::dynamic_pointer_cast<FusedBase>(n)) {
            for (const PipelineSpec& s : f->build_specs()) out.push_back(generate_pipeline(s));
            n = f->child;
        } else if (auto pn = std::dynamic_pointer_cast<PartitionNode>(n)) {
            n = pn->child;
        } else if (auto jn = std::dynamic_pointer_cast<JoinNode>(n)) {
            collect_kernels(jn->build_left ? jn->build_child : jn->probe_child, out);
            n = jn->build_left ? jn->probe_child : jn->build_child;
        } else {
            auto sn = std::dynamic_pointer_cast<SortNode>(n);
            n = sn ? sn->child : nullptr;
        }
    }
}

std::vector<GeneratedKernel> plan_kernels_for_build(const OperatorP& op, const std::vector<int>& assume) {
    ExecContext defaults; // build-time tuning: the defaults (constructing one makes no CUDA call)
    std::vector<GeneratedKernel> out;
    collect_kernels(build_node(op, &defaults, nullptr, true, assume), out);
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

// Device columns whose values are not stored in the Arrow layout of their type get a converted copy (aot_kernels.h
// launch_to_arrow_layout): INT32-backed int8 / int16 are narrowed, decimals stored in 4 or 8 bytes are sign-extended to Decimal128, and
// bit-packed booleans are given one byte per row.  Idempotent: a converted column has the layout it reports.  Returns whether it launched.
bool to_arrow_layout(Batch& b, ExecContext* ctx) {
    const size_t n = (size_t)b.n_rows;
    bool launched = false;
    for (Column& c : b.cols) {
        if (c.on_host || c.is_dict || !c.data) continue;
        int conv = -1, w = 0;
        if (c.type.id == TypeId::Bool && c.phys == Phys::Bitmap) {
            if (c.bool_bytes) { c.data = c.bool_bytes; c.phys = Phys::I8; continue; }
            conv = CB_BITS_TO_BYTES; w = 1;
        } else if (c.type.is_decimal() && c.phys == Phys::I32) { conv = CB_SEXT32_TO_128; w = 16; }
        else if (c.type.is_decimal() && c.phys == Phys::I64) { conv = CB_SEXT64_TO_128; w = 16; }
        else if (c.type.id == TypeId::Int8 && c.phys == Phys::I32) { conv = CB_NARROW32_TO_8; w = 1; }
        else if (c.type.id == TypeId::Int16 && c.phys == Phys::I32) { conv = CB_NARROW32_TO_16; w = 2; }
        if (conv < 0) continue;
        auto out = std::make_shared<DeviceBuf>(std::max<size_t>(n, 1) * (size_t)w);
        launch_to_arrow_layout(conv, c.data->ptr, (long long)n, out->ptr, ctx->stream);
        cuda_check(cudaGetLastError(), "to_arrow_layout launch");
        ctx->kernel_launches++;
        launched = true;
        c.data = out;
        c.phys = w == 16 ? Phys::I128 : w == 2 ? Phys::I16 : Phys::I8;
        if (c.type.id == TypeId::Bool) c.bool_bytes = out;
    }
    return launched;
}

// rows [row0, row0 + n_rows) of batch b as Arrow C Data arrays (the caller's spark.comet.batchSize slices a large batch, CometConf.scala:539-544)
void export_batch(Batch& b, ExecContext* ctx, ArrowArray* out_arrays, ArrowSchema* out_schemas, int n_cols, int64_t row0, int64_t n_rows) {
    TraceSpan ts("export_batch");
    if ((int)b.cols.size() != n_cols) throw PlanError("executePlan: caller passed " + std::to_string(n_cols) + " output slots, plan produces " + std::to_string(b.cols.size()) + " columns");
    if (row0 < 0 || n_rows < 0 || row0 + n_rows > b.n_rows) throw PlanError("export_batch: slice out of range");
    to_arrow_layout(b, ctx);
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
            // dictionary-coded strings: fetch the codes (1, 2 or 4 bytes each, as the source delivered them), spell the strings out on the host
            const size_t cw = (size_t)phys_bytes(c.phys);
            std::vector<uint8_t> raw_codes(n * cw + 8);
            if (n) cuda_check(cudaMemcpyAsync(raw_codes.data(), (const uint8_t*)c.data->ptr + r0 * cw, n * cw, cudaMemcpyDeviceToHost, ctx->stream), "D2H key codes");
            cuda_check(cudaStreamSynchronize(ctx->stream), "D2H sync");
            ctx->d2h_bytes += (int64_t)(n * cw);
            std::vector<int32_t> codes(n + 1);
            for (size_t r = 0; r < n; r++)
                codes[r] = cw == 1 ? (int32_t)(int8_t)raw_codes[r] : cw == 2 ? (int32_t)((const int16_t*)raw_codes.data())[r] : ((const int32_t*)raw_codes.data())[r];
            std::vector<uint8_t> vb = c.validity && n ? fetch_bits(ctx, c.validity->ptr, row0, n) : std::vector<uint8_t>((n + 7) / 8 + 8, 0xff);
            offs.resize((n + 1) * 4);
            int32_t* o = (int32_t*)offs.data();
            o[0] = 0;
            for (size_t r = 0; r < n; r++) {
                bool valid = (vb[r >> 3] >> (r & 7)) & 1;
                if (valid) { const std::string& sv = c.dict->values().at((size_t)codes[r]); data.insert(data.end(), sv.begin(), sv.end()); }
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
