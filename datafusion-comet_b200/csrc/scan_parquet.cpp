// scan_parquet.cpp -- native Parquet scan (NativeScan -> DataSourceExec(ParquetSource),
// native/core/src/parquet/parquet_exec.rs:60-200): the device pipeline over the host plans of scan_plan.cpp.
//
// Footers and page headers are parsed on the host (parquet.cpp, scan_plan.cpp); encoded pages cross PCIe as they sit in the file and
// every value byte is decoded on the device (parquet_kernels.cu) -- but for strings (turned into dictionary codes on the host) and
// DELTA_BYTE_ARRAY decimals (sequential by construction, re-encoded as PLAIN on the host).  d(p<=18) / INT64 decimals stay 8 bytes wide in HBM (the Parquet
// physical width) and the fused kernels read them as such.
//
// Memory.  A scan owns two SLOTS that alternate between consecutive batches, so that batch k+1's encoded bytes cross PCIe
// (copy stream) while batch k is decoded (decode stream) and consumed (plan stream).  Every byte a slot needs lives in three
// blocks that are allocated ONCE -- sized from the footers before the first batch -- and come from a process-wide cache, so
// the next plan over a similar file set (the next task of the same stage) starts with warm blocks:
//   chunk : the encoded column chunks of the batch (device)
//   work  : decoded columns handed to the consumer + decode temporaries (device, bump-allocated per batch)
//   meta  : page tables / dictionary remaps on their way to the device (pinned host)
// Nothing is allocated, freed or synchronised per batch beyond the one wait for the batch itself.  (Round 1 took these
// buffers from cudaMallocAsync per batch; one such call was measured at 577 ms when the pool had to grow next to a
// framework that holds most of HBM -- the end-to-end step time was hostage to it.)
#include "exec.h"

#include "parquet_kernels.h"
#include "scan_plan.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>

namespace cb200 {

// =================================================================================================
// block cache: device / pinned blocks survive their scan and are handed to the next one
// =================================================================================================
namespace {

struct ScanBlock {
    int device = 0;
    bool pinned = false;
    uint8_t* ptr = nullptr;
    size_t cap = 0;
};
using ScanBlockP = std::shared_ptr<ScanBlock>;

struct BlockCache {
    std::mutex mu;
    std::vector<ScanBlock*> free_list;
    static constexpr size_t MAX_CACHED = 12; // 2 slots x 3 blocks of two live plan shapes

    static void destroy(ScanBlock* b) {
        if (b->ptr) {
            if (b->pinned) cudaFreeHost(b->ptr);
            else { cudaSetDevice(b->device); cudaFree(b->ptr); }
        }
        delete b;
    }
    void give_back(ScanBlock* b) {
        ScanBlock* victim = nullptr;
        {
            std::lock_guard<std::mutex> lk(mu);
            free_list.push_back(b);
            if (free_list.size() > MAX_CACHED) { // drop the smallest: the big blocks are the expensive ones to make again
                auto it = std::min_element(free_list.begin(), free_list.end(), [](ScanBlock* a, ScanBlock* c) { return a->cap < c->cap; });
                victim = *it;
                free_list.erase(it);
            }
        }
        if (victim) destroy(victim);
    }
    ScanBlockP acquire(int device, bool pinned, size_t bytes) {
        bytes = std::max<size_t>(bytes, 4096);
        ScanBlock* got = nullptr;
        {
            std::lock_guard<std::mutex> lk(mu);
            size_t best = free_list.size();
            for (size_t i = 0; i < free_list.size(); i++) {
                ScanBlock* b = free_list[i];
                if (b->pinned != pinned || (!pinned && b->device != device) || b->cap < bytes) continue;
                if (b->cap > 2 * bytes + ((size_t)64 << 20)) continue; // do not spend a 6 GB block on a 1 MB request
                if (best == free_list.size() || b->cap < free_list[best]->cap) best = i;
            }
            if (best != free_list.size()) { got = free_list[best]; free_list.erase(free_list.begin() + (long)best); }
        }
        if (!got) {
            got = new ScanBlock();
            got->device = device;
            got->pinned = pinned;
            got->cap = (bytes + ((size_t)2 << 20) - 1) / ((size_t)2 << 20) * ((size_t)2 << 20);
            // pinned blocks are MAPPED: kernels read the page tables straight out of them (see bind_batch), so the tables never
            // queue on the H2D copy engine behind the next batch's bulk transfer
            cudaError_t e = pinned ? cudaHostAlloc((void**)&got->ptr, got->cap, cudaHostAllocMapped | cudaHostAllocPortable) : cudaMalloc((void**)&got->ptr, got->cap);
            if (e != cudaSuccess) {
                size_t want = got->cap;
                delete got;
                cudaGetLastError();
                throw ExecError(2, "", std::string("parquet scan: cannot allocate ") + std::to_string(want) + (pinned ? " pinned host" : " device") + " bytes: " + cudaGetErrorString(e));
            }
        }
        return ScanBlockP(got, [this](ScanBlock* b) { give_back(b); });
    }
};
BlockCache& block_cache() {
    static BlockCache* c = new BlockCache(); // never destroyed: blocks may outlive static destruction order, the driver reclaims them at exit
    return *c;
}

// streams + events + pinned flags of one scan, pooled per device (creating them costs ~1-2 ms per plan)
struct ScanRes {
    cudaStream_t copy_stream = nullptr, decode_stream = nullptr;
    cudaEvent_t decoded[2] = {nullptr, nullptr}, uploaded[2] = {nullptr, nullptr}, done[2] = {nullptr, nullptr}, consumer = nullptr;
    int* h_flags = nullptr;
    // Snappy: the columns of a batch are decompressed side by side (a column's index pass has one warp per page -- a few hundred
    // warps -- and would leave most SMs idle if the columns queued behind each other on the decode stream)
    static constexpr int N_SIDE = 4;
    cudaStream_t side[N_SIDE] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t side_begin = nullptr, side_done[N_SIDE] = {nullptr, nullptr, nullptr, nullptr};
};
std::mutex g_res_mu;
std::map<int, std::vector<ScanRes>> g_res_pool;

ScanRes acquire_res(int device) {
    {
        std::lock_guard<std::mutex> lk(g_res_mu);
        auto& fl = g_res_pool[device];
        if (!fl.empty()) { ScanRes r = fl.back(); fl.pop_back(); return r; }
    }
    ScanRes r;
    cuda_check(cudaStreamCreateWithFlags(&r.copy_stream, cudaStreamNonBlocking), "copy stream");
    cuda_check(cudaStreamCreateWithFlags(&r.decode_stream, cudaStreamNonBlocking), "decode stream");
    for (int i = 0; i < 2; i++) {
        cuda_check(cudaEventCreateWithFlags(&r.decoded[i], cudaEventDisableTiming), "event");
        cuda_check(cudaEventCreateWithFlags(&r.uploaded[i], cudaEventDisableTiming), "event");
        cuda_check(cudaEventCreateWithFlags(&r.done[i], cudaEventDisableTiming), "event");
    }
    cuda_check(cudaEventCreateWithFlags(&r.consumer, cudaEventDisableTiming), "event");
    cuda_check(cudaEventCreateWithFlags(&r.side_begin, cudaEventDisableTiming), "event");
    for (int i = 0; i < ScanRes::N_SIDE; i++) {
        cuda_check(cudaStreamCreateWithFlags(&r.side[i], cudaStreamNonBlocking), "side stream");
        cuda_check(cudaEventCreateWithFlags(&r.side_done[i], cudaEventDisableTiming), "event");
    }
    cuda_check(cudaMallocHost((void**)&r.h_flags, 64), "cudaMallocHost flags");
    return r;
}
void release_res(int device, const ScanRes& r) {
    std::lock_guard<std::mutex> lk(g_res_mu);
    g_res_pool[device].push_back(r);
}

} // namespace

// =================================================================================================
// the scan
// =================================================================================================
struct NativeScanSource : ExecNode {
    ExecContext* ctx;
    std::vector<std::string> files;
    std::vector<int64_t> file_start, file_length; // SparkPartitionedFile.start / length (0/0 = whole file)
    std::vector<StructField> fields;
    std::vector<ExprP> data_filters;

    std::vector<ScanFile> open_files;
    std::vector<FILE*> fh;                  // per file: its handle when the bytes are read from disk
    std::vector<Unit> all_units;
    BatchPlan plan;
    size_t next_batch = 0;
    bool opened = false;
    std::vector<DictionaryP> dicts;         // per column: the plan-wide dictionary of a string column

    struct Slot {
        ScanBlockP chunk, work, meta, staging;
        size_t work_used = 0, meta_used = 0;
        bool used = false;
        uint8_t* meta_dev = nullptr;        // the current batch's device mirror of the pinned page tables (in the work block)
        int* derr = nullptr;                // the current batch's decode error bits (PqErr)
    };
    Slot slots[2];
    ScanRes res;
    bool have_res = false;

    struct Prepared {
        Batch batch;
        int slot = 0;
        cudaEvent_t tr[4] = {nullptr, nullptr, nullptr, nullptr}; // CB200_TRACE: copy-stream begin/end, decode-stream begin/end
        ~Prepared() { for (auto e : tr) if (e) cudaEventDestroy(e); }
    };
    std::unique_ptr<Prepared> pending;
    int64_t n_issued = 0;

    void push_filters(const std::vector<ExprP>& preds) override {
        if (!opened) for (auto& p : preds) data_filters.push_back(p);
    }

    ~NativeScanSource() override {
        if (have_res) {
            cudaStreamSynchronize(res.copy_stream);
            cudaStreamSynchronize(res.decode_stream);
            release_res(ctx->device, res);
        }
        pending.reset();
        for (FILE* f : fh) if (f) fclose(f);
    }

    // ---- open: footers, pruning, batch plan, block sizes ---------------------------------------------------------------------
    void open_all() {
        TraceSpan ts("parquet.open");
        std::vector<PruneTerm> terms;
        const bool prune = getenv("CB200_NO_PRUNE") ? atoi(getenv("CB200_NO_PRUNE")) == 0 : true;
        if (prune) for (auto& f : data_filters) collect_prune_terms(f, terms);
        for (auto& path : files) {
            open_files.push_back(open_scan_file(path, fields));
            fh.push_back(open_files.back().mem ? nullptr : fopen(strip_file_scheme(path).c_str(), "rb"));
            if (!open_files.back().mem && !fh.back()) throw ExecError(3, "", "parquet: cannot open " + path);
        }
        Selection sel = select_row_groups(open_files, file_start, file_length, fields.size(), terms);
        all_units = std::move(sel.units);
        const PageSelection ps = select_pages(all_units, open_files, fields.size(), terms);
        for (size_t c = 0; c < fields.size(); c++) dicts.push_back(std::make_shared<Dictionary>());
        plan = plan_batches(all_units, open_files, fields, ctx->chunk_rows);
        if (trace_on()) fprintf(stderr, "[cb200 trace]   parquet scan: %zu row groups in %zu batches (%lld pruned by statistics, %lld data pages by the page index), chunk block %.1f MB, work block %.1f MB per slot\n",
                                all_units.size(), plan.batches.size(), (long long)sel.pruned_row_groups, (long long)ps.pruned_pages, plan.chunk_need / 1e6, plan.work_estimate / 1e6);
        ctx->scan_pruned_row_groups += sel.pruned_row_groups;
        ctx->scan_pruned_rows += sel.pruned_rows;
        ctx->scan_pruned_pages += ps.pruned_pages;
        ctx->scan_page_pruned_rows += ps.pruned_rows;
        opened = true;
    }

    void ensure_resources() {
        if (have_res) return;
        res = acquire_res(ctx->device);
        have_res = true;
        // a cached block may have been released by another plan whose last kernels are still in flight on ITS stream
        cuda_check(cudaDeviceSynchronize(), "scan start sync");
        for (auto& sl : slots) {
            sl.chunk = block_cache().acquire(ctx->device, false, plan.chunk_need);
            sl.work = block_cache().acquire(ctx->device, false, plan.work_estimate);
            sl.meta = block_cache().acquire(ctx->device, true, (size_t)4 << 20);
        }
    }

    uint8_t* meta_take(Slot& sl, size_t bytes) {
        bytes = align_up(bytes, 64);
        if (sl.meta_used + bytes > sl.meta->cap) throw ExecError(15, "", "internal: page-table block overflow");
        uint8_t* p = sl.meta->ptr + sl.meta_used;
        sl.meta_used += bytes;
        return p;
    }

    // ---- one batch ----------------------------------------------------------------------------------------------------------------
    std::unique_ptr<Prepared> issue() {
        if (next_batch >= plan.batches.size()) return nullptr;
        TraceSpan ts("parquet.issue");
        ensure_resources();
        auto pr = std::make_unique<Prepared>();
        pr->slot = (int)(n_issued++ & 1);
        const int si = pr->slot;
        Slot& sl = slots[si];
        const std::vector<Unit> units = batch_units(all_units, plan.batches[next_batch++]);
        const int64_t total = units.back().row0 + units.back().rows;
        Batch& out = pr->batch;
        out.n_rows = total;
        out.cols.assign(fields.size(), Column());
        const UploadPlan up = plan_uploads(units, open_files, fields.size());
        reuse_slot(si, up);
        if (trace_on()) {
            for (auto& e : pr->tr) cuda_check(cudaEventCreate(&e), "event");
            cuda_check(cudaEventRecord(pr->tr[0], res.copy_stream), "event record");
            cuda_check(cudaEventRecord(pr->tr[2], res.decode_stream), "event record");
        }
        double tt = now_ms();
        const std::vector<std::vector<ChunkLoc>> loc = upload(up, si);
        const double t_h2d = now_ms() - tt;
        // phase A: page tables on the host (reads only page headers)
        tt = now_ms();
        std::vector<ColPlan> plans;
        for (size_t c = 0; c < fields.size(); c++) plans.push_back(plan_column(open_files, fields[c], c, units, total, loc[c], dicts[c]));
        bind_buffers(plans, total, sl);
        const double t_pages = now_ms() - tt;
        // phase B: decode kernels
        tt = now_ms();
        launch(plans, total, out, si);
        const double t_launch = now_ms() - tt;
        if (trace_on()) fprintf(stderr, "[cb200 trace]   issue breakdown: h2d enqueue (%zu ranges) %.3f  page tables %.3f  launches %.3f ms; work %.1f MB\n", up.ranges.size(), t_h2d, t_pages, t_launch, sl.work_used / 1e6);
        cuda_check(cudaEventRecord(res.decoded[si], res.decode_stream), "event record");
        if (trace_on()) {
            cuda_check(cudaEventRecord(pr->tr[1], res.copy_stream), "event record");
            cuda_check(cudaEventRecord(pr->tr[3], res.decode_stream), "event record");
        }
        sl.used = true;
        cuda_check(cudaMemcpyAsync(&res.h_flags[si], sl.derr, 4, cudaMemcpyDeviceToHost, res.decode_stream), "parquet err");
        cuda_check(cudaEventRecord(res.done[si], res.decode_stream), "event record");
        return pr;
    }

    // everything queued on the slot two batches ago must be done with its blocks; the chunk / staging blocks must hold this batch
    void reuse_slot(int si, const UploadPlan& up) {
        Slot& sl = slots[si];
        if (sl.used) {
            cuda_check(cudaEventSynchronize(res.decoded[si]), "slot reuse"); // page tables / staging on the host side; long done (two batches back)
            cuda_check(cudaStreamWaitEvent(res.copy_stream, res.decoded[si], 0), "stream wait");
        }
        // the consumer's kernels over the slot's previous batch were queued before this call (the caller asks for batch k+1 only
        // when it is finished with batch k-1): order the decode stream behind them
        cuda_check(cudaEventRecord(res.consumer, ctx->stream), "event record");
        cuda_check(cudaStreamWaitEvent(res.decode_stream, res.consumer, 0), "stream wait");
        if (up.dev_total + 64 > sl.chunk->cap) { // cannot happen when the footers are honest; grow rather than fail
            cuda_check(cudaStreamSynchronize(res.copy_stream), "chunk growth");
            sl.chunk = block_cache().acquire(ctx->device, false, up.dev_total + up.dev_total / 8 + 65536);
        }
        bool any_file = false;
        for (auto& r : up.ranges) if (!open_files[r.file].mem) any_file = true;
        if (any_file && (!sl.staging || sl.staging->cap < up.dev_total)) sl.staging = block_cache().acquire(ctx->device, true, up.dev_total + up.dev_total / 8);
        sl.meta_used = 0;
        sl.work_used = 0;
    }

    // the batch's byte ranges onto the copy stream (ranges of files on disk are read into the pinned staging block first);
    // returns where every column chunk sits, [column][unit]
    std::vector<std::vector<ChunkLoc>> upload(const UploadPlan& up, int si) {
        Slot& sl = slots[si];
        auto host_of = [&](const UploadRange& r) -> const uint8_t* {
            const ScanFile& f = open_files[r.file];
            return f.mem ? f.mem + r.start : sl.staging->ptr + r.dev_off;
        };
        for (auto& r : up.ranges) {
            const size_t len = (size_t)(r.end - r.start);
            FILE* f = fh[r.file];
            if (f && (fseeko(f, (off_t)r.start, SEEK_SET) != 0 || fread(sl.staging->ptr + r.dev_off, 1, len, f) != len)) throw ExecError(3, "", "parquet: short read");
            cuda_check(cudaMemcpyAsync(sl.chunk->ptr + r.dev_off, host_of(r), len, cudaMemcpyHostToDevice, res.copy_stream), "H2D parquet range");
            ctx->h2d_bytes += (int64_t)len;
        }
        cuda_check(cudaEventRecord(res.uploaded[si], res.copy_stream), "event record");
        std::vector<std::vector<ChunkLoc>> loc(fields.size());
        for (size_t c = 0; c < fields.size(); c++) loc[c] = locate_chunks(up, c, host_of, sl.chunk->ptr);
        return loc;
    }

    // one bump allocation in the work block per device buffer, sized now that every page is known; page tables into the pinned block
    void bind_buffers(std::vector<ColPlan>& plans, int64_t total, Slot& sl) {
        size_t need = 1024, meta_need = 4096;
        for (auto& p : plans) meta_need += align_up(p.pages.size() * sizeof(PqPage), 64) + align_up(p.remap.size() * 4, 64) + align_up(p.hostdec.size(), 64) + align_up(p.segs.size() * sizeof(PqSeg), 64) + 256;
        std::vector<std::pair<uint8_t**, size_t>> reqs;
        uint8_t* derr = nullptr;
        reqs.push_back({&derr, 64});
        reqs.push_back({&sl.meta_dev, meta_need});
        for (auto& p : plans) buffer_requests(p, total, reqs);
        for (auto& r : reqs) need += align_up(r.second, 256) + 256;
        if (need > sl.work->cap) {
            // the estimate from the footers was short (unusual page / run structure): take a bigger block.  The old one stays alive
            // as long as a batch handed to the consumer still points into it.
            if (trace_on()) fprintf(stderr, "[cb200 trace]   work block grows %.1f -> %.1f MB\n", sl.work->cap / 1e6, (need + need / 8) / 1e6);
            sl.work = block_cache().acquire(ctx->device, false, need + need / 8);
            plan.work_estimate = std::max(plan.work_estimate, need + need / 8);
        }
        if (meta_need > sl.meta->cap) sl.meta = block_cache().acquire(ctx->device, true, meta_need + meta_need / 4);
        size_t off = 0;
        for (auto& r : reqs) { *r.first = sl.work->ptr + off; off += align_up(r.second, 256) + 256; }
        sl.work_used = off;
        sl.derr = (int*)derr;
        // tables: staged in the pinned block, pulled into the device mirror by ONE kernel that reads the mapped host memory.  (An
        // H2D memcpy would share the copy engine with the bulk transfer of the NEXT batch, which is already queued: measured,
        // every batch's decode then started a whole transfer late -- 17.7 ms per batch instead of the 14.75 ms the bytes take.)
        for (auto& p : plans) stage_tables(p, sl);
    }

    // `bytes` into the slot's pinned block; returns their address in the device mirror
    uint8_t* stage(Slot& sl, const void* p, size_t bytes) {
        uint8_t* pin = meta_take(sl, bytes);
        memcpy(pin, p, bytes);
        return sl.meta_dev + (pin - sl.meta->ptr);
    }

    // host-produced page bodies, page descriptors and the string dictionary remap of one column
    void stage_tables(ColPlan& cp, Slot& sl) {
        if (cp.pages.empty()) return;
        uint8_t* hostdec_dev = cp.hostdec.empty() ? nullptr : stage(sl, cp.hostdec.data(), cp.hostdec.size());
        std::vector<uint8_t>().swap(cp.hostdec);
        resolve_bodies(cp, hostdec_dev);
        cp.dpd = stage(sl, cp.pages.data(), cp.pages.size() * sizeof(PqPage));
        if (!cp.remap.empty()) cp.ddict = stage(sl, cp.remap.data(), cp.remap.size() * 4);
        if (!cp.segs.empty()) cp.dsegs = stage(sl, cp.segs.data(), cp.segs.size() * sizeof(PqSeg));
    }

    void launch(std::vector<ColPlan>& plans, int64_t total, Batch& out, int si) {
        Slot& sl = slots[si];
        cuda_check(cudaMemsetAsync(sl.derr, 0, 64, res.decode_stream), "memset parquet err");
        void* meta_host_dev = nullptr;
        cuda_check(cudaHostGetDevicePointer(&meta_host_dev, sl.meta->ptr, 0), "cudaHostGetDevicePointer");
        launch_pq_copy(sl.meta_dev, meta_host_dev, align_up(sl.meta_used, 16), res.decode_stream);
        ctx->kernel_launches++;
        cuda_check(cudaStreamWaitEvent(res.decode_stream, res.uploaded[si], 0), "stream wait"); // decode kernels start when the batch has landed
        launch_snappy(plans, sl.derr);
        for (size_t c = 0; c < fields.size(); c++) launch_column(c, plans[c], total, out.cols[c], sl);
    }

    // compressed columns first, spread over the side streams; the decode stream carries on when all of them are done
    void launch_snappy(std::vector<ColPlan>& plans, int* derr) {
        bool used[ScanRes::N_SIDE] = {false, false, false, false};
        int k = 0;
        for (auto& cp : plans) {
            if (!cp.any_compressed || cp.pages.empty()) continue;
            if (k == 0) cuda_check(cudaEventRecord(res.side_begin, res.decode_stream), "event record");
            const int sid = k++ % ScanRes::N_SIDE;
            if (!used[sid]) { cuda_check(cudaStreamWaitEvent(res.side[sid], res.side_begin, 0), "stream wait"); used[sid] = true; }
            launch_pq_snappy_segmented((PqPage*)cp.dpd, (int)cp.pages.size(), (unsigned*)cp.dckpt, (int)cp.n_segs_total, derr, res.side[sid]);
            ctx->kernel_launches += 3;
        }
        for (int i = 0; i < ScanRes::N_SIDE; i++) {
            if (!used[i]) continue;
            cuda_check(cudaEventRecord(res.side_done[i], res.side[i]), "event record");
            cuda_check(cudaStreamWaitEvent(res.decode_stream, res.side_done[i], 0), "stream wait");
        }
    }

    bool next(Batch& out) override {
        TraceSpan ts("parquet.next");
        if (!opened) open_all();
        std::unique_ptr<Prepared> cur = pending ? std::move(pending) : issue();
        if (!cur) return false;
        pending = issue(); // prefetch: its H2D overlaps this batch's decode + the consumer's kernels
        cuda_check(cudaEventSynchronize(res.done[cur->slot]), "parquet decode sync");
        if (trace_on() && cur->tr[0]) {
            cudaEventSynchronize(cur->tr[1]);
            float h2d = 0, dec = 0, lag = 0;
            cudaEventElapsedTime(&h2d, cur->tr[0], cur->tr[1]);
            cudaEventElapsedTime(&dec, cur->tr[2], cur->tr[3]);
            cudaEventElapsedTime(&lag, cur->tr[0], cur->tr[3]);
            fprintf(stderr, "[cb200 trace]   batch of %lld rows: copy stream %.3f ms, decode stream (waits + decode) %.3f ms, first upload -> decoded %.3f ms\n",
                    (long long)cur->batch.n_rows, h2d, dec, lag);
        }
        const int perr = res.h_flags[cur->slot];
        if (perr & PQ_ERR_NULL_ON_FAST_PATH) throw PlanError("parquet: a column chunk whose statistics say null_count = 0 contains NULLs (corrupt statistics)");
        if (perr & PQ_ERR_SNAPPY) throw PlanError("parquet: malformed Snappy page");
        if (perr & PQ_ERR_DICT_INDEX) throw ExecError(3, "", "parquet: dictionary index out of range (corrupt page)");
        if (perr & PQ_ERR_DELTA) throw PlanError("parquet: malformed DELTA_BINARY_PACKED page (block sizes, bit width, value count or a body past the page)");
        if (perr & PQ_ERR_BSS) throw PlanError("parquet: BYTE_STREAM_SPLIT page whose size is not (non-null values) x (value width)");
        if (perr & PQ_ERR_TRUNCATED) throw PlanError("parquet: truncated page (fewer encoded values than the page header declares)");
        if (perr & PQ_ERR_RLE) throw PlanError("parquet: malformed RLE / bit-packed stream (dictionary indices or definition levels)");
        out = std::move(cur->batch);
        return true;
    }

    DeviceBufP view(const Slot& sl, void* p, size_t bytes) const {
        auto b = std::make_shared<DeviceBuf>(p, bytes);
        b->owner = sl.work; // the block lives as long as a batch points into it
        return b;
    }

    void launch_column(size_t c, ColPlan& cp, int64_t total, Column& col, Slot& sl) {
        col.type = fields[c].type;
        col.phys = cp.phys;
        col.is_dict = cp.dict != nullptr;
        col.dict = cp.dict;
        col.data = view(sl, cp.out, cp.out_bytes);
        if (cp.pages.empty()) return;
        const cudaStream_t ds = res.decode_stream;
        int* derr = sl.derr;
        const int n_all = (int)cp.pages.size(), n_data = (int)cp.n_data;
        PqPage* data_pages = (PqPage*)cp.dpd;
        const PqPage* dict_pages = data_pages + n_data;
        uint8_t* dense = cp.null_aware ? cp.dense : !cp.segs.empty() ? cp.dcov : cp.out; // page-pruned: decoded into covered rows first
        launch_pq_resolve(data_pages, n_all, derr, ds);
        ctx->kernel_launches++;
        if (cp.n_dict_pages) { launch_pq_plain(dict_pages, (int)cp.n_dict_pages, cp.conv, cp.type_length, cp.ddict, derr, ds); ctx->kernel_launches++; }
        if (cp.optional && !cp.null_aware) { launch_pq_check_def_levels(data_pages, n_data, derr, ds); ctx->kernel_launches++; }
        if (cp.null_aware) {
            launch_pq_def_levels(data_pages, n_data, (PqRun*)cp.druns, (int*)cp.dcounts, cp.dvalid, (unsigned*)cp.didx, derr, ds);
            ctx->kernel_launches += 4;
            col.validity = view(sl, cp.validity, cp.validity_bytes);
            col.null_count = -1;
        }
        if (cp.conv >= 0) { launch_pq_plain(data_pages, n_data, cp.conv, cp.type_length, dense, derr, ds); ctx->kernel_launches++; }
        if (cp.run_base > 0) {
            launch_pq_rle_scan(data_pages, n_data, (PqRun*)cp.runs, (int*)cp.counts, derr, ds);
            launch_pq_rle_decode(data_pages, n_data, (const PqRun*)cp.runs, (const int*)cp.counts, cp.ddict, cp.out_w, dense, derr, ds);
            ctx->kernel_launches += 3;
        }
        if (cp.mb_base > 0) { // DELTA_BINARY_PACKED pages: header walk, miniblock sums, carries, decode
            launch_pq_dbp(data_pages, n_data, (PqMiniblock*)cp.dmb, cp.conv, dense, derr, ds);
            ctx->kernel_launches += 4;
        }
        if (!cp.segs.empty()) {
            launch_pq_select((const PqSeg*)cp.dsegs, (int)cp.segs.size(), total, cp.null_aware ? cp.dvalid : nullptr, (const unsigned*)cp.didx, dense, cp.out,
                             (unsigned*)cp.validity, cp.out_w, ds);
            ctx->kernel_launches++;
        } else if (cp.null_aware) {
            launch_pq_scatter(cp.dvalid, (const unsigned*)cp.didx, dense, cp.out, (unsigned*)cp.validity, total, cp.out_w, ds);
            ctx->kernel_launches++;
        }
    }
};

ExecNodeP make_native_scan(const OperatorP& op, ExecContext* ctx) {
    auto s = std::make_shared<NativeScanSource>();
    s->ctx = ctx;
    s->schema = op->schema;
    s->files = op->files;
    s->file_start = op->file_start;
    s->file_length = op->file_length;
    s->fields = op->required_schema;
    s->data_filters = op->data_filters;
    return s;
}

} // namespace cb200
