// abi.cpp -- extern "C" surface of libcomet_b200.so (include/comet_b200.h).
#include "../../include/comet_b200.h"

#include "abi_internal.h"
#include "parquet_kernels.h"
#include "exec_internal.h"
#include "jit.h"
#include "plan.h"
#include "proto_wire.h"

#include <cstring>
#include <functional>
#include <map>
#include <mutex>

using namespace cb200;

namespace {

struct CtxRes {
    cudaStream_t stream;
    int* d_err;
    int* h_err;
    cudaEvent_t ev0, ev1;
};
std::mutex g_pool_mu;
std::map<int, std::vector<CtxRes>> g_pool;

void parse_config(const uint8_t* cfg, size_t len, ExecContext& ctx) { // config.proto ConfigMap
    if (!cfg || !len) return;
    PbReader r(cfg, len);
    while (r.next()) {
        if (r.field != 1 || r.wire != 2) { r.skip(); continue; }
        PbReader e = r.sub();
        std::string k, v;
        while (e.next()) {
            if (e.field == 1) k = e.bytes();
            else if (e.field == 2) v = e.bytes();
            else e.skip();
        }
        if (k == "spark.comet.b200.chunkRows") ctx.chunk_rows = std::max<int64_t>(1024, atoll(v.c_str()));
        else if (k == "spark.comet.batchSize") ctx.batch_size = atoi(v.c_str()); // CometConf.scala:539
        else if (k == "spark.comet.b200.streamAgg.minRows") ctx.stream_agg_min_rows = atoll(v.c_str());
        else if (k == "spark.comet.b200.streamAgg.maxRatio") ctx.stream_agg_max_ratio = atof(v.c_str());
        else if (k == "spark.comet.b200.hashThreads") { int t = atoi(v.c_str()); if (t == 256 || t == 512 || t == 768 || t == 960) ctx.hash_threads = t; } // + the producer warp <= 1024 threads per CTA
    }
}

void start(cb200_plan* p) {
    if (p->started) return;
    TraceSpan ts("plan.start");
    ExecContext& ctx = p->ctx;
    cuda_check(cudaSetDevice(ctx.device), "cudaSetDevice");
    {
        // cudaGetDeviceProperties costs 2-6 ms per call (it walks the whole property table, PCI topology included): two
        // attributes, queried once per device, are all a plan needs
        struct DevInfo { int major = 0, minor = 0, sms = 0; bool known = false; };
        static DevInfo info[64];
        static std::mutex info_mu;
        std::lock_guard<std::mutex> lk(info_mu);
        if (ctx.device < 0 || ctx.device >= 64) throw ExecError(CB200_ERR_CUDA, "", "device ordinal out of range");
        DevInfo& di = info[ctx.device];
        if (!di.known) {
            cuda_check(cudaDeviceGetAttribute(&di.major, cudaDevAttrComputeCapabilityMajor, ctx.device), "cudaDeviceGetAttribute");
            cuda_check(cudaDeviceGetAttribute(&di.minor, cudaDevAttrComputeCapabilityMinor, ctx.device), "cudaDeviceGetAttribute");
            cuda_check(cudaDeviceGetAttribute(&di.sms, cudaDevAttrMultiProcessorCount, ctx.device), "cudaDeviceGetAttribute");
            di.known = true;
        }
        // sm_90a code runs on compute capability 9.0 only: the `a` features (and the cubins) do not carry forward
        if (di.major != 9 || di.minor != 0) throw ExecError(CB200_ERR_CUDA, "", "comet_b200 kernels are built for sm_90a; device is sm_" + std::to_string(di.major * 10 + di.minor));
        ctx.num_sms = di.sms;
    }
    {
        // per-plan CUDA resources come from a per-device free list: creating a stream, events and pinned /
        // device scratch costs ~2 ms per plan, which matters when a plan runs for 10 ms
        std::lock_guard<std::mutex> lk(g_pool_mu);
        auto& fl = g_pool[ctx.device];
        if (!fl.empty()) {
            CtxRes r = fl.back();
            fl.pop_back();
            ctx.stream = r.stream; ctx.d_err = r.d_err; ctx.h_err = r.h_err; ctx.ev0 = r.ev0; ctx.ev1 = r.ev1;
        }
    }
    if (!ctx.stream) {
        cuda_check(cudaStreamCreateWithFlags(&ctx.stream, cudaStreamNonBlocking), "cudaStreamCreate");
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, ctx.device) == cudaSuccess) {
            unsigned long long keep = ~0ull; // keep freed blocks cached in the pool
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
        cuda_check(cudaMalloc((void**)&ctx.d_err, 64), "cudaMalloc err");
        cuda_check(cudaMallocHost((void**)&ctx.h_err, 64), "cudaMallocHost err");
        cuda_check(cudaEventCreate(&ctx.ev0), "cudaEventCreate");
        cuda_check(cudaEventCreate(&ctx.ev1), "cudaEventCreate");
    }
    cuda_check(cudaMemsetAsync(ctx.d_err, 0, 64, ctx.stream), "memset err");
    set_alloc_stream(ctx.stream);
    p->root = build_exec(p->op, &ctx, &p->inputs);
    p->started = true;
}

DType dtype_from_ids(int type_id, int precision, int scale) {
    if (type_id < 0 || type_id > 13) throw Unsupported("type id " + std::to_string(type_id));
    DType d;
    d.id = (TypeId)type_id;
    d.precision = precision;
    d.scale = scale;
    return d;
}

} // namespace

extern "C" {

const char* cb200_version(void) { return "comet_b200 0.1.0 (sm_90a; reference apache/datafusion-comet 1.1.0 @2699f59b)"; }

int cb200_supports(const uint8_t* op_proto, size_t op_len, cb200_error* why) {
    return cb200_guarded(why, [&]() -> int {
        OperatorP op = decode_plan(op_proto, op_len);
        plan_kernels_for_build(op); // exercises fusion + code generation rules
        return 1;
    }, 0);
}

cb200_plan* cb200_create_plan(const uint8_t* op_proto, size_t op_len, const uint8_t* cfg_proto, size_t cfg_len, struct ArrowArrayStream** inputs,
                              int32_t n_inputs, int32_t partition, int32_t partition_count, int32_t batch_size, int32_t device_ordinal, cb200_error* err) {
    TraceSpan ts("create_plan");
    return cb200_guarded(err, [&]() -> cb200_plan* {
        auto p = std::unique_ptr<cb200_plan>(new cb200_plan());
        p->op = decode_plan(op_proto, op_len);
        p->ctx.device = device_ordinal;
        if (batch_size > 0) p->ctx.batch_size = batch_size;
        parse_config(cfg_proto, cfg_len, p->ctx);
        p->partition = partition;
        p->partition_count = partition_count;
        for (int i = 0; i < n_inputs; i++) {
            p->inputs.streams.push_back(inputs ? inputs[i] : nullptr);
            p->inputs.tables.push_back(nullptr);
        }
        return p.release();
    }, (cb200_plan*)nullptr);
}

int32_t cb200_plan_num_columns(cb200_plan* plan) { return plan ? (int32_t)plan->op->schema.size() : -1; }

static int64_t execute_common(cb200_plan* plan, cb200_error* err, const std::function<void(Batch&)>& sink) {
    TraceSpan ts("execute");
    return cb200_guarded(err, [&]() -> int64_t {
        if (!plan) throw PlanError("null plan handle");
        if (plan->finished) return -1;
        start(plan);
        cuda_check(cudaSetDevice(plan->ctx.device), "cudaSetDevice");
        set_alloc_stream(plan->ctx.stream);
        Batch b;
        if (!plan->root->next(b)) { plan->finished = true; return -1; }
        plan->last = std::move(b);
        sink(plan->last);
        return plan->last.n_rows;
    }, (int64_t)-2);
}

// A batch the plan produced is handed to the caller in slices of at most spark.comet.batchSize rows (CometConf.scala:539-544; the JVM side
// sizes its vectors for that), each a zero-offset Arrow batch like prepare_output's (jni_api.rs:674-742).
int64_t cb200_execute(cb200_plan* plan, struct ArrowArray* out_arrays, struct ArrowSchema* out_schemas, int32_t n_cols, cb200_error* err) {
    if (plan && plan->export_pending) {
        TraceSpan ts("execute(slice)");
        return cb200_guarded(err, [&]() -> int64_t {
            cuda_check(cudaSetDevice(plan->ctx.device), "cudaSetDevice");
            set_alloc_stream(plan->ctx.stream);
            const int64_t n = std::min<int64_t>(std::max(plan->ctx.batch_size, 1), plan->last.n_rows - plan->export_pos);
            export_batch(plan->last, &plan->ctx, out_arrays, out_schemas, n_cols, plan->export_pos, n);
            plan->export_pos += n;
            plan->export_pending = plan->export_pos < plan->last.n_rows;
            return n;
        }, (int64_t)-2);
    }
    int64_t first = 0;
    const int64_t rc = execute_common(plan, err, [&](Batch& b) {
        // a ShuffleWriter's batch is one unit: cb200_plan_partition_starts / cb200_exchange address its rows by partition offsets
        const bool whole = plan->op->kind == OpKind::ShuffleWriter;
        first = whole ? b.n_rows : std::min<int64_t>(std::max(plan->ctx.batch_size, 1), b.n_rows);
        export_batch(b, &plan->ctx, out_arrays, out_schemas, n_cols, 0, first);
        plan->export_pos = first;
        plan->export_pending = first < b.n_rows;
    });
    return rc < 0 ? rc : first;
}

int64_t cb200_execute_device(cb200_plan* plan, cb200_device_column* cols, int32_t n_cols, cb200_error* err) {
    if (plan && plan->export_pending)
        return cb200_guarded(err, [&]() -> int64_t { throw PlanError("cb200_execute_device: the current batch is still being handed out by cb200_execute"); }, (int64_t)-2);
    return execute_common(plan, err, [&](Batch& b) {
        if ((int)b.cols.size() != n_cols) throw PlanError("execute_device: plan produces " + std::to_string(b.cols.size()) + " columns");
        if (to_arrow_layout(b, &plan->ctx)) cuda_check(cudaStreamSynchronize(plan->ctx.stream), "to_arrow_layout"); // the caller reads the columns on its own stream
        for (int i = 0; i < n_cols; i++) {
            Column& c = b.cols[(size_t)i];
            cb200_device_column& o = cols[i];
            memset(&o, 0, sizeof(o));
            o.type_id = (int)c.type.id;
            o.precision = c.type.precision;
            o.scale = c.type.scale;
            o.value_width = c.type.id == TypeId::Bool ? 1 : c.type.arrow_width();
            if (c.on_host) {
                o.host_values = c.h_data.data();
                o.host_validity_bytes = c.h_valid.empty() ? nullptr : c.h_valid.data();
            } else {
                o.values = c.data ? c.data->ptr : nullptr;
                o.validity = c.validity ? c.validity->ptr : nullptr;
                o.validity_bytes = c.valid_bytes ? c.valid_bytes->ptr : nullptr;
                o.bool_bytes = c.bool_bytes ? c.bool_bytes->ptr : nullptr;
                if (c.is_dict) { o.n_dict = (int)c.dict->values().size(); o.value_width = phys_bytes(c.phys); }
            }
        }
    });
}

void cb200_release(cb200_plan* plan) {
    if (!plan) return;
    TraceSpan ts("release");
    try {
        if (plan->started) cudaSetDevice(plan->ctx.device);
        plan->last = Batch();
        plan->root.reset();
        if (plan->ctx.stream) {
            cudaStreamSynchronize(plan->ctx.stream); // stream-ordered frees above
            std::lock_guard<std::mutex> lk(g_pool_mu);
            g_pool[plan->ctx.device].push_back(CtxRes{plan->ctx.stream, plan->ctx.d_err, plan->ctx.h_err, plan->ctx.ev0, plan->ctx.ev1});
        }
        // streams that were never handed to a source still belong to us
        for (auto* s : plan->inputs.streams) if (s && s->release) s->release(s);
    } catch (...) {
    }
    delete plan;
}

cb200_table* cb200_table_create(int64_t n_rows) {
    auto* t = new cb200_table();
    t->t = std::make_shared<DeviceTable>();
    t->t->n_rows = n_rows;
    return t;
}

int cb200_table_add_column(cb200_table* t, int32_t type_id, int32_t precision, int32_t scale, int32_t value_width, const void* dev_values,
                           const void* dev_validity, int64_t null_count, const char* const* dict_values, int32_t n_dict, cb200_error* err) {
    return cb200_guarded(err, [&]() -> int {
        if (!t) throw PlanError("null table handle");
        Column c;
        c.type = dtype_from_ids(type_id, precision, scale);
        size_t n = (size_t)t->t->n_rows;
        if (n_dict > 0) {
            if (!c.type.is_string()) throw PlanError("dictionary values on a non-string column");
            c.is_dict = true;
            c.dict = std::make_shared<Dictionary>();
            for (int i = 0; i < n_dict; i++) c.dict->append(dict_values[i]);
            c.phys = value_width == 1 ? Phys::I8 : value_width == 2 ? Phys::I16 : Phys::I32;
            if (value_width != 1 && value_width != 2 && value_width != 4) throw PlanError("dictionary codes must be 1, 2 or 4 bytes wide");
        } else if (c.type.is_string()) {
            throw Unsupported("device string columns must be dictionary-encoded");
        } else if (c.type.is_decimal() && value_width == 8) {
            if (c.type.precision > 18) throw PlanError("8-byte decimals need precision <= 18");
            c.phys = Phys::I64;
        } else {
            int w = c.type.arrow_width();
            if (value_width != w) throw PlanError("value_width " + std::to_string(value_width) + " does not match " + c.type.str());
            c.phys = phys_of(c.type);
        }
        if (((uintptr_t)dev_values & 15) || ((uintptr_t)dev_validity & 15)) throw PlanError("device buffers must be 16-byte aligned");
        size_t bytes = value_width == 0 ? (n + 7) / 8 : n * (size_t)value_width;
        c.data = std::make_shared<DeviceBuf>((void*)dev_values, bytes);
        if (dev_validity && null_count != 0) c.validity = std::make_shared<DeviceBuf>((void*)dev_validity, (n + 7) / 8);
        c.null_count = null_count;
        t->t->cols.push_back(c);
        return 0;
    }, -1);
}

const char* cb200_plan_dict_value(cb200_plan* plan, int32_t col, int32_t i, int32_t* len) {
    if (!plan || col < 0 || col >= (int)plan->last.cols.size()) return nullptr;
    const Column& c = plan->last.cols[(size_t)col];
    if (!c.is_dict || !c.dict || i < 0 || i >= (int)c.dict->values().size()) return nullptr;
    const std::string& v = c.dict->values()[(size_t)i];
    if (len) *len = (int32_t)v.size();
    return v.data();
}

int cb200_table_add_column_bytes(cb200_table* t, int32_t type_id, int32_t precision, int32_t scale, int32_t value_width, const void* dev_values,
                                 const void* dev_validity_bytes, const char* const* dict_values, int32_t n_dict, cb200_error* err) {
    return cb200_guarded(err, [&]() -> int {
        if (!t) throw PlanError("null table handle");
        size_t n = (size_t)t->t->n_rows;
        bool is_bool = type_id == (int)TypeId::Bool;
        // reuse the validation of the bitmap form, then swap in the byte forms
        int rc = cb200_table_add_column(t, type_id, precision, scale, is_bool ? 0 : value_width, is_bool ? nullptr : dev_values, nullptr, 0, dict_values, n_dict, err);
        if (rc != 0) throw PlanError(err ? err->message : "add_column failed");
        Column& c = t->t->cols.back();
        if (is_bool) {
            if (value_width != 1) throw PlanError("byte-per-row booleans need value_width 1");
            c.data = nullptr;
            c.bool_bytes = std::make_shared<DeviceBuf>((void*)dev_values, n);
            t->t->needs_packing = true;
        }
        if (dev_validity_bytes) {
            c.valid_bytes = std::make_shared<DeviceBuf>((void*)dev_validity_bytes, n);
            c.null_count = -1;
            t->t->needs_packing = true;
        }
        return 0;
    }, -1);
}

int cb200_plan_bind_table(cb200_plan* plan, int32_t input_index, cb200_table* t, cb200_error* err) {
    return cb200_guarded(err, [&]() -> int {
        if (!plan || !t) throw PlanError("null handle");
        if (plan->started) throw PlanError("tables must be bound before the first execute");
        if (input_index < 0 || input_index >= (int)plan->inputs.tables.size()) throw PlanError("input index out of range");
        plan->inputs.tables[(size_t)input_index] = t->t;
        return 0;
    }, -1);
}

void cb200_table_release(cb200_table* t) { delete t; }

int32_t cb200_plan_partition_starts(cb200_plan* plan, int64_t* starts, int32_t cap) {
    if (!plan) return -1;
    const auto& ps = plan->ctx.partition_starts;
    for (size_t i = 0; i < ps.size() && (int32_t)i < cap; i++) starts[i] = ps[i];
    return (int32_t)ps.size();
}

int64_t cb200_plan_kernel_launches(cb200_plan* plan) { return plan ? plan->ctx.kernel_launches : -1; }

int64_t cb200_release_cached_memory(int32_t device_ordinal) {
    try {
        if (cudaSetDevice(device_ordinal) != cudaSuccess) return 0;
        return (int64_t)release_cached_device_memory();
    } catch (...) { return 0; }
}

int cb200_plan_stats(cb200_plan* plan, cb200_stats* out) {
    if (!plan || !out) return -1;
    const ExecContext& c = plan->ctx;
    out->kernel_launches = c.kernel_launches;
    out->pipeline_launches = c.pipeline_launches;
    out->pipeline_ms = c.pipeline_ms;
    out->pipeline_rows = c.pipeline_rows;
    out->h2d_bytes = c.h2d_bytes;
    out->d2h_bytes = c.d2h_bytes;
    out->scan_pruned_row_groups = c.scan_pruned_row_groups;
    out->scan_pruned_rows = c.scan_pruned_rows;
    out->agg_strategies = c.agg_strategies;
    out->scan_pruned_pages = c.scan_pruned_pages;
    out->scan_page_pruned_rows = c.scan_page_pruned_rows;
    out->sort_rows = c.sort_rows;
    out->sort_passes = c.sort_passes;
    out->sort_pass_rows = c.sort_pass_rows;
    out->sort_select_rows = c.sort_select_rows;
    out->join_build_rows = c.join_build_rows;
    out->join_probe_rows = c.join_probe_rows;
    out->join_out_rows = c.join_out_rows;
    out->agg_range_levels = c.agg_range_levels;
    out->agg_range_reruns = c.agg_range_reruns;
    out->join_cond_pairs = c.join_cond_pairs;
    out->partition_ids_ms = c.partition_ids_ms;
    out->partition_place_ms = c.partition_place_ms;
    out->partition_gather_ms = c.partition_gather_ms;
    return 0;
}

void cb200_reset_range_profiles(void) { reset_range_profiles(); }

int cb200_compile_plan(const uint8_t* op_proto, size_t op_len, char* keys_out, size_t keys_cap, cb200_error* err) {
    return cb200_guarded(err, [&]() -> int {
        OperatorP op = decode_plan(op_proto, op_len);
        auto ks = plan_kernels_for_build(op);
        std::string keys;
        for (auto& g : ks) {
            jit_get(g, false);
            keys += (keys.empty() ? "" : ",") + g.key;
        }
        if (keys_out && keys_cap) snprintf(keys_out, keys_cap, "%s", keys.c_str());
        return (int)ks.size();
    }, -1);
}

int cb200_compile_plan_assume(const uint8_t* op_proto, size_t op_len, const int32_t* assume_bits, int32_t n_assume, int32_t source_index,
                              char* src_out, size_t src_cap, cb200_error* err) {
    return cb200_guarded(err, [&]() -> int {
        OperatorP op = decode_plan(op_proto, op_len);
        std::vector<int> as(assume_bits, assume_bits + n_assume);
        auto ks = plan_kernels_for_build(op, as);
        for (auto& g : ks) jit_get(g, false);
        if (src_out && src_cap && source_index >= 0 && source_index < (int)ks.size()) snprintf(src_out, src_cap, "%s", ks[(size_t)source_index].source.c_str());
        return (int)ks.size();
    }, -1);
}

int cb200_register_memory_file(const char* name, const void* data, size_t len) {
    if (!name) return -1;
    register_memory_file(name, (const uint8_t*)data, len);
    return 0;
}

int64_t cb200_snappy_decompress(const uint8_t* comp, size_t comp_len, uint8_t* out, size_t uncompressed_len, int32_t device_ordinal, int32_t* path_taken,
                                cb200_error* err) {
    return cb200_guarded(err, [&]() -> int64_t {
        if (!comp || (!out && uncompressed_len) || comp_len >= ((size_t)1 << 31) || uncompressed_len >= ((size_t)1 << 31)) throw PlanError("cb200_snappy_decompress: bad arguments");
        cuda_check(cudaSetDevice(device_ordinal), "cudaSetDevice");
        cudaStream_t st = nullptr; // legacy default stream: a diagnostic entry point, not a hot path
        set_alloc_stream(st);
        DeviceBuf dcomp(comp_len + 64), dout(uncompressed_len + 64), dpage(sizeof(PqPage)), derr(64);
        const int n_segs = (int)((uncompressed_len + PQ_SNAPPY_SEG - 1) / PQ_SNAPPY_SEG);
        DeviceBuf dck((size_t)(n_segs + 1) * 4);
        PqPage pg;
        memset(&pg, 0, sizeof(pg));
        pg.body = (unsigned char*)dout.ptr;
        pg.body_bytes = (int)uncompressed_len;
        pg.comp = (const unsigned char*)dcomp.ptr;
        pg.comp_bytes = (int)comp_len;
        pg.seg_base = 0;
        pg.n_segs = n_segs;
        cuda_check(cudaMemsetAsync(dcomp.ptr, 0, comp_len + 64, st), "memset");
        cuda_check(cudaMemcpyAsync(dcomp.ptr, comp, comp_len, cudaMemcpyHostToDevice, st), "copy in");
        cuda_check(cudaMemcpyAsync(dpage.ptr, &pg, sizeof(pg), cudaMemcpyHostToDevice, st), "copy page");
        cuda_check(cudaMemsetAsync(derr.ptr, 0, 64, st), "memset err");
        launch_pq_snappy_segmented((PqPage*)dpage.ptr, 1, (unsigned*)dck.ptr, n_segs, (int*)derr.ptr, st);
        int e = 0;
        cuda_check(cudaMemcpyAsync(&e, derr.ptr, 4, cudaMemcpyDeviceToHost, st), "read err");
        cuda_check(cudaMemcpyAsync(&pg, dpage.ptr, sizeof(pg), cudaMemcpyDeviceToHost, st), "read page");
        if (uncompressed_len) cuda_check(cudaMemcpyAsync(out, dout.ptr, uncompressed_len, cudaMemcpyDeviceToHost, st), "copy out");
        cuda_check(cudaStreamSynchronize(st), "sync");
        if (path_taken) *path_taken = (pg.flags & PQ_PAGE_SN_SERIAL) ? 1 : 0;
        if (e) throw ExecError(14, "", "malformed Snappy stream (device error flags " + std::to_string(e) + ")");
        return (int64_t)uncompressed_len;
    }, (int64_t)-1);
}

int cb200_parquet_describe(const char* path, char* out, size_t cap, cb200_error* err) {
    return cb200_guarded(err, [&]() -> int {
        std::string s = describe_parquet(path ? path : "");
        if (out && cap) snprintf(out, cap, "%s", s.c_str());
        return (int)s.size();
    }, -1);
}

int cb200_plan_kernel_source(const uint8_t* op_proto, size_t op_len, int32_t index, char* out, size_t cap, cb200_error* err) {
    return cb200_guarded(err, [&]() -> int {
        OperatorP op = decode_plan(op_proto, op_len);
        auto ks = plan_kernels_for_build(op);
        if (index < 0 || index >= (int)ks.size()) throw PlanError("kernel index out of range");
        const std::string& s = ks[(size_t)index].source;
        if (out && cap) snprintf(out, cap, "%s", s.c_str());
        return (int)s.size();
    }, -1);
}

} // extern "C"
