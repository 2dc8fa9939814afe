// exec.h -- executor: pull-based operator tree over device batches.
//
// Mirrors what the reference builds in PhysicalPlanner::create_plan (native/core/src/execution/
// planner.rs:1211) but with pipeline fusion: every maximal chain Scan -> (Filter|Projection)* ->
// {output | HashAggregate} becomes ONE JIT-specialised kernel launch per device chunk.
#pragma once
#include "arrow_abi.h"
#include "codegen.h"
#include "jit.h"
#include "plan.h"

#include <cuda_runtime.h>
#include <climits>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

namespace cb200 {

struct ExecError : std::runtime_error {
    int code;
    std::string error_class;
    ExecError(int c, const std::string& cls, const std::string& msg) : std::runtime_error(msg), code(c), error_class(cls) {}
};

void cuda_check(cudaError_t e, const char* what);

// CB200_TRACE=1: wall-clock spans to stderr (the reference's spark.comet.tracing.enabled analogue,
// native/common/src/tracing.rs:27-96)
struct TraceSpan {
    const char* name;
    double t0;
    explicit TraceSpan(const char* n);
    ~TraceSpan();
};
bool trace_on();
double now_ms();
void set_alloc_stream(cudaStream_t s); // stream used by DeviceBuf allocations made on this thread
size_t release_cached_device_memory();  // frees the library's recycled large blocks on the current device; returns the bytes released
void reset_range_profiles();            // forgets the value ranges dense aggregates left for later plans with the same pipeline (agg.cpp)

struct DeviceBuf {
    void* ptr = nullptr;
    size_t bytes = 0;
    bool owned = true;
    cudaStream_t stream = nullptr;
    std::shared_ptr<void> owner;               // non-owning views: the block this pointer lives in (kept alive with the view)
    DeviceBuf() {}
    DeviceBuf(size_t n);                       // cudaMalloc, padded
    DeviceBuf(void* p, size_t n) : ptr(p), bytes(n), owned(false) {}
    ~DeviceBuf();
    DeviceBuf(const DeviceBuf&) = delete;
    DeviceBuf& operator=(const DeviceBuf&) = delete;
};
using DeviceBufP = std::shared_ptr<DeviceBuf>;

// The string dictionary of a dictionary-coded column (host copy): code i stands for values()[i].  Entries are only ever added, so a
// code keeps its meaning as the dictionary grows.
class Dictionary {
  public:
    const std::vector<std::string>& values() const { return values_; }
    // the code of the first entry equal to v; v is appended when there is none
    int32_t intern(std::string v) {
        auto it = index_.find(v);
        if (it != index_.end()) return it->second;
        if (values_.size() >= (size_t)INT32_MAX) throw Unsupported("more than 2^31 distinct strings in one dictionary");
        const int32_t code = (int32_t)values_.size();
        index_.emplace(v, code);
        values_.push_back(std::move(v));
        return code;
    }
    // v as a new entry even if an equal one exists: a caller's dictionary may repeat a value, and each code keeps its own entry
    void append(std::string v) {
        index_.emplace(v, (int32_t)values_.size()); // no-op for a repeat: intern keeps finding the first
        values_.push_back(std::move(v));
    }
    // the code of the first entry equal to v, or -1 when there is none (nothing is added)
    int32_t find(const std::string& v) const {
        auto it = index_.find(v);
        return it == index_.end() ? -1 : it->second;
    }

  private:
    std::vector<std::string> values_;
    std::unordered_map<std::string, int32_t> index_; // value -> code of its first entry
};
using DictionaryP = std::shared_ptr<Dictionary>;

// A device column.  Which layouts `phys` takes for each type, and which source produces each, is listed in DESIGN.md
// ("Data layout in HBM"); phys_bytes(phys) is the width of one row of `data`, dictionary codes included.
struct Column {
    DType type;
    Phys phys = Phys::I32;          // physical encoding of `data` (device) -- see codegen.h
    bool is_dict = false;           // data holds dictionary codes (type = String)
    DictionaryP dict;
    DeviceBufP data, validity;      // device (validity: Arrow bitmap) ...
    DeviceBufP offsets, chars;      // ... device Utf8 (offsets int32[n+1], chars)
    DeviceBufP valid_bytes;         // optional byte-per-row validity (exchange-friendly form; see gather_columns / cb200_table_add_column_bytes)
    DeviceBufP bool_bytes;          // optional byte-per-row form of a boolean column
    int64_t null_count = 0;
    // host-resident alternative (small aggregate results)
    bool on_host = false;
    std::vector<uint8_t> h_data;        // fixed-width values or chars
    std::vector<uint8_t> h_valid;       // one byte per row; empty = all valid
    std::vector<int32_t> h_offsets;     // Utf8
};

struct Batch {
    int64_t n_rows = 0;
    std::vector<Column> cols;
};

struct ExecContext {
    int device = 0;
    cudaStream_t stream = nullptr;
    int num_sms = 132;        // H100 SXM; start() reads the device's count
    int64_t chunk_rows = 1ll << 26;
    int hash_threads = 512;   // consumer threads per CTA of the hash-aggregate kernel (tuning knob)
    // Partial hash aggregates over inputs of at least this many rows sample whether equal keys are adjacent and, if so, emit one state
    // row per run instead of building a key table (spark.comet.b200.streamAgg.minRows; -1 disables, 0 = always sample)
    int64_t stream_agg_min_rows = 4 << 20;
    double stream_agg_max_ratio = 0.5; // state rows per input row above which the key table is used (spark.comet.b200.streamAgg.maxRatio)
    int batch_size = 8192;
    int* d_err = nullptr;   // device error flags
    int* h_err = nullptr;   // pinned host mirror
    int64_t kernel_launches = 0;
    // measurement (bench.py / cb200_plan_stats): CUDA events around each fused pipeline kernel, on the
    // stream the kernel is launched on
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    bool ev_pending = false;
    double pipeline_ms = 0;       // sum of fused-pipeline kernel durations
    int64_t pipeline_launches = 0;
    int64_t pipeline_rows = 0;    // rows those launches scanned
    int64_t h2d_bytes = 0, d2h_bytes = 0;
    int64_t scan_pruned_row_groups = 0, scan_pruned_rows = 0; // Parquet row groups skipped by statistics (parquet_exec.rs:143-196)
    int64_t scan_pruned_pages = 0, scan_page_pruned_rows = 0;  // data pages / rows of kept row groups skipped by the page index
    int64_t agg_strategies = 0;   // CB200_AGG_* bits of the aggregate strategies that ran
    int64_t agg_range_levels = 0; // CB200_RANGE_* bits of the dense launches kept
    int64_t agg_range_reruns = 0; // dense launches discarded by value-mask validation
    int64_t sort_rows = 0, sort_passes = 0, sort_pass_rows = 0; // rows Sort operators radix-sorted, the digit passes they ran, rows moved
    int64_t sort_select_rows = 0; // rows TopK's radix select read (one read per digit step)
    int64_t join_build_rows = 0, join_probe_rows = 0, join_out_rows = 0; // hash, sort-merge and nested-loop joins: rows drained from the build side, rows probed, rows out
    int64_t join_cond_pairs = 0;  // candidate (probe row, build row) pairs a join condition was evaluated on
    double partition_ids_ms = 0, partition_place_ms = 0, partition_gather_ms = 0; // ShuffleWriter stages, device time by CUDA events
    int64_t agg_table_grows = 0;  // IdRows::grow calls that moved groups already handed out to a larger array
    int64_t agg_stream_reruns = 0; // stream launches discarded because their runs outnumbered the state rows, then repeated
    std::vector<int64_t> partition_starts; // last ShuffleWriter batch: partition p = rows [starts[p], starts[p+1])
    void check_device_errors() { raise_device_errors(take_device_errors()); }
    int take_device_errors();           // synchronises; returns the error flags the kernels raised so far and clears them
    void raise_device_errors(int e);    // throws the error the flags `e` stand for (none: returns)
    void collect_timing();
};

struct ExecNode {
    std::vector<DType> schema;
    virtual ~ExecNode() {}
    virtual bool next(Batch& out) = 0; // false = end of stream
    // the node's children in plan order (a join: left, then right, whichever side builds)
    virtual std::vector<std::shared_ptr<ExecNode>> children() const { return {}; }
    // build time: the pipelines this node may launch, for inputs without nulls and with dictionary-encoded strings
    virtual std::vector<PipelineSpec> build_specs() const { return {}; }
    // predicates (over this node's output columns) that the consumer applies to every row anyway: a source may use them to skip
    // data that cannot pass (Parquet row groups whose statistics rule them out)
    virtual void push_filters(const std::vector<ExprP>&) {}
    // rows this node will still produce, if it knows (-1: unknown): lets a hash aggregate size its table once instead of growing it
    virtual int64_t rows_hint() const { return -1; }
};
using ExecNodeP = std::shared_ptr<ExecNode>;

struct DeviceTable { // caller-owned device-resident columns bound as a plan input (bench "value" path)
    int64_t n_rows = 0;
    std::vector<Column> cols;
    bool needs_packing = false; // some columns were given byte-per-row validity / booleans: packed to Arrow bitmaps at first use
};

// Build the executor tree for a decoded plan.  `inputs` are consumed in Scan order.
struct PlanInputs {
    std::vector<ArrowArrayStream*> streams;
    std::vector<std::shared_ptr<DeviceTable>> tables; // parallel to streams; non-null entry overrides
};
ExecNodeP build_exec(const OperatorP& op, ExecContext* ctx, PlanInputs* inputs);

// native Parquet scan (scan_parquet.cpp)
ExecNodeP make_native_scan(const OperatorP& op, ExecContext* ctx);

// Export helpers (host-visible Arrow C Data); to_arrow_layout gives every device column of b the Arrow layout of its type
bool to_arrow_layout(Batch& b, ExecContext* ctx); // true if it launched conversions (on ctx->stream)
void export_batch(Batch& b, ExecContext* ctx, ArrowArray* out_arrays, ArrowSchema* out_schemas, int n_cols, int64_t row0, int64_t n_rows);

// Debug / build-time: generate (and NVRTC-compile, no device needed) the kernels a plan would use,
// assuming inputs without nulls and dictionary-encoded string keys.
void register_memory_file(const std::string& name, const uint8_t* p, size_t n); // p == nullptr unregisters
std::string describe_parquet(const std::string& path);

std::vector<GeneratedKernel> plan_kernels_for_build(const OperatorP& op, const std::vector<int>& assume_bits = {});

} // namespace cb200
