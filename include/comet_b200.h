/*
 * comet_b200.h -- C ABI of libcomet_b200.so: the H100-native drop-in for the hot path of
 * apache/datafusion-comet's native layer (scan -> filter -> project -> hash aggregate).
 *
 * The entry points are exactly what the reference's JNI surface binds for this path; each one names
 * the reference interface it replaces (paths relative to the reference tree).  Plain pointers and
 * sizes only: a Rust `ExecutionPlan` shim (extern "C"), a JNI stub or ctypes can call it directly.
 * INTEGRATION.md shows the reference-side bindings.
 *
 * Threading (same contract as the reference, jni_api.rs:194-223): one plan handle is driven by one
 * thread at a time; any number of handles may run concurrently (each owns a CUDA stream + arena).
 * Errors never unwind across the ABI: calls return a code and fill `cb200_error`
 * (jni-bridge/src/errors.rs:832-850 `try_unwrap_or_throw` is the reference's equivalent).
 */
#ifndef COMET_B200_H
#define COMET_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

struct ArrowArray;       /* Arrow C Data interface  */
struct ArrowSchema;
struct ArrowArrayStream; /* Arrow C Stream interface */

typedef struct cb200_plan cb200_plan;
typedef struct cb200_table cb200_table;

/* error codes */
#define CB200_OK 0
#define CB200_ERR_UNSUPPORTED 1  /* plan uses an operator/expression outside the GPU hot path: fall back */
#define CB200_ERR_CUDA 2
#define CB200_ERR_INPUT 3        /* Arrow stream / schema problem */
#define CB200_ERR_PLAN 4         /* malformed plan */
#define CB200_ERR_JIT 5
#define CB200_ERR_SPARK 10       /* Spark-visible runtime error; error_class carries the Spark error class */

typedef struct cb200_error {
    int32_t code;
    char error_class[64];  /* e.g. "ARITHMETIC_OVERFLOW" (errors.rs:507-519 carries the same class to the JVM) */
    char message[952];
} cb200_error;

const char* cb200_version(void);

/* 1 if the serialized `spark.spark_operator.Operator` can run on the GPU path, 0 otherwise (`why`
 * explains).  Lets the caller keep the CPU path for everything else -- the role CometExecRule's
 * fallback tagging plays on the JVM side (spark/src/main/scala/org/apache/comet/rules/). */
int cb200_supports(const uint8_t* op_proto, size_t op_len, cb200_error* why);

/* Replaces Native.createPlan (spark/src/main/scala/org/apache/comet/Native.scala:60-79,
 * native/core/src/execution/jni_api.rs:371-394).  `op_proto` is the same prost-encoded
 * spark.spark_operator.Operator the JVM sends; `cfg_proto` the spark.spark_config.ConfigMap (may be
 * NULL).  `inputs[i]` feeds the i-th Scan in plan order; ownership of each stream moves to the plan
 * (planner.rs:1725-1737).  An entry may be NULL if a device table is bound before the first execute.
 * Returns NULL on error. */
cb200_plan* cb200_create_plan(const uint8_t* op_proto, size_t op_len, const uint8_t* cfg_proto, size_t cfg_len,
                              struct ArrowArrayStream** inputs, int32_t n_inputs, int32_t partition,
                              int32_t partition_count, int32_t batch_size, int32_t device_ordinal, cb200_error* err);

/* number of columns every output batch has */
int32_t cb200_plan_num_columns(cb200_plan* plan);

/* Replaces Native.executePlan (Native.scala:98-103, jni_api.rs:767-775): produce the next output
 * batch into caller-allocated ArrowArray/ArrowSchema structs (moved, release callbacks set).  Returns
 * the row count, -1 at end of stream (jni_api.rs:891,933), -2 on error.  A batch never has more than
 * spark.comet.batchSize rows (CometConf.scala:539-544; `batch_size` of cb200_create_plan when > 0): larger
 * results leave in consecutive zero-offset slices (jni_api.rs:716-732), except the batch of a ShuffleWriter
 * plan, which cb200_plan_partition_starts / cb200_exchange address as a whole. */
int64_t cb200_execute(cb200_plan* plan, struct ArrowArray* out_arrays, struct ArrowSchema* out_schemas,
                      int32_t n_cols, cb200_error* err);

/* Replaces Native.releasePlan (jni_api.rs:961).  Safe mid-stream. */
void cb200_release(cb200_plan* plan);

/* ---- device-resident inputs / outputs (no reference equivalent: the reference has no device) --------
 * Columns already in HBM can be bound as the input of a Scan instead of an Arrow stream; this is the
 * "inputs resident in HBM" leg of bench.py.  Buffers stay owned by the caller, must be 16-byte aligned
 * and readable 16 bytes past the last element (TMA bulk copies round sizes up to 16 B). */
cb200_table* cb200_table_create(int64_t n_rows);
/* type_id: spark_expression.DataType.DataTypeId (types.proto:43-66).  value_width: bytes per value in
 * `dev_values` (0 = bit-packed booleans; 1/2/4 for dictionary codes of a STRING column when
 * n_dict > 0; 8 allowed for DECIMAL with precision <= 18).  dev_validity: Arrow bitmap or NULL. */
int cb200_table_add_column(cb200_table* t, int32_t type_id, int32_t precision, int32_t scale, int32_t value_width,
                           const void* dev_values, const void* dev_validity, int64_t null_count,
                           const char* const* dict_values, int32_t n_dict, cb200_error* err);
/* Same, for columns in the exchange-friendly form cb200_execute_device reports for ShuffleWriter plans:
 * validity as one byte per row (`dev_validity_bytes`, may be NULL) and BOOL values as one byte per row
 * (value_width = 1).  The library packs them to Arrow bitmaps on the plan's stream at first use. */
int cb200_table_add_column_bytes(cb200_table* t, int32_t type_id, int32_t precision, int32_t scale, int32_t value_width,
                                 const void* dev_values, const void* dev_validity_bytes, const char* const* dict_values,
                                 int32_t n_dict, cb200_error* err);
int cb200_plan_bind_table(cb200_plan* plan, int32_t input_index, cb200_table* t, cb200_error* err);
void cb200_table_release(cb200_table* t);

typedef struct cb200_device_column {
    /* value_width: bytes per value of `values` -- the Arrow width of the type (BOOL: one byte per row, DECIMAL: 16), or the width of
     * the codes (1, 2 or 4) of a dictionary-coded STRING column */
    int32_t type_id, precision, scale, value_width;
    const void* values;    /* device pointer (NULL when the column lives on the host: small aggregate results) */
    const void* validity;  /* device Arrow bitmap or NULL */
    const void* host_values;
    const uint8_t* host_validity_bytes; /* one byte per row, or NULL */
    const void* validity_bytes;  /* device, one byte per row (ShuffleWriter plans: segments slice at any row) or NULL */
    const void* bool_bytes;      /* device, BOOL values one byte per row (ShuffleWriter plans) or NULL */
    int32_t n_dict;              /* dictionary-coded STRING column: number of dictionary entries (values = codes of value_width bytes) */
    int32_t pad;
} cb200_device_column;
/* i-th dictionary string of output column `col` of the last batch (valid until the next call on the plan) */
const char* cb200_plan_dict_value(cb200_plan* plan, int32_t col, int32_t i, int32_t* len);
/* Like cb200_execute but leaves fixed-width results where they are (valid until the next call on the
 * plan).  Returns rows, -1 at end, -2 on error. */
int64_t cb200_execute_device(cb200_plan* plan, cb200_device_column* cols, int32_t n_cols, cb200_error* err);

/* Plans rooted at a ShuffleWriter (operator.proto:688, partitioning.proto; at most 16 384 partitions, cb200_supports refuses more)
 * return their child's rows reordered by partition id, stable within a partition.  The partition id of a row is:
 *   HashPartition (at most 8 key columns):  pmod(murmur3(keys, seed 42), num_partitions) -- multi_partition.rs:265-330
 *   SinglePartition:                        0
 *   RoundRobinPartition:                    pmod(murmur3(first max_hash_columns columns, all when <= 0), num_partitions)
 *                                           -- multi_partition.rs:386-430
 *   RangePartition:                         the number of boundary rows <= the row under the sort orders (repeated sort
 *                                           columns dropped) -- multi_partition.rs:333-380; with fewer than num_partitions - 1
 *                                           boundary rows the last partitions are empty.
 * After each cb200_execute / cb200_execute_device
 * this returns the num_partitions+1 row offsets of that batch (the map-side of the exchange; the reference writes
 * the same segments as per-partition IPC blocks).  Returns the number of entries. */
int32_t cb200_plan_partition_starts(cb200_plan* plan, int64_t* starts, int32_t cap);

/* ---- multi-GPU: one process per GPU, NCCL over NVLink / NVSwitch --------------------------------------------------------------
 * The path shards by partition with no collective except ONE exchange step: the hash-repartition of partial aggregate state between
 * Partial and Final (SURVEY 8e; the reference's shuffle, native/shuffle/src/partitioners/multi_partition.rs:265-330, followed by
 * Spark's block fetch).  A caller with N GPUs on one box creates one communicator per process: rank 0 draws the id and hands the
 * 128 bytes to the others over whatever control channel it has (the JVM driver, torch.distributed, a file). */
#define CB200_UNIQUE_ID_BYTES 128
typedef struct cb200_comm cb200_comm;
int cb200_comm_unique_id(uint8_t* id_out /* CB200_UNIQUE_ID_BYTES */, cb200_error* err);
cb200_comm* cb200_comm_create(const uint8_t* id, int32_t rank, int32_t world, int32_t device_ordinal, cb200_error* err);
void cb200_comm_destroy(cb200_comm* comm);
int32_t cb200_comm_rank(cb200_comm* comm);
int32_t cb200_comm_world(cb200_comm* comm);
const char* cb200_nccl_info(void); /* which NCCL the library resolved, for logs */

typedef struct cb200_exchange_stats {
    int64_t rows_sent, rows_received;
    int64_t bytes_sent, bytes_received; /* payload bytes incl. the segment this rank keeps */
    double payload_ms;                  /* CUDA-event duration of the grouped send/recv on the communicator's stream */
} cb200_exchange_stats;
/* The exchange itself.  `map_plan` is a ShuffleWriter plan with num_partitions = world whose last cb200_execute /
 * cb200_execute_device batch is still alive: its rows are ordered by partition id (cb200_plan_partition_starts: pmod(murmur3(keys,
 * 42), world) for HashPartitioning, the number of boundary rows <= the row for RangePartitioning, so that rank r receives the r-th
 * range of a global order, and murmur3 over the first columns for RoundRobinPartitioning).  Every rank calls
 * this exactly once per map plan, collectively -- also when its map plan produced no batch (an empty partition, a filter that removed
 * every row): that rank takes part with zero rows of the plan's output schema.  Rank r gets back a device table (owned by the
 * library, release with cb200_table_release) holding partition r of every rank, sources in rank order, rows in their map-side order
 * -- ready to be bound as the input of the Final plan with cb200_plan_bind_table.
 * Every column travels as its values (the Arrow width of its type, BOOL one byte per row) plus one validity byte per row, whether or
 * not the local column has NULLs, so every rank moves the same list of buffers and every received column has validity:
 * bytes_sent = rows x sum(width + 1).  Fixed-width columns only (aggregate state: keys, sums, counts, flags): a plan with string
 * columns (CB200_ERR_UNSUPPORTED), a plan that is not a ShuffleWriter or whose num_partitions is not the world size, a plan created
 * for another device than the communicator's, and a plan that was never executed (CB200_ERR_PLAN) are refused before any collective, so a refusal leaves no peer waiting.
 * Only the last batch moves: a map plan that emits more than one batch (a ShuffleWriter over a Scan larger than
 * spark.comet.b200.chunkRows, or over a join) is not exchanged whole.  A ShuffleWriter over a grouped Partial emits one batch.
 * Returns NULL on error. */
cb200_table* cb200_exchange(cb200_comm* comm, cb200_plan* map_plan, int64_t* n_rows_out, cb200_exchange_stats* stats, cb200_error* err);
/* receive layout of that exchange from the gathered N x N count matrix (counts[s * world + p] = rows rank s holds for rank p):
 * fills recv_counts / recv_offsets (either may be NULL), returns the rows rank `me` receives.  Pure host arithmetic. */
int64_t cb200_exchange_layout(const int64_t* counts, int32_t world, int32_t me, int64_t* recv_counts, int64_t* recv_offsets);
/* All-gather of one small host payload per rank (the serialized state batch of a dense / ungrouped Partial aggregate: a handful of
 * rows; merged by the Final plan with merge_batch semantics, not by an all-reduce).  `out` has world slots of slot_bytes (a multiple
 * of 16, >= n_bytes + 8); sizes_out[r] = payload length of rank r.  One NCCL collective, one synchronisation. */
int cb200_comm_allgather_small(cb200_comm* comm, const void* payload, int64_t n_bytes, int64_t slot_bytes, void* out, int64_t* sizes_out,
                               cb200_error* err);

/* kernels launched so far by this plan (bench.py reports it as gpu_launches) */
int64_t cb200_plan_kernel_launches(cb200_plan* plan);

/* ---- native Parquet scan --------------------------------------------------------------------------------------
 * NativeScan plans (operator.proto:141-185) name files; besides plain paths / file:// URLs the library accepts
 * "memory://<name>" for a Parquet file image the caller holds in (ideally pinned) host memory -- what a Spark
 * executor has after fetching an object-store range.  Encoded pages are copied H2D as they are and decoded on
 * the device.  `data` = NULL unregisters. */
int cb200_register_memory_file(const char* name, const void* data, size_t len);
/* One raw Snappy buffer through the scan's device decompressor (index pass + 64 KB segments + serial fallback, csrc/parquet_kernels.cu),
 * host in / host out.  Returns the bytes produced (= `uncompressed_len`) or -1.  `path_taken` (may be NULL): 0 segmented, 1 the page
 * went to the serial kernel.  For tests and diagnostics: lets hand-made streams (elements across a 64 KB boundary, references into an
 * earlier segment, malformed input) reach kernels that Parquet writers never exercise.  Reference: the `snap` crate behind the
 * third-party parquet reader (native/core/Cargo.toml:40). */
int64_t cb200_snappy_decompress(const uint8_t* comp, size_t comp_len, uint8_t* out, size_t uncompressed_len, int32_t device_ordinal, int32_t* path_taken,
                                cb200_error* err);
/* JSON description of a Parquet file's footer as this library parsed it (tests compare it with pyarrow). */
int cb200_parquet_describe(const char* path, char* out, size_t cap, cb200_error* err);

/* Measurement: the library times every fused pipeline kernel with CUDA events on its own stream. */
typedef struct cb200_stats {
    int64_t kernel_launches;   /* all kernels (pipelines, fold/finalize, helpers) */
    int64_t pipeline_launches; /* fused pipeline kernels only */
    double pipeline_ms;        /* sum of their device durations */
    int64_t pipeline_rows;     /* input rows those launches scanned */
    int64_t h2d_bytes;         /* host->device bytes copied by Arrow-stream sources */
    int64_t d2h_bytes;         /* device->host bytes copied by cb200_execute */
    int64_t scan_pruned_row_groups; /* Parquet row groups skipped because their statistics rule the pushed filters out */
    int64_t scan_pruned_rows;
    int64_t agg_strategies;    /* OR of CB200_AGG_* over the plan's aggregates: which accumulation strategies ran */
    int64_t scan_pruned_pages; /* Parquet data pages of read columns not uploaded because the page index rules the pushed filters out */
    int64_t scan_page_pruned_rows; /* rows of row groups the statistics kept that the page index ruled out */
    int64_t sort_rows;         /* rows Sort operators built keys for and radix-sorted (TopK: every chunk and every merge with the candidates) */
    int64_t sort_passes;       /* radix passes they ran: one per 8-bit key digit that is not the same in every row */
    int64_t sort_pass_rows;    /* rows those passes moved, summed over the passes */
    int64_t sort_select_rows;  /* rows TopK's radix select read, summed over its digit steps */
    int64_t join_build_rows;   /* rows HashJoin, SortMergeJoin and BroadcastNestedLoopJoin operators drained from their build side */
    int64_t join_probe_rows;   /* probe-side (streamed-side) rows they looked up or paired */
    int64_t join_out_rows;     /* rows they emitted */
    int64_t agg_range_levels;  /* OR of CB200_RANGE_* over the dense aggregate launches that were kept: which value-range assumptions ran */
    int64_t agg_range_reruns;  /* dense aggregate launches discarded because their input broke the value range the kernel assumed */
    int64_t join_cond_pairs;   /* candidate pairs their join condition was evaluated on: pairs with equal keys (HashJoin, SortMergeJoin), every
                                  (probe row, build row) pair (BroadcastNestedLoopJoin: n * m per probe batch when the build side has rows) */
    double partition_ids_ms;    /* ShuffleWriter stages, device time between CUDA events on the plan's stream, summed over batches: */
    double partition_place_ms;  /*   the partition ids, their stable counting sort (histogram, scan, placement) */
    double partition_gather_ms; /*   and the gather of the columns into partition order */
} cb200_stats;
#define CB200_AGG_DENSE 1      /* thread-private accumulators over dictionary / bool key codes (and ungrouped aggregates) */
#define CB200_AGG_TABLE 2      /* global key table */
#define CB200_AGG_STREAM 4     /* one state row per run of equal keys */
#define CB200_AGG_MIGRATED 8   /* a dense aggregate outgrew its group limit and moved to hashing mid-stream */
#define CB200_RANGE_TIGHT 1    /* kernel specialised to the observed value bits + 2 */
#define CB200_RANGE_TYPE 2     /* kernel specialised to the declared decimal precision */
#define CB200_RANGE_SAFE 4     /* fully checked kernel, no value-range assumption */
int cb200_plan_stats(cb200_plan* plan, cb200_stats* out);

/* The library recycles device blocks >= 1 MiB on a per-device free list instead of returning them to the driver (a query step
 * allocates the same multi-GB buffers again and again; see csrc/exec.cpp DeviceBuf).  This gives them back, e.g. before another
 * framework in the same process needs the memory.  Returns the bytes released.  No reference equivalent (the reference's memory
 * pools are host-side, native/core/src/execution/memory_pools/). */
int64_t cb200_release_cached_memory(int32_t device_ordinal);

/* A dense decimal aggregate over a batch of more than 2 Mi rows leaves the value ranges it observed for the next plan with the same
 * pipeline, which then starts from them instead of sampling (a guess every launch still validates).  This forgets them, so that what
 * a plan runs does not depend on the plans before it: for tests and diagnostics. */
void cb200_reset_range_profiles(void);

/* Build-time: generate and NVRTC-compile (sm_90a; needs no GPU) every pipeline kernel the plan would
 * use for null-free inputs; cubins land in the JIT cache that ships with the library.  Writes the
 * comma-separated kernel keys to `keys_out`.  Returns the number of kernels, <0 on error. */
int cb200_compile_plan(const uint8_t* op_proto, size_t op_len, char* keys_out, size_t keys_cap, cb200_error* err);
/* Same with value-range assumptions for the scan's decimal columns (assume_bits[i] > 0: |column i| < 2^bits,
 * validated at run time by the kernels' value masks): pre-compiles the range-specialised variant a known
 * workload will select after sampling.  Optionally returns the source of kernel `source_index`. */
int cb200_compile_plan_assume(const uint8_t* op_proto, size_t op_len, const int32_t* assume_bits, int32_t n_assume,
                              int32_t source_index, char* src_out, size_t src_cap, cb200_error* err);
/* Same, but returns the generated CUDA source of kernel `index` (for inspection / nvcc -Xptxas -v). */
int cb200_plan_kernel_source(const uint8_t* op_proto, size_t op_len, int32_t index, char* out, size_t cap, cb200_error* err);

#ifdef __cplusplus
}
#endif
#endif
