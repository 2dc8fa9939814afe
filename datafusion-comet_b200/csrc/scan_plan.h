// scan_plan.h -- host planning of the native Parquet scan: which row groups are read, how they form batches, which byte ranges cross
// PCIe, and the page tables of every column of a batch.  Pure computation over footers and page headers: these functions keep no
// scan state and never call the CUDA runtime; scan_parquet.cpp runs the device pipeline over what they return.
#pragma once
#include "exec.h"
#include "parquet.h"
#include "parquet_pages.h"

#include <unordered_map>
#include <utility>

namespace cb200 {

inline size_t align_up(size_t n, size_t a) { return (n + a - 1) / a * a; }

// ---- files ---------------------------------------------------------------------------------------------------------------------
std::string strip_file_scheme(const std::string& path);

struct ScanFile {
    pq::FileMeta meta;
    const uint8_t* mem = nullptr; // memory:// image; nullptr: the bytes are read from disk
    size_t mem_len = 0;
    std::vector<int> leaf_of;     // per output column: leaf index in this file
    const pq::SchemaElement& leaf(size_t c) const { return meta.leaf(leaf_of[c]); }
    const pq::ColumnChunkMeta& chunk(size_t rg, size_t c) const { return meta.row_groups[rg].columns[(size_t)leaf_of[c]]; }
};
ScanFile open_scan_file(const std::string& path, const std::vector<StructField>& fields);

// ---- row groups ----------------------------------------------------------------------------------------------------------------
// conjuncts `column <op> literal` of the pushed-down filters, evaluated against chunk statistics
struct PruneTerm {
    int col;          // index into required_schema
    ExprKind op;      // Eq, Lt, LtEq, Gt, GtEq (column on the left), IsNotNull
    bool is_float = false;
    __int128 ival = 0;
    double fval = 0;
};
void collect_prune_terms(const ExprP& e, std::vector<PruneTerm>& out);
// true = the statistics prove that no row of the chunk satisfies the term
bool term_excludes(const PruneTerm& t, const pq::SchemaElement& se, const pq::ColumnChunkMeta& cc);

struct Unit { size_t file, rg; int64_t rows, row0; }; // one row group; row0: its first row within its batch
struct Selection {
    std::vector<Unit> units;
    int64_t pruned_row_groups = 0, pruned_rows = 0;
};
// the row groups a scan reads: those a file split owns, minus those the statistics rule out
Selection select_row_groups(const std::vector<ScanFile>& files, const std::vector<int64_t>& file_start, const std::vector<int64_t>& file_length,
                            size_t n_cols, const std::vector<PruneTerm>& terms);

// ---- batches -------------------------------------------------------------------------------------------------------------------
struct BatchPlan {
    std::vector<std::pair<size_t, size_t>> batches; // [first unit, end unit) of every batch
    size_t chunk_need = 0;                          // per slot: encoded bytes of the largest batch, exact
    size_t work_estimate = 0;                       // per slot: decoded columns + decode temporaries, estimated
};
BatchPlan plan_batches(const std::vector<Unit>& units, const std::vector<ScanFile>& files, const std::vector<StructField>& fields, int64_t chunk_rows);
// the units of one batch, each with its first row within the batch
std::vector<Unit> batch_units(const std::vector<Unit>& units, std::pair<size_t, size_t> batch);

// ---- upload ranges -------------------------------------------------------------------------------------------------------------
struct UploadRange { size_t file; int64_t start, end; size_t dev_off; };
struct ChunkAt { size_t range; int64_t off; }; // a column chunk inside an upload range
struct UploadPlan {
    std::vector<UploadRange> ranges;
    std::vector<std::vector<ChunkAt>> chunk_at; // [column][unit]
    size_t dev_total = 0;                       // device bytes of all ranges, each 256-byte aligned
};
UploadPlan plan_uploads(const std::vector<Unit>& units, const std::vector<ScanFile>& files, size_t n_cols);

// ---- columns -------------------------------------------------------------------------------------------------------------------
// The plan-wide dictionary of one string column.  Dictionary pages and PLAIN pages both intern through it, so a value gets the same
// code whichever encoding, file or batch it comes from; codes are handed out in first-occurrence order.
struct StringInterner {
    DictionaryP dict = std::make_shared<Dictionary>();
    std::unordered_map<std::string, int32_t> index; // value -> code, in step with dict->values
    int32_t code(std::string v);
};

struct ChunkLoc { const uint8_t* host; unsigned char* dev; }; // one column chunk of a batch: its bytes on the host and where they land on the device

// one column of one batch: page tables on the host, then the device buffers they refer to
struct ColPlan {
    int conv = 0, out_w = 0, type_length = 0;
    Phys phys = Phys::I32;
    DictionaryP dict;             // string columns: the plan-wide dictionary the codes index
    std::vector<PqPage> pages;    // data pages, then fixed-width dictionary pages
    size_t n_data = 0, n_dict_pages = 0;
    std::vector<int32_t> remap;   // string columns: combined code remap tables
    int64_t run_base = 0, def_run_base = 0, dict_elems = 0;
    size_t unc_bytes = 0;
    int64_t n_segs_total = 0;     // Snappy: 64 KB output segments over all compressed pages (checkpoint table entries)
    std::vector<uint8_t> hostdec; // page bodies produced on the host, 16-byte aligned each; shipped with the page tables
    bool optional = false, null_aware = false, any_compressed = false;
    // device buffers, bound by the scan (buffer_requests)
    uint8_t *out = nullptr, *dunc = nullptr, *dpd = nullptr, *ddict = nullptr, *dense = nullptr, *dvalid = nullptr, *didx = nullptr, *druns = nullptr,
            *dcounts = nullptr, *validity = nullptr, *runs = nullptr, *counts = nullptr, *dckpt = nullptr;
    size_t out_bytes = 0, validity_bytes = 0;
};

ColPlan plan_column(const std::vector<ScanFile>& files, const StructField& field, size_t c, const std::vector<Unit>& units, int64_t total,
                    const std::vector<ChunkLoc>& loc, StringInterner& strings);
// every device buffer of a column, as (where the pointer goes, bytes)
void buffer_requests(ColPlan& cp, int64_t total, std::vector<std::pair<uint8_t**, size_t>>& reqs);
// Page bodies whose buffer has no device address at plan time hold an offset into it; this turns them into addresses, once `cp.dunc`
// is bound and the host-produced bytes are staged at `hostdec_dev`.
void resolve_bodies(ColPlan& cp, uint8_t* hostdec_dev);

} // namespace cb200
