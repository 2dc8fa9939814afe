// scan_plan.h -- host planning of the native Parquet scan: which row groups are read, how they form batches, which byte ranges cross
// PCIe, and the page tables of every column of a batch.  Pure computation over footers and page headers: these functions keep no
// scan state and never call the CUDA runtime; scan_parquet.cpp runs the device pipeline over what they return.
#pragma once
#include "exec.h"
#include "parquet.h"
#include "parquet_pages.h"

#include <memory>
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
// the statistics of a column chunk or of one page: min / max (PLAIN-encoded values; nullptr = not known) and whether every value is NULL
struct StatVals {
    const std::string* min = nullptr;
    const std::string* max = nullptr;
    bool all_null = false;
};
// true = the statistics prove that no row they describe satisfies the term (all NULL: no term holds; else min / max decide)
bool stats_exclude(const PruneTerm& t, const pq::SchemaElement& se, const StatVals& s);
// the same for a whole column chunk
bool term_excludes(const PruneTerm& t, const pq::SchemaElement& se, const pq::ColumnChunkMeta& cc);

// The rows of one row group that the page index cannot rule out, and per read column the data pages that hold them.  A column decodes
// those pages into "covered" rows (the rows of its selected pages back to back); `segs` maps selected rows to covered rows.
struct ColumnWindow {
    std::vector<int> pages;    // into the chunk's offset_index, ascending
    int64_t covered = 0;       // rows of those pages
    std::vector<PqSeg> segs;   // out_row: among the unit's selected rows; cov_row: among its covered rows
};
struct RowSelection {
    std::vector<std::pair<int64_t, int64_t>> ranges; // [begin, end) rows of the row group, sorted and disjoint
    std::vector<ColumnWindow> cols;                  // per read column
};
// one row group; rows: the rows it emits (all of them, or the selected ones); row0: its first row within its batch
struct Unit {
    size_t file, rg;
    int64_t rows, row0;
    std::shared_ptr<const RowSelection> sel = nullptr; // nullptr: the whole row group
};
struct Selection {
    std::vector<Unit> units;
    int64_t pruned_row_groups = 0, pruned_rows = 0;
};
// the row groups a scan reads: those a file split owns, minus those the statistics rule out
Selection select_row_groups(const std::vector<ScanFile>& files, const std::vector<int64_t>& file_start, const std::vector<int64_t>& file_length,
                            size_t n_cols, const std::vector<PruneTerm>& terms);

// ---- pages ---------------------------------------------------------------------------------------------------------------------
struct PageSelection {
    int64_t pruned_pages = 0;       // data pages of read columns that are not uploaded
    int64_t pruned_rows = 0;        // rows of the given units that are not emitted
    int64_t dropped_row_groups = 0; // units none of whose pages survive
};
// Attaches a row selection to every unit whose page index rules rows out, and drops the units it rules out entirely.  A row leaves
// only when the ColumnIndex of its page, in some term's column, proves that term false.  Applies to a unit whose term columns all have
// a ColumnIndex and whose read columns all have an OffsetIndex; every other unit stays whole.
PageSelection select_pages(std::vector<Unit>& units, const std::vector<ScanFile>& files, size_t n_cols, const std::vector<PruneTerm>& terms);

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
struct PieceAt { int64_t start, end; size_t range; int64_t off; }; // file bytes [start, end) of a page-pruned chunk inside an upload range
struct ChunkAt {   // a column chunk inside an upload range
    size_t range;
    int64_t off;
    std::vector<PieceAt> pieces = {}; // page-pruned unit: its dictionary page, then its runs of selected data pages (range / off unused)
};
struct UploadPlan {
    std::vector<UploadRange> ranges;
    std::vector<std::vector<ChunkAt>> chunk_at; // [column][unit]
    size_t dev_total = 0;                       // device bytes of all ranges, each 256-byte aligned
};
// Whole row groups upload whole column chunks; a page-pruned one uploads its dictionary pages and its runs of selected data pages.
UploadPlan plan_uploads(const std::vector<Unit>& units, const std::vector<ScanFile>& files, size_t n_cols);

// ---- columns -------------------------------------------------------------------------------------------------------------------
// The plan-wide dictionary of one string column.  Dictionary pages and PLAIN pages both intern through it, so a value gets the same
// code whichever encoding, file or batch it comes from; codes are handed out in first-occurrence order.
struct StringInterner {
    DictionaryP dict = std::make_shared<Dictionary>();
    std::unordered_map<std::string, int32_t> index; // value -> code, in step with dict->values
    int32_t code(std::string v);
};

// one column chunk of a batch: its bytes on the host and where they land on the device; for a page-pruned unit, those of each piece
struct PieceLoc { int64_t start, end; const uint8_t* host; unsigned char* dev; };
struct ChunkLoc {
    const uint8_t* host;
    unsigned char* dev;
    std::vector<PieceLoc> pieces = {};
};
// the ChunkLocs of column c: `host_of(range)` is the host address of an upload range's first byte, `dev_base` the device block
template <typename HostOf> std::vector<ChunkLoc> locate_chunks(const UploadPlan& up, size_t c, HostOf host_of, unsigned char* dev_base) {
    std::vector<ChunkLoc> loc;
    for (const ChunkAt& at : up.chunk_at[c]) {
        const UploadRange& r = up.ranges[at.range];
        ChunkLoc l{host_of(r) + at.off, dev_base + r.dev_off + at.off};
        for (const PieceAt& p : at.pieces) {
            const UploadRange& pr = up.ranges[p.range];
            l.pieces.push_back({p.start, p.end, host_of(pr) + p.off, dev_base + pr.dev_off + p.off});
        }
        loc.push_back(std::move(l));
    }
    return loc;
}

// one column of one batch: page tables on the host, then the device buffers they refer to
struct ColPlan {
    int conv = 0, out_w = 0, type_length = 0;
    Phys phys = Phys::I32;
    DictionaryP dict;             // string columns: the plan-wide dictionary the codes index
    std::vector<PqPage> pages;    // data pages, then fixed-width dictionary pages
    size_t n_data = 0, n_dict_pages = 0;
    std::vector<int32_t> remap;   // string columns: combined code remap tables
    int64_t run_base = 0, def_run_base = 0, dict_elems = 0;
    int64_t mb_base = 0;          // DELTA_BINARY_PACKED: miniblock table entries over all pages
    size_t unc_bytes = 0;
    int64_t n_segs_total = 0;     // Snappy: 64 KB output segments over all compressed pages (checkpoint table entries)
    std::vector<uint8_t> hostdec; // page bodies produced on the host, 16-byte aligned each; shipped with the page tables
    bool optional = false, null_aware = false, any_compressed = false;
    // page-pruned units: the pages decode into `covered` rows (PqPage::dst_row counts them), `segs` picks the batch's rows out of them.
    // Empty when the covered rows are the batch's rows: the pages decode straight into `out`.
    int64_t covered = 0;
    std::vector<PqSeg> segs;
    // device buffers, bound by the scan (buffer_requests)
    uint8_t *out = nullptr, *dunc = nullptr, *dpd = nullptr, *ddict = nullptr, *dense = nullptr, *dvalid = nullptr, *didx = nullptr, *druns = nullptr,
            *dcounts = nullptr, *validity = nullptr, *runs = nullptr, *counts = nullptr, *dckpt = nullptr, *dmb = nullptr, *dcov = nullptr, *dsegs = nullptr;
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
