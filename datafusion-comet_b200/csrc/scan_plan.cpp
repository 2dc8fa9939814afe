// scan_plan.cpp -- host planning of the native Parquet scan (scan_plan.h).
//
// Row groups come from the footers: a file split owns the row groups that start inside it, and the pushed-down filters drop those
// whose min/max statistics rule them out (parquet_exec.rs:143-196).  Page tables come from the page headers; only string values, DELTA_BYTE_ARRAY
// decimals and pages of the host codecs are touched on the host, every other value byte is decoded on the device.
#include "scan_plan.h"

#include "device/cb_delta.h"
#include "device/cb_snappy.h"
#include "host_codecs.h"

#include <algorithm>
#include <cstring>
#include <map>
#include <mutex>

namespace cb200 {

// ---- files ----------------------------------------------------------------------------------------------------------
static std::mutex g_memfile_mu;
static std::map<std::string, std::pair<const uint8_t*, size_t>> g_memfiles;
void register_memory_file(const std::string& name, const uint8_t* p, size_t n) {
    std::lock_guard<std::mutex> lk(g_memfile_mu);
    if (p) g_memfiles[name] = {p, n};
    else g_memfiles.erase(name);
}
std::string strip_file_scheme(const std::string& p) { return p.compare(0, 7, "file://") == 0 ? p.substr(7) : p; }

// footer of a file path or of a memory:// image (then *mem / *mem_len point at the image)
static pq::FileMeta open_parquet(const std::string& path, const uint8_t** mem, size_t* mem_len) {
    *mem = nullptr;
    *mem_len = 0;
    const std::string pre = "memory://";
    if (path.compare(0, pre.size(), pre) != 0) {
        int64_t sz = 0;
        pq::FileMeta m = pq::read_footer(strip_file_scheme(path), &sz);
        pq::read_page_indexes(m, strip_file_scheme(path), sz);
        return m;
    }
    std::lock_guard<std::mutex> lk(g_memfile_mu);
    auto it = g_memfiles.find(path.substr(pre.size()));
    if (it == g_memfiles.end()) throw ExecError(3, "", "parquet: memory file '" + path + "' is not registered");
    *mem = it->second.first;
    *mem_len = it->second.second;
    pq::FileMeta m = pq::parse_footer(*mem, *mem_len);
    pq::read_page_indexes(m, *mem, *mem_len);
    return m;
}

std::string describe_parquet(const std::string& path) {
    const uint8_t* mem;
    size_t len;
    return pq::describe(open_parquet(path, &mem, &len));
}

ScanFile open_scan_file(const std::string& path, const std::vector<StructField>& fields) {
    ScanFile f;
    f.meta = open_parquet(path, &f.mem, &f.mem_len);
    for (auto& fd : fields) {
        int li = f.meta.leaf_index(fd.name);
        if (li < 0) throw Unsupported("parquet: column '" + fd.name + "' missing from " + path + " (schema evolution / default values are out of scope)");
        f.leaf_of.push_back(li);
    }
    return f;
}

// ---- row groups -----------------------------------------------------------------------------------------------------
void collect_prune_terms(const ExprP& e, std::vector<PruneTerm>& out) {
    if (e->kind == ExprKind::And) {
        for (auto& c : e->children) collect_prune_terms(c, out);
        return;
    }
    if (e->kind == ExprKind::IsNotNull && e->children[0]->kind == ExprKind::Bound) {
        PruneTerm t;
        t.col = e->children[0]->index;
        t.op = ExprKind::IsNotNull;
        out.push_back(t);
        return;
    }
    ExprKind k = e->kind;
    if (!(k == ExprKind::Eq || k == ExprKind::Lt || k == ExprKind::LtEq || k == ExprKind::Gt || k == ExprKind::GtEq)) return;
    const Expr *l = e->children[0].get(), *r = e->children[1].get();
    if (l->kind == ExprKind::Literal && r->kind == ExprKind::Bound) { // literal <op> column: mirror
        std::swap(l, r);
        k = k == ExprKind::Lt ? ExprKind::Gt : k == ExprKind::LtEq ? ExprKind::GtEq : k == ExprKind::Gt ? ExprKind::Lt : k == ExprKind::GtEq ? ExprKind::LtEq : k;
    }
    if (l->kind != ExprKind::Bound || r->kind != ExprKind::Literal || r->lit_null) return;
    PruneTerm t;
    t.col = l->index;
    t.op = k;
    const DType& ty = l->type;
    if (ty.is_integer() || ty.id == TypeId::Date || ty.id == TypeId::Timestamp || ty.id == TypeId::TimestampNtz) t.ival = r->lit_i64;
    else if (ty.is_decimal() && r->type.is_decimal() && r->type.scale == ty.scale) t.ival = (__int128)r->lit_dec;
    else if (ty.id == TypeId::Float64 || ty.id == TypeId::Float32) { t.is_float = true; t.fval = r->lit_f64; if (t.fval != t.fval) return; }
    else return;
    out.push_back(t);
}

// decode a statistics value (PLAIN-encoded single value) of a leaf; false = cannot use it
static bool stat_value(const pq::SchemaElement& se, const std::string& raw, bool* is_float, __int128* iv, double* fv) {
    *is_float = false;
    switch (se.type) {
    case pq::INT32: { if (raw.size() != 4) return false; int32_t v; memcpy(&v, raw.data(), 4); *iv = v; return true; }
    case pq::INT64: { if (raw.size() != 8) return false; int64_t v; memcpy(&v, raw.data(), 8); *iv = v; return true; }
    case pq::FLOAT: { if (raw.size() != 4) return false; float v; memcpy(&v, raw.data(), 4); *is_float = true; *fv = v; return v == v; }
    case pq::DOUBLE: { if (raw.size() != 8) return false; double v; memcpy(&v, raw.data(), 8); *is_float = true; *fv = v; return v == v; }
    case pq::FIXED_LEN_BYTE_ARRAY: { // big-endian two's complement decimal
        if (raw.empty() || raw.size() > 16) return false;
        __int128 v = (signed char)raw[0] < 0 ? -1 : 0;
        for (unsigned char ch : raw) v = (v << 8) | ch;
        *iv = v;
        return true;
    }
    default: return false;
    }
}

bool term_excludes(const PruneTerm& t, const pq::SchemaElement& se, const pq::ColumnChunkMeta& cc) {
    StatVals s;
    if (cc.has_min_max) { s.min = &cc.min_value; s.max = &cc.max_value; }
    // a chunk's null_count rules out IsNotNull only: comparison terms on a chunk are decided by its min / max alone
    s.all_null = t.op == ExprKind::IsNotNull && cc.null_count >= 0 && cc.null_count == cc.num_values && cc.num_values > 0;
    return stats_exclude(t, se, s);
}

bool stats_exclude(const PruneTerm& t, const pq::SchemaElement& se, const StatVals& s) {
    if (s.all_null) return true; // a comparison with NULL is never true
    if (t.op == ExprKind::IsNotNull || !s.min || !s.max) return false;
    bool fmin, fmax;
    __int128 imin = 0, imax = 0;
    double dmin = 0, dmax = 0;
    if (!stat_value(se, *s.min, &fmin, &imin, &dmin) || !stat_value(se, *s.max, &fmax, &imax, &dmax)) return false;
    if (fmin != t.is_float) return false;
    if (t.is_float) {
        // float statistics may be written with -0.0 / +0.0 either way; comparisons below treat them as equal, which is safe
        switch (t.op) {
        case ExprKind::Eq: return t.fval < dmin || t.fval > dmax;
        case ExprKind::Lt: return !(dmin < t.fval);
        case ExprKind::LtEq: return !(dmin <= t.fval);
        case ExprKind::Gt: return !(dmax > t.fval);
        case ExprKind::GtEq: return !(dmax >= t.fval);
        default: return false;
        }
    }
    switch (t.op) {
    case ExprKind::Eq: return t.ival < imin || t.ival > imax;
    case ExprKind::Lt: return !(imin < t.ival);
    case ExprKind::LtEq: return !(imin <= t.ival);
    case ExprKind::Gt: return !(imax > t.ival);
    case ExprKind::GtEq: return !(imax >= t.ival);
    default: return false;
    }
}

Selection select_row_groups(const std::vector<ScanFile>& files, const std::vector<int64_t>& file_start, const std::vector<int64_t>& file_length,
                            size_t n_cols, const std::vector<PruneTerm>& terms) {
    Selection s;
    for (size_t fi = 0; fi < files.size(); fi++) {
        const ScanFile& f = files[fi];
        const int64_t r0 = fi < file_start.size() ? file_start[fi] : 0, rl = fi < file_length.size() ? file_length[fi] : 0;
        for (size_t g = 0; g < f.meta.row_groups.size(); g++) {
            const pq::RowGroupMeta& rg = f.meta.row_groups[g];
            if (rg.num_rows <= 0 || rg.columns.empty()) continue;
            if (rl > 0) { // a file split owns the row groups that START inside it (DataFusion's range rule for ParquetSource)
                const int64_t off = rg.columns[0].start();
                if (off < r0 || off >= r0 + rl) continue;
            }
            bool excluded = false;
            for (auto& t : terms) {
                if (t.col < 0 || t.col >= (int)n_cols) continue;
                if (term_excludes(t, f.leaf((size_t)t.col), f.chunk(g, (size_t)t.col))) { excluded = true; break; }
            }
            if (excluded) { s.pruned_row_groups++; s.pruned_rows += rg.num_rows; continue; }
            s.units.push_back({fi, g, rg.num_rows, 0});
        }
    }
    return s;
}

// ---- pages ----------------------------------------------------------------------------------------------------------
// [first row, end row) of page i of a chunk's offset index
static std::pair<int64_t, int64_t> page_rows(const std::vector<pq::PageLocation>& loc, size_t i, int64_t rg_rows) {
    return {loc[i].first_row_index, i + 1 < loc.size() ? loc[i + 1].first_row_index : rg_rows};
}

// the pages of one column that overlap `ranges`, their covered rows and the segments that map selected rows onto them
static ColumnWindow column_window(const std::vector<pq::PageLocation>& loc, int64_t rg_rows, const std::vector<std::pair<int64_t, int64_t>>& ranges) {
    ColumnWindow w;
    std::vector<int64_t> cov_at(loc.size(), -1); // covered row of a selected page's first row
    size_t r = 0;
    for (size_t i = 0; i < loc.size(); i++) {
        const auto [p0, p1] = page_rows(loc, i, rg_rows);
        while (r < ranges.size() && ranges[r].second <= p0) r++;
        if (r < ranges.size() && ranges[r].first < p1) {
            cov_at[i] = w.covered;
            w.pages.push_back((int)i);
            w.covered += p1 - p0;
        }
    }
    int64_t out = 0;
    size_t i = 0;
    for (const auto& [a, b] : ranges) { // every page a range touches is selected, and they are consecutive: one segment per range
        while (page_rows(loc, i, rg_rows).second <= a) i++;
        w.segs.push_back({out, cov_at[i] + (a - loc[i].first_row_index), b - a});
        out += b - a;
    }
    return w;
}

PageSelection select_pages(std::vector<Unit>& units, const std::vector<ScanFile>& files, size_t n_cols, const std::vector<PruneTerm>& terms) {
    PageSelection ps;
    if (terms.empty()) return ps;
    std::vector<Unit> kept;
    for (Unit& u : units) {
        const ScanFile& f = files[u.file];
        const int64_t n = f.meta.row_groups[u.rg].num_rows;
        bool usable = !u.sel;
        for (size_t c = 0; c < n_cols && usable; c++) usable = !f.chunk(u.rg, c).offset_index.empty();
        for (auto& t : terms)
            if (usable && t.col >= 0 && t.col < (int)n_cols) usable = !f.chunk(u.rg, (size_t)t.col).column_index.null_pages.empty();
        if (!usable) { kept.push_back(u); continue; }
        // the rows some term's page statistics rule out, merged; the selection is what is left
        std::vector<std::pair<int64_t, int64_t>> out;
        for (auto& t : terms) {
            if (t.col < 0 || t.col >= (int)n_cols) continue;
            const pq::ColumnChunkMeta& cc = f.chunk(u.rg, (size_t)t.col);
            const pq::ColumnIndex& ci = cc.column_index;
            for (size_t i = 0; i < cc.offset_index.size(); i++) {
                StatVals s;
                if (ci.null_pages[i]) s.all_null = true;
                else { s.min = &ci.min_values[i]; s.max = &ci.max_values[i]; }
                if (stats_exclude(t, f.leaf((size_t)t.col), s)) out.push_back(page_rows(cc.offset_index, i, n));
            }
        }
        std::sort(out.begin(), out.end());
        auto sel = std::make_shared<RowSelection>();
        int64_t at = 0, rows = 0;
        for (const auto& [a, b] : out) {
            if (a > at) { sel->ranges.push_back({at, a}); rows += a - at; }
            at = std::max(at, b);
        }
        if (at < n) { sel->ranges.push_back({at, n}); rows += n - at; }
        if (rows == n) { kept.push_back(u); continue; }
        int64_t pages = 0;
        for (size_t c = 0; c < n_cols; c++) pages += (int64_t)f.chunk(u.rg, c).offset_index.size();
        ps.pruned_rows += n - rows;
        if (rows == 0) { ps.pruned_pages += pages; ps.dropped_row_groups++; continue; }
        for (size_t c = 0; c < n_cols; c++) {
            sel->cols.push_back(column_window(f.chunk(u.rg, c).offset_index, n, sel->ranges));
            pages -= (int64_t)sel->cols.back().pages.size();
        }
        ps.pruned_pages += pages;
        u.rows = rows;
        u.sel = std::move(sel);
        kept.push_back(u);
    }
    units = std::move(kept);
    return ps;
}

// ---- batches --------------------------------------------------------------------------------------------------------
static void unit_ranges(const ScanFile& f, const Unit& unit, size_t u, size_t n_cols, UploadPlan& up);

BatchPlan plan_batches(const std::vector<Unit>& units, const std::vector<ScanFile>& files, const std::vector<StructField>& fields, int64_t chunk_rows) {
    BatchPlan bp;
    // greedy fill up to chunk_rows; the FIRST batch is a sixteenth of that: nothing overlaps its upload, so it should be short
    // (the blocks are sized for the largest batch, so batches of different sizes cost nothing)
    int64_t total_rows = 0;
    for (auto& x : units) total_rows += x.rows;
    for (size_t u = 0; u < units.size();) {
        int64_t cap = chunk_rows;
        if (bp.batches.empty() && total_rows > 2 * chunk_rows) cap = std::max<int64_t>(chunk_rows / 16, 1);
        size_t e = u;
        int64_t rows = 0;
        while (e < units.size() && (e == u || rows + units[e].rows <= cap)) rows += units[e++].rows;
        bp.batches.push_back({u, e});
        u = e;
    }
    // block sizes: encoded bytes exactly (from the chunk metadata), decoded bytes + temporaries as an estimate that
    // the scan re-checks per batch (a slot grows once if the estimate was short)
    for (auto& b : bp.batches) {
        size_t enc = 0, work = 4096;
        int64_t rows = 0;
        for (size_t i = b.first; i < b.second; i++) {
            rows += units[i].rows;
            if (units[i].sel) { // page-pruned: its upload ranges exactly, and the uncompressed bytes of its share of the chunks
                UploadPlan one;
                one.chunk_at.assign(fields.size(), std::vector<ChunkAt>(1));
                unit_ranges(files[units[i].file], units[i], 0, fields.size(), one);
                for (auto& r : one.ranges) enc += align_up((size_t)(r.end - r.start), 256) + 256;
            }
            for (size_t c = 0; c < fields.size(); c++) {
                const pq::ColumnChunkMeta& cc = files[units[i].file].chunk(units[i].rg, c);
                if (!units[i].sel) enc += align_up((size_t)std::max<int64_t>(cc.total_compressed, 0), 256) + 256;
                if (cc.codec != pq::UNCOMPRESSED) work += (size_t)std::max<int64_t>(cc.total_uncompressed, 0) + 64 * 1024;
            }
        }
        for (size_t c = 0; c < fields.size(); c++) {
            const DType& t = fields[c].type;
            const size_t w = t.is_decimal() ? (t.precision <= 18 ? 8 : 16) : t.is_string() ? 4 : (size_t)std::max(t.arrow_width(), 1);
            bool nulls = false, dict_encoded = false, delta = false;
            int64_t cov = 0; // rows the column's pages decode into
            for (size_t i = b.first; i < b.second; i++) {
                const ScanFile& f = files[units[i].file];
                const pq::ColumnChunkMeta& cc = f.chunk(units[i].rg, c);
                cov += units[i].sel ? units[i].sel->cols[c].covered : units[i].rows;
                if (f.leaf(c).repetition == 1 && cc.null_count != 0) nulls = true;
                for (int enc : cc.encodings) {
                    if (enc == pq::RLE_DICTIONARY || enc == pq::PLAIN_DICTIONARY) dict_encoded = true;
                    if (enc == pq::DELTA_BINARY_PACKED) delta = true;
                }
            }
            work += (size_t)rows * w + 4096;                                  // decoded column
            if (cov != rows) work += (size_t)cov * w + 4096;                  // page-pruned: the covered rows it is selected from
            work += (b.second - b.first) * 96 * 1024;                         // page tables / dictionaries
            if (dict_encoded) work += (size_t)cov * 4 + (b.second - b.first) * 16 * 2048; // run table: (values / 8 + 64) runs of 32 bytes per page
            if (nulls) work += (size_t)cov * (w + 5 + 4) + 65536;             // dense values + validity bytes + indices + level runs
            if (delta) work += ((size_t)cov / 16 + (b.second - b.first) * 256) * sizeof(PqMiniblock); // miniblock table: values / 32 + 2 entries per page
        }
        bp.chunk_need = std::max(bp.chunk_need, enc + 65536);
        bp.work_estimate = std::max(bp.work_estimate, work + work / 16);
    }
    return bp;
}

std::vector<Unit> batch_units(const std::vector<Unit>& units, std::pair<size_t, size_t> batch) {
    std::vector<Unit> out(units.begin() + (long)batch.first, units.begin() + (long)batch.second);
    int64_t row0 = 0;
    for (auto& u : out) { u.row0 = row0; row0 += u.rows; }
    return out;
}

// ---- upload ranges --------------------------------------------------------------------------------------------------
// Per row group, the selected column chunks sorted by file offset and merged into byte ranges (gaps of unselected columns up to
// 64 KB ride along) -- PCIe moves few large copies faster than many chunk-sized ones (measured: 49 GB/s at 1.8 MB per copy,
// 54 GB/s at 12 MB).
// The file bytes a page-pruned unit reads of column c: what precedes the first data page (the dictionary page), then every run of
// selected data pages.
static std::vector<std::pair<int64_t, int64_t>> chunk_pieces(const pq::ColumnChunkMeta& cc, const ColumnWindow& w) {
    std::vector<std::pair<int64_t, int64_t>> out;
    const auto& loc = cc.offset_index;
    if (loc[0].offset > cc.start()) out.push_back({cc.start(), loc[0].offset});
    for (size_t k = 0; k < w.pages.size(); k++) {
        const pq::PageLocation& p = loc[(size_t)w.pages[k]];
        const bool next_to_last = k > 0 && w.pages[k] == w.pages[k - 1] + 1 && out.back().second == p.offset;
        if (next_to_last) out.back().second = p.offset + p.compressed_page_size;
        else out.push_back({p.offset, p.offset + p.compressed_page_size});
    }
    return out;
}

// the upload ranges of unit u, appended to `up`
static void unit_ranges(const ScanFile& f, const Unit& unit, size_t u, size_t n_cols, UploadPlan& up) {
    struct Item { int64_t start, end; size_t col; long piece; }; // piece -1: the whole chunk
    std::vector<Item> items;
    for (size_t c = 0; c < n_cols; c++) {
        const pq::ColumnChunkMeta& cc = f.chunk(unit.rg, c);
        if (cc.total_compressed < 0 || cc.start() < 0) throw PlanError("parquet: negative column chunk offset / size");
        if (f.mem && (size_t)cc.start() + (size_t)cc.total_compressed > f.mem_len) throw PlanError("parquet: column chunk beyond the end of the file image");
        if (!unit.sel) { items.push_back({cc.start(), cc.start() + cc.total_compressed, c, -1}); continue; }
        const auto pieces = chunk_pieces(cc, unit.sel->cols[c]);
        for (size_t k = 0; k < pieces.size(); k++) items.push_back({pieces[k].first, pieces[k].second, c, (long)k});
    }
    std::sort(items.begin(), items.end(), [](const Item& a, const Item& b) { return a.start != b.start ? a.start < b.start : a.col != b.col ? a.col < b.col : a.piece < b.piece; });
    bool open_range = false;
    for (auto& it : items) {
        // a gap of up to 64 KB rides along; chunks may also overlap (the same column projected twice)
        if (open_range && it.start - up.ranges.back().end <= 65536) up.ranges.back().end = std::max(up.ranges.back().end, it.end);
        else { up.ranges.push_back({unit.file, it.start, it.end, 0}); open_range = true; }
        const size_t r = up.ranges.size() - 1;
        const int64_t off = it.start - up.ranges.back().start;
        ChunkAt& at = up.chunk_at[it.col][u];
        if (it.piece < 0) { at.range = r; at.off = off; continue; }
        if (it.piece == 0) { at.range = r; at.off = off; }
        at.pieces.push_back({it.start, it.end, r, off});
    }
}

UploadPlan plan_uploads(const std::vector<Unit>& units, const std::vector<ScanFile>& files, size_t n_cols) {
    UploadPlan up;
    up.chunk_at.assign(n_cols, std::vector<ChunkAt>(units.size()));
    for (size_t u = 0; u < units.size(); u++) unit_ranges(files[units[u].file], units[u], u, n_cols, up);
    for (auto& r : up.ranges) { r.dev_off = up.dev_total; up.dev_total += align_up((size_t)(r.end - r.start), 256); }
    return up;
}

// ---- columns --------------------------------------------------------------------------------------------------------
static void check_annotations(const pq::SchemaElement& se, const DType& t) {
    // SchemaElement.converted_type / logicalType decide what the physical bytes MEAN; a mismatch must not be read silently
    const int ct = se.converted_type;
    if (t.id == TypeId::Timestamp || t.id == TypeId::TimestampNtz) {
        const bool millis = ct == 9 || se.ts_unit == 1, nanos = se.ts_unit == 3;
        if (millis || nanos) throw Unsupported(std::string("parquet: TIMESTAMP_") + (millis ? "MILLIS" : "NANOS") + " column '" + se.name + "' (only microsecond timestamps are decoded; unit conversion is out of scope)");
    }
    if (ct == 13 || ct == 14 || (se.int_bits >= 32 && se.int_signed == 0)) throw Unsupported("parquet: unsigned 32/64-bit integer column '" + se.name + "'");
    if ((ct == 11 || ct == 12 || (se.int_bits > 0 && se.int_bits < 32 && se.int_signed == 0)) && !(t.id == TypeId::Int32 || t.id == TypeId::Int64 || t.id == TypeId::Int16))
        throw Unsupported("parquet: unsigned 8/16-bit integer column '" + se.name + "' read as " + t.str());
    if (t.is_decimal()) {
        if (se.scale != t.scale) throw Unsupported("parquet decimal scale differs from the requested type (schema adapter casts are out of scope)");
        if (se.precision > 0 && se.precision > t.precision) throw Unsupported("parquet: decimal(" + std::to_string(se.precision) + ") column '" + se.name + "' read as " + t.str());
        if (ct != 5 && !se.logical_decimal) throw Unsupported("parquet: column '" + se.name + "' carries no DECIMAL annotation but is read as " + t.str());
    }
}

// the conversion from the leaf's physical type to the requested type
static void column_type(const pq::SchemaElement& se, const DType& t, ColPlan& cp) {
    cp.type_length = se.type_length;
    switch (se.type) {
    case pq::INT32:
        if (!(t.is_integer() || t.id == TypeId::Date || (t.is_decimal() && t.precision <= 9))) throw Unsupported("parquet INT32 -> " + t.str());
        if (t.id == TypeId::Int64) { cp.conv = PQ_I32_TO_I64; cp.out_w = 8; cp.phys = Phys::I64; }
        else { cp.conv = PQ_COPY32; cp.out_w = 4; cp.phys = Phys::I32; }
        break;
    case pq::INT64:
        if (!(t.id == TypeId::Int64 || t.id == TypeId::Timestamp || t.id == TypeId::TimestampNtz || (t.is_decimal() && t.precision <= 18)))
            throw Unsupported("parquet INT64 -> " + t.str());
        cp.conv = PQ_COPY64; cp.out_w = 8; cp.phys = Phys::I64;
        break;
    case pq::FLOAT: if (t.id != TypeId::Float32) throw Unsupported("parquet FLOAT -> " + t.str()); cp.conv = PQ_COPY32; cp.out_w = 4; cp.phys = Phys::F32; break;
    case pq::DOUBLE: if (t.id != TypeId::Float64) throw Unsupported("parquet DOUBLE -> " + t.str()); cp.conv = PQ_COPY64; cp.out_w = 8; cp.phys = Phys::F64; break;
    case pq::FIXED_LEN_BYTE_ARRAY:
        if (!t.is_decimal() || se.type_length > 16) throw Unsupported("parquet FIXED_LEN_BYTE_ARRAY -> " + t.str());
        if (t.precision <= 18) { cp.conv = PQ_FLBA_TO_I64; cp.out_w = 8; cp.phys = Phys::I64; }
        else { cp.conv = PQ_FLBA_TO_I128; cp.out_w = 16; cp.phys = Phys::I128; }
        break;
    case pq::BYTE_ARRAY:
        if (!t.is_string()) throw Unsupported("parquet BYTE_ARRAY -> " + t.str());
        cp.conv = -1; cp.out_w = 4; cp.phys = Phys::I32; // dictionary codes
        break;
    default: throw Unsupported("parquet physical type " + std::to_string(se.type));
    }
}

namespace {

// the bytes of a page that one codec applies to: a whole v1 page, a v2 values section, a dictionary page
struct Section {
    const uint8_t* host;  // the stored bytes on the host ...
    unsigned char* dev;   // ... and where they land on the device
    int comp, unc;        // stored / uncompressed size
    int codec;            // pq::UNCOMPRESSED for a v2 values section stored as is
};

// appends the uncompressed bytes of `s` (any codec but UNCOMPRESSED) to `out`, then `pad` zero bytes
void decompress_on_host(const Section& s, std::vector<uint8_t>& out, size_t pad, const char* what) {
    if (s.unc < 0 || s.comp < 0) throw PlanError("parquet: negative page size");
    const size_t off = out.size();
    out.resize(off + (size_t)s.unc + pad, 0);
    if (s.codec != pq::SNAPPY) host_decompress(s.codec, s.host, (size_t)s.comp, out.data() + off, (size_t)s.unc);
    else if (cb::snappy_decode_serial(s.host, s.comp, out.data() + off, s.unc) != s.unc) throw PlanError(std::string("parquet: malformed Snappy ") + what);
}

// [u32 length][bytes] values of a BYTE_ARRAY section
struct ByteArrays {
    const uint8_t *p, *e;
    const char* truncated; // the error a value running past the section raises
    bool more() const { return p < e; }
    std::string next() {
        if (e - p < 4) throw PlanError(truncated);
        uint32_t len;
        memcpy(&len, p, 4);
        p += 4;
        if (len > (size_t)(e - p)) throw PlanError(truncated);
        std::string v((const char*)p, len);
        p += len;
        return v;
    }
};

// a DELTA_BINARY_PACKED section of at most `cap` values (device/cb_delta.h) at p, as 32-bit lengths; advances p past it
std::vector<int32_t> delta_lengths(const uint8_t*& p, const uint8_t* e, long long cap, const char* what) {
    cb::DbpHeader h;
    if (cb::dbp_header(p, e, h) != 0 || h.total > cap) throw PlanError(std::string("parquet: malformed DELTA_BINARY_PACKED ") + what);
    std::vector<cb::i64> v((size_t)h.total + 1);
    long long n = 0;
    const uint8_t* q = cb::dbp_decode_serial(p, e, 32, v.data(), cap, &n);
    if (!q) throw PlanError(std::string("parquet: malformed DELTA_BINARY_PACKED ") + what);
    p = q;
    std::vector<int32_t> out((size_t)n);
    for (long long i = 0; i < n; i++) {
        out[(size_t)i] = (int32_t)v[(size_t)i];
        if (out[(size_t)i] < 0) throw PlanError(std::string("parquet: negative length in ") + what);
    }
    return out;
}

// The values of a BYTE_ARRAY / FIXED_LEN_BYTE_ARRAY section in order, in any byte-array value encoding: PLAIN ([u32 length][bytes]),
// DELTA_LENGTH_BYTE_ARRAY (DELTA_BINARY_PACKED lengths, then the bytes back to back) or DELTA_BYTE_ARRAY (DELTA_BINARY_PACKED prefix
// lengths, then the suffixes as DELTA_LENGTH_BYTE_ARRAY; a value is the previous value's first `prefix` bytes + its suffix).  At most
// `cap` values (the page's row count).
template <typename F> void for_each_byte_array(int encoding, const uint8_t* p, const uint8_t* e, long long cap, F f) {
    if (encoding == pq::PLAIN) {
        ByteArrays vals{p, e, "parquet: truncated PLAIN string page"};
        while (vals.more()) f(vals.next());
        return;
    }
    std::vector<int32_t> prefix;
    if (encoding == pq::DELTA_BYTE_ARRAY) prefix = delta_lengths(p, e, cap, "prefix lengths");
    const std::vector<int32_t> len = delta_lengths(p, e, cap, "lengths");
    if (encoding == pq::DELTA_BYTE_ARRAY && prefix.size() != len.size()) throw PlanError("parquet: DELTA_BYTE_ARRAY prefix and suffix counts differ");
    std::string v;
    for (size_t i = 0; i < len.size(); i++) {
        if ((size_t)len[i] > (size_t)(e - p)) throw PlanError("parquet: truncated DELTA_LENGTH_BYTE_ARRAY / DELTA_BYTE_ARRAY page");
        if (encoding == pq::DELTA_BYTE_ARRAY) {
            if ((size_t)prefix[i] > v.size()) throw PlanError("parquet: DELTA_BYTE_ARRAY prefix longer than the previous value");
            v.resize((size_t)prefix[i]);
            v.append((const char*)p, (size_t)len[i]);
        } else v.assign((const char*)p, (size_t)len[i]);
        p += len[i];
        f(v);
    }
}

// a body kept as an offset until resolve_bodies
void set_body_offset(PqPage& d, size_t off) { d.body = (unsigned char*)(uintptr_t)off; }

// the page tables of one column over the chunks of a batch
class ColumnPlanner {
  public:
    ColumnPlanner(const pq::SchemaElement& se, const StructField& field, size_t c, Dictionary& strings, ColPlan& cp)
        : se(se), field(field), c(c), strings(strings), cp(cp) {}

    void chunk(const ScanFile& f, const Unit& unit, const ChunkLoc& at) {
        const pq::SchemaElement& use = f.leaf(c);
        if (use.type != se.type || use.type_length != se.type_length) throw Unsupported("parquet: column '" + field.name + "' changes physical type between files");
        if (&use != &se) check_annotations(use, field.type);
        const bool optional = use.repetition == 1;
        cp.optional = cp.optional || optional;
        const pq::ColumnChunkMeta& cc = f.chunk(unit.rg, c);
        if (optional && cc.null_count != 0) nulls_possible = true; // unknown (-1) counts as possible
        if (cc.codec != pq::UNCOMPRESSED && cc.codec != pq::SNAPPY && !host_codec_supported(cc.codec))
            throw Unsupported("parquet codec " + std::to_string(cc.codec) + " (UNCOMPRESSED and SNAPPY are decompressed on the device, ZSTD / LZ4 / LZ4_RAW / GZIP on the host; BROTLI / LZO are not read)");
        const int64_t rg_rows = f.meta.row_groups[unit.rg].num_rows;
        if (cc.num_values != rg_rows) throw Unsupported("parquet: repeated column (num_values != num_rows)");
        const int64_t cov0 = row; // pages decode into covered rows: the batch's rows unless a unit before this one is page-pruned
        dict_off = -1;
        dict_size = 0;
        if (!unit.sel) {
            for (auto& pg : pq::walk_pages(at.host, (size_t)cc.total_compressed, cc.num_values)) {
                const Section s{at.host + pg.data_offset, at.dev + pg.data_offset, pg.compressed_size, pg.uncompressed_size, cc.codec};
                if (pg.type == pq::DICTIONARY_PAGE) dictionary_page(pg, s);
                else if (pg.type == pq::DATA_PAGE || pg.type == pq::DATA_PAGE_V2) data_page(pg, s, optional);
            }
            if (row != cov0 + rg_rows) throw PlanError("parquet: data pages of column '" + field.name + "' do not add up to the row group's row count");
            add_seg({unit.row0, cov0, unit.rows});
            return;
        }
        // page-pruned: the dictionary page in front of the first data page, then the selected data pages where the offset index puts them
        const ColumnWindow& w = unit.sel->cols[c];
        const auto& loc = cc.offset_index;
        if (loc[0].offset > cc.start()) {
            const auto [h, d] = piece(at, cc.start(), loc[0].offset - cc.start());
            for (auto& pg : pq::walk_pages(h, (size_t)(loc[0].offset - cc.start()), 1)) {
                const Section s{h + pg.data_offset, d + pg.data_offset, pg.compressed_size, pg.uncompressed_size, cc.codec};
                if (pg.type == pq::DICTIONARY_PAGE) dictionary_page(pg, s);
                else if (pg.type == pq::DATA_PAGE || pg.type == pq::DATA_PAGE_V2) throw PlanError("parquet: column '" + field.name + "' has a data page in front of the first page its offset index lists");
            }
        }
        for (int i : w.pages) {
            const pq::PageLocation& pl = loc[(size_t)i];
            const int64_t span = ((size_t)i + 1 < loc.size() ? loc[(size_t)i + 1].first_row_index : rg_rows) - pl.first_row_index;
            const auto [h, d] = piece(at, pl.offset, pl.compressed_page_size);
            const std::vector<pq::PageInfo> one = pq::walk_pages(h, (size_t)pl.compressed_page_size, 1);
            if (one.size() != 1 || (one[0].type != pq::DATA_PAGE && one[0].type != pq::DATA_PAGE_V2) || one[0].num_values != span ||
                one[0].data_offset + one[0].compressed_size != pl.compressed_page_size)
                throw PlanError("parquet: a page header of column '" + field.name + "' contradicts its offset index");
            const pq::PageInfo& pg = one[0];
            data_page(pg, Section{h + pg.data_offset, d + pg.data_offset, pg.compressed_size, pg.uncompressed_size, cc.codec}, optional);
        }
        if (row != cov0 + w.covered) throw PlanError("parquet: selected data pages of column '" + field.name + "' do not add up to their rows");
        for (const PqSeg& s : w.segs) add_seg({unit.row0 + s.out_row, cov0 + s.cov_row, s.count});
    }

    void finish(int64_t total) {
        cp.n_data = cp.pages.size();
        cp.n_dict_pages = dict_pages.size();
        cp.pages.insert(cp.pages.end(), dict_pages.begin(), dict_pages.end()); // one upload for every descriptor of this column
        for (auto& d : cp.pages) { d.seg_base = (int)cp.n_segs_total; cp.n_segs_total += d.n_segs; } // n_segs = 0 unless Snappy
        // the covered rows are the batch's rows exactly when no unit is page-pruned in this column: no selection step then
        cp.covered = row;
        if (row == total) cp.segs.clear();
        // definition levels: the statistics' null_count == 0 selects the verify-only fast path; otherwise values are decoded
        // densely and scattered to their rows
        cp.null_aware = cp.optional && nulls_possible;
        if (cp.null_aware && row >= (int64_t)1 << 32) throw Unsupported("parquet: NULL-aware decode of more than 2^32 rows per batch (lower spark.comet.b200.chunkRows)");
    }

  private:
    const pq::SchemaElement& se;
    const StructField& field;
    const size_t c;
    Dictionary& strings; // the column's plan-wide dictionary (string columns)
    ColPlan& cp;
    std::vector<PqPage> dict_pages; // fixed-width dictionary pages (decoded into the combined dictionary)
    std::vector<uint8_t> scratch;
    bool nulls_possible = false;
    int64_t row = 0, dict_off = -1; // next output row / the current chunk's dictionary in the combined one
    int dict_size = 0;

    // host / device address of the file bytes [off, off + len) of a page-pruned chunk
    std::pair<const uint8_t*, unsigned char*> piece(const ChunkLoc& at, int64_t off, int64_t len) const {
        for (const PieceLoc& p : at.pieces)
            if (p.start <= off && off + len <= p.end) return {p.host + (off - p.start), p.dev + (off - p.start)};
        throw PlanError("parquet: a selected page of column '" + field.name + "' was not uploaded");
    }

    // appends a segment, extending the last one when they are contiguous in both row spaces
    void add_seg(const PqSeg& s) {
        if (s.count <= 0) return;
        if (!cp.segs.empty()) {
            PqSeg& b = cp.segs.back();
            if (b.out_row + b.count == s.out_row && b.cov_row + b.count == s.cov_row) { b.count += s.count; return; }
        }
        cp.segs.push_back(s);
    }

    // uncompressed bytes of a section on the host, valid until the next call
    std::pair<const uint8_t*, size_t> host_section(const Section& s, const char* what) {
        if (s.codec == pq::UNCOMPRESSED) return {s.host, (size_t)s.comp};
        scratch.clear();
        decompress_on_host(s, scratch, 16, what);
        return {scratch.data(), (size_t)s.unc};
    }

    // a body produced on the host at cp.hostdec[off, end): padded to 16 bytes with >= 8 spare bytes for the unaligned-word loads
    void host_body(PqPage& d, size_t off) {
        const size_t n = cp.hostdec.size() - off;
        cp.hostdec.resize(off + (n + 31) / 16 * 16, 0);
        set_body_offset(d, off);
        d.body_bytes = (int)n;
        d.flags |= PQ_PAGE_HOSTDEC;
    }

    // UNCOMPRESSED: the body is read where it landed; SNAPPY: decompressed on the device into `dunc`; other codecs: on the host
    void place_body(PqPage& d, const Section& s) {
        if (s.codec == pq::UNCOMPRESSED) {
            d.body = s.dev;
            d.body_bytes = s.comp;
        } else if (s.codec == pq::SNAPPY) {
            d.comp = s.dev;
            d.comp_bytes = s.comp;
            set_body_offset(d, cp.unc_bytes);
            d.body_bytes = s.unc;
            d.n_segs = (s.unc + PQ_SNAPPY_SEG - 1) / PQ_SNAPPY_SEG; // checkpoint entries of the segmented Snappy decoder
            cp.unc_bytes += ((size_t)s.unc + 31) / 16 * 16;       // 16-byte aligned, >= 8 spare bytes for the unaligned-word loads
            cp.any_compressed = true;
        } else {
            const size_t off = cp.hostdec.size();
            decompress_on_host(s, cp.hostdec, 0, "page");
            host_body(d, off);
        }
    }

    // String pages that are not dictionary-encoded (PLAIN: a writer's dictionary fallback; DELTA_LENGTH_BYTE_ARRAY / DELTA_BYTE_ARRAY).
    // Strings live on the device as codes of the plan-wide dictionary only, so the host -- which already parses every string
    // dictionary page -- turns the page's values into codes: the page the device sees is [levels as written][int32 codes], PLAIN.
    // DELTA_BYTE_ARRAY decimals (FIXED_LEN_BYTE_ARRAY) are sequential by construction -- every value starts with a prefix of the one
    // before -- and come out the same way as [levels as written][type_length-byte big-endian values], a PLAIN page.
    void place_host_values(PqPage& d, const Section& s, int encoding) {
        const auto b = host_section(s, "page");
        size_t pre = 0;
        if (d.flags & PQ_PAGE_V1_LEVELS) { // [u32 byte length][RLE definition levels] stay as they are
            if (b.second < 4) throw PlanError("parquet: data page shorter than its level header");
            uint32_t ll;
            memcpy(&ll, b.first, 4);
            if ((size_t)ll + 4 > b.second) throw PlanError("parquet: definition levels exceed the page");
            pre = 4 + ll;
        }
        const size_t off = cp.hostdec.size();
        cp.hostdec.insert(cp.hostdec.end(), b.first, b.first + pre);
        if (se.type == pq::BYTE_ARRAY) {
            for_each_byte_array(encoding, b.first + pre, b.first + b.second, d.num_values, [&](std::string v) {
                const int32_t code = strings.intern(std::move(v));
                const uint8_t* code_bytes = (const uint8_t*)&code;
                cp.hostdec.insert(cp.hostdec.end(), code_bytes, code_bytes + 4);
            });
            cp.conv = PQ_COPY32; // k_pq_plain copies the codes of PLAIN pages; dictionary pages of the same column go through k_pq_rle_decode
        } else {
            for_each_byte_array(encoding, b.first + pre, b.first + b.second, d.num_values, [&](const std::string& v) {
                if (v.size() != (size_t)se.type_length) throw PlanError("parquet: DELTA_BYTE_ARRAY value of column '" + field.name + "' is not type_length bytes long");
                cp.hostdec.insert(cp.hostdec.end(), (const uint8_t*)v.data(), (const uint8_t*)v.data() + v.size());
            });
        }
        host_body(d, off);
    }

    void dictionary_page(const pq::PageInfo& pg, const Section& s) {
        dict_size = (int)pg.num_values;
        dict_off = cp.dict_elems;
        if (se.type == pq::BYTE_ARRAY) { // strings: unified with the plan-wide dictionary on the host; the device gets the code remap table
            const auto b = host_section(s, "dictionary page");
            ByteArrays vals{b.first, b.first + b.second, "parquet: truncated dictionary page"};
            for (int k = 0; k < dict_size; k++) cp.remap.push_back(strings.intern(vals.next()));
        } else {
            PqPage dp{};
            place_body(dp, s);
            dp.num_values = dict_size;
            dp.dst_row = cp.dict_elems; // decoded into the combined dictionary at this element offset
            dict_pages.push_back(dp);
        }
        cp.dict_elems += dict_size;
    }

    void data_page(const pq::PageInfo& pg, const Section& s, bool optional) {
        PqPage d{};
        d.dst_row = row;
        d.num_values = (int)pg.num_values;
        Section vals = s;
        if (pg.type == pq::DATA_PAGE) {
            // v1: [u32 length + definition levels (optional columns)] [values], compressed as one block
            if (optional) d.flags |= PQ_PAGE_V1_LEVELS;
            // the level decoders read the RLE / bit-packed hybrid behind a u32 length; deprecated BIT_PACKED levels have neither
            if (optional && pg.def_encoding != pq::RLE)
                throw Unsupported("parquet definition level encoding " + std::to_string(pg.def_encoding) + " (column '" + field.name + "'): only RLE levels are read");
        } else {
            // v2: repetition + definition levels sit uncompressed in front of the (optionally compressed) values
            const int lv = pg.rep_levels_bytes + pg.def_levels_bytes;
            if (lv > pg.compressed_size || lv > pg.uncompressed_size) throw PlanError("parquet: data page v2 level sizes exceed the page");
            // every row of an optional column has a level; without any, the page would read as a required column's (Arrow refuses it too)
            if (optional && pg.def_levels_bytes <= 0 && pg.num_values > 0)
                throw PlanError("parquet: data page v2 of optional column '" + field.name + "' has no definition levels");
            d.def_ptr = s.dev + pg.rep_levels_bytes;
            d.def_bytes = pg.def_levels_bytes;
            vals = {s.host + lv, s.dev + lv, s.comp - lv, s.unc - lv, pg.v2_compressed ? s.codec : (int)pq::UNCOMPRESSED};
        }
        const int enc = pg.encoding;
        const bool dict = enc == pq::RLE_DICTIONARY || enc == pq::PLAIN_DICTIONARY;
        const bool fixed_int = se.type == pq::INT32 || se.type == pq::INT64;
        const bool on_host = (se.type == pq::BYTE_ARRAY && (enc == pq::PLAIN || enc == pq::DELTA_LENGTH_BYTE_ARRAY || enc == pq::DELTA_BYTE_ARRAY)) ||
                             (se.type == pq::FIXED_LEN_BYTE_ARRAY && enc == pq::DELTA_BYTE_ARRAY);
        if (!(dict || on_host || enc == pq::PLAIN || (enc == pq::DELTA_BINARY_PACKED && fixed_int) || (enc == pq::BYTE_STREAM_SPLIT && se.type != pq::BYTE_ARRAY)))
            throw Unsupported("parquet value encoding " + std::to_string(enc) + " on physical type " + std::to_string(se.type) + " (column '" + field.name + "')");
        if (on_host) place_host_values(d, vals, enc);
        else place_body(d, vals);
        if (enc == pq::PLAIN || on_host) {
            d.encoding = PQ_ENC_PLAIN;
        } else if (enc == pq::DELTA_BINARY_PACKED) {
            d.encoding = PQ_ENC_DBP;
            d.mb_base = cp.mb_base;
            d.mb_cap = (int)(pg.num_values / 32 + 2); // entry 0 = the first value, then miniblocks of >= 32 values each
            cp.mb_base += d.mb_cap;
        } else if (enc == pq::BYTE_STREAM_SPLIT) {
            d.encoding = PQ_ENC_BSS;
        } else {
            if (dict_off < 0) throw PlanError("parquet: dictionary-encoded page without a dictionary page");
            d.encoding = PQ_ENC_DICT;
            d.run_base = cp.run_base;
            d.max_runs = (int)(pg.num_values / 8 + 64);
            d.dict_off = dict_off;
            d.dict_size = dict_size;
            cp.run_base += d.max_runs;
        }
        if (optional) {
            d.def_run_base = cp.def_run_base;
            d.def_max_runs = (int)(pg.num_values / 8 + 64);
            cp.def_run_base += d.def_max_runs;
        }
        row += pg.num_values;
        cp.pages.push_back(d);
    }
};

} // namespace

ColPlan plan_column(const std::vector<ScanFile>& files, const StructField& field, size_t c, const std::vector<Unit>& units, int64_t total,
                    const std::vector<ChunkLoc>& loc, const DictionaryP& dict) {
    ColPlan cp;
    const pq::SchemaElement& se = files[units[0].file].leaf(c);
    column_type(se, field.type, cp);
    check_annotations(se, field.type);
    if (se.type == pq::BYTE_ARRAY) cp.dict = dict;
    ColumnPlanner p(se, field, c, *dict, cp);
    for (size_t u = 0; u < units.size(); u++) p.chunk(files[units[u].file], units[u], loc[u]);
    p.finish(total);
    return cp;
}

void buffer_requests(ColPlan& cp, int64_t total, std::vector<std::pair<uint8_t**, size_t>>& reqs) {
    const size_t n = (size_t)std::max<int64_t>(total, 1);
    const size_t nc = cp.segs.empty() ? n : (size_t)std::max<int64_t>(cp.covered, 1); // rows the pages decode into
    cp.out_bytes = n * (size_t)cp.out_w;
    reqs.push_back({&cp.out, cp.out_bytes});
    if (cp.pages.empty()) return;
    if (cp.any_compressed) {
        reqs.push_back({&cp.dunc, cp.unc_bytes + 64});
        reqs.push_back({&cp.dckpt, (size_t)(cp.n_segs_total + 1) * 4});
    }
    if (cp.dict_elems > 0 && cp.remap.empty()) reqs.push_back({&cp.ddict, (size_t)cp.dict_elems * (size_t)cp.out_w + 16}); // string dictionaries: the remap table in the mirror IS the dictionary
    if (!cp.segs.empty() && !cp.null_aware) reqs.push_back({&cp.dcov, nc * (size_t)cp.out_w});
    if (cp.null_aware) {
        reqs.push_back({&cp.dense, nc * (size_t)cp.out_w});
        reqs.push_back({&cp.dvalid, nc + 64});
        reqs.push_back({&cp.didx, nc * 4 + 64});
        reqs.push_back({&cp.druns, (size_t)std::max<int64_t>(cp.def_run_base, 1) * sizeof(PqRun)});
        reqs.push_back({&cp.dcounts, cp.n_data * 4 + 16});
        cp.validity_bytes = (n + 31) / 32 * 4 + 16;
        reqs.push_back({&cp.validity, cp.validity_bytes});
    }
    if (cp.mb_base > 0) reqs.push_back({&cp.dmb, (size_t)cp.mb_base * sizeof(PqMiniblock)});
    if (cp.run_base > 0) {
        reqs.push_back({&cp.runs, (size_t)cp.run_base * sizeof(PqRun)});
        reqs.push_back({&cp.counts, cp.n_data * 4 + 16});
    }
}

// The one place page-body offsets become addresses: Snappy pages (comp set) into the column's decompression buffer, pages produced on
// the host (PQ_PAGE_HOSTDEC) into the staged copy of cp.hostdec.  Every other body already holds its device address.
void resolve_bodies(ColPlan& cp, uint8_t* hostdec_dev) {
    for (auto& d : cp.pages) {
        uint8_t* base = d.comp ? cp.dunc : (d.flags & PQ_PAGE_HOSTDEC) ? hostdec_dev : nullptr;
        if (base) d.body = base + (size_t)(uintptr_t)d.body;
    }
}

} // namespace cb200
