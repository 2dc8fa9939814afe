// page_index_test.cpp -- test-only driver of page-index pruning in the Parquet scan planner (scan_plan.cpp), linked without the CUDA
// runtime by tests/test_parquet_pageindex_cpu.py.  pi_plan() plans a NativeScan operator the way the scan does -- row groups by
// statistics, then rows by the page index -- and returns JSON.
#include "scan_plan.h"

#include <cstdio>
#include <sstream>

using namespace cb200;

static std::vector<uint8_t> read_file(const std::string& path) {
    std::vector<uint8_t> b;
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) throw PlanError("cannot open " + path);
    uint8_t buf[1 << 16];
    for (size_t n; (n = fread(buf, 1, sizeof(buf), f)) > 0;) b.insert(b.end(), buf, buf + n);
    fclose(f);
    return b;
}

static std::string hex(const std::string& s) {
    static const char* d = "0123456789abcdef";
    std::string o;
    for (unsigned char ch : s) { o += d[ch >> 4]; o += d[ch & 15]; }
    return o;
}

template <typename T, typename F> static void list(std::ostringstream& o, const std::vector<T>& v, F f) {
    o << "[";
    for (size_t i = 0; i < v.size(); i++) { o << (i ? ", " : ""); f(v[i]); }
    o << "]";
}

static void segs_json(std::ostringstream& o, const std::vector<PqSeg>& segs) {
    list(o, segs, [&](const PqSeg& s) { o << "[" << s.out_row << ", " << s.cov_row << ", " << s.count << "]"; });
}

// `plan`: an encoded NativeScan operator; `no_prune`: plan as CB200_NO_PRUNE=1 does.  Returns {"pruned_row_groups", "pruned_rows",
// "pruned_pages", "page_pruned_rows", "units": [{"file", "rg", "rows", "ranges", "columns": [{"pages", "covered", "segs"}]}],
// "batches": [{"units": [[file, rg, rows, row0]], "upload_bytes", "dev_total", "columns": [{"covered", "segs", "pages": [[dst_row,
// num_values]]}]}]} or {"error": message}; valid until the next call.
extern "C" const char* pi_plan(const uint8_t* plan, size_t len, long long chunk_rows, int no_prune) {
    static std::string out;
    std::ostringstream o;
    try {
        OperatorP op = decode_plan(plan, len);
        if (op->kind != OpKind::NativeScan) throw PlanError("not a NativeScan operator");
        const std::vector<StructField>& fields = op->required_schema;
        std::vector<ScanFile> files;
        std::vector<std::vector<uint8_t>> images;
        for (auto& path : op->files) {
            files.push_back(open_scan_file(path, fields));
            images.push_back(read_file(strip_file_scheme(path)));
        }
        std::vector<PruneTerm> terms;
        if (!no_prune) for (auto& f : op->data_filters) collect_prune_terms(f, terms);
        Selection sel = select_row_groups(files, op->file_start, op->file_length, fields.size(), terms);
        const PageSelection ps = select_pages(sel.units, files, fields.size(), terms);
        o << "{\"pruned_row_groups\": " << sel.pruned_row_groups << ", \"pruned_rows\": " << sel.pruned_rows << ", \"pruned_pages\": " << ps.pruned_pages
          << ", \"page_pruned_rows\": " << ps.pruned_rows << ", \"dropped_row_groups\": " << ps.dropped_row_groups << ", \"units\": ";
        list(o, sel.units, [&](const Unit& u) {
            o << "{\"file\": " << u.file << ", \"rg\": " << u.rg << ", \"rows\": " << u.rows << ", \"ranges\": ";
            if (!u.sel) { o << "null, \"columns\": null}"; return; }
            list(o, u.sel->ranges, [&](const std::pair<int64_t, int64_t>& r) { o << "[" << r.first << ", " << r.second << "]"; });
            o << ", \"columns\": ";
            list(o, u.sel->cols, [&](const ColumnWindow& w) {
                o << "{\"pages\": ";
                list(o, w.pages, [&](int p) { o << p; });
                o << ", \"covered\": " << w.covered << ", \"segs\": ";
                segs_json(o, w.segs);
                o << "}";
            });
            o << "}";
        });
        const BatchPlan bp = plan_batches(sel.units, files, fields, chunk_rows);
        std::vector<DictionaryP> dicts;
        for (size_t c = 0; c < fields.size(); c++) dicts.push_back(std::make_shared<Dictionary>());
        o << ", \"chunk_need\": " << bp.chunk_need << ", \"batches\": [";
        for (size_t b = 0; b < bp.batches.size(); b++) {
            const std::vector<Unit> units = batch_units(sel.units, bp.batches[b]);
            const int64_t total = units.back().row0 + units.back().rows;
            const UploadPlan up = plan_uploads(units, files, fields.size());
            int64_t upload = 0;
            for (auto& r : up.ranges) upload += r.end - r.start;
            o << (b ? ", " : "") << "{\"units\": ";
            list(o, units, [&](const Unit& u) { o << "[" << u.file << ", " << u.rg << ", " << u.rows << ", " << u.row0 << "]"; });
            o << ", \"upload_bytes\": " << upload << ", \"dev_total\": " << up.dev_total << ", \"columns\": [";
            for (size_t c = 0; c < fields.size(); c++) {
                // device addresses are only recorded; host addresses point into the file images
                const std::vector<ChunkLoc> loc = locate_chunks(up, c, [&](const UploadRange& r) { return images[r.file].data() + r.start; }, (unsigned char*)(uintptr_t)4096);
                ColPlan cp = plan_column(files, fields[c], c, units, total, loc, dicts[c]);
                o << (c ? ", " : "") << "{\"covered\": " << cp.covered << ", \"null_aware\": " << (cp.null_aware ? 1 : 0) << ", \"segs\": ";
                segs_json(o, cp.segs);
                o << ", \"pages\": ";
                std::vector<PqPage> data(cp.pages.begin(), cp.pages.begin() + (long)cp.n_data);
                list(o, data, [&](const PqPage& d) { o << "[" << d.dst_row << ", " << d.num_values << "]"; });
                o << "}";
            }
            o << "]}";
        }
        o << "]}";
        out = o.str();
    } catch (const std::exception& e) {
        out = "{\"error\": \"" + hex(e.what()) + "\"}";
    }
    return out.c_str();
}
