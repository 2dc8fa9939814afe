// scan_plan_test.cpp -- test-only driver of the Parquet scan planner (scan_plan.cpp), linked without the CUDA runtime by
// tests/test_parquet_cpu.py.  sp_plan() plans every batch of a NativeScan operator the way the scan does and returns JSON.
#include "scan_plan.h"

#include <cstdio>
#include <cstring>
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

// one column of one batch: its page table (data pages first), and for host-encoded PLAIN string pages the codes they carry
static void column_json(std::ostringstream& o, ColPlan& cp) {
    resolve_bodies(cp, cp.hostdec.data()); // host-produced bodies now point into cp.hostdec
    o << "{\"conv\": " << cp.conv << ", \"n_data\": " << cp.n_data << ", \"dict_elems\": " << cp.dict_elems << ", \"remap\": [";
    for (size_t i = 0; i < cp.remap.size(); i++) o << (i ? ", " : "") << cp.remap[i];
    o << "], \"pages\": [";
    for (size_t i = 0; i < cp.pages.size(); i++) {
        const PqPage& d = cp.pages[i];
        o << (i ? ", " : "") << "{\"dst_row\": " << d.dst_row << ", \"num_values\": " << d.num_values << ", \"encoding\": " << d.encoding
          << ", \"dict_off\": " << d.dict_off << ", \"dict_size\": " << d.dict_size << ", \"flags\": " << d.flags << ", \"body_bytes\": " << d.body_bytes
          << ", \"comp_bytes\": " << d.comp_bytes << ", \"def_bytes\": " << d.def_bytes;
        if (cp.dict && d.encoding == 0 && (d.flags & PQ_PAGE_HOSTDEC)) { // PLAIN string page: [levels][int32 codes]
            size_t pre = 0;
            if (d.flags & PQ_PAGE_V1_LEVELS) { uint32_t ll; memcpy(&ll, d.body, 4); pre = 4 + ll; }
            o << ", \"codes\": [";
            for (size_t k = pre; k + 4 <= (size_t)d.body_bytes; k += 4) { int32_t v; memcpy(&v, d.body + k, 4); o << (k > pre ? ", " : "") << v; }
            o << "]";
        }
        o << "}";
    }
    o << "]}";
}

// `plan`: an encoded NativeScan operator.  Returns {"pruned_row_groups", "pruned_rows", "batches": [{"units": [[file, rg, rows, row0]],
// "columns": [...]}], "dictionaries": [[hex values] per column]} or {"error": message}; valid until the next call.
extern "C" const char* sp_plan(const uint8_t* plan, size_t len, long long chunk_rows) {
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
        for (auto& f : op->data_filters) collect_prune_terms(f, terms);
        const Selection sel = select_row_groups(files, op->file_start, op->file_length, fields.size(), terms);
        const BatchPlan bp = plan_batches(sel.units, files, fields, chunk_rows);
        std::vector<StringInterner> strings(fields.size());
        o << "{\"pruned_row_groups\": " << sel.pruned_row_groups << ", \"pruned_rows\": " << sel.pruned_rows << ", \"batches\": [";
        for (size_t b = 0; b < bp.batches.size(); b++) {
            const std::vector<Unit> units = batch_units(sel.units, bp.batches[b]);
            const int64_t total = units.back().row0 + units.back().rows;
            const UploadPlan up = plan_uploads(units, files, fields.size());
            o << (b ? ", " : "") << "{\"units\": [";
            for (size_t u = 0; u < units.size(); u++) o << (u ? ", " : "") << "[" << units[u].file << ", " << units[u].rg << ", " << units[u].rows << ", " << units[u].row0 << "]";
            o << "], \"columns\": [";
            for (size_t c = 0; c < fields.size(); c++) {
                std::vector<ChunkLoc> loc;
                for (const ChunkAt& at : up.chunk_at[c]) {
                    const UploadRange& r = up.ranges[at.range];
                    loc.push_back({images[r.file].data() + r.start + at.off, (unsigned char*)(uintptr_t)(4096 + r.dev_off + at.off)}); // device addresses are only recorded
                }
                ColPlan cp = plan_column(files, fields[c], c, units, total, loc, strings[c]);
                o << (c ? ", " : "");
                column_json(o, cp);
            }
            o << "]}";
        }
        o << "], \"dictionaries\": [";
        for (size_t c = 0; c < strings.size(); c++) {
            o << (c ? ", " : "") << "[";
            for (size_t k = 0; k < strings[c].dict->values.size(); k++) o << (k ? ", " : "") << "\"" << hex(strings[c].dict->values[k]) << "\"";
            o << "]";
        }
        o << "]}";
        out = o.str();
    } catch (const std::exception& e) {
        out = "{\"error\": \"" + hex(e.what()) + "\"}";
    }
    return out.c_str();
}
