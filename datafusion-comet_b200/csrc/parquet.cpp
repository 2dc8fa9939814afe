// parquet.cpp -- Thrift compact protocol reader + Parquet footer / page-header structures (host side).
#include "parquet.h"
#include "exec.h"

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <sstream>
#include <stdexcept>

namespace cb200 {
namespace pq {

namespace {

struct TReader { // Thrift compact protocol (THRIFT-110)
    const uint8_t* p;
    const uint8_t* end;
    uint64_t varint() {
        uint64_t v = 0;
        int shift = 0;
        while (true) {
            if (p >= end) throw PlanError("parquet: truncated thrift varint");
            uint8_t b = *p++;
            v |= (uint64_t)(b & 0x7f) << shift;
            if (!(b & 0x80)) return v;
            shift += 7;
            if (shift > 63) throw PlanError("parquet: thrift varint too long");
        }
    }
    int64_t zigzag() { uint64_t v = varint(); return (int64_t)(v >> 1) ^ -(int64_t)(v & 1); }
    std::string binary() {
        uint64_t n = varint();
        if ((uint64_t)(end - p) < n) throw PlanError("parquet: truncated thrift binary");
        std::string s((const char*)p, (size_t)n);
        p += n;
        return s;
    }
    // field header: returns type (0 = stop); id in *fid
    int field(int16_t* fid, int16_t last) {
        if (p >= end) throw PlanError("parquet: truncated thrift struct");
        uint8_t b = *p++;
        if (b == 0) return 0;
        int type = b & 0x0f, delta = b >> 4;
        *fid = delta ? (int16_t)(last + delta) : (int16_t)zigzag();
        return type;
    }
    void list_header(int* elem_type, uint32_t* size) {
        if (p >= end) throw PlanError("parquet: truncated thrift list");
        uint8_t b = *p++;
        *elem_type = b & 0x0f;
        *size = b >> 4;
        if (*size == 15) *size = (uint32_t)varint();
    }
    void need(size_t n) const { if ((size_t)(end - p) < n) throw PlanError("parquet: truncated thrift value"); }
    void skip(int type, int depth = 0) {
        if (depth > 64) throw PlanError("parquet: thrift structure nested too deeply");
        switch (type) {
        case 1: case 2: break;          // bool encoded in the field header
        case 3: need(1); p++; break;    // byte
        case 4: case 5: case 6: zigzag(); break;
        case 7: need(8); p += 8; break; // double
        case 8: binary(); break;
        case 9: case 10: {
            int et; uint32_t n;
            list_header(&et, &n);
            if (n > (uint64_t)(end - p)) throw PlanError("parquet: thrift list longer than its buffer"); // every element takes at least one byte
            for (uint32_t i = 0; i < n; i++) {
                if (et == 1 || et == 2) { need(1); p++; } // bools in lists take one byte each
                else skip(et, depth + 1);
            }
            break;
        }
        case 11: {
            uint32_t n = (uint32_t)varint();
            if (n) {
                need(1);
                uint8_t kv = *p++;
                if (n > (uint64_t)(end - p) + 1) throw PlanError("parquet: thrift map longer than its buffer");
                for (uint32_t i = 0; i < n; i++) { skip(kv >> 4, depth + 1); skip(kv & 0x0f, depth + 1); }
            }
            break;
        }
        case 12: {
            int16_t fid = 0, last = 0;
            int t;
            while ((t = field(&fid, last)) != 0) { skip(t, depth + 1); last = fid; }
            break;
        }
        default: throw PlanError("parquet: unknown thrift type " + std::to_string(type));
        }
    }
    // element count of a list whose elements take at least one byte each
    uint32_t list_of(int* elem_type) {
        uint32_t n;
        list_header(elem_type, &n);
        if (n > (uint64_t)(end - p)) throw PlanError("parquet: thrift list longer than its buffer");
        return n;
    }
};

#define FOR_FIELDS(r)                 \
    int16_t fid = 0, last = 0;        \
    int t;                            \
    while ((t = (r).field(&fid, last)) != 0)

SchemaElement parse_schema_element(TReader& r) {
    SchemaElement e;
    FOR_FIELDS(r) {
        switch (fid) {
        case 1: e.type = (int)r.zigzag(); break;
        case 2: e.type_length = (int)r.zigzag(); break;
        case 3: e.repetition = (int)r.zigzag(); break;
        case 4: e.name = r.binary(); break;
        case 5: e.num_children = (int)r.zigzag(); break;
        case 6: e.converted_type = (int)r.zigzag(); break;
        case 7: e.scale = (int)r.zigzag(); break;
        case 8: e.precision = (int)r.zigzag(); break;
        case 10: { // LogicalType union: 5 DECIMAL, 8 TIMESTAMP{2: unit{1 MILLIS, 2 MICROS, 3 NANOS}}, 10 INTEGER{1 bitWidth, 2 isSigned}
            int16_t f2 = 0, l2 = 0; int t2;
            while ((t2 = r.field(&f2, l2)) != 0) {
                if (f2 == 5) { e.logical_decimal = true; r.skip(t2); }
                else if (f2 == 8 && t2 == 12) {
                    int16_t f3 = 0, l3 = 0; int t3;
                    while ((t3 = r.field(&f3, l3)) != 0) {
                        if (f3 == 2 && t3 == 12) {
                            int16_t f4 = 0, l4 = 0; int t4;
                            while ((t4 = r.field(&f4, l4)) != 0) { if (f4 >= 1 && f4 <= 3) e.ts_unit = f4; r.skip(t4); l4 = f4; }
                        } else r.skip(t3);
                        l3 = f3;
                    }
                } else if (f2 == 10 && t2 == 12) {
                    int16_t f3 = 0, l3 = 0; int t3;
                    while ((t3 = r.field(&f3, l3)) != 0) {
                        if (f3 == 1 && t3 == 3) { r.need(1); e.int_bits = (int)(signed char)*r.p++; }
                        else if (f3 == 2 && (t3 == 1 || t3 == 2)) e.int_signed = t3 == 1 ? 1 : 0;
                        else r.skip(t3);
                        l3 = f3;
                    }
                } else r.skip(t2);
                l2 = f2;
            }
            break;
        }
        default: r.skip(t);
        }
        last = fid;
    }
    return e;
}

// Statistics (parquet.thrift): 1 max / 2 min are the deprecated signed-byte-order pair (ignored), 3 null_count,
// 5 max_value / 6 min_value follow the column's own sort order
void parse_statistics(TReader& r, ColumnChunkMeta& m) {
    bool have_min = false, have_max = false;
    FOR_FIELDS(r) {
        if (fid == 3) m.null_count = r.zigzag();
        else if (fid == 5 && t == 8) { m.max_value = r.binary(); have_max = true; }
        else if (fid == 6 && t == 8) { m.min_value = r.binary(); have_min = true; }
        else r.skip(t);
        last = fid;
    }
    m.has_min_max = have_min && have_max;
}

ColumnChunkMeta parse_column_meta(TReader& r) {
    ColumnChunkMeta m;
    FOR_FIELDS(r) {
        switch (fid) {
        case 1: m.type = (int)r.zigzag(); break;
        case 2: { int et; uint32_t n = r.list_of(&et); for (uint32_t i = 0; i < n; i++) m.encodings.push_back((int)r.zigzag()); break; }
        case 3: { int et; uint32_t n = r.list_of(&et); for (uint32_t i = 0; i < n; i++) m.path.push_back(r.binary()); break; }
        case 4: m.codec = (int)r.zigzag(); break;
        case 5: m.num_values = r.zigzag(); break;
        case 6: m.total_uncompressed = r.zigzag(); break;
        case 7: m.total_compressed = r.zigzag(); break;
        case 9: m.data_page_offset = r.zigzag(); break;
        case 11: m.dictionary_page_offset = r.zigzag(); break;
        case 12: parse_statistics(r, m); break;
        default: r.skip(t);
        }
        last = fid;
    }
    return m;
}

ColumnChunkMeta parse_column_chunk(TReader& r) {
    ColumnChunkMeta m;
    int64_t oi_off = -1, ci_off = -1;
    int32_t oi_len = 0, ci_len = 0;
    FOR_FIELDS(r) {
        switch (fid) {
        case 3: m = parse_column_meta(r); break;
        case 4: oi_off = r.zigzag(); break;
        case 5: oi_len = (int32_t)r.zigzag(); break;
        case 6: ci_off = r.zigzag(); break;
        case 7: ci_len = (int32_t)r.zigzag(); break;
        default: r.skip(t);
        }
        last = fid;
    }
    m.offset_index_offset = oi_off;
    m.offset_index_length = oi_len;
    m.column_index_offset = ci_off;
    m.column_index_length = ci_len;
    return m;
}

// the index of one column chunk is used only if it tiles the chunk: pages inside [start, start + total_compressed) in file order,
// first rows 0 = f0 < f1 < ... < num_rows, and a ColumnIndex entry per page
bool offset_index_valid(const ColumnChunkMeta& cc, int64_t num_rows) {
    const auto& loc = cc.offset_index;
    if (loc.empty() || loc[0].first_row_index != 0) return false;
    const int64_t lo = cc.start(), hi = lo + cc.total_compressed;
    int64_t prev_end = lo;
    for (size_t i = 0; i < loc.size(); i++) {
        if (loc[i].compressed_page_size <= 0 || loc[i].offset < prev_end || loc[i].offset + loc[i].compressed_page_size > hi) return false;
        if (loc[i].first_row_index >= num_rows || (i && loc[i].first_row_index <= loc[i - 1].first_row_index)) return false;
        prev_end = loc[i].offset + loc[i].compressed_page_size;
    }
    return true;
}

void load_page_indexes(FileMeta& m, const uint8_t* span, int64_t span_lo, int64_t span_hi) {
    for (auto& rg : m.row_groups)
        for (auto& cc : rg.columns) {
            auto in_span = [&](int64_t off, int32_t len) { return off >= span_lo && len > 0 && off + len <= span_hi; };
            if (in_span(cc.offset_index_offset, cc.offset_index_length)) {
                try { cc.offset_index = parse_offset_index(span + (cc.offset_index_offset - span_lo), (size_t)cc.offset_index_length); }
                catch (const PlanError&) { cc.offset_index.clear(); }
                if (!offset_index_valid(cc, rg.num_rows)) cc.offset_index.clear();
            }
            if (!cc.offset_index.empty() && in_span(cc.column_index_offset, cc.column_index_length)) {
                try { cc.column_index = parse_column_index(span + (cc.column_index_offset - span_lo), (size_t)cc.column_index_length); }
                catch (const PlanError&) { cc.column_index = ColumnIndex(); }
                if (cc.column_index.null_pages.size() != cc.offset_index.size()) cc.column_index = ColumnIndex();
            }
        }
}

// [lo, hi): the bytes that hold every page index of the file (they sit together in front of the footer); false if there are none
bool page_index_span(const FileMeta& m, int64_t file_size, int64_t* lo, int64_t* hi) {
    *lo = INT64_MAX;
    *hi = -1;
    for (auto& rg : m.row_groups)
        for (auto& cc : rg.columns)
            for (auto [off, len] : {std::pair<int64_t, int64_t>{cc.offset_index_offset, cc.offset_index_length}, {cc.column_index_offset, cc.column_index_length}})
                if (off >= 0 && len > 0 && off + len <= file_size) { *lo = std::min(*lo, off); *hi = std::max(*hi, off + len); }
    return *hi > *lo && *hi - *lo <= ((int64_t)1 << 30);
}

RowGroupMeta parse_row_group(TReader& r) {
    RowGroupMeta g;
    FOR_FIELDS(r) {
        switch (fid) {
        case 1: { int et; uint32_t n = r.list_of(&et); for (uint32_t i = 0; i < n; i++) g.columns.push_back(parse_column_chunk(r)); break; }
        case 3: g.num_rows = r.zigzag(); break;
        default: r.skip(t);
        }
        last = fid;
    }
    return g;
}

} // namespace

int FileMeta::leaf_index(const std::string& name) const {
    for (size_t i = 1; i < schema.size(); i++) if (schema[i].name == name) return (int)i - 1;
    return -1;
}

FileMeta parse_footer(const uint8_t* file, size_t len) {
    if (len < 12 || memcmp(file + len - 4, "PAR1", 4) != 0) throw PlanError("parquet: missing PAR1 footer magic (encrypted files are out of scope)");
    uint32_t flen;
    memcpy(&flen, file + len - 8, 4);
    if ((size_t)flen + 8 > len) throw PlanError("parquet: footer larger than the bytes provided");
    TReader r{file + len - 8 - flen, file + len - 8};
    FileMeta m;
    FOR_FIELDS(r) {
        switch (fid) {
        case 2: { int et; uint32_t n = r.list_of(&et); for (uint32_t i = 0; i < n; i++) m.schema.push_back(parse_schema_element(r)); break; }
        case 3: m.num_rows = r.zigzag(); break;
        case 4: { int et; uint32_t n = r.list_of(&et); for (uint32_t i = 0; i < n; i++) m.row_groups.push_back(parse_row_group(r)); break; }
        default: r.skip(t);
        }
        last = fid;
    }
    if (m.schema.empty()) throw PlanError("parquet: empty schema");
    for (size_t i = 1; i < m.schema.size(); i++)
        if (m.schema[i].num_children > 0) throw Unsupported("nested Parquet schemas (struct/list/map columns) are outside the GPU hot path");
    return m;
}

FileMeta read_footer(const std::string& path, int64_t* file_size) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) throw ExecError(3, "", "parquet: cannot open " + path);
    fseek(f, 0, SEEK_END);
    long sz = ftell(f);
    if (file_size) *file_size = sz;
    // metadata size hint: 512 KiB (parquet_exec.rs:221-266 sets the same hint), grow if the footer is larger
    size_t want = (size_t)std::min<long>(sz, 512 * 1024);
    std::vector<uint8_t> tail(want);
    fseek(f, sz - (long)want, SEEK_SET);
    if (fread(tail.data(), 1, want, f) != want) { fclose(f); throw ExecError(3, "", "parquet: short read on " + path); }
    uint32_t flen = 0;
    if (want >= 8) memcpy(&flen, tail.data() + want - 8, 4);
    if ((size_t)flen + 8 > want) {
        want = (size_t)flen + 8;
        if ((long)want > sz) { fclose(f); throw PlanError("parquet: corrupt footer length"); }
        tail.resize(want);
        fseek(f, sz - (long)want, SEEK_SET);
        if (fread(tail.data(), 1, want, f) != want) { fclose(f); throw ExecError(3, "", "parquet: short read on " + path); }
    }
    fclose(f);
    return parse_footer(tail.data(), tail.size());
}

// OffsetIndex: 1 page_locations list<PageLocation{1 offset, 2 compressed_page_size, 3 first_row_index}>
std::vector<PageLocation> parse_offset_index(const uint8_t* p, size_t len) {
    TReader r{p, p + len};
    std::vector<PageLocation> out;
    FOR_FIELDS(r) {
        if (fid == 1 && t == 9) {
            int et;
            const uint32_t n = r.list_of(&et);
            if (et != 12) throw PlanError("parquet: OffsetIndex page_locations is not a list of structs");
            for (uint32_t i = 0; i < n; i++) {
                PageLocation pl;
                int16_t f2 = 0, l2 = 0; int t2;
                while ((t2 = r.field(&f2, l2)) != 0) {
                    if (f2 == 1) pl.offset = r.zigzag();
                    else if (f2 == 2) pl.compressed_page_size = (int32_t)r.zigzag();
                    else if (f2 == 3) pl.first_row_index = r.zigzag();
                    else r.skip(t2);
                    l2 = f2;
                }
                out.push_back(pl);
            }
        } else r.skip(t);
        last = fid;
    }
    return out;
}

// ColumnIndex: 1 null_pages list<bool>, 2 min_values / 3 max_values list<binary>, 4 boundary_order, 5 null_counts (not used).  The lists
// must be equally long, or the index is not used.
ColumnIndex parse_column_index(const uint8_t* p, size_t len) {
    TReader r{p, p + len};
    ColumnIndex ci;
    FOR_FIELDS(r) {
        int et;
        if (fid == 1 && t == 9) {
            const uint32_t n = r.list_of(&et);
            if (et != 1 && et != 2) throw PlanError("parquet: ColumnIndex null_pages is not a list of bools");
            for (uint32_t i = 0; i < n; i++) ci.null_pages.push_back(*r.p++ == 1); // a bool in a list is one byte: 1 true, anything else false
        } else if ((fid == 2 || fid == 3) && t == 9) {
            const uint32_t n = r.list_of(&et);
            if (et != 8) throw PlanError("parquet: ColumnIndex min / max values are not binary");
            auto& v = fid == 2 ? ci.min_values : ci.max_values;
            for (uint32_t i = 0; i < n; i++) v.push_back(r.binary());
        } else r.skip(t);
        last = fid;
    }
    if (ci.min_values.size() != ci.null_pages.size() || ci.max_values.size() != ci.null_pages.size()) throw PlanError("parquet: ColumnIndex lists differ in length");
    return ci;
}

void read_page_indexes(FileMeta& m, const uint8_t* file, size_t file_len) {
    int64_t lo, hi;
    if (page_index_span(m, (int64_t)file_len, &lo, &hi)) load_page_indexes(m, file + lo, lo, hi);
}

void read_page_indexes(FileMeta& m, const std::string& path, int64_t file_size) {
    int64_t lo, hi;
    if (!page_index_span(m, file_size, &lo, &hi)) return;
    std::vector<uint8_t> span((size_t)(hi - lo));
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) throw ExecError(3, "", "parquet: cannot open " + path);
    const bool ok = fseeko(f, (off_t)lo, SEEK_SET) == 0 && fread(span.data(), 1, span.size(), f) == span.size();
    fclose(f);
    if (!ok) throw ExecError(3, "", "parquet: short read on " + path);
    load_page_indexes(m, span.data(), lo, hi);
}

std::vector<PageInfo> walk_pages(const uint8_t* chunk, size_t len, int64_t num_values) {
    std::vector<PageInfo> pages;
    size_t pos = 0;
    int64_t seen = 0;
    while (pos < len && seen < num_values) {
        TReader r{chunk + pos, chunk + len};
        PageInfo pg;
        pg.header_offset = (int64_t)pos;
        FOR_FIELDS(r) {
            switch (fid) {
            case 1: pg.type = (int)r.zigzag(); break;
            case 2: pg.uncompressed_size = (int32_t)r.zigzag(); break;
            case 3: pg.compressed_size = (int32_t)r.zigzag(); break;
            case 5: { // DataPageHeader
                int16_t f2 = 0, l2 = 0; int t2;
                while ((t2 = r.field(&f2, l2)) != 0) {
                    if (f2 == 1) pg.num_values = r.zigzag();
                    else if (f2 == 2) pg.encoding = (int)r.zigzag();
                    else if (f2 == 3) pg.def_encoding = (int)r.zigzag();
                    else r.skip(t2);
                    l2 = f2;
                }
                break;
            }
            case 7: { // DictionaryPageHeader
                int16_t f2 = 0, l2 = 0; int t2;
                while ((t2 = r.field(&f2, l2)) != 0) {
                    if (f2 == 1) pg.num_values = r.zigzag();
                    else if (f2 == 2) pg.encoding = (int)r.zigzag();
                    else r.skip(t2);
                    l2 = f2;
                }
                break;
            }
            case 8: { // DataPageHeaderV2
                int16_t f2 = 0, l2 = 0; int t2;
                while ((t2 = r.field(&f2, l2)) != 0) {
                    if (f2 == 1) pg.num_values = r.zigzag();
                    else if (f2 == 2) pg.num_nulls = r.zigzag();
                    else if (f2 == 4) pg.encoding = (int)r.zigzag();
                    else if (f2 == 5) pg.def_levels_bytes = (int32_t)r.zigzag();
                    else if (f2 == 6) pg.rep_levels_bytes = (int32_t)r.zigzag();
                    else if (f2 == 7) pg.v2_compressed = (t2 == 1);
                    else r.skip(t2);
                    l2 = f2;
                }
                break;
            }
            default: r.skip(t);
            }
            last = fid;
        }
        pg.data_offset = (int64_t)(r.p - chunk);
        if (pg.compressed_size < 0 || (size_t)pg.data_offset + (size_t)pg.compressed_size > len) throw PlanError("parquet: page runs past its column chunk");
        if (pg.type == DATA_PAGE || pg.type == DATA_PAGE_V2) seen += pg.num_values;
        pages.push_back(pg);
        pos = (size_t)pg.data_offset + (size_t)pg.compressed_size;
    }
    return pages;
}

std::string describe(const FileMeta& m) {
    std::ostringstream o;
    o << "{\"num_rows\": " << m.num_rows << ", \"columns\": [";
    for (size_t i = 1; i < m.schema.size(); i++) {
        const auto& e = m.schema[i];
        o << (i > 1 ? ", " : "") << "{\"name\": \"" << e.name << "\", \"type\": " << e.type << ", \"type_length\": " << e.type_length << ", \"precision\": "
          << e.precision << ", \"scale\": " << e.scale << ", \"converted_type\": " << e.converted_type << "}";
    }
    o << "], \"row_groups\": [";
    for (size_t g = 0; g < m.row_groups.size(); g++) {
        const auto& rg = m.row_groups[g];
        o << (g ? ", " : "") << "{\"num_rows\": " << rg.num_rows << ", \"columns\": [";
        for (size_t c = 0; c < rg.columns.size(); c++) {
            const auto& cc = rg.columns[c];
            o << (c ? ", " : "") << "{\"codec\": " << cc.codec << ", \"num_values\": " << cc.num_values << ", \"total_compressed\": " << cc.total_compressed
              << ", \"data_page_offset\": " << cc.data_page_offset << ", \"dictionary_page_offset\": " << cc.dictionary_page_offset << ", \"null_count\": "
              << cc.null_count << ", \"encodings\": [";
            for (size_t k = 0; k < cc.encodings.size(); k++) o << (k ? "," : "") << cc.encodings[k];
            o << "]}";
        }
        o << "]}";
    }
    o << "]}";
    return o.str();
}

} // namespace pq
} // namespace cb200
