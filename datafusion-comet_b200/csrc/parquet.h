// parquet.h -- host side of the native Parquet scan: footer + page-header parsing (Thrift compact protocol) and the
// page table handed to the device decode kernels (parquet_kernels.cu).
//
// Replaces, for flat schemas, what the reference gets from the third-party `parquet` crate 58.4.0 through
// DataFusion's ParquetSource (native/core/src/parquet/parquet_exec.rs:60-200): metadata is parsed on the host
// (it is tiny and sequential), every value byte is decoded on the device.  Restated from the Apache Parquet
// format specification (parquet.thrift, Encodings.md); the crate's source is not under the reference tree.
#pragma once
#include "plan.h"

#include <cstdint>
#include <string>
#include <vector>

namespace cb200 {
namespace pq {

enum PhysType { BOOLEAN = 0, INT32 = 1, INT64 = 2, INT96 = 3, FLOAT = 4, DOUBLE = 5, BYTE_ARRAY = 6, FIXED_LEN_BYTE_ARRAY = 7 };
enum Encoding { PLAIN = 0, PLAIN_DICTIONARY = 2, RLE = 3, BIT_PACKED = 4, DELTA_BINARY_PACKED = 5, DELTA_LENGTH_BYTE_ARRAY = 6, DELTA_BYTE_ARRAY = 7, RLE_DICTIONARY = 8,
                BYTE_STREAM_SPLIT = 9 };
enum Codec { UNCOMPRESSED = 0, SNAPPY = 1, GZIP = 2, LZO = 3, BROTLI = 4, LZ4 = 5, ZSTD = 6, LZ4_RAW = 7 };
enum PageType { DATA_PAGE = 0, INDEX_PAGE = 1, DICTIONARY_PAGE = 2, DATA_PAGE_V2 = 3 };

struct SchemaElement {
    int type = -1, type_length = 0, repetition = 0, num_children = 0, converted_type = -1, scale = 0, precision = 0;
    // LogicalType (field 10): what the physical bytes mean where converted_type is absent or too coarse
    int ts_unit = 0;       // TIMESTAMP: 1 MILLIS, 2 MICROS, 3 NANOS (0 = not a logical timestamp)
    int int_bits = 0;      // INTEGER: bit width (0 = not a logical integer)
    int int_signed = 1;
    bool logical_decimal = false;
    std::string name;
};
// OffsetIndex.page_locations (parquet.thrift): where one data page of a column chunk sits, header included, and its first row
struct PageLocation {
    int64_t offset = 0;
    int32_t compressed_page_size = 0;
    int64_t first_row_index = 0;
};
// ColumnIndex (parquet.thrift): per data page, whether it holds only NULLs and its min / max (PLAIN-encoded, like chunk statistics;
// meaningless for an all-NULL page)
struct ColumnIndex {
    std::vector<uint8_t> null_pages;
    std::vector<std::string> min_values, max_values;
};
struct ColumnChunkMeta {
    int type = 0, codec = 0;
    std::vector<int> encodings;
    std::vector<std::string> path;
    int64_t num_values = 0, total_uncompressed = 0, total_compressed = 0, data_page_offset = 0, dictionary_page_offset = -1;
    int64_t null_count = -1; // statistics, -1 unknown
    bool has_min_max = false; // statistics min_value / max_value (fields 5, 6: the type's own sort order), PLAIN-encoded
    std::string min_value, max_value;
    int64_t offset_index_offset = -1, column_index_offset = -1; // ColumnChunk fields 4-7: the page index, stored outside the footer
    int32_t offset_index_length = 0, column_index_length = 0;
    // the page index as read_page_indexes left it: empty unless present and valid (offset_index: pages inside the chunk, first rows
    // 0 < ... < num_rows; column_index: as many pages as offset_index)
    std::vector<PageLocation> offset_index;
    ColumnIndex column_index;
    int64_t start() const { return dictionary_page_offset > 0 && dictionary_page_offset < data_page_offset ? dictionary_page_offset : data_page_offset; }
};
struct RowGroupMeta {
    int64_t num_rows = 0;
    std::vector<ColumnChunkMeta> columns;
};
struct FileMeta {
    int64_t num_rows = 0;
    std::vector<SchemaElement> schema; // schema[0] = root
    std::vector<RowGroupMeta> row_groups;
    int leaf_index(const std::string& name) const; // flat schemas: position among the leaves, -1 if absent
    const SchemaElement& leaf(int i) const { return schema[(size_t)i + 1]; }
};

struct PageInfo {
    int type = 0;                 // PageType
    int encoding = 0;             // value encoding
    int def_encoding = RLE;
    int64_t num_values = 0;       // incl. nulls
    int64_t header_offset = 0;    // relative to the chunk start
    int64_t data_offset = 0;      // first byte after the header, relative to the chunk start
    int32_t compressed_size = 0, uncompressed_size = 0;
    int32_t def_levels_bytes = 0; // v2: byte length of the definition levels (uncompressed, before the values)
    int32_t rep_levels_bytes = 0;
    bool v2_compressed = true;
    int64_t num_nulls = -1;
};

FileMeta parse_footer(const uint8_t* file, size_t file_len);               // whole file image or at least its tail
FileMeta read_footer(const std::string& path, int64_t* file_size);
// The page indexes of every column chunk that has them, from the whole file image / from the file.  An index that does not parse
// or fails validation is left out: that chunk is read whole.
void read_page_indexes(FileMeta& m, const uint8_t* file, size_t file_len);
void read_page_indexes(FileMeta& m, const std::string& path, int64_t file_size);
std::vector<PageLocation> parse_offset_index(const uint8_t* p, size_t len);
ColumnIndex parse_column_index(const uint8_t* p, size_t len);
// walk the page headers of one column chunk (bytes = the chunk, [0, total_compressed))
std::vector<PageInfo> walk_pages(const uint8_t* chunk, size_t len, int64_t num_values);
std::string describe(const FileMeta& m); // JSON, for tests

} // namespace pq
} // namespace cb200
