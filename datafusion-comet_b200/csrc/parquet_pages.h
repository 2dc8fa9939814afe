// parquet_pages.h -- the page tables the host plans (scan_plan.cpp) and the device decode kernels read (parquet_kernels.cu).
// Plain data, no CUDA runtime: the planner is built and tested without it.
#pragma once
#include <cstdint>

namespace cb200 {

// PqPage::flags.  V1_LEVELS: body starts with [u32 byte length][RLE definition levels] (DataPage v1 of an optional column).  SN_*: set by the
// Snappy index / segment kernels (the page needs the serial decoder / is malformed).  HOSTDEC (host bookkeeping only): the body was produced
// on the host -- decompressed (csrc/host_codecs.h) or PLAIN strings turned into dictionary codes -- and travels with the page tables.
enum { PQ_PAGE_V1_LEVELS = 1, PQ_PAGE_SN_SERIAL = 2, PQ_PAGE_SN_BAD = 4, PQ_PAGE_HOSTDEC = 8 };

// Bits the decode kernels set in the scan's error word.
enum PqErr {
    PQ_ERR_RLE = 1,               // malformed RLE / bit-packed stream, or more runs than the page's run table holds
    PQ_ERR_NULL_ON_FAST_PATH = 2, // a NULL in a chunk whose statistics say null_count = 0
    PQ_ERR_DICT_INDEX = 4,        // dictionary index out of range
    PQ_ERR_SNAPPY = 8,            // malformed Snappy page
    PQ_ERR_TRUNCATED = 16,        // fewer encoded values than the page header declares
    PQ_ERR_DELTA = 32,            // malformed DELTA_BINARY_PACKED page (sizes, bit width, value count, body past the page, table overflow)
    PQ_ERR_BSS = 64,              // BYTE_STREAM_SPLIT page whose size is not (non-null values) x (value width)
};

// PqPage::encoding: the Parquet value encoding the device decodes the page by.  Pages the host re-encoded (strings, DELTA_BYTE_ARRAY
// decimals) are PQ_ENC_PLAIN; PLAIN_DICTIONARY pages are PQ_ENC_DICT.
enum { PQ_ENC_PLAIN = 0, PQ_ENC_DBP = 5, PQ_ENC_DICT = 8, PQ_ENC_BSS = 9 };

// One page of a column chunk resident on the device.  The host fills what the page HEADER tells it; everything
// that lives inside the (possibly compressed) page body is resolved on the device by k_pq_resolve.
struct PqPage {
    unsigned char* body;          // v1: page body (levels + values); v2: the values section.  Snappy pages: where the decompressor writes
    int body_bytes;               // uncompressed size of `body`
    const unsigned char* comp;    // Snappy-compressed source, nullptr when `body` already holds the bytes
    int comp_bytes;
    int flags;
    const unsigned char* def_ptr; // definition levels (RLE/bit-packed hybrid, bit width 1); v2: set by the host
    int def_bytes;
    const unsigned char* values;  // resolved: encoded values (non-null values only)
    int values_bytes;
    long long dst_row;            // first output row of this page
    int num_values;               // rows of the page (incl. NULLs)
    int nonnull;                  // resolved: encoded values present
    int encoding;                 // PQ_ENC_*
    long long run_base;           // value runs: first entry of this page in the run table, capacity
    int max_runs;
    long long def_run_base;       // definition-level runs (NULL-aware path)
    int def_max_runs;
    long long dict_off;           // element offset of this page's dictionary inside the column's combined dictionary buffer
    int dict_size;
    int seg_base;                 // Snappy pages: first entry of this page in the column's checkpoint table (one entry per 64 KB of output)
    int n_segs;
    long long mb_base;            // DELTA_BINARY_PACKED: first entry of this page in the column's miniblock table, capacity (num_values / 32 + 2),
    int mb_cap;                   //   entries the header walk wrote
    int mb_count;
};

// One DELTA_BINARY_PACKED miniblock, written by the header walk.  Entry 0 of a page is the first value, stored as a lone delta from
// zero, so every value of the page is a prefix sum of deltas; `carry` is the sum of all deltas before the entry's first value.
struct PqMiniblock {
    const unsigned char* src;     // packed deltas
    long long min_delta;
    long long carry;
    int out_idx;                  // index of the entry's first value within the page's non-null values
    int count;                    // values
    int bit_width;
    int nbytes;                   // body bytes (the packed deltas are read inside them only)
};

struct PqRun {              // one run of the RLE / bit-packed hybrid
    long long out_row;      // absolute output row of the run's first value
    const unsigned char* src; // packed data (bit-packed runs)
    int count;              // values in the run
    unsigned value;         // RLE runs: the repeated value
    int bit_packed;
    int bit_width;
};

enum PqConv { PQ_COPY32, PQ_COPY64, PQ_I32_TO_I64, PQ_FLBA_TO_I64, PQ_FLBA_TO_I128 };

// segmented Snappy decoder: one checkpoint table entry per PQ_SNAPPY_SEG bytes of a page's output
constexpr int PQ_SNAPPY_SEG = 65536;

} // namespace cb200
