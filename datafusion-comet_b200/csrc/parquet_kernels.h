// parquet_kernels.h -- device-side Parquet page decode: Snappy decompression, PLAIN, BYTE_STREAM_SPLIT, DELTA_BINARY_PACKED, RLE_DICTIONARY, definition
// levels (validity + NULL scatter).
#pragma once
#include "parquet_pages.h"

#include <cuda_runtime.h>
#include <cstddef>

namespace cb200 {

// dst[0, bytes) = src[0, bytes) with SM loads/stores (bytes a multiple of 16, both 16-byte aligned).  `src` may be mapped pinned
// host memory: small tables reach the device without queueing on a copy engine.
void launch_pq_copy(void* dst, const void* src, size_t bytes, cudaStream_t st);
// Snappy, segmented: `ckpt` has room for n_segs_total entries (sum of PqPage::n_segs, n_segs = ceil(body_bytes / PQ_SNAPPY_SEG)); pages
// with comp == nullptr are skipped
void launch_pq_snappy_segmented(PqPage* pages_dev, int n_pages, unsigned* ckpt_dev, int n_segs_total, int* err, cudaStream_t st);
// locate levels / values inside every page body; nonnull = num_values
void launch_pq_resolve(PqPage* pages_dev, int n_pages, cudaStream_t st);
// PLAIN and BYTE_STREAM_SPLIT fixed-width pages -> out[dst_row + k] for the page's k-th encoded value (element width given by the conversion)
void launch_pq_plain(const PqPage* pages_dev, int n_pages, int conv, int flba_len, void* out, int* err, cudaStream_t st);
// DELTA_BINARY_PACKED INT32 / INT64 pages (conv PQ_COPY32 / PQ_COPY64 / PQ_I32_TO_I64) -> out[dst_row + k], like PLAIN.  `table` holds
// every page's miniblock entries at [mb_base, mb_base + mb_cap); four launches (header walk, sums, carries, decode)
void launch_pq_dbp(PqPage* pages_dev, int n_pages, PqMiniblock* table, int conv, void* out, int* err, cudaStream_t st);
// RLE_DICTIONARY pages: (1) scan run headers, one thread per page
void launch_pq_rle_scan(const PqPage* pages_dev, int n_pages, PqRun* runs, int* run_counts, int* err, cudaStream_t st);
// (2) decode runs (warp per run) and gather through the dictionary: dict_width 4/8/16 bytes per entry
void launch_pq_rle_decode(const PqPage* pages_dev, int n_pages, const PqRun* runs, const int* run_counts, const void* dict, int dict_width, void* out, int* err,
                          cudaStream_t st);
// definition levels of flat optional columns (max level 1)
//   fast path (statistics promise no NULLs): verify it (PQ_ERR_NULL_ON_FAST_PATH otherwise)
void launch_pq_check_def_levels(const PqPage* pages_dev, int n_pages, int* err, cudaStream_t st);
//   NULL-aware path: valid[row] = level, idx[row] = dst_row(page) + number of non-null rows before `row` in its page, pages[].nonnull
void launch_pq_def_levels(PqPage* pages_dev, int n_pages, PqRun* runs, int* run_counts, unsigned char* valid, unsigned* idx, int* err, cudaStream_t st);
//   out[row] = valid[row] ? dense[idx[row]] : 0 ; bitmap = Arrow validity (total rows, width 4/8/16 bytes)
void launch_pq_scatter(const unsigned char* valid, const unsigned* idx, const void* dense, void* out, unsigned* bitmap, long long total, int width, cudaStream_t st);

} // namespace cb200
