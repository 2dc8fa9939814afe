// aot_kernels.h -- host-callable launchers of the plan-independent sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "device/cb_strpred.h"

namespace cb200 {

void launch_bitmap_append(uint32_t* dst, long long dst_off, const uint8_t* src, long long src_off, long long n, cudaStream_t st);
void launch_bytes_to_bitmap(const uint8_t* bytes, long long n, uint32_t* out, cudaStream_t st);
// string predicate d over dictionary entries [first, n) -> mask bits [first, n) (bit i & 31 of word i >> 5).  Entry i is
// chars[offsets[i - first], offsets[i - first + 1]).  first must be a multiple of 32: each warp writes whole words of its own.
void launch_str_pred(const cb::StrPredDev& d, const int* offsets, const unsigned char* chars, long long first, long long n, unsigned* mask, cudaStream_t st);
void launch_remap_codes(const void* in, int in_width, long long n, const int* table, int table_len, int* out, cudaStream_t st);

enum { CB_DICT_FULL = 1, CB_DICT_COLLISION = 2 };
struct StringDictDev {
    unsigned long long* tags; // [capacity] 0 = empty
    int* slot_code;           // [capacity]
    long long capacity;       // power of two
    int* n_codes;             // running number of codes
    int max_codes;
    long long* code_off;      // [max_codes]
    int* code_len;            // [max_codes]
    unsigned char* bytes;     // string storage
    long long bytes_cap;
    unsigned long long* bytes_used;
    int* err;
};
void launch_dict_encode(const StringDictDev& d, const int* offsets, const unsigned char* chars, const unsigned char* validity, long long n,
                        int* row_slot, int* codes, cudaStream_t st);

// hash partitioning (ShuffleWriter with HashPartition): murmur3 seed 42 chained over the key columns, pmod, stable counting sort
// HK_BOOL reads an Arrow bitmap, HK_BOOL8 one byte per row; HK_DEC_SMALL_32 is a decimal(p <= 9) stored as INT32 (hashed as its i64)
enum { HK_BOOL, HK_I8, HK_I16, HK_I32, HK_I64, HK_F32, HK_F64, HK_DEC_SMALL_128, HK_DEC_LARGE_128, HK_DEC_SMALL_64 = HK_I64, HK_DEC_LARGE_64 = 9,
       HK_DICT8 = 10, HK_DICT16, HK_DICT32, HK_UTF8, HK_DEC_SMALL_32, HK_BOOL8 };
struct HashKeyCol {
    int kind;
    const void* data;
    const unsigned char* validity; // Arrow bitmap or nullptr
    const int* dict_offsets;       // dictionary / utf8 offsets
    const unsigned char* dict_chars;
};
struct HashKeyCols {
    int n;
    HashKeyCol col[8];
};
long long partition_chunks(long long n); // entries per partition of launch_partition's chunk_tmp scratch
// n_parts <= CB_MAX_HASH_PARTITIONS: three of the kernels keep one counter per partition in shared memory (8 bytes each at most)
enum { CB_MAX_HASH_PARTITIONS = 16384 };
// returns the first error of the launches (a launch the device refuses is reported here, not by a later synchronisation)
cudaError_t launch_partition(const HashKeyCols& kc, long long n, unsigned n_parts, unsigned* hashes, unsigned* pids, int* block_hist, long long* block_base,
                      long long* chunk_tmp, long long* starts, long long* row_idx, cudaStream_t st);
void launch_gather(const void* in, int width, const long long* row_idx, long long n, void* out, cudaStream_t st);
void launch_gather_bits(const void* in_bits, const long long* row_idx, long long n, void* out_bytes, cudaStream_t st);

// device values -> the Arrow layout of their logical type, rows [0, n): what the hand-off (Arrow export, cb200_execute_device) gives out
enum { CB_SEXT32_TO_128, CB_SEXT64_TO_128, CB_NARROW32_TO_8, CB_NARROW32_TO_16, CB_BITS_TO_BYTES };
void launch_to_arrow_layout(int conv, const void* in, long long n, void* out, cudaStream_t st);

// stream compaction (hash-aggregate results): per-1024-row-block counts + exclusive scan, then one scatter per column
void launch_key_presence(const unsigned long long* keys, long long n, unsigned char* present, cudaStream_t st);
void launch_compact_plan(const unsigned char* present, long long n, int* counts, long long* offsets, long long* total, cudaStream_t st);
void launch_compact_scatter(const unsigned char* present, long long n, const long long* offsets, const void* in, int width, void* out, cudaStream_t st);

// exclusive prefix sum of u32 counts, in place, in chunks of `chunk` entries (power of two, <= 4096): data[i] becomes the
// offset inside its chunk, chunk_off[i / chunk] the offset of the chunk, *total the grand total (select pipelines)
void launch_scan_u32(unsigned* data, long long m, int chunk, unsigned* chunk_off, long long* total, cudaStream_t st);

} // namespace cb200
