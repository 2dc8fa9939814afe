// aot_kernels.h -- host-callable launchers of the plan-independent sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "device/cb_sortkey.h"
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

// hash partitioning (ShuffleWriter with HashPartition): murmur3 seed 42 chained over the key columns, pmod, stable counting sort.
// Key columns are read by their HK_* layout (device/cb_sortkey.h); HK_DEC_SMALL_32 is hashed as its i64.
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
// out[i] = in[row_idx[i]] (width bytes per row), i < n; 64-bit (partitioning) or 32-bit (sort) row indices
void launch_gather(const void* in, int width, const long long* row_idx, long long n, void* out, cudaStream_t st);
void launch_gather(const void* in, int width, const unsigned* row_idx, long long n, void* out, cudaStream_t st);
void launch_gather_bits(const void* in_bits, const long long* row_idx, long long n, void* out_bytes, cudaStream_t st);
void launch_gather_bits(const void* in_bits, const unsigned* row_idx, long long n, void* out_bytes, cudaStream_t st);
// the same for NULL-extended join output: row index CB_NULL_ROW gives zero bytes (launch_gather_or_null) or 0 (launch_gather_bits_or_null).
// in_bits == nullptr (a column without a validity bitmap) reads as all set.
enum : unsigned { CB_NULL_ROW = 0xffffffffu };
void launch_gather_or_null(const void* in, int width, const unsigned* row_idx, long long n, void* out, cudaStream_t st);
void launch_gather_bits_or_null(const void* in_bits, const unsigned* row_idx, long long n, void* out_bytes, cudaStream_t st);

// ---- sort (SortExec / TopK): packed row keys (device/cb_sortkey.h), stable LSD radix sort of (key, row index) ----------------------------
// k_sort_keys: kc.words 64-bit words per row into keys[n * words]; and_or[0, words) ANDs and and_or[words, 2 * words) ORs them over
// all rows (the caller sets them to ~0 and 0 first): a digit equal in every row needs no pass.
void launch_sort_keys(const cb::SortKeyCols& kc, long long n, unsigned long long* keys, unsigned long long* and_or, cudaStream_t st);
// scratch of launch_sort_passes for n rows of `words` words: the key / index buffers come in pairs (keys[0] holds the input keys);
// hist holds 256 x sort_tiles(n) entries, chunk_off 256 x sort_tiles(n) / 4096 + 1, total one
struct RadixScratch {
    unsigned long long* keys[2];
    unsigned* idx[2];
    unsigned* hist;
    unsigned* chunk_off;
    long long* total;
};
long long sort_tiles(long long n);
// one stable counting-sort pass per digit in digits[0, n_digits) (8-bit digit d = bits [8d, 8d + 8) of the row key), least significant
// first; n < 2^32.  The first pass reads row i's index as i; no digits: idx[0] = 0, 1, ... .  *result: which buffer pair holds the
// sorted keys and indices.  Returns the first launch error.
cudaError_t launch_sort_passes(const RadixScratch& s, int words, long long n, const int* digits, int n_digits, int* result, cudaStream_t st);
// TopK selection.  A row key k "matches" when (k[j] & mask[j]) == want[j] for every word j.
struct SortSelectKey {
    unsigned long long mask[cb::SK_MAX_WORDS], want[cb::SK_MAX_WORDS];
};
// hist[256] += the histogram of digit `digit` over the matching rows (an MSD radix select step)
cudaError_t launch_sort_select_hist(const unsigned long long* keys, int words, long long n, const SortSelectKey& p, int digit, unsigned* hist, cudaStream_t st);
// keep[i] = row i is among the first rows of the stable order up to the selected key p.want: its key is smaller, or equal and fewer
// than r equal rows precede it.  eq (n + 16 bytes), counts / offsets (n / 1024 + 1 entries) and total are scratch (launch_compact_plan).
cudaError_t launch_sort_select_keep(const unsigned long long* keys, int words, long long n, const SortSelectKey& p, long long r, unsigned char* eq,
                                    int* counts, long long* offsets, long long* total, unsigned char* keep, cudaStream_t st);
void launch_sort_iota(unsigned* idx, long long n, cudaStream_t st); // idx[i] = i

// ---- hash join: build keys sorted by the radix sort, one table slot per distinct key, probe by lookup ------------------------------------
// Row keys are the sort's (device/cb_sortkey.h), `words` words per row, every key field with a null bit that is set on a valid value:
// a key has no NULL field iff (k[j] & nullmask[j]) == nullmask[j] for every word.  The build side's keys[m] are sorted with their row
// indices rows[m]; run r of equal keys is sorted rows [run_start[r], run_start[r + 1]).  slots[mask + 1]: 0 = empty, otherwise
// (hash tag << 32) | (run + 1).
struct JoinTable {
    const unsigned long long* keys;
    const unsigned* rows;
    const unsigned* run_start;
    unsigned long long* slots;
    unsigned long long mask;
    int words;
    unsigned long long nullmask[cb::SK_MAX_WORDS];
};
// head[i] = 1 where sorted key i differs from key i - 1 (row 0 always): the run heads
void launch_join_heads(const unsigned long long* keys, int words, long long m, unsigned char* head, cudaStream_t st);
// every run r < n_runs whose key has no NULL field gets one slot
void launch_join_insert(const JoinTable& t, long long n_runs, cudaStream_t st);
enum { CB_JOIN_COUNT = 0, CB_JOIN_SEMI = 1, CB_JOIN_ANTI = 2, CB_JOIN_OUTER = 3 };
// one lookup per probe key (NULL fields match nothing).  CB_JOIN_COUNT: counts[i] = matching build rows, run_of[i] = their run (~0 when
// none), *total += the sum of counts (64-bit; the caller zeroes it).  CB_JOIN_OUTER: the same, but a row without a match counts 1.
// CB_JOIN_SEMI / ANTI: keep[i] = a match exists / none does.  hit (n_runs bytes, or nullptr): hit[run] = 1 for every run found.
void launch_join_probe(const JoinTable& t, const unsigned long long* keys, long long n, int mode, unsigned* counts, unsigned* run_of,
                       unsigned long long* total, unsigned char* keep, unsigned char* hit, cudaStream_t st);
// join pairs at output positions [o0, o1): probe row i's matches occupy [off_i, off_i + count_i), off_i = offs[i] + chunk_off[i / 4096]
// (launch_scan_u32 over the counts); probe_idx[p - o0] = i, build_idx[p - o0] = the build row, in build input order.  outer: a row
// without a match gives one pair whose build row is CB_NULL_ROW.
void launch_join_emit(const JoinTable& t, const unsigned* run_of, const unsigned* offs, const unsigned* chunk_off, long long n, long long o0,
                      long long o1, bool outer, unsigned* probe_idx, unsigned* build_idx, cudaStream_t st);
// keep[rows[p]] = 1 for every sorted build position p < m whose run (run_start[0, n_runs)) has no hit: the build rows no probe row matched,
// NULL keys included (their runs are not in the table)
void launch_join_unmatched(const unsigned* run_start, long long n_runs, const unsigned* rows, const unsigned char* hit, long long m,
                           unsigned char* keep, cudaStream_t st);
// Join conditions.  bits: one pass bit per pair of a probe batch (bit p & 31 of word p >> 5).  mark: the pairs of a slice whose first
// pair is a multiple of 32 (bits points at its first word): clears the bit of every pair whose build row is CB_NULL_ROW, then for every
// pair still set stores passed[probe row] = 1 and, if build_hit is given, build_hit[build row] = 1; *candidates += its pairs whose build
// row is not CB_NULL_ROW.
void launch_join_cond_mark(unsigned* bits, const unsigned* probe_idx, const unsigned* build_idx, long long k, unsigned char* passed,
                           unsigned char* build_hit, unsigned long long* candidates, cudaStream_t st);
// resolve: pairs [o0, o0 + k) once `passed` is final: keep[j] = pair o0 + j passed, or (outer) it is the first pair of a probe row that
// passed nothing -- offs / chunk_off as in launch_join_emit -- whose build_idx[j] then becomes CB_NULL_ROW
void launch_join_cond_resolve(const unsigned* bits, long long o0, const unsigned* probe_idx, unsigned* build_idx, long long k, const unsigned* offs,
                              const unsigned* chunk_off, const unsigned char* passed, bool outer, unsigned char* keep, cudaStream_t st);
// Nested-loop join.  The pairs of a group of probe rows from row0 against m build rows (0 < m < 2^32) are numbered probe-row major:
// position p is (row0 + p / m, p % m).  inv = floor((2^64 - 1) / m) replaces the divide.  pairs: probe_idx[j], build_idx[j] = pair p0 + j,
// j < k.
void launch_nlj_pairs(long long p0, long long k, unsigned row0, unsigned m, unsigned long long inv, unsigned* probe_idx, unsigned* build_idx,
                      cudaStream_t st);
// resolve (launch_join_cond_resolve for the arithmetic pairs, writing them too): pairs [p0, p0 + k) of the group once `passed` is final;
// bits: the group's pass bits from bit 0.  keep[j] = pair p0 + j passed, or (outer) it is build row 0 of a probe row that passed nothing,
// whose build_idx[j] then becomes CB_NULL_ROW.
void launch_nlj_cond_resolve(const unsigned* bits, long long p0, long long k, unsigned row0, unsigned m, unsigned long long inv,
                             const unsigned char* passed, bool outer, unsigned* probe_idx, unsigned* build_idx, unsigned char* keep, cudaStream_t st);
// out[i] = !flags[i], i < n
void launch_flags_not(const unsigned char* flags, long long n, unsigned char* out, cudaStream_t st);

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
