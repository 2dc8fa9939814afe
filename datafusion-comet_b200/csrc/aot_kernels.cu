// aot_kernels.cu -- ahead-of-time sm_90a kernels that do not depend on the plan: Arrow buffer
// normalisation (bitmap append at arbitrary bit offsets, byte->bitmap packing), dictionary code
// remapping and the device-side string dictionary builder used to turn Utf8 group keys into dense
// codes.  (Plan-dependent kernels are JIT-specialised: device/cb_kernels.cuh.)
#include "aot_kernels.h"
#include "device/cb_math.h"
#include "device/cb_rangepart.h"
#include "device/cb_strpred.h"

#include <algorithm>

namespace cb200 {
using namespace cb;

// ---- bitmap append: dst[dst_off .. dst_off+n) = src[src_off ..) (src == nullptr -> ones) -----------
// dst must be zero-initialised; one thread per 32 destination bits, boundary words via atomicOr.
__global__ void k_bitmap_append(u32* dst, i64 dst_off, const u8* src, i64 src_off, i64 n) {
    i64 first_word = dst_off >> 5, last_word = (dst_off + n - 1) >> 5;
    i64 w = first_word + (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (w > last_word) return;
    u32 bits = 0;
    i64 lo = w << 5;
    for (int b = 0; b < 32; b++) {
        i64 d = lo + b;
        if (d < dst_off || d >= dst_off + n) continue;
        i64 s = src_off + (d - dst_off);
        u32 bit = src ? ((src[s >> 3] >> (s & 7)) & 1u) : 1u;
        bits |= bit << b;
    }
    if (w == first_word || w == last_word) atomicOr(&dst[w], bits);
    else dst[w] = bits;
}
void launch_bitmap_append(u32* dst, i64 dst_off, const u8* src, i64 src_off, i64 n, cudaStream_t st) {
    if (n <= 0) return;
    i64 words = ((dst_off + n - 1) >> 5) - (dst_off >> 5) + 1;
    int threads = 256;
    k_bitmap_append<<<(unsigned)((words + threads - 1) / threads), threads, 0, st>>>(dst, dst_off, src, src_off, n);
}

// ---- validity bytes (1 per row) -> Arrow bitmap -------------------------------------------------
__global__ void k_bytes_to_bitmap(const u8* bytes, i64 n, u32* out) {
    i64 w = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (w * 32 >= n) return;
    u32 bits = 0;
    for (int b = 0; b < 32; b++) {
        i64 i = w * 32 + b;
        if (i < n && bytes[i]) bits |= 1u << b;
    }
    out[w] = bits;
}
void launch_bytes_to_bitmap(const u8* bytes, i64 n, u32* out, cudaStream_t st) {
    if (n <= 0) return;
    i64 words = (n + 31) / 32;
    k_bytes_to_bitmap<<<(unsigned)((words + 255) / 256), 256, 0, st>>>(bytes, n, out);
}

// ---- dictionary code remap (batch dictionary -> plan-global dictionary) ------------------------------
template <typename T> __global__ void k_remap_codes(const T* in, i64 n, const i32* table, i32 table_len, i32* out) {
    i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    i32 c = (i32)in[i];
    out[i] = (c >= 0 && c < table_len) ? table[c] : 0;
}
void launch_remap_codes(const void* in, int in_width, i64 n, const i32* table, i32 table_len, i32* out, cudaStream_t st) {
    if (n <= 0) return;
    unsigned blocks = (unsigned)((n + 255) / 256);
    if (in_width == 1) k_remap_codes<signed char><<<blocks, 256, 0, st>>>((const signed char*)in, n, table, table_len, out);
    else if (in_width == 2) k_remap_codes<short><<<blocks, 256, 0, st>>>((const short*)in, n, table, table_len, out);
    else k_remap_codes<i32><<<blocks, 256, 0, st>>>((const i32*)in, n, table, table_len, out);
}

// ---- string predicate over dictionary entries -> one bit per code ---------------------------------------------------------------------
// One thread per entry; a warp's 32 entries are one mask word (first is a multiple of 32), written whole by the ballot: no atomics and no
// read-modify-write of a word another launch owns.  Bits past n are 0 in the last word; the next launch over a grown dictionary starts
// at that word again.
__global__ void k_str_pred(StrPredDev d, const i32* off, const u8* chars, i64 first, i64 n, u32* mask) {
    const i64 i = first + (i64)blockIdx.x * blockDim.x + threadIdx.x;
    bool bit = false;
    if (i < n) {
        const i64 k = i - first;
        bit = sp_eval(d, chars + off[k], off[k + 1] - off[k]);
    }
    const u32 w = __ballot_sync(0xffffffffu, bit);
    if ((threadIdx.x & 31) == 0 && i < n) mask[i >> 5] = w;
}
void launch_str_pred(const StrPredDev& d, const int* offsets, const unsigned char* chars, i64 first, i64 n, unsigned* mask, cudaStream_t st) {
    if (n <= first) return;
    const int threads = 256;
    k_str_pred<<<(unsigned)((n - first + threads - 1) / threads), threads, 0, st>>>(d, offsets, chars, first, n, mask);
}

// ---- device string dictionary -----------------------------------------------------------------------
// Open-addressing table keyed by a 64-bit hash of the bytes; each claimed slot owns a dense code and
// a copy of the string.  Pass 1 claims / finds slots (codes handed out by atomicAdd), pass 2 verifies
// the bytes against the stored copy (a 64-bit hash collision between different strings raises
// CB_DICT_COLLISION instead of silently merging two groups) and writes the code column.
__device__ __forceinline__ u64 hash_bytes64(const u8* p, i32 len) {
    u32 a = mm3_bytes(p, len, 42u), b = mm3_bytes(p, len, 0x9747b28cu);
    u64 h = ((u64)a << 32) | b;
    return h == 0 ? 1 : h; // 0 = empty slot
}
__global__ void k_dict_insert(StringDictDev d, const i32* offsets, const u8* chars, const u8* validity, i64 n, i32* row_slot) {
    i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (validity && !((validity[i >> 3] >> (i & 7)) & 1)) { row_slot[i] = -1; return; }
    const u8* p = chars + offsets[i];
    i32 len = offsets[i + 1] - offsets[i];
    u64 h = hash_bytes64(p, len);
    u32 mask = (u32)d.capacity - 1;
    u32 s = (u32)(h ^ (h >> 32)) & mask;
    for (u32 probe = 0; probe <= mask; probe++, s = (s + 1) & mask) {
        u64 prev = atomicCAS((unsigned long long*)&d.tags[s], 0ull, (unsigned long long)h);
        if (prev == 0) { // claimed: allocate a code and copy the bytes
            i32 code = atomicAdd(d.n_codes, 1);
            if (code >= d.max_codes) { atomicOr(d.err, CB_DICT_FULL); row_slot[i] = -1; return; }
            i64 off = (i64)atomicAdd((unsigned long long*)d.bytes_used, (unsigned long long)len);
            if (off + len > d.bytes_cap) { atomicOr(d.err, CB_DICT_FULL); row_slot[i] = -1; return; }
            for (i32 k = 0; k < len; k++) d.bytes[off + k] = p[k];
            d.code_off[code] = off;
            d.code_len[code] = len;
            d.slot_code[s] = code;
            row_slot[i] = (i32)s;
            return;
        }
        if (prev == h) { row_slot[i] = (i32)s; return; }
    }
    atomicOr(d.err, CB_DICT_FULL);
    row_slot[i] = -1;
}
__global__ void k_dict_resolve(StringDictDev d, const i32* offsets, const u8* chars, i64 n, const i32* row_slot, i32* codes) {
    i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    i32 s = row_slot[i];
    if (s < 0) { codes[i] = 0; return; }
    i32 code = d.slot_code[s];
    i32 len = offsets[i + 1] - offsets[i];
    const u8* p = chars + offsets[i];
    bool same = d.code_len[code] == len;
    const u8* q = d.bytes + d.code_off[code];
    for (i32 k = 0; same && k < len; k++) same = p[k] == q[k];
    if (!same) atomicOr(d.err, CB_DICT_COLLISION);
    codes[i] = code;
}
void launch_dict_encode(const StringDictDev& d, const i32* offsets, const u8* chars, const u8* validity, i64 n, i32* row_slot, i32* codes,
                        cudaStream_t st) {
    if (n <= 0) return;
    unsigned blocks = (unsigned)((n + 255) / 256);
    k_dict_insert<<<blocks, 256, 0, st>>>(d, offsets, chars, validity, n, row_slot);
    k_dict_resolve<<<blocks, 256, 0, st>>>(d, offsets, chars, n, row_slot, codes);
}

} // namespace cb200

// ---- stream compaction of sparse (hash-table ordered) result columns ---------------------------------------------
namespace cb200 {
using namespace cb;

__global__ void k_block_counts(const u8* present, i64 n, i32* counts) {
    __shared__ i32 s;
    if (threadIdx.x == 0) s = 0;
    __syncthreads();
    i64 i = (i64)blockIdx.x * 1024 + threadIdx.x;
    int c = 0;
    for (int k = 0; k < 4; k++, i += 256) if (i < n && present[i]) c++;
    for (int m = 16; m >= 1; m >>= 1) c += __shfl_xor_sync(0xffffffffu, c, m);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s, c);
    __syncthreads();
    if (threadIdx.x == 0) counts[blockIdx.x] = s;
}
// single-CTA exclusive scan of the per-block counts (<= a few million entries); total written to *total
__global__ void k_scan_counts(const i32* counts, i64 nb, i64* offsets, i64* total) {
    __shared__ i64 carry;
    __shared__ i64 wsum[32];
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (i64 base = 0; base < nb; base += 1024) {
        i64 i = base + threadIdx.x;
        i64 v = i < nb ? counts[i] : 0, x = v;
        int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
        for (int d = 1; d < 32; d <<= 1) { i64 y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
        if (lane == 31) wsum[w] = x;
        __syncthreads();
        if (w == 0) {
            i64 t = wsum[lane], u = t;
            for (int d = 1; d < 32; d <<= 1) { i64 y = __shfl_up_sync(0xffffffffu, u, d); if (lane >= d) u += y; }
            wsum[lane] = u - t; // exclusive
        }
        __syncthreads();
        i64 excl = carry + wsum[w] + x - v;
        if (i < nb) offsets[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}
// out[offsets[block] + rank within block] = in[i] for present rows; one launch per column (width bytes per row)
__global__ void k_compact_scatter(const u8* present, i64 n, const i64* offsets, const u8* in, int width, u8* out) {
    __shared__ i32 wcount[8];
    i64 blk0 = (i64)blockIdx.x * 1024;
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    i64 base = offsets[blockIdx.x];
    for (int k = 0; k < 4; k++) { // rows blk0 + k*256 + tid: (k, warp, lane) order == row order
        i64 i = blk0 + (i64)k * 256 + threadIdx.x;
        bool keep = i < n && present[i];
        u32 bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) wcount[w] = __popc(bal);
        __syncthreads();
        i64 off = base;
        int tot = 0;
        for (int j = 0; j < 8; j++) { if (j < w) off += wcount[j]; tot += wcount[j]; }
        if (keep) {
            i64 o = off + __popc(bal & ((1u << lane) - 1u));
            const u8* src = in + i * width;
            u8* dst = out + o * width;
            if (width == 16) *reinterpret_cast<ulonglong2*>(dst) = *reinterpret_cast<const ulonglong2*>(src);
            else if (width == 8) *reinterpret_cast<u64*>(dst) = *reinterpret_cast<const u64*>(src);
            else if (width == 4) *reinterpret_cast<u32*>(dst) = *reinterpret_cast<const u32*>(src);
            else for (int b = 0; b < width; b++) dst[b] = src[b];
        }
        base += tot;
        __syncthreads();
    }
}

__global__ void k_key_presence(const unsigned long long* keys, i64 n, u8* present) {
    i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) present[i] = keys[i] != 0xffffffffffffffffull;
}
void launch_key_presence(const unsigned long long* keys, i64 n, u8* present, cudaStream_t st) {
    if (n > 0) k_key_presence<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(keys, n, present);
}
void launch_compact_plan(const u8* present, i64 n, i32* counts, i64* offsets, i64* total, cudaStream_t st) {
    i64 nb = (n + 1023) / 1024;
    if (nb <= 0) return;
    k_block_counts<<<(unsigned)nb, 256, 0, st>>>(present, n, counts);
    k_scan_counts<<<1, 1024, 0, st>>>(counts, nb, offsets, total);
}
void launch_compact_scatter(const u8* present, i64 n, const i64* offsets, const void* in, int width, void* out, cudaStream_t st) {
    i64 nb = (n + 1023) / 1024;
    if (nb <= 0) return;
    k_compact_scatter<<<(unsigned)nb, 256, 0, st>>>(present, n, offsets, (const u8*)in, width, (u8*)out);
}

} // namespace cb200

// ---- hash partitioning: Spark murmur3 (seed 42) over the key columns, pmod, stable counting sort ---------------------
// Replaces native/shuffle/src/partitioners/multi_partition.rs:265-330 (hash + pmod) and :54-99 (counting sort).
namespace cb200 {
using namespace cb;

__device__ __forceinline__ bool bit_at(const u8* bm, i64 i) { return (bm[i >> 3] >> (i & 7)) & 1; }

// h chained over row i's key columns by Spark's murmur3 rules
__device__ __forceinline__ u32 hash_key_cols(const HashKeyCols& kc, i64 i, u32 h) {
    for (int c = 0; c < kc.n; c++) {
        const HashKeyCol& k = kc.col[c];
        if (k.validity && !bit_at(k.validity, i)) continue; // NULL leaves the running hash unchanged (utils.rs:38-42)
        const u8* d = (const u8*)k.data;
        switch (k.kind) {
        case HK_BOOL: h = mm3_i32(bit_at(d, i) ? 1 : 0, h); break;
        case HK_BOOL8: h = mm3_i32(d[i] ? 1 : 0, h); break;
        case HK_I8: h = mm3_i32((i32)((const signed char*)d)[i], h); break;
        case HK_I16: h = mm3_i32((i32)((const short*)d)[i], h); break;
        case HK_I32: h = mm3_i32(((const i32*)d)[i], h); break;
        case HK_I64: h = mm3_i64(((const i64*)d)[i], h); break;
        case HK_F32: { float f = ((const float*)d)[i]; if (f == 0.0f) f = 0.0f; h = mm3_i32((i32)__float_as_uint(f == 0.0f ? 0.0f : f), h); break; }
        case HK_F64: { double f = ((const double*)d)[i]; h = mm3_i64(f == 0.0 ? 0ll : __double_as_longlong(f), h); break; }
        case HK_DEC_SMALL_128: h = mm3_i64((i64)((const i128*)d)[i].lo, h); break; // d(p<=18): hashed as i64 (utils.rs:159-196)
        case HK_DEC_LARGE_128: h = mm3_i128(((const i128*)d)[i], h); break;        // d(p>18): 16 LE bytes (utils.rs:199-226)
        case HK_DEC_LARGE_64: h = mm3_i128(i128_from_i64(((const i64*)d)[i]), h); break;
        case HK_DEC_SMALL_32: h = mm3_i64((i64)((const i32*)d)[i], h); break;
        case HK_DICT8: case HK_DICT16: case HK_DICT32: {
            i32 code = k.kind == HK_DICT8 ? (i32)((const signed char*)d)[i] : k.kind == HK_DICT16 ? (i32)((const short*)d)[i] : ((const i32*)d)[i];
            i32 o0 = k.dict_offsets[code], o1 = k.dict_offsets[code + 1];
            h = mm3_bytes(k.dict_chars + o0, o1 - o0, h);
            break;
        }
        case HK_UTF8: {
            i32 o0 = k.dict_offsets[i], o1 = k.dict_offsets[i + 1];
            h = mm3_bytes(k.dict_chars + o0, o1 - o0, h);
            break;
        }
        }
    }
    return h;
}

__global__ void k_partition_ids(HashKeyCols kc, i64 n, u32 n_parts, u32* hashes, u32* pids) {
    i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u32 h = hash_key_cols(kc, i, 42u); // spark seed (multi_partition.rs:298)
    if (hashes) hashes[i] = h;
    pids[i] = pmod_u32(h, n_parts);
}

// one group of at most 8 columns of a longer hash chain (round-robin partitioning over more columns): the first group starts from the
// seed, the others from hashes[i]; the last writes pids[i] = pmod, the others the running hash back to hashes[i]
__global__ void k_partition_ids_chain(HashKeyCols kc, i64 n, u32 n_parts, int first, int last, u32* hashes, u32* pids) {
    i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u32 h = hash_key_cols(kc, i, first ? 42u : hashes[i]);
    if (last) pids[i] = pmod_u32(h, n_parts);
    else hashes[i] = h;
}

// Range partitioning: pids[i] = the number of boundary rows <= row i's packed key (device/cb_rangepart.h).  The key has W words, a
// template constant, so it is built and compared in registers.  The top level of the search (all boundary rows, or every 2^shift-th)
// is staged in shared memory once per CTA of a grid-stride loop; with shift > 0 the search ends in `bounds`, which stays in L2.
template <int W>
__global__ void __launch_bounds__(256) k_range_pids(SortKeyCols kc, i64 n, const u64* top, u32 n_top, int shift, const u64* bounds, u32 nb, u32* pids) {
    extern __shared__ u64 s_top[];
    for (u32 j = threadIdx.x; j < n_top * (u32)W; j += blockDim.x) s_top[j] = top[j];
    __syncthreads();
    for (i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (i64)gridDim.x * blockDim.x) {
        u64 w[W] = {};
        if (!sk_row_reg<W>(kc, i, w)) atomicOr(kc.err, 1 << 5);
        pids[i] = rp_pid<W>(s_top, n_top, shift, bounds, nb, w);
    }
}

// per-1024-row-block histogram of partition ids -> block_hist[block][n_parts]
__global__ void k_pid_block_hist(const u32* pids, i64 n, u32 n_parts, i32* block_hist) {
    extern __shared__ i32 sh[];
    for (u32 p = threadIdx.x; p < n_parts; p += blockDim.x) sh[p] = 0;
    __syncthreads();
    i64 i0 = (i64)blockIdx.x * 1024;
    for (int k = threadIdx.x; k < 1024; k += blockDim.x) { i64 i = i0 + k; if (i < n) atomicAdd(&sh[pids[i]], 1); }
    __syncthreads();
    for (u32 p = threadIdx.x; p < n_parts; p += blockDim.x) block_hist[(size_t)blockIdx.x * n_parts + p] = sh[p];
}
// exclusive scan in (partition-major, block-minor) order: out position of the first row of (block, partition).
// Three small kernels over CHUNKS of 1024 row blocks (a single-CTA scan took 13 ms for the 183 K row blocks of a 187 M-row batch):
//   k_pid_chunk_totals : rows of (chunk, partition)                       -- one CTA per chunk, one warp per partition at a time
//   k_pid_chunk_scan   : partition starts + first position of (chunk, partition); tiny (chunks x partitions)
//   k_pid_block_bases  : first position of (block, partition) by a warp scan over the chunk's blocks
#define PID_CHUNK 1024
__global__ void k_pid_chunk_totals(const i32* block_hist, i64 n_blocks, u32 n_parts, i64* chunk_tot) {
    const i64 b0 = (i64)blockIdx.x * PID_CHUNK;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (u32 p = warp; p < n_parts; p += nw) {
        i64 t = 0;
        for (int k = lane; k < PID_CHUNK; k += 32) { const i64 b = b0 + k; if (b < n_blocks) t += block_hist[(size_t)b * n_parts + p]; }
#pragma unroll
        for (int o = 16; o; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (lane == 0) chunk_tot[(size_t)blockIdx.x * n_parts + p] = t;
    }
}
__global__ void k_pid_chunk_scan(i64* chunk_tot, i64 n_chunks, u32 n_parts, i64* starts) {
    extern __shared__ i64 totals[];
    for (u32 p = threadIdx.x; p < n_parts; p += blockDim.x) {
        i64 t = 0;
        for (i64 c = 0; c < n_chunks; c++) t += chunk_tot[(size_t)c * n_parts + p];
        totals[p] = t;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        i64 run = 0;
        for (u32 p = 0; p < n_parts; p++) { starts[p] = run; run += totals[p]; }
        starts[n_parts] = run;
    }
    __syncthreads();
    for (u32 p = threadIdx.x; p < n_parts; p += blockDim.x) { // in place: totals -> exclusive bases
        i64 run = starts[p];
        for (i64 c = 0; c < n_chunks; c++) { const i64 t = chunk_tot[(size_t)c * n_parts + p]; chunk_tot[(size_t)c * n_parts + p] = run; run += t; }
    }
}
__global__ void k_pid_block_bases(const i32* block_hist, i64 n_blocks, u32 n_parts, const i64* chunk_base, i64* block_base) {
    const i64 b0 = (i64)blockIdx.x * PID_CHUNK;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (u32 p = warp; p < n_parts; p += nw) {
        i64 run = chunk_base[(size_t)blockIdx.x * n_parts + p];
        for (int k = 0; k < PID_CHUNK; k += 32) {
            const i64 b = b0 + k + lane;
            const i64 v = b < n_blocks ? (i64)block_hist[(size_t)b * n_parts + p] : 0;
            i64 incl = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const i64 up = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += up; }
            if (b < n_blocks) block_base[(size_t)b * n_parts + p] = run + incl - v;
            run += __shfl_sync(0xffffffffu, incl, 31);
        }
    }
}
// stable placement: rows of a block are visited in row order by ONE warp-sized sweep per 32 rows
__global__ void k_pid_place(const u32* pids, i64 n, u32 n_parts, const i64* block_base, i64* row_idx) {
    extern __shared__ i64 cursor[]; // [n_parts] running output position for this block
    for (u32 p = threadIdx.x; p < n_parts; p += blockDim.x) cursor[p] = block_base[(size_t)blockIdx.x * n_parts + p];
    __syncthreads();
    if (threadIdx.x >= 32) return; // a single warp walks the block in row order: keeps the sort stable
    i64 i0 = (i64)blockIdx.x * 1024;
    int lane = threadIdx.x;
    for (int k = 0; k < 32; k++) {
        i64 i = i0 + k * 32 + lane;
        bool in = i < n;
        u32 pid = in ? pids[i] : 0xffffffffu;
        u32 peers = __match_any_sync(0xffffffffu, pid);
        int rank = __popc(peers & ((1u << lane) - 1u));
        int leader = __ffs(peers) - 1;
        i64 base = 0;
        if (in && lane == leader) { base = cursor[pid]; cursor[pid] = base + __popc(peers); }
        base = __shfl_sync(0xffffffffu, base, leader);
        if (in) row_idx[base + rank] = i;
        __syncwarp();
    }
}
template <typename T, typename I> __global__ void k_gather_rows(const T* in, const I* row_idx, i64 n, T* out) {
    i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[row_idx[i]];
}
template <typename I> __global__ void k_gather_bits(const u8* in_bits, const I* row_idx, i64 n, u8* out_bytes) {
    i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out_bytes[i] = bit_at(in_bits, (i64)row_idx[i]) ? 1 : 0;
}

// the gathers of NULL-extended join columns: row index CB_NULL_ROW gives zero value bytes and a clear bit.  Kept apart from the gathers
// above, which Sort, repartitioning and inner joins run.
template <typename T> __global__ void k_gather_rows_or_null(const T* in, const u32* row_idx, i64 n, T* out) {
    i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { const u32 r = row_idx[i]; out[i] = r == CB_NULL_ROW ? T{} : in[r]; }
}
__global__ void k_gather_bits_or_null(const u8* in_bits, const u32* row_idx, i64 n, u8* out_bytes) {
    i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { const u32 r = row_idx[i]; out_bytes[i] = r != CB_NULL_ROW && (!in_bits || bit_at(in_bits, (i64)r)) ? 1 : 0; }
}

i64 partition_chunks(i64 n) { const i64 nb = (n + 1023) / 1024; return (nb + PID_CHUNK - 1) / PID_CHUNK; }
// one counter per partition in shared memory: above the default 48 KB a kernel has to opt in
static cudaError_t partition_smem_setup(u32 n_parts, int& smem32, int& smem64) {
    if (n_parts == 0 || n_parts > (u32)CB_MAX_HASH_PARTITIONS) return cudaErrorInvalidValue;
    smem32 = (int)(n_parts * sizeof(i32)), smem64 = (int)(n_parts * sizeof(i64));
    cudaError_t e = cudaSuccess;
    if (smem32 > 48 * 1024) e = cudaFuncSetAttribute((const void*)k_pid_block_hist, cudaFuncAttributeMaxDynamicSharedMemorySize, smem32);
    if (smem64 > 48 * 1024 && e == cudaSuccess) e = cudaFuncSetAttribute((const void*)k_pid_chunk_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, smem64);
    if (smem64 > 48 * 1024 && e == cudaSuccess) e = cudaFuncSetAttribute((const void*)k_pid_place, cudaFuncAttributeMaxDynamicSharedMemorySize, smem64);
    return e;
}
cudaError_t launch_partition_ids(const HashKeyCols& kc, i64 n, u32 n_parts, u32* hashes, u32* pids, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    if (n_parts == 0 || n_parts > (u32)CB_MAX_HASH_PARTITIONS) return cudaErrorInvalidValue;
    k_partition_ids<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(kc, n, n_parts, hashes, pids);
    return cudaGetLastError();
}
cudaError_t launch_partition_place(const u32* pids, i64 n, u32 n_parts, i32* block_hist, i64* block_base, i64* chunk_tmp, i64* starts, i64* row_idx,
                                   cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    int smem32 = 0, smem64 = 0;
    cudaError_t e = partition_smem_setup(n_parts, smem32, smem64);
    if (e != cudaSuccess) return e;
    const i64 nb = (n + 1023) / 1024, nc = partition_chunks(n);
    k_pid_block_hist<<<(unsigned)nb, 256, smem32, st>>>(pids, n, n_parts, block_hist);
    k_pid_chunk_totals<<<(unsigned)nc, 256, 0, st>>>(block_hist, nb, n_parts, chunk_tmp);
    k_pid_chunk_scan<<<1, 256, smem64, st>>>(chunk_tmp, nc, n_parts, starts);
    k_pid_block_bases<<<(unsigned)nc, 256, 0, st>>>(block_hist, nb, n_parts, chunk_tmp, block_base);
    k_pid_place<<<(unsigned)nb, 64, smem64, st>>>(pids, n, n_parts, block_base, row_idx);
    return cudaGetLastError();
}
cudaError_t launch_partition_ids_chain(const HashKeyCols& kc, i64 n, u32 n_parts, bool first, bool last, u32* hashes, u32* pids, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    k_partition_ids_chain<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(kc, n, n_parts, first, last, hashes, pids);
    return cudaGetLastError();
}
template <int W> static cudaError_t range_pids(const SortKeyCols& kc, i64 n, const u64* top, u32 n_top, int shift, const u64* bounds, u32 nb, u32* pids,
                                               cudaStream_t st) {
    const size_t smem = (size_t)n_top * W * 8;
    // grid-stride over one wave: as many CTAs as fit on the device at once with this much shared memory each
    int dev = 0, sms = 0, per_sm = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_range_pids<W>, 256, smem);
    if (e != cudaSuccess) return e;
    const i64 blocks = std::min<i64>((n + 255) / 256, (i64)std::max(1, sms * per_sm));
    k_range_pids<W><<<(unsigned)blocks, 256, smem, st>>>(kc, n, top, n_top, shift, bounds, nb, pids);
    return cudaGetLastError();
}
cudaError_t launch_range_pids(const SortKeyCols& kc, i64 n, const u64* top, u32 n_top, int shift, const u64* bounds, u32 nb, u32* pids, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    if ((size_t)n_top * kc.words * 8 > CB_RANGE_TOP_BYTES) return cudaErrorInvalidValue;
    switch (kc.words) {
    case 1: return range_pids<1>(kc, n, top, n_top, shift, bounds, nb, pids, st);
    case 2: return range_pids<2>(kc, n, top, n_top, shift, bounds, nb, pids, st);
    case 3: return range_pids<3>(kc, n, top, n_top, shift, bounds, nb, pids, st);
    case 4: return range_pids<4>(kc, n, top, n_top, shift, bounds, nb, pids, st);
    default: return cudaErrorInvalidValue;
    }
}
template <typename I> static void gather_rows(const void* in, int width, const I* row_idx, i64 n, void* out, cudaStream_t st) {
    if (n <= 0) return;
    unsigned blocks = (unsigned)((n + 255) / 256);
    if (width == 16) k_gather_rows<ulonglong2, I><<<blocks, 256, 0, st>>>((const ulonglong2*)in, row_idx, n, (ulonglong2*)out);
    else if (width == 8) k_gather_rows<u64, I><<<blocks, 256, 0, st>>>((const u64*)in, row_idx, n, (u64*)out);
    else if (width == 4) k_gather_rows<u32, I><<<blocks, 256, 0, st>>>((const u32*)in, row_idx, n, (u32*)out);
    else if (width == 2) k_gather_rows<u16, I><<<blocks, 256, 0, st>>>((const u16*)in, row_idx, n, (u16*)out);
    else k_gather_rows<u8, I><<<blocks, 256, 0, st>>>((const u8*)in, row_idx, n, (u8*)out);
}
void launch_gather(const void* in, int width, const i64* row_idx, i64 n, void* out, cudaStream_t st) { gather_rows(in, width, row_idx, n, out, st); }
void launch_gather(const void* in, int width, const u32* row_idx, i64 n, void* out, cudaStream_t st) { gather_rows(in, width, row_idx, n, out, st); }
void launch_gather_bits(const void* in_bits, const i64* row_idx, i64 n, void* out_bytes, cudaStream_t st) {
    if (n > 0) k_gather_bits<i64><<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const u8*)in_bits, row_idx, n, (u8*)out_bytes);
}
void launch_gather_bits(const void* in_bits, const u32* row_idx, i64 n, void* out_bytes, cudaStream_t st) {
    if (n > 0) k_gather_bits<u32><<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const u8*)in_bits, row_idx, n, (u8*)out_bytes);
}

void launch_gather_or_null(const void* in, int width, const u32* row_idx, i64 n, void* out, cudaStream_t st) {
    if (n <= 0) return;
    unsigned blocks = (unsigned)((n + 255) / 256);
    if (width == 16) k_gather_rows_or_null<ulonglong2><<<blocks, 256, 0, st>>>((const ulonglong2*)in, row_idx, n, (ulonglong2*)out);
    else if (width == 8) k_gather_rows_or_null<u64><<<blocks, 256, 0, st>>>((const u64*)in, row_idx, n, (u64*)out);
    else if (width == 4) k_gather_rows_or_null<u32><<<blocks, 256, 0, st>>>((const u32*)in, row_idx, n, (u32*)out);
    else if (width == 2) k_gather_rows_or_null<u16><<<blocks, 256, 0, st>>>((const u16*)in, row_idx, n, (u16*)out);
    else k_gather_rows_or_null<u8><<<blocks, 256, 0, st>>>((const u8*)in, row_idx, n, (u8*)out);
}
void launch_gather_bits_or_null(const void* in_bits, const u32* row_idx, i64 n, void* out_bytes, cudaStream_t st) {
    if (n > 0) k_gather_bits_or_null<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const u8*)in_bits, row_idx, n, (u8*)out_bytes);
}

// ---- sort: packed row keys, stable LSD radix sort -----------------------------------------------------------------------------------------
// Keys are `W` 64-bit words per row (device/cb_sortkey.h), word 0 the most significant.  A pass sorts by one 8-bit digit, stably, over
// tiles of SORT_TILE rows:
//   k_sort_hist     : digit histogram of each tile, digit-major: hist[digit * n_tiles + tile]
//   launch_scan_u32 : the select pipelines' chunked exclusive scan over that array, which in this order is the first output position of
//                     (digit, tile) -- flat and coalesced (the partitioner's per-partition scan reads [tile][digit] with a 1 KB stride)
//   k_sort_scatter  : moves keys and row indices; each of the 8 warps of a tile owns 512 consecutive rows, counts its digits, takes its
//                     base from the warps before it, then walks its rows in order (a __match_any_sync rank per 32 rows): stable.
//                     The tile is put in digit order in shared memory first and written out from there in runs.
#define SORT_TILE 4096
__global__ void __launch_bounds__(256) k_sort_keys(SortKeyCols kc, i64 n, u64* keys, u64* and_or) {
    __shared__ u64 s_and[8][SK_MAX_WORDS], s_or[8][SK_MAX_WORDS];
    u64 a[SK_MAX_WORDS] = {~0ull, ~0ull, ~0ull, ~0ull}, o[SK_MAX_WORDS] = {0, 0, 0, 0};
    const int W = kc.words;
    for (i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (i64)gridDim.x * blockDim.x) {
        u64 w[SK_MAX_WORDS] = {0, 0, 0, 0};
        if (!sk_row(kc, i, w)) atomicOr(kc.err, 1 << 5);
#pragma unroll
        for (int j = 0; j < SK_MAX_WORDS; j++) {
            if (j < W) keys[i * W + j] = w[j];
            a[j] &= w[j];
            o[j] |= w[j];
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int j = 0; j < SK_MAX_WORDS; j++) {
#pragma unroll
        for (int m = 16; m; m >>= 1) { a[j] &= __shfl_xor_sync(0xffffffffu, a[j], m); o[j] |= __shfl_xor_sync(0xffffffffu, o[j], m); }
        if (lane == 0) { s_and[warp][j] = a[j]; s_or[warp][j] = o[j]; }
    }
    __syncthreads();
    if (threadIdx.x < W) {
        u64 ba = ~0ull, bo = 0;
        for (int k = 0; k < 8; k++) { ba &= s_and[k][threadIdx.x]; bo |= s_or[k][threadIdx.x]; }
        atomicAnd(&and_or[threadIdx.x], ba);
        atomicOr(&and_or[W + threadIdx.x], bo);
    }
}
void launch_sort_keys(const SortKeyCols& kc, i64 n, u64* keys, u64* and_or, cudaStream_t st) {
    if (n <= 0) return;
    const i64 blocks = std::min<i64>((n + 255) / 256, 132 * 16); // grid-stride: one and / or per block
    k_sort_keys<<<(unsigned)blocks, 256, 0, st>>>(kc, n, keys, and_or);
}

template <int W> __global__ void __launch_bounds__(256) k_sort_hist(const u64* keys, i64 n, int digit, i64 n_tiles, u32* hist) {
    __shared__ u32 h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int word = W - 1 - (digit >> 3), sh = (digit & 7) * 8;
    const i64 i0 = (i64)blockIdx.x * SORT_TILE;
#pragma unroll 4
    for (int k = threadIdx.x; k < SORT_TILE; k += 256) {
        const i64 i = i0 + k;
        if (i < n) atomicAdd(&h[(keys[i * W + word] >> sh) & 255u], 1u);
    }
    __syncthreads();
    hist[(i64)threadIdx.x * n_tiles + blockIdx.x] = h[threadIdx.x];
}

// rows of a warp: r0 + k * 32 + lane, k < SORT_ITEMS; keys are staged in registers GROUP rows at a time.  Each row goes first to its
// place in the tile ordered by digit (shared memory), and from there to the output: consecutive threads write consecutive positions of
// a digit's run, instead of one scattered 8-byte key and 4-byte index per row.
#define SORT_ITEMS (SORT_TILE / 8 / 32)
template <int W> constexpr size_t sort_scatter_smem() { return (size_t)SORT_TILE * (8 * W + 4); }
template <int W>
__global__ void __launch_bounds__(256, 2) k_sort_scatter(const u64* kin, const u32* iin, i64 n, int digit, i64 n_tiles, const u32* hist,
                                                      const u32* chunk_off, u64* kout, u32* iout) {
    constexpr int GROUP = W <= 2 ? SORT_ITEMS : SORT_ITEMS / 2;
    extern __shared__ u64 sm[];     // [W][SORT_TILE] key words, then [SORT_TILE] row indices: the tile in digit order
    u64* skey = sm;
    u32* sidx = (u32*)(sm + (size_t)W * SORT_TILE);
    __shared__ u32 cur[8][256];     // per warp: digit count, then the warp's next tile position of each digit
    __shared__ u32 dstart[256];     // tile position of each digit's first row
    __shared__ u32 gbase[256];      // output position of each digit's first row
    __shared__ u32 wsum[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int w = 0; w < 8; w++) cur[w][threadIdx.x] = 0;
    __syncthreads();
    const int word = W - 1 - (digit >> 3), sh = (digit & 7) * 8;
    const i64 t0 = (i64)blockIdx.x * SORT_TILE, r0 = t0 + warp * (SORT_TILE / 8);
    u32 dg[SORT_ITEMS];
#pragma unroll
    for (int k = 0; k < SORT_ITEMS; k++) {
        const i64 i = r0 + k * 32 + lane;
        dg[k] = i < n ? (u32)(kin[i * W + word] >> sh) & 255u : 256u + lane; // rows past the end match nobody
    }
#pragma unroll
    for (int k = 0; k < SORT_ITEMS; k++)
        if (dg[k] < 256u) atomicAdd(&cur[warp][dg[k]], 1u);
    __syncthreads();
    { // thread t: digit t.  Tile start of the digit = exclusive scan over digits; each warp's start after the warps before it
        const u32 t = threadIdx.x;
        u32 c[8], tot = 0;
#pragma unroll
        for (int w = 0; w < 8; w++) { c[w] = cur[w][t]; tot += c[w]; }
        u32 incl = tot;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const u32 up = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += up; }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        u32 run = incl - tot;
        for (int w = 0; w < warp; w++) run += wsum[w];
        dstart[t] = run;
        const i64 at = (i64)t * n_tiles + blockIdx.x;
        gbase[t] = hist[at] + chunk_off[at >> 12];
#pragma unroll
        for (int w = 0; w < 8; w++) { cur[w][t] = run; run += c[w]; }
    }
    __syncthreads();
#pragma unroll
    for (int g = 0; g < SORT_ITEMS; g += GROUP) {
        u64 key[GROUP][W];
        u32 id[GROUP];
#pragma unroll
        for (int k = 0; k < GROUP; k++) {
            const i64 i = r0 + (g + k) * 32 + lane;
            if (i < n) {
#pragma unroll
                for (int j = 0; j < W; j++) key[k][j] = kin[i * W + j];
                id[k] = iin ? iin[i] : (u32)i;
            }
        }
#pragma unroll
        for (int k = 0; k < GROUP; k++) {
            const u32 d = dg[g + k];
            const u32 peers = __match_any_sync(0xffffffffu, d);
            const int leader = __ffs(peers) - 1;
            u32 base = 0;
            if (d < 256u && lane == leader) { base = cur[warp][d]; cur[warp][d] = base + __popc(peers); }
            base = __shfl_sync(0xffffffffu, base, leader);
            if (d < 256u) {
                const u32 l = base + __popc(peers & ((1u << lane) - 1u));
#pragma unroll
                for (int j = 0; j < W; j++) skey[j * SORT_TILE + l] = key[k][j];
                sidx[l] = id[k];
            }
            __syncwarp();
        }
    }
    __syncthreads();
    const int rows = (int)min((i64)SORT_TILE, n - t0);
    for (int l = threadIdx.x; l < rows; l += 256) {
        u64 kw[W], dw = 0;
#pragma unroll
        for (int j = 0; j < W; j++) { kw[j] = skey[j * SORT_TILE + l]; if (j == word) dw = kw[j]; }
        const u32 d = (u32)(dw >> sh) & 255u;
        const i64 o = (i64)gbase[d] + (l - (int)dstart[d]);
#pragma unroll
        for (int j = 0; j < W; j++) kout[o * W + j] = kw[j];
        iout[o] = sidx[l];
    }
}
// ---- TopK selection: the key of the k-th row by an MSD radix select, then the rows before it in the stable order ------------------------
// k_sort_select_hist: histogram of one digit over the rows whose key equals `want` under `mask` (the digits decided so far); one read of
// the digit's word per row, shared-memory bins, one global add per bin and block.
template <int W> __global__ void __launch_bounds__(256) k_sort_select_hist(const u64* keys, i64 n, SortSelectKey p, int digit, u32* hist) {
    __shared__ u32 h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int word = W - 1 - (digit >> 3), sh = (digit & 7) * 8;
    for (i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (i64)gridDim.x * blockDim.x) {
        bool match = true;
#pragma unroll
        for (int j = 0; j < W; j++) match &= (keys[i * W + j] & p.mask[j]) == p.want[j];
        if (match) atomicAdd(&h[(keys[i * W + word] >> sh) & 255u], 1u);
    }
    __syncthreads();
    if (h[threadIdx.x]) atomicAdd(&hist[threadIdx.x], h[threadIdx.x]);
}
template <int W> __device__ __forceinline__ int sort_key_cmp(const u64* k, const SortSelectKey& p) { // -1 / 0 / 1: k against p.want
#pragma unroll
    for (int j = 0; j < W; j++)
        if (k[j] != p.want[j]) return k[j] < p.want[j] ? -1 : 1;
    return 0;
}
// eq[i] = row i's key equals the selected key
template <int W> __global__ void k_sort_select_eq(const u64* keys, i64 n, SortSelectKey p, u8* eq) {
    const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) eq[i] = sort_key_cmp<W>(keys + i * W, p) == 0;
}
// keep[i] = key < selected, or key == selected and fewer than `r` equal rows come before it (eq_before: per 1024-row block, from
// launch_compact_plan over eq).  Rows of a block in the (k, warp, lane) order k_compact_scatter uses: row order.
template <int W> __global__ void k_sort_select_keep(const u64* keys, i64 n, SortSelectKey p, const i64* eq_before, i64 r, u8* keep) {
    __shared__ i32 wcount[8];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    i64 before = eq_before[blockIdx.x];
    for (int k = 0; k < 4; k++) {
        const i64 i = (i64)blockIdx.x * 1024 + k * 256 + threadIdx.x;
        const int c = i < n ? sort_key_cmp<W>(keys + i * W, p) : 1;
        const u32 bal = __ballot_sync(0xffffffffu, c == 0);
        if (lane == 0) wcount[w] = __popc(bal);
        __syncthreads();
        i64 off = before;
        int tot = 0;
        for (int j = 0; j < 8; j++) { if (j < w) off += wcount[j]; tot += wcount[j]; }
        if (i < n) keep[i] = c < 0 || (c == 0 && off + __popc(bal & ((1u << lane) - 1u)) < r);
        before += tot;
        __syncthreads();
    }
}
template <int W> static void select_hist(const u64* keys, i64 n, const SortSelectKey& p, int digit, u32* hist, cudaStream_t st) {
    const i64 blocks = std::min<i64>((n + 255) / 256, 132 * 8);
    k_sort_select_hist<W><<<(unsigned)blocks, 256, 0, st>>>(keys, n, p, digit, hist);
}
template <int W> static void select_keep(const u64* keys, i64 n, const SortSelectKey& p, i64 r, u8* eq, i32* counts, i64* offsets, i64* total, u8* keep,
                                         cudaStream_t st) {
    k_sort_select_eq<W><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(keys, n, p, eq);
    launch_compact_plan(eq, n, counts, offsets, total, st);
    k_sort_select_keep<W><<<(unsigned)((n + 1023) / 1024), 256, 0, st>>>(keys, n, p, offsets, r, keep);
}
cudaError_t launch_sort_select_hist(const u64* keys, int words, i64 n, const SortSelectKey& p, int digit, u32* hist, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    switch (words) {
    case 1: select_hist<1>(keys, n, p, digit, hist, st); break;
    case 2: select_hist<2>(keys, n, p, digit, hist, st); break;
    case 3: select_hist<3>(keys, n, p, digit, hist, st); break;
    default: select_hist<4>(keys, n, p, digit, hist, st); break;
    }
    return cudaGetLastError();
}
cudaError_t launch_sort_select_keep(const u64* keys, int words, i64 n, const SortSelectKey& p, i64 r, u8* eq, i32* counts, i64* offsets, i64* total,
                                    u8* keep, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    switch (words) {
    case 1: select_keep<1>(keys, n, p, r, eq, counts, offsets, total, keep, st); break;
    case 2: select_keep<2>(keys, n, p, r, eq, counts, offsets, total, keep, st); break;
    case 3: select_keep<3>(keys, n, p, r, eq, counts, offsets, total, keep, st); break;
    default: select_keep<4>(keys, n, p, r, eq, counts, offsets, total, keep, st); break;
    }
    return cudaGetLastError();
}
__global__ void k_sort_iota(u32* idx, i64 n) {
    const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) idx[i] = (u32)i;
}
void launch_sort_iota(unsigned* idx, i64 n, cudaStream_t st) {
    if (n > 0) k_sort_iota<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(idx, n);
}

i64 sort_tiles(i64 n) { return (n + SORT_TILE - 1) / SORT_TILE; }

// ---- hash join ------------------------------------------------------------------------------------------------------------------------------
// The build side's row keys are radix-sorted, so equal keys form runs in build input order.  Each distinct key (run) owns one slot of an
// open-addressing table, found by linear probing from its hash; a slot stores a 32-bit tag of the hash and the run, and a tag hit is
// confirmed against the run's key words, so two keys are never merged and no collision can fail the query.  The hash and the NULL test
// are join_hash / join_no_null (device/cb_sortkey.h).
__global__ void k_join_heads(const u64* keys, int W, i64 m, u8* head) {
    const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    bool h = i == 0;
    for (int j = 0; j < W && !h; j++) h = keys[i * W + j] != keys[(i - 1) * W + j];
    head[i] = h;
}
__global__ void k_join_insert(JoinTable t, i64 n_runs) {
    const i64 r = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_runs) return;
    const u64* k = t.keys + (i64)t.run_start[r] * t.words;
    if (!join_no_null(k, t.nullmask, t.words)) return;
    const u64 h = join_hash(k, t.words), v = ((h >> 32) << 32) | (u64)(r + 1);
    for (u64 s = h & t.mask;; s = (s + 1) & t.mask) // capacity >= 2 x runs: a free slot exists
        if (atomicCAS((unsigned long long*)&t.slots[s], 0ull, (unsigned long long)v) == 0ull) return;
}
// the run of key k, or -1
__device__ __forceinline__ i64 join_find(const JoinTable& t, const u64* k) {
    if (!join_no_null(k, t.nullmask, t.words)) return -1;
    const u64 h = join_hash(k, t.words);
    const u32 tag = (u32)(h >> 32);
    for (u64 s = h & t.mask;; s = (s + 1) & t.mask) {
        const u64 v = t.slots[s];
        if (v == 0) return -1;
        if ((u32)(v >> 32) != tag) continue;
        const i64 r = (i64)(u32)v - 1;
        const u64* b = t.keys + (i64)t.run_start[r] * t.words;
        bool eq = true;
#pragma unroll
        for (int j = 0; j < SK_MAX_WORDS; j++)
            if (j < t.words) eq &= b[j] == k[j];
        if (eq) return r;
    }
}
__global__ void __launch_bounds__(256) k_join_probe(JoinTable t, const u64* keys, i64 n, int mode, u32* counts, u32* run_of, u64* total, u8* keep,
                                                    u8* hit) {
    const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    const bool pairs = mode == CB_JOIN_COUNT || mode == CB_JOIN_OUTER;
    u64 c = 0;
    if (i < n) {
        u64 k[SK_MAX_WORDS];
#pragma unroll
        for (int j = 0; j < SK_MAX_WORDS; j++) k[j] = j < t.words ? keys[i * t.words + j] : 0;
        const i64 r = join_find(t, k);
        if (pairs) {
            c = r < 0 ? (mode == CB_JOIN_OUTER ? 1 : 0) : t.run_start[r + 1] - t.run_start[r];
            counts[i] = (u32)c;
            run_of[i] = r < 0 ? 0xffffffffu : (u32)r;
            if (hit && r >= 0) hit[r] = 1; // plain stores: every writer stores the same value
        } else keep[i] = (r >= 0) == (mode == CB_JOIN_SEMI);
    }
    if (!pairs) return;
#pragma unroll
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd((unsigned long long*)total, (unsigned long long)c);
}
__global__ void k_join_emit(JoinTable t, const u32* run_of, const u32* offs, const u32* chunk_off, i64 n, i64 o0, i64 o1, int outer, u32* probe_idx,
                            u32* build_idx) {
    const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u32 r = run_of[i];
    const i64 off = (i64)offs[i] + chunk_off[i >> 12];
    if (r == 0xffffffffu) { // no match: an outer join's one NULL-extended pair
        if (outer && off >= o0 && off < o1) { probe_idx[off - o0] = (u32)i; build_idx[off - o0] = CB_NULL_ROW; }
        return;
    }
    const i64 b0 = t.run_start[r], c = (i64)t.run_start[r + 1] - b0;
    const i64 lo = max(off, o0), hi = min(off + c, o1);
    for (i64 p = lo; p < hi; p++) {
        probe_idx[p - o0] = (u32)i;
        build_idx[p - o0] = t.rows[b0 + (p - off)];
    }
}
// keep[rows[p]] = the run holding sorted position p was never hit.  The run is found by binary search over run_start, one thread per
// position: a run may hold most of the build side.
__global__ void k_join_unmatched(const u32* run_start, i64 n_runs, const u32* rows, const u8* hit, i64 m, u8* keep) {
    const i64 p = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    i64 lo = 0, hi = n_runs - 1; // the last run starting at or before p
    while (lo < hi) {
        const i64 mid = (lo + hi + 1) >> 1;
        if ((i64)run_start[mid] <= p) lo = mid;
        else hi = mid - 1;
    }
    keep[rows[p]] = !hit[lo];
}
// ---- join conditions: from one pass bit per candidate pair to the rows the join type keeps ---------------------------------------------------
// One thread per pair of a slice whose first pair is a multiple of 32, so each warp owns whole words of the pass bits.  A pair whose build
// row is CB_NULL_ROW is no candidate (an outer join's slot of a probe row without a match): its bit is cleared, whatever the condition
// gave on its NULLs.  A passing pair sets its probe row's `passed` byte and, with build_hit, its build row's: plain stores, every writer
// stores 1.
__global__ void __launch_bounds__(256) k_join_cond_mark(u32* bits, const u32* probe_idx, const u32* build_idx, i64 k, u8* passed, u8* build_hit,
                                                        u64* candidates) {
    const i64 j = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if ((j & ~(i64)31) >= k) return; // whole warps only: the ballots below take every lane
    const bool in = j < k;
    const u32 b = in ? build_idx[j] : CB_NULL_ROW;
    const bool cand = b != CB_NULL_ROW;
    const bool pass = cand && ((bits[j >> 5] >> (j & 31)) & 1u);
    const u32 word = __ballot_sync(0xffffffffu, pass), n_cand = __popc(__ballot_sync(0xffffffffu, cand));
    if ((threadIdx.x & 31) == 0) {
        bits[j >> 5] = word;
        if (n_cand) atomicAdd((unsigned long long*)candidates, (unsigned long long)n_cand);
    }
    if (pass) {
        passed[probe_idx[j]] = 1;
        if (build_hit) build_hit[b] = 1;
    }
}
// pairs [o0, o0 + k) of a probe batch after its pass bits are final: keep[j] = the pair passed, or (outer) it is the first pair of a probe
// row that passed nothing, which becomes that row's NULL-extended row (build_idx[j] = CB_NULL_ROW)
__global__ void __launch_bounds__(256) k_join_cond_resolve(const u32* bits, i64 o0, const u32* probe_idx, u32* build_idx, i64 k, const u32* offs,
                                                           const u32* chunk_off, const u8* passed, int outer, u8* keep) {
    const i64 j = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    const i64 p = o0 + j;
    const bool pass = (bits[p >> 5] >> (p & 31)) & 1u;
    bool kept = pass;
    if (!pass && outer) {
        const u32 i = probe_idx[j];
        if (!passed[i] && p == (i64)offs[i] + chunk_off[i >> 12]) { kept = true; build_idx[j] = CB_NULL_ROW; }
    }
    keep[j] = kept;
}
// ---- nested-loop join: pair position p of a group is (probe row row0 + p / m, build row p % m) -------------------------------------------
// p / m without a 64-bit divide: inv = floor((2^64 - 1) / m) gives inv * m in (2^64 - 1 - m, 2^64), so mulhi(p, inv) is p / m or one less;
// one compare of the remainder corrects it.  Exact for every p < 2^64 and 0 < m < 2^32.
__device__ __forceinline__ u32 nlj_divmod(u64 p, u32 m, u64 inv, u32& r) {
    u64 q = __umul64hi(p, inv);
    u64 rem = p - q * m;
    if (rem >= m) { q++; rem -= m; }
    r = (u32)rem;
    return (u32)q;
}
__global__ void __launch_bounds__(256) k_nlj_pairs(i64 p0, i64 k, u32 row0, u32 m, u64 inv, u32* probe_idx, u32* build_idx) {
    const i64 j = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    u32 r;
    const u32 q = nlj_divmod((u64)(p0 + j), m, inv, r);
    probe_idx[j] = row0 + q;
    build_idx[j] = r;
}
// k_join_cond_resolve's arithmetic sibling, which also writes the pairs: keep[j] = pair p0 + j passed, or (outer) it is the first pair
// (build row 0) of a probe row that passed nothing, whose build row then becomes CB_NULL_ROW
__global__ void __launch_bounds__(256) k_nlj_cond_resolve(const u32* bits, i64 p0, i64 k, u32 row0, u32 m, u64 inv, const u8* passed, int outer,
                                                          u32* probe_idx, u32* build_idx, u8* keep) {
    const i64 j = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    const i64 p = p0 + j;
    u32 r;
    const u32 i = row0 + nlj_divmod((u64)p, m, inv, r);
    const bool pass = (bits[p >> 5] >> (p & 31)) & 1u;
    bool kept = pass;
    if (!pass && outer && r == 0 && !passed[i]) { kept = true; r = CB_NULL_ROW; }
    probe_idx[j] = i;
    build_idx[j] = r;
    keep[j] = kept;
}
void launch_nlj_pairs(i64 p0, i64 k, unsigned row0, unsigned m, unsigned long long inv, unsigned* probe_idx, unsigned* build_idx, cudaStream_t st) {
    if (k > 0) k_nlj_pairs<<<(unsigned)((k + 255) / 256), 256, 0, st>>>(p0, k, row0, m, (u64)inv, probe_idx, build_idx);
}
void launch_nlj_cond_resolve(const unsigned* bits, i64 p0, i64 k, unsigned row0, unsigned m, unsigned long long inv, const u8* passed, bool outer,
                             unsigned* probe_idx, unsigned* build_idx, u8* keep, cudaStream_t st) {
    if (k > 0)
        k_nlj_cond_resolve<<<(unsigned)((k + 255) / 256), 256, 0, st>>>(bits, p0, k, row0, m, (u64)inv, passed, outer, probe_idx, build_idx, keep);
}
__global__ void k_flags_not(const u8* flags, i64 n, u8* out) {
    const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = !flags[i];
}
void launch_join_cond_mark(unsigned* bits, const unsigned* probe_idx, const unsigned* build_idx, i64 k, u8* passed, u8* build_hit,
                           unsigned long long* candidates, cudaStream_t st) {
    if (k > 0) k_join_cond_mark<<<(unsigned)((k + 255) / 256), 256, 0, st>>>(bits, probe_idx, build_idx, k, passed, build_hit, (u64*)candidates);
}
void launch_join_cond_resolve(const unsigned* bits, i64 o0, const unsigned* probe_idx, unsigned* build_idx, i64 k, const unsigned* offs,
                              const unsigned* chunk_off, const u8* passed, bool outer, u8* keep, cudaStream_t st) {
    if (k > 0)
        k_join_cond_resolve<<<(unsigned)((k + 255) / 256), 256, 0, st>>>(bits, o0, probe_idx, build_idx, k, offs, chunk_off, passed, outer, keep);
}
void launch_flags_not(const u8* flags, i64 n, u8* out, cudaStream_t st) {
    if (n > 0) k_flags_not<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(flags, n, out);
}
void launch_join_heads(const u64* keys, int words, i64 m, u8* head, cudaStream_t st) {
    if (m > 0) k_join_heads<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(keys, words, m, head);
}
void launch_join_insert(const JoinTable& t, i64 n_runs, cudaStream_t st) {
    if (n_runs > 0) k_join_insert<<<(unsigned)((n_runs + 255) / 256), 256, 0, st>>>(t, n_runs);
}
void launch_join_probe(const JoinTable& t, const u64* keys, i64 n, int mode, u32* counts, u32* run_of, u64* total, u8* keep, u8* hit, cudaStream_t st) {
    if (n > 0) k_join_probe<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(t, keys, n, mode, counts, run_of, total, keep, hit);
}
void launch_join_emit(const JoinTable& t, const u32* run_of, const u32* offs, const u32* chunk_off, i64 n, i64 o0, i64 o1, bool outer, u32* probe_idx,
                      u32* build_idx, cudaStream_t st) {
    if (n > 0 && o1 > o0) k_join_emit<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(t, run_of, offs, chunk_off, n, o0, o1, outer, probe_idx, build_idx);
}
void launch_join_unmatched(const u32* run_start, i64 n_runs, const u32* rows, const u8* hit, i64 m, u8* keep, cudaStream_t st) {
    if (m > 0) k_join_unmatched<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(run_start, n_runs, rows, hit, m, keep);
}

template <int W> static cudaError_t sort_pass(const RadixScratch& s, i64 n, int digit, int from, bool first, cudaStream_t st) {
    const i64 nt = sort_tiles(n);
    k_sort_hist<W><<<(unsigned)nt, 256, 0, st>>>(s.keys[from], n, digit, nt, s.hist);
    launch_scan_u32(s.hist, 256 * nt, 4096, s.chunk_off, s.total, st);
    constexpr size_t smem = sort_scatter_smem<W>();
    const cudaError_t e = cudaFuncSetAttribute((const void*)k_sort_scatter<W>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); // > 48 KB
    if (e != cudaSuccess) return e;
    k_sort_scatter<W><<<(unsigned)nt, 256, smem, st>>>(s.keys[from], first ? nullptr : s.idx[from], n, digit, nt, s.hist, s.chunk_off,
                                                       s.keys[from ^ 1], s.idx[from ^ 1]);
    return cudaGetLastError();
}
cudaError_t launch_sort_passes(const RadixScratch& s, int words, i64 n, const int* digits, int n_digits, int* result, cudaStream_t st) {
    *result = 0;
    if (n <= 0) return cudaSuccess;
    if (n >= (i64)1 << 32 || words < 1 || words > SK_MAX_WORDS) return cudaErrorInvalidValue;
    if (n_digits == 0) k_sort_iota<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(s.idx[0], n);
    int from = 0;
    for (int p = 0; p < n_digits; p++, from ^= 1) {
        cudaError_t e;
        switch (words) {
        case 1: e = sort_pass<1>(s, n, digits[p], from, p == 0, st); break;
        case 2: e = sort_pass<2>(s, n, digits[p], from, p == 0, st); break;
        case 3: e = sort_pass<3>(s, n, digits[p], from, p == 0, st); break;
        default: e = sort_pass<4>(s, n, digits[p], from, p == 0, st); break;
        }
        if (e != cudaSuccess) return e;
    }
    *result = from;
    return cudaGetLastError();
}

// ---- device values -> Arrow layout (hand-off) ----------------------------------------------------------------------------------------
// The scan and the device tables keep some columns narrower or wider than Arrow does: INT32-backed int8 / int16 / decimal(p <= 9) 4 bytes
// per row, decimal(p <= 18) 8 bytes, booleans as bitmaps.  Decimals are sign-extended to Decimal128, ints narrowed (the scan wrote them
// from values of the narrow type), booleans spelled out one byte per row.
__global__ void k_to_arrow_layout(int conv, const u8* in, i64 n, u8* out) {
    const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    switch (conv) {
    case CB_SEXT32_TO_128: { const i64 v = ((const i32*)in)[i]; ((i64*)out)[2 * i] = v; ((i64*)out)[2 * i + 1] = v >> 63; break; }
    case CB_SEXT64_TO_128: { const i64 v = ((const i64*)in)[i]; ((i64*)out)[2 * i] = v; ((i64*)out)[2 * i + 1] = v >> 63; break; }
    case CB_NARROW32_TO_8: ((signed char*)out)[i] = (signed char)((const i32*)in)[i]; break;
    case CB_NARROW32_TO_16: ((short*)out)[i] = (short)((const i32*)in)[i]; break;
    case CB_BITS_TO_BYTES: out[i] = bit_at(in, i) ? 1 : 0; break;
    }
}
void launch_to_arrow_layout(int conv, const void* in, i64 n, void* out, cudaStream_t st) {
    if (n > 0) k_to_arrow_layout<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(conv, (const u8*)in, n, (u8*)out);
}

// ---- chunked exclusive scan (select pipelines: per-(tile, warp) kept-row counts -> output offsets) ------------------------
// one block per chunk of 4096 entries: 256 threads x 16 consecutive entries, warp shuffles + one shared-memory hop
__global__ void __launch_bounds__(256) k_scan_chunks(u32* data, long long m, u32* chunk_tot) {
    __shared__ u32 wsum[8];
    const long long base = (long long)blockIdx.x * 4096 + threadIdx.x * 16;
    u32 v[16], local = 0;
#pragma unroll
    for (int k = 0; k < 16; k++) { v[k] = base + k < m ? data[base + k] : 0u; local += v[k]; }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 incl = local;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { u32 t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    u32 wbase = 0, total = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) { if (w < warp) wbase += wsum[w]; total += wsum[w]; }
    u32 excl = wbase + incl - local;
#pragma unroll
    for (int k = 0; k < 16; k++) { if (base + k < m) data[base + k] = excl; excl += v[k]; }
    if (threadIdx.x == 0) chunk_tot[blockIdx.x] = total;
}
// single block: exclusive scan of the chunk totals (any count, running carry), grand total
__global__ void __launch_bounds__(1024) k_scan_totals(u32* chunk_tot, int n_chunks, long long* total_out) {
    __shared__ unsigned long long wsum[32];
    __shared__ unsigned long long carry_s;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (int base = 0; base < n_chunks; base += 1024) {
        const int i = base + threadIdx.x;
        const unsigned long long v = i < n_chunks ? chunk_tot[i] : 0ull;
        unsigned long long incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { unsigned long long t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        unsigned long long wbase = 0, total = 0;
        for (int w = 0; w < 32; w++) { if (w < warp) wbase += wsum[w]; total += wsum[w]; }
        const unsigned long long carry = carry_s;
        if (i < n_chunks) chunk_tot[i] = (u32)(carry + wbase + incl - v); // < 2^32: the caller bounds the row count
        __syncthreads();
        if (threadIdx.x == 0) carry_s = carry + total;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total_out = (long long)carry_s;
}
void launch_scan_u32(unsigned* data, long long m, int chunk, unsigned* chunk_off, long long* total, cudaStream_t st) {
    (void)chunk; // fixed at 4096 (CB_SCAN_CHUNK in device/cb_params.h)
    const int n_chunks = (int)((m + 4095) / 4096);
    if (n_chunks > 0) k_scan_chunks<<<n_chunks, 256, 0, st>>>(data, m, chunk_off);
    k_scan_totals<<<1, 1024, 0, st>>>(chunk_off, n_chunks, total);
}

} // namespace cb200
