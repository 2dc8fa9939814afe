// aot_kernels.cu -- ahead-of-time sm_90a kernels that do not depend on the plan: Arrow buffer
// normalisation (bitmap append at arbitrary bit offsets, byte->bitmap packing), dictionary code
// remapping and the device-side string dictionary builder used to turn Utf8 group keys into dense
// codes.  (Plan-dependent kernels are JIT-specialised: device/cb_kernels.cuh.)
#include "aot_kernels.h"
#include "device/cb_math.h"

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

__global__ void k_partition_ids(HashKeyCols kc, i64 n, u32 n_parts, u32* hashes, u32* pids) {
    i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    u32 h = 42u; // spark seed (multi_partition.rs:298)
    for (int c = 0; c < kc.n; c++) {
        const HashKeyCol& k = kc.col[c];
        if (k.validity && !bit_at(k.validity, i)) continue; // NULL leaves the running hash unchanged (utils.rs:38-42)
        const u8* d = (const u8*)k.data;
        switch (k.kind) {
        case HK_BOOL: h = mm3_i32(bit_at(d, i) ? 1 : 0, h); break;
        case HK_I8: h = mm3_i32((i32)((const signed char*)d)[i], h); break;
        case HK_I16: h = mm3_i32((i32)((const short*)d)[i], h); break;
        case HK_I32: h = mm3_i32(((const i32*)d)[i], h); break;
        case HK_I64: h = mm3_i64(((const i64*)d)[i], h); break;
        case HK_F32: { float f = ((const float*)d)[i]; if (f == 0.0f) f = 0.0f; h = mm3_i32((i32)__float_as_uint(f == 0.0f ? 0.0f : f), h); break; }
        case HK_F64: { double f = ((const double*)d)[i]; h = mm3_i64(f == 0.0 ? 0ll : __double_as_longlong(f), h); break; }
        case HK_DEC_SMALL_128: h = mm3_i64((i64)((const i128*)d)[i].lo, h); break; // d(p<=18): hashed as i64 (utils.rs:159-196)
        case HK_DEC_LARGE_128: h = mm3_i128(((const i128*)d)[i], h); break;        // d(p>18): 16 LE bytes (utils.rs:199-226)
        case HK_DEC_LARGE_64: h = mm3_i128(i128_from_i64(((const i64*)d)[i]), h); break;
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
    if (hashes) hashes[i] = h;
    pids[i] = pmod_u32(h, n_parts);
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
template <typename T> __global__ void k_gather_rows(const T* in, const i64* row_idx, i64 n, T* out) {
    i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[row_idx[i]];
}
__global__ void k_gather_bits(const u8* in_bits, const i64* row_idx, i64 n, u8* out_bytes) {
    i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out_bytes[i] = bit_at(in_bits, row_idx[i]) ? 1 : 0;
}

i64 partition_chunks(i64 n) { const i64 nb = (n + 1023) / 1024; return (nb + PID_CHUNK - 1) / PID_CHUNK; }
void launch_partition(const HashKeyCols& kc, i64 n, u32 n_parts, u32* hashes, u32* pids, i32* block_hist, i64* block_base, i64* chunk_tmp, i64* starts,
                      i64* row_idx, cudaStream_t st) {
    if (n <= 0) return;
    i64 nb = (n + 1023) / 1024;
    const i64 nc = partition_chunks(n);
    k_partition_ids<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(kc, n, n_parts, hashes, pids);
    k_pid_block_hist<<<(unsigned)nb, 256, n_parts * sizeof(i32), st>>>(pids, n, n_parts, block_hist);
    k_pid_chunk_totals<<<(unsigned)nc, 256, 0, st>>>(block_hist, nb, n_parts, chunk_tmp);
    k_pid_chunk_scan<<<1, 256, n_parts * sizeof(i64), st>>>(chunk_tmp, nc, n_parts, starts);
    k_pid_block_bases<<<(unsigned)nc, 256, 0, st>>>(block_hist, nb, n_parts, chunk_tmp, block_base);
    k_pid_place<<<(unsigned)nb, 64, n_parts * sizeof(i64), st>>>(pids, n, n_parts, block_base, row_idx);
}
void launch_gather(const void* in, int width, const i64* row_idx, i64 n, void* out, cudaStream_t st) {
    if (n <= 0) return;
    unsigned blocks = (unsigned)((n + 255) / 256);
    if (width == 16) k_gather_rows<ulonglong2><<<blocks, 256, 0, st>>>((const ulonglong2*)in, row_idx, n, (ulonglong2*)out);
    else if (width == 8) k_gather_rows<u64><<<blocks, 256, 0, st>>>((const u64*)in, row_idx, n, (u64*)out);
    else if (width == 4) k_gather_rows<u32><<<blocks, 256, 0, st>>>((const u32*)in, row_idx, n, (u32*)out);
    else if (width == 2) k_gather_rows<u16><<<blocks, 256, 0, st>>>((const u16*)in, row_idx, n, (u16*)out);
    else k_gather_rows<u8><<<blocks, 256, 0, st>>>((const u8*)in, row_idx, n, (u8*)out);
}
void launch_gather_bits(const void* in_bits, const i64* row_idx, i64 n, void* out_bytes, cudaStream_t st) {
    if (n > 0) k_gather_bits<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const u8*)in_bits, row_idx, n, (u8*)out_bytes);
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
