// parquet_kernels.cu -- Parquet page decode on sm_90a.
//
// Encodings per the Apache Parquet specification (Encodings.md): PLAIN and BYTE_STREAM_SPLIT for fixed-width physical
// types, DELTA_BINARY_PACKED for INT32 / INT64, RLE/bit-packed hybrid for dictionary indices (RLE_DICTIONARY: 1 byte bit
// width, then runs) and for definition levels.  The reference reaches the third-party `parquet` crate for this
// (native/core/src/parquet/parquet_exec.rs:139-141); its source is not under the reference tree, so the
// decoders follow the format specification and are checked against pyarrow-written files.
#include "parquet_kernels.h"
#include "device/cb_math.h"
#include "device/cb_delta.h"
#include "device/cb_snappy.h"
#include <algorithm>

namespace cb200 {
using namespace cb;

// page bytes start at arbitrary offsets: assemble unaligned little-endian words from aligned loads
__device__ __forceinline__ u64 load_u64_unaligned(const u8* p) {
    size_t a = (size_t)p;
    const u64* q = (const u64*)(a & ~(size_t)7);
    int sh = (int)(a & 7) * 8;
    u64 lo = q[0];
    if (sh == 0) return lo;
    u64 hi = q[1];
    return (lo >> sh) | (hi << (64 - sh));
}
__device__ __forceinline__ u32 load_u32_unaligned(const u8* p) {
    size_t a = (size_t)p;
    const u32* q = (const u32*)(a & ~(size_t)3);
    int sh = (int)(a & 3) * 8;
    u32 lo = q[0];
    if (sh == 0) return lo;
    u32 hi = q[1];
    return (lo >> sh) | (hi << (32 - sh));
}

__global__ void k_pq_copy(uint4* dst, const uint4* src, size_t n16) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) dst[i] = src[i];
}
void launch_pq_copy(void* dst, const void* src, size_t bytes, cudaStream_t st) {
    const size_t n16 = bytes / 16;
    if (n16 == 0) return;
    const unsigned blocks = (unsigned)std::min<size_t>((n16 + 255) / 256, 296);
    k_pq_copy<<<blocks, 256, 0, st>>>((uint4*)dst, (const uint4*)src, n16);
}

// ---- Snappy --------------------------------------------------------------------------------------------------
// One warp per page.  Elements are inherently sequential (each tag's position depends on the previous one), so
// lane 0 parses the tag and broadcasts it in two registers; the bytes are moved by the whole warp.  What makes a
// serial decoder slow on a GPU is the latency of every dependent access, so both ends are kept in shared memory:
//   * a 512-byte window of the compressed input, refilled with one coalesced 16-byte load per lane;
//   * a 16 KB ring of the most recent output: a back-reference within it (almost all of them -- the reference
//     compressor never looks back more than 64 KB, typical matches are far closer) is served without the
//     store -> L2 -> load round trip.  Older references fall back to L2 loads of the page's own output.
// A copy whose distance is shorter than its length repeats a pattern that lies entirely before the write position,
// so every lane computes its source independently; element semantics are those of device/cb_snappy.h (host-tested).
constexpr int SN_RING = 16384, SN_WIN = 512, SN_WARPS = 4;
// A lone warp issues one dependent instruction every ~4.5 cycles, so the cost of a page is (elements x instructions
// per element): positions are 32-bit offsets (a page is < 2 GiB), the common shapes -- a literal or a copy of at
// most 32 bytes -- take one predicated step without a loop, and validation is a handful of compares.
__global__ void __launch_bounds__(SN_WARPS * 32) k_pq_snappy(PqPage* pages, int n_pages, int* err, int only_flagged) {
    extern __shared__ __align__(16) u8 sn_smem[];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int warp = blockIdx.x * SN_WARPS + wib;
    if (warp >= n_pages) return; // warps are independent: no block-wide barrier below
    const PqPage pg = pages[warp];
    if (!pg.comp) return;
    if (only_flagged && (pg.flags & (PQ_PAGE_SN_SERIAL | PQ_PAGE_SN_BAD)) != PQ_PAGE_SN_SERIAL) return; // the segmented decoder did (or rejected) this page
    u8* ring = sn_smem + wib * (SN_RING + SN_WIN);
    u8* win = ring + SN_RING;
    const u8* in = pg.comp;
    const u32 n = (u32)pg.comp_bytes;
    u8* out = pg.body;
    u64 ulen64 = 0;
    long long pre = 0;
    if (lane == 0) pre = snappy_preamble(in, n, ulen64);
    pre = __shfl_sync(0xffffffffu, pre, 0);
    ulen64 = __shfl_sync(0xffffffffu, ulen64, 0);
    if (pre < 0 || ulen64 != (u64)pg.body_bytes) { if (lane == 0) atomicOr(err, PQ_ERR_SNAPPY); return; }
    const u32 ulen = (u32)ulen64;
    // the window holds input bytes [wbase, wbase + SN_WIN) where wbase is `in`-relative and 16-byte aligned in memory
    const u32 misalign = (u32)((size_t)in & 15);
    u32 pos = (u32)pre, o = 0;
    int wbase = -SN_WIN - 16; // nothing loaded yet
    bool bad = false;
    while (pos < n) {
        u32 wp = pos - (u32)wbase; // offset of the element inside the window
        if (wp + 5 > (u32)SN_WIN) { // an element header is at most 5 bytes
            wbase = (int)((pos + misalign) & ~15u) - (int)misalign;
            const int lo = wbase + lane * 16;
            uint4 v = make_uint4(0u, 0u, 0u, 0u);
            if (lo < (int)n) v = *(const uint4*)(in + lo); // reads < 16 bytes outside the page: inside the padded chunk buffer
            __syncwarp();
            ((uint4*)win)[lane] = v;
            __syncwarp();
            wp = pos - (u32)wbase;
        }
        u32 w0 = 0xffffffffu, w1 = 0;
        if (lane == 0) {
            const u8* p = win + wp;
            const u32 tag = p[0], t = tag & 3u;
            u32 len, src = 0, hdr;
            if (t == 0) {
                hdr = 1; len = tag >> 2;
                if (len >= 60) {
                    const u32 extra = len - 59;
                    const u32 raw = (u32)p[1] | ((u32)p[2] << 8) | ((u32)p[3] << 16) | ((u32)p[4] << 24);
                    len = extra == 4 ? raw : raw & ((1u << (8 * extra)) - 1u);
                    hdr += extra;
                }
                len += 1;
                if (len < (1u << 27) && len <= ulen - o && hdr + len <= n - pos) w0 = len | (hdr << 27);
            } else {
                if (t == 1) { hdr = 2; len = ((tag >> 2) & 7u) + 4; src = ((tag >> 5) << 8) | p[1]; }
                else if (t == 2) { hdr = 3; len = (tag >> 2) + 1; src = (u32)p[1] | ((u32)p[2] << 8); }
                else { hdr = 5; len = (tag >> 2) + 1; src = (u32)p[1] | ((u32)p[2] << 8) | ((u32)p[3] << 16) | ((u32)p[4] << 24); }
                if (src - 1u < o && len <= ulen - o && hdr <= n - pos) { w0 = len | (hdr << 27) | (1u << 30); w1 = src; }
            }
        }
        w0 = __shfl_sync(0xffffffffu, w0, 0);
        if (w0 == 0xffffffffu) { bad = true; break; }
        const u32 len = w0 & ((1u << 27) - 1), hdr = (w0 >> 27) & 7u;
        if (!(w0 & (1u << 30))) {
            if (wp + hdr + len <= (u32)SN_WIN) { // short literal: already in the window
                for (u32 i = lane; i < len; i += 32) {
                    const u8 b = win[wp + hdr + i];
                    out[o + i] = b;
                    ring[(o + i) & (SN_RING - 1)] = b;
                }
            } else {
                const u8* s = in + pos + hdr;
                for (u32 i = lane; i < len; i += 32) {
                    const u8 b = s[i];
                    out[o + i] = b;
                    ring[(o + i) & (SN_RING - 1)] = b;
                }
            }
            pos += hdr + len;
        } else {
            const u32 d = __shfl_sync(0xffffffffu, w1, 0);
            const bool near = d + 64 <= (u32)SN_RING; // the source still sits in the ring and this copy (<= 64 bytes) does not overwrite it
            if (d >= len) { // no overlap with the bytes being written
                for (u32 i = lane; i < len; i += 32) {
                    const u32 sp = o - d + i;
                    const u8 b = near ? ring[sp & (SN_RING - 1)] : __ldcg(out + sp);
                    out[o + i] = b;
                    ring[(o + i) & (SN_RING - 1)] = b;
                }
            } else { // pattern of period d, entirely before the write position
                for (u32 i = lane; i < len; i += 32) {
                    const u32 sp = o - d + i % d;
                    const u8 b = near ? ring[sp & (SN_RING - 1)] : __ldcg(out + sp);
                    out[o + i] = b;
                    ring[(o + i) & (SN_RING - 1)] = b;
                }
            }
            pos += hdr;
        }
        __syncwarp(); // the next element may read what this one wrote
        o += len;
    }
    if ((bad || o != ulen) && lane == 0) atomicOr(err, PQ_ERR_SNAPPY);
}
// ---- Snappy, segmented ------------------------------------------------------------------------------------------------------------
// One warp per page leaves most of the GPU idle (a batch has a few hundred pages) and a page of small elements -- PLAIN INT64
// decimals compress to a literal + copy pair per value -- took ~80 ms.  The stock compressor works on independent 64 KB fragments
// of the input: no element straddles, and no back-reference crosses, a 64 KB boundary of the OUTPUT.  So:
//   k_pq_snappy_index  (warp per page)     walks the element chain WITHOUT moving bytes -- every lane parses the element that would
//                      start at its byte of a 32-byte window, the chain is followed through the lanes' answers with one shuffle pair
//                      per element -- and records the input position of every 64 KB output boundary (checkpoint table);
//   k_pq_snappy_seg    (warp per segment)  decodes [checkpoint s, checkpoint s + 1) exactly like the serial kernel: 16 x more warps
//                      per 1 MB page;
//   k_pq_snappy        (only_flagged)      pages that do not have that shape (an element across a boundary, a reference into an
//                      earlier segment: legal Snappy, never produced by the stock compressor) are redone serially.
constexpr int SX_WARPS = 8, SX_RING = 8192;

// element starting at w[0] (w points into a window with >= 5 readable bytes): bytes to the next element / bytes produced; adv == 0: malformed
__device__ __forceinline__ void sn_elem_len(const u8* w, u32& adv, u32& out) {
    const u32 tag = w[0], t = tag & 3u;
    if (t == 0) {
        u32 len = tag >> 2, hdr = 1;
        if (len >= 60) {
            const u32 extra = len - 59;
            const u32 raw = (u32)w[1] | ((u32)w[2] << 8) | ((u32)w[3] << 16) | ((u32)w[4] << 24);
            len = extra == 4 ? raw : raw & ((1u << (8 * extra)) - 1u);
            hdr += extra;
        }
        if (len >= (1u << 30)) { adv = 0; out = 0; return; }
        out = len + 1;
        adv = hdr + out;
    } else if (t == 1) { adv = 2; out = ((tag >> 2) & 7u) + 4; }
    else { adv = t == 2 ? 3 : 5; out = (tag >> 2) + 1; }
}

// Index pass.  A warp looks at SXI_W input bytes at a time.  Every byte position is treated as if an element started there: nxt =
// where the following element would start, sum = output bytes it produces.  Lane l owns the 32 positions of block l and collapses
// the chains inside it with one backward sweep (the entry of a later position is final when an earlier one needs it), so every
// position knows where its chain leaves its block; the TRUE chain -- the one from position 0 -- then hops from block to block in
// at most 32 dependent shared-memory lookups.  All candidate chains are computed although one is real: that is what makes the
// sweep parallel.  (Following the chain element by element with a shuffle pair each took 25 ms for a page of 4-byte elements,
// pointer jumping over all 1024 positions 10 ms.)  Only a window that contains a 64 KB output boundary is walked element by element.
constexpr int SXI_WARPS = 8, SXI_W = 512; // 4.9 KB of shared memory per warp: the sweep is a chain of dependent shared-memory accesses (ncu: 0.09 IPC per
                                             // scheduler at 12 warps per SM with 1 KB windows), so what it needs is resident warps
constexpr u32 SXI_INVALID = 0xffffffffu;

__global__ void __launch_bounds__(SXI_WARPS * 32) k_pq_snappy_index(PqPage* pages, int n_pages, u32* ckpt, int* err) {
    extern __shared__ __align__(16) u8 sxi_smem[];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int warp = blockIdx.x * SXI_WARPS + wib;
    if (warp >= n_pages) return;
    const PqPage pg = pages[warp];
    if (!pg.comp) return;
    u8* base = sxi_smem + (size_t)wib * (SXI_W + 32 + (SXI_W + 32) * 8);
    u8* win = base;                                              // SXI_W + 32 input bytes
    u32* s_nxt = reinterpret_cast<u32*>(base + SXI_W + 32);      // [SXI_W + 32] (skewed)
    u32* s_sum = s_nxt + SXI_W + 32;                             // [SXI_W + 32]
    const u8* in = pg.comp;
    const u32 n = (u32)pg.comp_bytes;
    u64 ulen64 = 0;
    long long pre = 0;
    if (lane == 0) pre = snappy_preamble(in, n, ulen64);
    pre = __shfl_sync(0xffffffffu, pre, 0);
    ulen64 = __shfl_sync(0xffffffffu, ulen64, 0);
    if (pre < 0 || ulen64 != (u64)pg.body_bytes) { if (lane == 0) { atomicOr(err, PQ_ERR_SNAPPY); atomicOr(&pages[warp].flags, PQ_PAGE_SN_BAD); } return; }
    u32* ck = ckpt + pg.seg_base;
    const u32 misalign = (u32)((size_t)in & 15);
    const u32 body = (u32)pg.body_bytes;
    u32 pos = (u32)pre, o = 0, bnd = 0;
    int k = 0;           // next checkpoint to record (output offset bnd = k * PQ_SNAPPY_SEG)
    int status = 0;      // 1: irregular (serial decoder), 2: malformed
    while (pos < n && status == 0) {
        if (o == bnd) { if (lane == 0 && k < pg.n_segs) ck[k] = pos; k++; bnd += (u32)PQ_SNAPPY_SEG; }
        else if (o > bnd) { status = 1; break; }                 // an element straddles a 64 KB output boundary
        // ---- window: input bytes [pos, pos + SXI_W + 4), 16-byte aligned loads ----
        const int wbase = (int)((pos + misalign) & ~15u) - (int)misalign; // <= pos, pos - wbase < 16
        __syncwarp();
        for (int j = lane; j < (SXI_W + 32) / 16; j += 32) {
            const int lo = wbase + j * 16;
            uint4 v = make_uint4(0u, 0u, 0u, 0u);
            if (lo < (int)n) v = *(const uint4*)(in + lo);       // < 16 bytes outside the page: inside the padded chunk buffer
            ((uint4*)win)[j] = v;
        }
        __syncwarp();
        const u32 woff = pos - (u32)wbase;                       // window byte of position 0
        const u32 L = min((u32)SXI_W - 16u, n - pos);            // positions examined (the loads above cover L + 4 bytes from any woff < 16)
        // ---- lane l owns the 32 positions [32 l, 32 l + 32): one backward sweep collapses the chains inside its block, so that
        //      s_nxt / s_sum of a position say where its chain LEAVES the block and what it produced until then (a later position's
        //      entry is final when an earlier one needs it).  Entries are skewed by one word per block: a warp-wide access to the same
        //      k of every block would otherwise hit one bank 32 times.
        {
            constexpr u32 BLK = SXI_W / 32;
            const u32 b0 = (u32)lane * BLK, bend = b0 + BLK;
#pragma unroll 4
            for (int kk = (int)BLK - 1; kk >= 0; kk--) {
                const u32 i = b0 + (u32)kk;
                u32 adv = 0, out = 0;
                if (i < L) sn_elem_len(win + woff + i, adv, out);
                const bool ok = i < L && adv != 0 && adv <= n - (pos + i);
                u32 nxt = SXI_INVALID, sum = 0;
                if (ok) {
                    const u32 t = i + adv;
                    if (t < bend && t < L) { const u32 ti = t + t / BLK; nxt = s_nxt[ti]; sum = out + s_sum[ti]; }
                    else { nxt = t; sum = out; }
                }
                const u32 ii = i + i / BLK;
                s_nxt[ii] = nxt;
                s_sum[ii] = sum;
            }
        }
        __syncwarp();
        // ---- the true chain starts at position 0 and hops from block to block: at most 32 dependent lookups ----
        u32 E = 0, S = 0;
        while (E < L) {
            const u32 ei = E + E / (SXI_W / 32);
            const u32 nx = s_nxt[ei];
            S += s_sum[ei];
            if (nx == SXI_INVALID || S > body) { E = SXI_INVALID; break; }
            E = nx;
        }
        if (E == SXI_INVALID || E < L || S > body - o) { status = 2; break; } // (E < L cannot happen: the walk only stops past L)
        if (o + S <= bnd) { o += S; pos += E; continue; }         // no boundary strictly inside this window's chain (landing on it: recorded above, next trip)
        // ---- a 64 KB boundary lies inside: walk element by element (32 candidate positions at a time) until it is reached ----
        while (pos < n && o < bnd && status == 0) {
            u32 adv, out;
            const u32 wp = pos - (u32)wbase;
            if (wp + 36 > (u32)SXI_W + 32u) break;               // left the window: reload (outer loop)
            sn_elem_len(win + wp + lane, adv, out);
            if (pos + lane >= n) { adv = 0; out = 0; }
            u32 cur = 0;
            while (cur < 32u && pos + cur < n && o < bnd) {
                const u32 a = __shfl_sync(0xffffffffu, adv, cur), ou = __shfl_sync(0xffffffffu, out, cur);
                if (a == 0 || a > n - (pos + cur) || ou > body - o) { status = 2; break; }
                o += ou;
                cur += a;
            }
            pos += cur;
        }
    }
    if (status == 0 && (o != body || k != pg.n_segs)) status = (o == body && pos == n && k < pg.n_segs) ? 1 : 2;
    if (lane == 0) {
        if (status == 2) { atomicOr(err, PQ_ERR_SNAPPY); atomicOr(&pages[warp].flags, PQ_PAGE_SN_BAD); }
        else if (status == 1) atomicOr(&pages[warp].flags, PQ_PAGE_SN_SERIAL);
    }
}

__global__ void __launch_bounds__(SX_WARPS * 32) k_pq_snappy_seg(PqPage* pages, int n_pages, const u32* ckpt, int n_segs_total, int* err) {
    extern __shared__ __align__(16) u8 sn_smem[];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int seg_global = blockIdx.x * SX_WARPS + wib;
    if (seg_global >= n_segs_total) return;
    // which page: the last one whose seg_base <= seg_global (pages without segments repeat their successor's base)
    int lo = 0, hi = n_pages - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (pages[mid].seg_base <= seg_global) lo = mid; else hi = mid - 1; }
    const PqPage pg = pages[lo];
    const int sidx = seg_global - pg.seg_base;
    if (!pg.comp || sidx >= pg.n_segs || (pg.flags & (PQ_PAGE_SN_SERIAL | PQ_PAGE_SN_BAD))) return;
    u8* ring = sn_smem + wib * (SX_RING + SN_WIN);
    u8* win = ring + SX_RING;
    const u8* in = pg.comp;
    const u32 n = sidx + 1 < pg.n_segs ? ckpt[pg.seg_base + sidx + 1] : (u32)pg.comp_bytes; // end of this segment's input
    const u32 o0 = (u32)sidx * (u32)PQ_SNAPPY_SEG;
    const u32 oend = min((u32)pg.body_bytes, o0 + (u32)PQ_SNAPPY_SEG);
    u8* out = pg.body;
    const u32 misalign = (u32)((size_t)in & 15);
    u32 pos = ckpt[pg.seg_base + sidx], o = o0;
    int wbase = -SN_WIN - 16;
    int status = 0;
    // 32 candidate elements are parsed at once (lane l: the element that would start at input byte pos + l); the true chain is then
    // followed through the lanes' answers -- two shuffles per element instead of ~60 dependent instructions of one lane parsing it
    while (pos < n && status == 0) {
        u32 wp = pos - (u32)wbase;
        if (wp + 36 > (u32)SN_WIN) { // the window must hold the 32 candidate tags and 4 bytes after each
            wbase = (int)((pos + misalign) & ~15u) - (int)misalign;
            const int l0 = wbase + lane * 16;
            uint4 v = make_uint4(0u, 0u, 0u, 0u);
            if (l0 < (int)pg.comp_bytes) v = *(const uint4*)(in + l0);
            __syncwarp();
            ((uint4*)win)[lane] = v;
            __syncwarp();
            wp = pos - (u32)wbase;
        }
        u32 w0 = 0xffffffffu, w1 = 0; // this lane's candidate: len | hdr << 27 | copy << 30, copy distance
        if (pos + lane < n) {
            const u8* p = win + wp + lane;
            const u32 tag = p[0], t = tag & 3u, room = n - (pos + lane);
            u32 len, hdr;
            if (t == 0) {
                hdr = 1; len = tag >> 2;
                if (len >= 60) {
                    const u32 extra = len - 59;
                    const u32 raw = (u32)p[1] | ((u32)p[2] << 8) | ((u32)p[3] << 16) | ((u32)p[4] << 24);
                    len = extra == 4 ? raw : raw & ((1u << (8 * extra)) - 1u);
                    hdr += extra;
                }
                len += 1;
                if (len < (1u << 27) && hdr <= room && len <= room - hdr) w0 = len | (hdr << 27);
            } else {
                if (t == 1) { hdr = 2; len = ((tag >> 2) & 7u) + 4; w1 = ((tag >> 5) << 8) | p[1]; }
                else if (t == 2) { hdr = 3; len = (tag >> 2) + 1; w1 = (u32)p[1] | ((u32)p[2] << 8); }
                else { hdr = 5; len = (tag >> 2) + 1; w1 = (u32)p[1] | ((u32)p[2] << 8) | ((u32)p[3] << 16) | ((u32)p[4] << 24); }
                if (hdr <= room) w0 = len | (hdr << 27) | (1u << 30);
            }
        }
        u32 cur = 0;
        while (cur < 32u && pos + cur < n) {
            const u32 e0 = __shfl_sync(0xffffffffu, w0, cur), d = __shfl_sync(0xffffffffu, w1, cur);
            if (e0 == 0xffffffffu) { status = 2; break; }
            const u32 len = e0 & ((1u << 27) - 1), hdr = (e0 >> 27) & 7u;
            if (len > oend - o) { status = 2; break; }
            if (!(e0 & (1u << 30))) {
                const u32 lp = wp + cur + hdr; // literal bytes: in the window when short, else straight from the page
                if (len <= 32u && lp + len <= (u32)SN_WIN) { // the common shape: one predicated step, no loop
                    if (lane < len) {
                        const u8 b = win[lp + lane];
                        out[o + lane] = b;
                        ring[(o + lane) & (SX_RING - 1)] = b;
                    }
                } else if (lp + len <= (u32)SN_WIN) {
                    for (u32 i = lane; i < len; i += 32) {
                        const u8 b = win[lp + i];
                        out[o + i] = b;
                        ring[(o + i) & (SX_RING - 1)] = b;
                    }
                } else {
                    const u8* s = in + pos + cur + hdr;
                    for (u32 i = lane; i < len; i += 32) {
                        const u8 b = s[i];
                        out[o + i] = b;
                        ring[(o + i) & (SX_RING - 1)] = b;
                    }
                }
                cur += hdr + len;
            } else {
                if (d - 1u >= o - o0) { status = d - 1u < o ? 1 : 2; break; } // reaches into an earlier segment (legal, not ours to race on) / before the page
                const bool near = d + 64 <= (u32)SX_RING;
                if (len <= 32u && near) { // the common shape: a short copy out of the ring
                    if (lane < len) {
                        const u8 b = ring[(o - d + (d >= len ? lane : lane % d)) & (SX_RING - 1)];
                        out[o + lane] = b;
                        ring[(o + lane) & (SX_RING - 1)] = b;
                    }
                } else if (d >= len) {
                    for (u32 i = lane; i < len; i += 32) {
                        const u32 sp = o - d + i;
                        const u8 b = near ? ring[sp & (SX_RING - 1)] : __ldcg(out + sp);
                        out[o + i] = b;
                        ring[(o + i) & (SX_RING - 1)] = b;
                    }
                } else {
                    for (u32 i = lane; i < len; i += 32) {
                        const u32 sp = o - d + i % d;
                        const u8 b = near ? ring[sp & (SX_RING - 1)] : __ldcg(out + sp);
                        out[o + i] = b;
                        ring[(o + i) & (SX_RING - 1)] = b;
                    }
                }
                cur += hdr;
            }
            __syncwarp(); // the next element may read what this one wrote
            o += len;
        }
        pos += cur;
    }
    if (status == 0 && o != oend) status = 2;
    if (lane == 0) {
        if (status == 2) { atomicOr(err, PQ_ERR_SNAPPY); atomicOr(&pages[lo].flags, PQ_PAGE_SN_BAD); }
        else if (status == 1) atomicOr(&pages[lo].flags, PQ_PAGE_SN_SERIAL);
    }
}

void launch_pq_snappy_segmented(PqPage* pages, int n_pages, unsigned* ckpt, int n_segs_total, int* err, cudaStream_t st) {
    if (n_pages <= 0) return;
    const int smem_i = SXI_WARPS * (SXI_W + 32 + (SXI_W + 32) * 8);
    cudaFuncSetAttribute(k_pq_snappy_index, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_i);
    k_pq_snappy_index<<<(n_pages + SXI_WARPS - 1) / SXI_WARPS, SXI_WARPS * 32, smem_i, st>>>(pages, n_pages, ckpt, err);
    if (n_segs_total > 0) {
        const int smem = SX_WARPS * (SX_RING + SN_WIN);
        cudaFuncSetAttribute(k_pq_snappy_seg, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        k_pq_snappy_seg<<<(n_segs_total + SX_WARPS - 1) / SX_WARPS, SX_WARPS * 32, smem, st>>>(pages, n_pages, ckpt, n_segs_total, err);
    }
    const int smem1 = SN_WARPS * (SN_RING + SN_WIN);
    cudaFuncSetAttribute(k_pq_snappy, cudaFuncAttributeMaxDynamicSharedMemorySize, smem1);
    k_pq_snappy<<<(n_pages + SN_WARPS - 1) / SN_WARPS, SN_WARPS * 32, smem1, st>>>(pages, n_pages, err, 1); // irregular pages only
}

// ---- locate levels / values inside the page body ------------------------------------------------------------------------
__global__ void k_pq_resolve(PqPage* pages, int n_pages) {
    int pi = blockIdx.x * blockDim.x + threadIdx.x;
    if (pi >= n_pages) return;
    PqPage pg = pages[pi];
    const u8* v = pg.body;
    int left = pg.body_bytes;
    if (pg.flags & PQ_PAGE_V1_LEVELS) {
        u32 dl = left >= 4 ? ((u32)v[0] | ((u32)v[1] << 8) | ((u32)v[2] << 16) | ((u32)v[3] << 24)) : 0u;
        if (left < 4 || dl > (u32)(left - 4)) dl = 0; // malformed: the level decoders will report the row-count mismatch
        pages[pi].def_ptr = v + 4;
        pages[pi].def_bytes = (int)dl;
        v += 4 + dl;
        left -= 4 + (int)dl;
    }
    pages[pi].values = v;
    pages[pi].values_bytes = left;
    pages[pi].nonnull = pg.num_values;
}
void launch_pq_resolve(PqPage* pages, int n_pages, cudaStream_t st) {
    if (n_pages > 0) k_pq_resolve<<<(n_pages + 127) / 128, 128, 0, st>>>(pages, n_pages);
}

// ---- PLAIN / BYTE_STREAM_SPLIT ---------------------------------------------------------------------------------
// One conversion for every layout: byte(k) returns byte k of the value being converted (little-endian for the numeric types,
// big-endian two's complement of flba_len bytes for FIXED_LEN_BYTE_ARRAY decimals).
template <int CONV, typename B> __device__ __forceinline__ void pq_store(u8* out, long long row, int flba_len, B byte) {
    if (CONV == PQ_COPY32 || CONV == PQ_I32_TO_I64) {
        const u32 v = (u32)byte(0) | ((u32)byte(1) << 8) | ((u32)byte(2) << 16) | ((u32)byte(3) << 24);
        if (CONV == PQ_COPY32) ((u32*)out)[row] = v;
        else ((i64*)out)[row] = (i64)(i32)v;
    } else if (CONV == PQ_COPY64) {
        u64 v = 0;
        for (int k = 0; k < 8; k++) v |= (u64)byte(k) << (8 * k);
        ((u64*)out)[row] = v;
    } else {
        u64 hi = (byte(0) & 0x80) ? ~0ull : 0ull, lo = hi;
        for (int k = 0; k < flba_len; k++) {
            hi = (hi << 8) | (lo >> 56);
            lo = (lo << 8) | byte(k);
        }
        if (CONV == PQ_FLBA_TO_I64) ((i64*)out)[row] = (i64)lo;
        else ((i128*)out)[row] = mk128(lo, (i64)hi);
    }
}

// PLAIN: value i at values[i * w, i * w + w).  BYTE_STREAM_SPLIT: byte k of value i at values[k * N + i], N = the page's non-null values.
template <int CONV> __global__ void k_pq_plain(const PqPage* pages, int flba_len, u8* out, int* err) {
    const PqPage pg = pages[blockIdx.y];
    const bool bss = pg.encoding == PQ_ENC_BSS;
    if (pg.encoding != PQ_ENC_PLAIN && !bss) return; // dictionary / delta pages have their own kernels
    const u8* src = pg.values;
    const int w = CONV == PQ_COPY32 || CONV == PQ_I32_TO_I64 ? 4 : CONV == PQ_COPY64 ? 8 : flba_len;
    const long long n = pg.nonnull;
    int count;
    if (bss) { // the streams' length follows from N: any other size is malformed and is not read at all
        if (n * w != (long long)pg.values_bytes) { if (blockIdx.x == 0 && threadIdx.x == 0) atomicOr(err, PQ_ERR_BSS); return; }
        count = (int)n;
    } else {
        const int have = w > 0 ? pg.values_bytes / w : 0;   // never read beyond the page, whatever the header claims
        count = pg.nonnull < have ? pg.nonnull : have;
        if (pg.nonnull > have && blockIdx.x == 0 && threadIdx.x == 0) atomicOr(err, PQ_ERR_TRUNCATED); // short page: the rows it cannot fill must not pass silently
    }
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
        long long row = pg.dst_row + i;
        if (bss) pq_store<CONV>(out, row, flba_len, [&](int k) -> u8 { return src[(size_t)k * (size_t)n + (size_t)i]; });
        else if (CONV == PQ_COPY32) ((u32*)out)[row] = load_u32_unaligned(src + (size_t)i * 4);
        else if (CONV == PQ_COPY64) ((u64*)out)[row] = load_u64_unaligned(src + (size_t)i * 8);
        else if (CONV == PQ_I32_TO_I64) ((i64*)out)[row] = (i64)(i32)load_u32_unaligned(src + (size_t)i * 4);
        else { const u8* b = src + (size_t)i * flba_len; pq_store<CONV>(out, row, flba_len, [&](int k) -> u8 { return b[k]; }); }
    }
}
void launch_pq_plain(const PqPage* pages, int n_pages, int conv, int flba_len, void* out, int* err, cudaStream_t st) {
    if (n_pages <= 0) return;
    dim3 grid(64, (unsigned)n_pages), block(256);
    switch (conv) {
    case PQ_COPY32: k_pq_plain<PQ_COPY32><<<grid, block, 0, st>>>(pages, flba_len, (u8*)out, err); break;
    case PQ_COPY64: k_pq_plain<PQ_COPY64><<<grid, block, 0, st>>>(pages, flba_len, (u8*)out, err); break;
    case PQ_I32_TO_I64: k_pq_plain<PQ_I32_TO_I64><<<grid, block, 0, st>>>(pages, flba_len, (u8*)out, err); break;
    case PQ_FLBA_TO_I64: k_pq_plain<PQ_FLBA_TO_I64><<<grid, block, 0, st>>>(pages, flba_len, (u8*)out, err); break;
    default: k_pq_plain<PQ_FLBA_TO_I128><<<grid, block, 0, st>>>(pages, flba_len, (u8*)out, err); break;
    }
}

// ---- DELTA_BINARY_PACKED ---------------------------------------------------------------------------------------------
// (1) walk   one thread per page reads only the block headers (device/cb_delta.h) into the page's miniblock table; entry 0 is the
//            first value as a delta from zero
// (2) sum    warp per entry: sum of its deltas (min delta + packed)
// (3) carry  block per page: exclusive scan of the sums -> each entry's carry
// (4) decode warp per entry: unpack again, warp prefix sum + carry, convert, store into the same dense buffer PLAIN pages use
// The packed bytes are read twice and the values written once; all arithmetic wraps in 64 bits, an INT32 page keeps the low 32.

// the i-th packed delta of an entry: two aligned words when 16 bytes of the body remain, else byte by byte (cb_delta.h)
__device__ __forceinline__ u64 dbp_get(const PqMiniblock& m, int i) {
    const int bw = m.bit_width;
    if (bw == 0) return 0;
    const long long bit = (long long)i * bw, byte = bit >> 3;
    if (byte + 16 > m.nbytes) return dbp_unpack(m.src, m.nbytes, i, bw);
    const int sh = (int)(bit & 7);
    const u64 lo = load_u64_unaligned(m.src + byte); // aligned words inside [body - 7, body + nbytes): the page's own bytes
    const u64 hi = m.src[byte + 8];
    const u64 v = (lo >> sh) | (sh ? hi << (64 - sh) : 0ull);
    return bw == 64 ? v : v & ((1ull << bw) - 1ull);
}

__global__ void k_pq_dbp_walk(PqPage* pages, int n_pages, PqMiniblock* table, int type_bits, int* err) {
    const int pi = blockIdx.x * blockDim.x + threadIdx.x;
    if (pi >= n_pages) return;
    const PqPage pg = pages[pi];
    if (pg.encoding != PQ_ENC_DBP) return;
    PqMiniblock* t = table + pg.mb_base;
    const int cap = pg.mb_cap;
    const u8* end = pg.values + pg.values_bytes;
    DbpHeader h;
    int n = 0;
    bool bad = dbp_header(pg.values, end, h) != 0 || h.total != (long long)pg.nonnull; // the header must count exactly the non-null values
    if (!bad && h.total > 0) {
        PqMiniblock first;
        first.src = nullptr; first.min_delta = (i64)h.first; first.carry = 0; first.out_idx = 0; first.count = 1; first.bit_width = 0; first.nbytes = 0;
        if (cap > 0) t[0] = first;
        n = 1;
        const u8* e = dbp_walk(h, end, type_bits, [&](long long idx, long long cnt, int bw, u64 min_delta, const u8* src, long long nbytes) {
            if (n < cap) {
                PqMiniblock m;
                m.src = src; m.min_delta = (i64)min_delta; m.carry = 0; m.out_idx = (int)idx; m.count = (int)cnt; m.bit_width = bw; m.nbytes = (int)nbytes;
                t[n] = m;
            }
            n++;
        });
        bad = e == nullptr || n > cap;
    }
    if (bad) { atomicOr(err, PQ_ERR_DELTA); n = 0; }
    pages[pi].mb_count = n;
}

__global__ void k_pq_dbp_sum(const PqPage* pages, PqMiniblock* table) {
    const PqPage pg = pages[blockIdx.y];
    if (pg.encoding != PQ_ENC_DBP) return;
    PqMiniblock* t = table + pg.mb_base;
    const int lane = threadIdx.x & 31, warps_per_block = blockDim.x >> 5;
    for (int e = blockIdx.x * warps_per_block + (threadIdx.x >> 5); e < pg.mb_count; e += gridDim.x * warps_per_block) {
        const PqMiniblock m = t[e];
        u64 s = 0;
        for (int i = lane; i < m.count; i += 32) s += (u64)m.min_delta + dbp_get(m, i);
        for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
        if (lane == 0) t[e].carry = (i64)s;
    }
}

__global__ void k_pq_dbp_carry(const PqPage* pages, PqMiniblock* table) {
    const PqPage pg = pages[blockIdx.x];
    if (pg.encoding != PQ_ENC_DBP) return;
    __shared__ u64 warp_sums[8];
    PqMiniblock* t = table + pg.mb_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u64 carry = 0;
    for (int base = 0; base < pg.mb_count; base += 256) {
        const int e = base + threadIdx.x;
        const u64 s = e < pg.mb_count ? (u64)t[e].carry : 0ull;
        u64 incl = s;
        for (int d = 1; d < 32; d <<= 1) { const u64 x = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += x; }
        if (lane == 31) warp_sums[warp] = incl;
        __syncthreads();
        u64 wbase = 0, total = 0;
        for (int w = 0; w < 8; w++) { if (w < warp) wbase += warp_sums[w]; total += warp_sums[w]; }
        if (e < pg.mb_count) t[e].carry = (i64)(carry + wbase + incl - s);
        carry += total;
        __syncthreads();
    }
}

template <int CONV> __global__ void k_pq_dbp_decode(const PqPage* pages, const PqMiniblock* table, u8* out) {
    const PqPage pg = pages[blockIdx.y];
    if (pg.encoding != PQ_ENC_DBP) return;
    const PqMiniblock* t = table + pg.mb_base;
    const int lane = threadIdx.x & 31, warps_per_block = blockDim.x >> 5;
    for (int e = blockIdx.x * warps_per_block + (threadIdx.x >> 5); e < pg.mb_count; e += gridDim.x * warps_per_block) {
        const PqMiniblock m = t[e];
        u64 run = (u64)m.carry;
        for (int base = 0; base < m.count; base += 32) {
            const int i = base + lane;
            const u64 d = i < m.count ? (u64)m.min_delta + dbp_get(m, i) : 0ull;
            u64 incl = d;
            for (int k = 1; k < 32; k <<= 1) { const u64 x = __shfl_up_sync(0xffffffffu, incl, k); if (lane >= k) incl += x; }
            if (i < m.count) {
                const u64 v = run + incl;
                const long long row = pg.dst_row + m.out_idx + i;
                if (CONV == PQ_COPY32) ((u32*)out)[row] = (u32)v;
                else if (CONV == PQ_COPY64) ((u64*)out)[row] = v;
                else ((i64*)out)[row] = (i64)(i32)(u32)v; // PQ_I32_TO_I64: wraps at 2^32, then widens
            }
            run += __shfl_sync(0xffffffffu, incl, 31);
        }
    }
}

void launch_pq_dbp(PqPage* pages, int n_pages, PqMiniblock* table, int conv, void* out, int* err, cudaStream_t st) {
    if (n_pages <= 0) return;
    const int type_bits = conv == PQ_COPY64 ? 64 : 32;
    k_pq_dbp_walk<<<(n_pages + 63) / 64, 64, 0, st>>>(pages, n_pages, table, type_bits, err);
    const dim3 grid(32, (unsigned)n_pages), block(256);
    k_pq_dbp_sum<<<grid, block, 0, st>>>(pages, table);
    k_pq_dbp_carry<<<n_pages, 256, 0, st>>>(pages, table);
    if (conv == PQ_COPY32) k_pq_dbp_decode<PQ_COPY32><<<grid, block, 0, st>>>(pages, table, (u8*)out);
    else if (conv == PQ_COPY64) k_pq_dbp_decode<PQ_COPY64><<<grid, block, 0, st>>>(pages, table, (u8*)out);
    else k_pq_dbp_decode<PQ_I32_TO_I64><<<grid, block, 0, st>>>(pages, table, (u8*)out);
}

// ---- RLE / bit-packed hybrid ------------------------------------------------------------------------------------------
// walk the run headers of [p, end): calls f(is_bit_packed, count, value, data_ptr); returns values seen
template <typename F> __device__ long long walk_hybrid(const u8* p, const u8* end, int bit_width, long long max_values, F f) {
    long long seen = 0;
    const int vbytes = (bit_width + 7) / 8;
    while (p < end && seen < max_values) {
        u32 header = 0;
        int shift = 0;
        while (p < end) { // ULEB128
            u8 b = *p++;
            header |= (u32)(b & 0x7f) << shift;
            shift += 7;
            if (!(b & 0x80)) break;
        }
        if (header & 1) { // bit-packed: (header >> 1) groups of 8 values
            long long count = (long long)(header >> 1) * 8;
            long long take = count < max_values - seen ? count : max_values - seen;
            f(1, (int)take, 0u, p);
            p += (size_t)(header >> 1) * bit_width;
            seen += take;
        } else {
            long long count = header >> 1;
            u32 v = 0;
            for (int k = 0; k < vbytes && p + k < end; k++) v |= (u32)p[k] << (8 * k);
            p += vbytes;
            long long take = count < max_values - seen ? count : max_values - seen;
            f(0, (int)take, v, p);
            seen += take;
        }
    }
    return seen;
}

// LEVELS = false: the dictionary indices of the page (first byte = bit width);  true: its definition levels (bit width 1)
template <bool LEVELS> __global__ void k_pq_rle_scan(const PqPage* pages, int n_pages, PqRun* runs, int* run_counts, int* err) {
    int pi = blockIdx.x * blockDim.x + threadIdx.x;
    if (pi >= n_pages) return;
    const PqPage pg = pages[pi];
    if (LEVELS ? pg.def_bytes <= 0 : pg.encoding != PQ_ENC_DICT) { run_counts[pi] = 0; return; }
    const u8* p = LEVELS ? pg.def_ptr : pg.values;
    const u8* end = p + (LEVELS ? pg.def_bytes : pg.values_bytes);
    int bw = 1;
    if (!LEVELS) bw = p < end ? *p++ : 0; // RLE_DICTIONARY: the first byte is the index bit width
    const long long want = LEVELS ? pg.num_values : pg.nonnull;
    const int cap = LEVELS ? pg.def_max_runs : pg.max_runs;
    PqRun* out = runs + (LEVELS ? pg.def_run_base : pg.run_base);
    int n = 0;
    bool truncated = false;
    long long row = pg.dst_row;
    long long seen = bw > 32 ? -1 : walk_hybrid(p, end, bw, want, [&](int packed, int count, u32 value, const u8* data) {
        if (n < cap) {
            PqRun r;
            r.out_row = row;
            r.src = data;
            r.count = count;
            r.value = value;
            r.bit_packed = packed;
            r.bit_width = bw;
            if (packed && data + ((long long)count * bw + 7) / 8 > end) { r.count = 0; truncated = true; } // truncated page: never read beyond it
            out[n] = r;
        }
        n++;
        row += count;
    });
    if (n > cap || seen != want) atomicOr(err, PQ_ERR_RLE);
    if (truncated) atomicOr(err, PQ_ERR_TRUNCATED);
    run_counts[pi] = n < cap ? n : cap;
}
void launch_pq_rle_scan(const PqPage* pages, int n_pages, PqRun* runs, int* run_counts, int* err, cudaStream_t st) {
    if (n_pages > 0) k_pq_rle_scan<false><<<(n_pages + 63) / 64, 64, 0, st>>>(pages, n_pages, runs, run_counts, err);
}

template <int DW> __device__ __forceinline__ void store_dict(const void* dict, int dict_size, u32 idx, void* out, long long row, int* err) {
    if ((int)idx >= dict_size) { atomicOr(err, PQ_ERR_DICT_INDEX); idx = 0; }
    if (DW == 4) ((u32*)out)[row] = ((const u32*)dict)[idx];
    else if (DW == 8) ((u64*)out)[row] = ((const u64*)dict)[idx];
    else ((ulonglong2*)out)[row] = ((const ulonglong2*)dict)[idx];
}
// one warp per run; blockIdx.y = page
template <int DW> __global__ void k_pq_rle_decode(const PqPage* pages, const PqRun* runs, const int* run_counts, const void* dict_all, void* out, int* err) {
    const PqPage pg = pages[blockIdx.y];
    if (pg.encoding != PQ_ENC_DICT) return;
    const void* dict = (const u8*)dict_all + (size_t)pg.dict_off * DW;
    const int dict_size = pg.dict_size;
    const int n_runs = run_counts[blockIdx.y];
    const int lane = threadIdx.x & 31, warps_per_block = blockDim.x >> 5;
    for (int ri = blockIdx.x * warps_per_block + (threadIdx.x >> 5); ri < n_runs; ri += gridDim.x * warps_per_block) {
        const PqRun r = runs[pg.run_base + ri];
        if (!r.bit_packed) {
            for (int i = lane; i < r.count; i += 32) store_dict<DW>(dict, dict_size, r.value, out, r.out_row + i, err);
        } else {
            const u8* src = r.src;
            const int bw = r.bit_width;
            const long long nbytes = ((long long)r.count * bw + 7) / 8;
            const u32 mask = bw >= 32 ? 0xffffffffu : ((1u << bw) - 1u);
            for (int i = lane; i < r.count; i += 32) {
                long long bit = (long long)i * bw;
                const u8* q = src + (bit >> 3);
                u64 w = 0;
                for (int k = 0; k < 5; k++) if ((bit >> 3) + k < nbytes) w |= (u64)q[k] << (8 * k); // bw <= 32: value spans at most 5 bytes
                u32 idx = (u32)(w >> (bit & 7)) & mask;
                store_dict<DW>(dict, dict_size, idx, out, r.out_row + i, err);
            }
        }
    }
}
void launch_pq_rle_decode(const PqPage* pages, int n_pages, const PqRun* runs, const int* run_counts, const void* dict, int dict_width, void* out, int* err,
                          cudaStream_t st) {
    if (n_pages <= 0) return;
    dim3 grid(32, (unsigned)n_pages), block(256);
    if (dict_width == 4) k_pq_rle_decode<4><<<grid, block, 0, st>>>(pages, runs, run_counts, dict, out, err);
    else if (dict_width == 8) k_pq_rle_decode<8><<<grid, block, 0, st>>>(pages, runs, run_counts, dict, out, err);
    else k_pq_rle_decode<16><<<grid, block, 0, st>>>(pages, runs, run_counts, dict, out, err);
}

// ---- definition levels (flat optional columns: bit width 1) ---------------------------------------------------------------
// fast path: the chunk statistics promise null_count == 0 -- verify it, one thread per page (run headers only for RLE runs)
__global__ void k_pq_check_def(const PqPage* pages, int n_pages, int* err) {
    int pi = blockIdx.x * blockDim.x + threadIdx.x;
    if (pi >= n_pages) return;
    const PqPage pg = pages[pi];
    if (pg.def_bytes <= 0) return;
    const u8* p = pg.def_ptr;
    const u8* end = p + pg.def_bytes;
    bool bad = false;
    long long seen = walk_hybrid(p, end, 1, pg.num_values, [&](int packed, int count, u32 value, const u8* data) {
        if (!packed) { if (value != 1u) bad = true; }
        else for (int i = 0; i < count && data + (i >> 3) < end; i++) if (!((data[i >> 3] >> (i & 7)) & 1)) { bad = true; break; }
    });
    if (bad) atomicOr(err, PQ_ERR_NULL_ON_FAST_PATH);
    if (seen != pg.num_values) atomicOr(err, PQ_ERR_RLE);
}
void launch_pq_check_def_levels(const PqPage* pages, int n_pages, int* err, cudaStream_t st) {
    if (n_pages > 0) k_pq_check_def<<<(n_pages + 63) / 64, 64, 0, st>>>(pages, n_pages, err);
}

// NULL-aware path, step 2: expand the level runs to one validity byte per row (warp per run; blockIdx.y = page)
__global__ void k_pq_def_expand(const PqPage* pages, const PqRun* runs, const int* run_counts, u8* valid) {
    const PqPage pg = pages[blockIdx.y];
    const int n_runs = run_counts[blockIdx.y];
    const int lane = threadIdx.x & 31, warps_per_block = blockDim.x >> 5;
    for (int ri = blockIdx.x * warps_per_block + (threadIdx.x >> 5); ri < n_runs; ri += gridDim.x * warps_per_block) {
        const PqRun r = runs[pg.def_run_base + ri];
        if (!r.bit_packed) for (int i = lane; i < r.count; i += 32) valid[r.out_row + i] = (u8)(r.value & 1u);
        else for (int i = lane; i < r.count; i += 32) valid[r.out_row + i] = (u8)((r.src[i >> 3] >> (i & 7)) & 1);
    }
}
// step 3: per page, idx[row] = dst_row + (non-null rows of the page before `row`): where the row's value sits in the
// densely decoded value stream.  One block per page, running carry across 2048-row tiles.
__global__ void k_pq_def_index(PqPage* pages, u8* valid, u32* idx) {
    const PqPage pg = pages[blockIdx.x];
    __shared__ u32 warp_sums[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 carry = 0;
    const bool all_valid = pg.def_bytes <= 0; // required column mixed into an optional one across files: no levels, everything present
    for (long long base = 0; base < pg.num_values; base += 2048) {
        const long long r0 = pg.dst_row + base + (long long)threadIdx.x * 8;
        u32 v[8], local = 0;
        for (int k = 0; k < 8; k++) {
            const bool in = base + threadIdx.x * 8 + k < pg.num_values;
            v[k] = in ? (all_valid ? 1u : (u32)valid[r0 + k]) : 0u;
            local += v[k];
        }
        u32 incl = local;
        for (int d = 1; d < 32; d <<= 1) { u32 t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
        if (lane == 31) warp_sums[warp] = incl;
        __syncthreads();
        u32 wbase = 0, total = 0;
        for (int w = 0; w < 8; w++) { if (w < warp) wbase += warp_sums[w]; total += warp_sums[w]; }
        u32 excl = carry + wbase + incl - local;
        for (int k = 0; k < 8; k++) {
            if (base + threadIdx.x * 8 + k < pg.num_values) {
                idx[r0 + k] = (u32)pg.dst_row + excl;
                if (all_valid) valid[r0 + k] = 1;
            }
            excl += v[k];
        }
        carry += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) pages[blockIdx.x].nonnull = (int)carry;
}
void launch_pq_def_levels(PqPage* pages, int n_pages, PqRun* runs, int* run_counts, unsigned char* valid, unsigned* idx, int* err, cudaStream_t st) {
    if (n_pages <= 0) return;
    k_pq_rle_scan<true><<<(n_pages + 63) / 64, 64, 0, st>>>(pages, n_pages, runs, run_counts, err);
    k_pq_def_expand<<<dim3(32, (unsigned)n_pages), 256, 0, st>>>(pages, runs, run_counts, valid);
    k_pq_def_index<<<n_pages, 256, 0, st>>>(pages, valid, idx);
}

// step 4 (after the values were decoded densely): scatter to row positions, zero the NULL slots, build the Arrow bitmap
template <int W> __global__ void k_pq_scatter(const u8* valid, const u32* idx, const u8* dense, u8* out, u32* bitmap, long long total) {
    const long long n32 = (total + 31) / 32 * 32;
    for (long long row = blockIdx.x * (long long)blockDim.x + threadIdx.x; row < n32; row += (long long)gridDim.x * blockDim.x) {
        const bool ok = row < total && valid[row] != 0;
        if (row < total) {
            if (W == 4) ((u32*)out)[row] = ok ? ((const u32*)dense)[idx[row]] : 0u;
            else if (W == 8) ((u64*)out)[row] = ok ? ((const u64*)dense)[idx[row]] : 0ull;
            else ((ulonglong2*)out)[row] = ok ? ((const ulonglong2*)dense)[idx[row]] : make_ulonglong2(0ull, 0ull);
        }
        const u32 word = __ballot_sync(0xffffffffu, ok);
        if ((threadIdx.x & 31) == 0) bitmap[row >> 5] = word;
    }
}
void launch_pq_scatter(const unsigned char* valid, const unsigned* idx, const void* dense, void* out, unsigned* bitmap, long long total, int width, cudaStream_t st) {
    if (total <= 0) return;
    const int blocks = (int)std::min<long long>((total + 255) / 256, 132 * 16); // grid-stride: 16 CTAs per H100 SM
    if (width == 4) k_pq_scatter<4><<<blocks, 256, 0, st>>>(valid, idx, (const u8*)dense, (u8*)out, bitmap, total);
    else if (width == 8) k_pq_scatter<8><<<blocks, 256, 0, st>>>(valid, idx, (const u8*)dense, (u8*)out, bitmap, total);
    else k_pq_scatter<16><<<blocks, 256, 0, st>>>(valid, idx, (const u8*)dense, (u8*)out, bitmap, total);
}

} // namespace cb200
