// cb_delta.h -- DELTA_BINARY_PACKED (parquet-format Encodings.md) header / block walk shared by the device decoder
// (parquet_kernels.cu: one thread per page walks the block headers into a miniblock table) and the host, which decodes the
// length / prefix sections of DELTA_LENGTH_BYTE_ARRAY and DELTA_BYTE_ARRAY string pages with it (scan_plan.cpp).
//
// Format: <block size in values> <miniblocks per block> <total value count> <first value (zigzag)>, all ULEB128; then blocks of
// <min delta (zigzag ULEB128)> <one bit-width byte per miniblock> <bit-packed miniblocks, LSB first>.  value[i] = value[i - 1] +
// min_delta + packed delta, wrapping in the physical type's width.  The last block holds as many miniblocks as carry values; the
// bit-width bytes of the others may hold anything and those miniblocks have no body bytes.  A used miniblock is always stored at
// full length (values per miniblock x bit width / 8 bytes), padding included.
#ifndef CB_DELTA_H
#define CB_DELTA_H
#include "cb_math.h"

namespace cb {

constexpr long long DBP_MAX_BLOCK = 1 << 20; // values per block; larger headers are treated as malformed

// ULEB128 of at most 64 bits at p (never reads at or beyond end); advances p, false on truncation / overflow
CB_HD bool dbp_uleb(const u8*& p, const u8* end, u64& v) {
    v = 0;
    for (int shift = 0; shift < 70 && p < end; shift += 7) {
        const u8 b = *p++;
        if (shift == 63 && (b & 0x7e)) return false;
        v |= (u64)(b & 0x7f) << shift;
        if (!(b & 0x80)) return true;
    }
    return false;
}
CB_HD u64 dbp_unzigzag(u64 z) { return (z >> 1) ^ (0ull - (z & 1)); }

struct DbpHeader {
    long long block, per_mb, total; // values per block / per miniblock, values of the page
    int mbs;                         // miniblocks per block
    u64 first;                       // the first value (two's complement, wrapping)
    const u8* blocks;                // first block header
};

// 0 = ok; -1 = malformed (sizes that break the rule "block a multiple of 128, miniblock a multiple of 32", truncated header)
CB_HD int dbp_header(const u8* p, const u8* end, DbpHeader& h) {
    u64 block, mbs, total, first;
    if (!dbp_uleb(p, end, block) || !dbp_uleb(p, end, mbs) || !dbp_uleb(p, end, total) || !dbp_uleb(p, end, first)) return -1;
    if (block == 0 || block % 128 != 0 || block > (u64)DBP_MAX_BLOCK || mbs == 0 || block % mbs != 0 || (block / mbs) % 32 != 0) return -1;
    if (total > 0x7fffffffull) return -1;
    h.block = (long long)block;
    h.mbs = (int)mbs;
    h.per_mb = (long long)(block / mbs);
    h.total = (long long)total;
    h.first = dbp_unzigzag(first);
    h.blocks = p;
    return 0;
}

// Walks the blocks of a stream whose header is `h`, calling on_mb(first value index, values, bit width, min delta, body, body bytes) for
// every miniblock that carries values (value index 1 is the first delta).  Returns the position after the stream, or nullptr when a
// used miniblock's width exceeds type_bits or a header / body runs past `end`.
template <typename F> CB_HD const u8* dbp_walk(const DbpHeader& h, const u8* end, int type_bits, F on_mb) {
    const u8* p = h.blocks;
    long long left = h.total > 0 ? h.total - 1 : 0, idx = 1;
    while (left > 0) {
        u64 zmin;
        if (!dbp_uleb(p, end, zmin) || end - p < h.mbs) return nullptr;
        const u64 min_delta = dbp_unzigzag(zmin);
        const u8* widths = p;
        p += h.mbs;
        for (int m = 0; m < h.mbs && left > 0; m++) {
            const int bw = widths[m];
            if (bw > type_bits) return nullptr;
            const long long nbytes = h.per_mb * bw / 8;
            if (end - p < nbytes) return nullptr;
            const long long cnt = left < h.per_mb ? left : h.per_mb;
            on_mb(idx, cnt, bw, min_delta, p, nbytes);
            p += nbytes;
            idx += cnt;
            left -= cnt;
        }
    }
    return p;
}

// the i-th packed value of a miniblock body of `nbytes` bytes (bit width 0..64); reads only inside the body
CB_HD u64 dbp_unpack(const u8* src, long long nbytes, long long i, int bw) {
    if (bw == 0) return 0;
    const long long bit = i * bw, byte = bit >> 3;
    const int sh = (int)(bit & 7);
    u64 lo = 0;
    u8 hi = 0;
    for (int k = 0; k < 8; k++) if (byte + k < nbytes) lo |= (u64)src[byte + k] << (8 * k);
    if (byte + 8 < nbytes) hi = src[byte + 8];
    u64 v = (lo >> sh) | (sh ? (u64)hi << (64 - sh) : 0ull);
    return bw == 64 ? v : v & ((1ull << bw) - 1ull);
}

// Serial decode (the host's; also the definition the device kernels are tested against).  out[0, total) gets the values, wrapping
// in 64 bits (an INT32 page's values are the low 32 bits).  Returns the position after the stream, or nullptr when the stream is
// malformed or holds more than `cap` values; *count = the header's value count.
CB_HD const u8* dbp_decode_serial(const u8* p, const u8* end, int type_bits, i64* out, long long cap, long long* count) {
    DbpHeader h;
    *count = 0;
    if (dbp_header(p, end, h) != 0 || h.total > cap) return nullptr;
    *count = h.total;
    if (h.total == 0) return h.blocks;
    u64 v = h.first;
    out[0] = (i64)v;
    return dbp_walk(h, end, type_bits, [&](long long idx, long long cnt, int bw, u64 min_delta, const u8* src, long long nbytes) {
        for (long long k = 0; k < cnt; k++) {
            v += min_delta + dbp_unpack(src, nbytes, k, bw);
            out[idx + k] = (i64)v;
        }
    });
}

} // namespace cb
#endif
