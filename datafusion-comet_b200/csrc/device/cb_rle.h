// cb_rle.h -- RLE / bit-packed hybrid (parquet-format Encodings.md) run walk and the unpack of one bit-packed value, shared by the
// device decoders of dictionary indices and definition levels (parquet_kernels.cu) and a host test driver (rle_test.cpp).
//
// Format: runs until the stream ends, each a ULEB128 header h.  h & 1: bit-packed, (h >> 1) groups of 8 values, (h >> 1) x bit width
// bytes, LSB first.  Otherwise an RLE run of (h >> 1) copies of one value stored in ceil(bit width / 8) little-endian bytes.
#ifndef CB_RLE_H
#define CB_RLE_H
#include "cb_math.h"

namespace cb {

// walk_hybrid's results below zero
enum { HYB_MALFORMED = -1, HYB_TRUNCATED = -2 };

// Walks the runs of [p, end) until max_values values were seen or the stream ends, calling f(is_bit_packed, count, value, data) for
// every run with count > 0 (count is cut to the values still wanted).  Returns the values seen, HYB_MALFORMED for a bit width above
// 32, a run header that does not end inside the stream or an RLE value past its end, and HYB_TRUNCATED for a bit-packed run whose
// wanted values lie past the end.  f is never called for such a run, so it only ever sees bytes inside [p, end).
template <typename F> CB_HD long long walk_hybrid(const u8* p, const u8* end, int bit_width, long long max_values, F f) {
    if (bit_width < 0 || bit_width > 32) return HYB_MALFORMED;
    long long seen = 0;
    const int vbytes = (bit_width + 7) / 8;
    while (p < end && seen < max_values) {
        u64 header = 0;
        bool ended = false;
        for (int shift = 0; shift < 35 && p < end; shift += 7) { // ULEB128 of at most 32 bits
            const u8 b = *p++;
            header |= (u64)(b & 0x7f) << shift;
            if (!(b & 0x80)) { ended = true; break; }
        }
        if (!ended || header >> 32) return HYB_MALFORMED;
        const long long count = (long long)(header >> 1) * ((header & 1) ? 8 : 1);
        const long long take = count < max_values - seen ? count : max_values - seen;
        if (header & 1) {
            const long long bytes = (long long)(header >> 1) * bit_width, left = (long long)(end - p);
            if ((take * bit_width + 7) / 8 > left) return HYB_TRUNCATED;
            if (take > 0) f(1, (int)take, 0u, p);
            p += bytes < left ? bytes : left; // padding of the last group may be cut off at the end of the stream
        } else {
            if (vbytes > end - p) return HYB_MALFORMED;
            u32 v = 0;
            for (int k = 0; k < vbytes; k++) v |= (u32)p[k] << (8 * k);
            p += vbytes;
            if (take > 0) f(0, (int)take, v, p);
        }
        seen += take;
    }
    return seen;
}

// value i of a bit-packed run of bit width bw <= 32 whose bytes are src[0, nbytes): never reads at or beyond src + nbytes
CB_HD u32 hybrid_unpack(const u8* src, long long nbytes, long long i, int bw) {
    const long long bit = i * bw;
    const u8* q = src + (bit >> 3);
    u64 w = 0;
    for (int k = 0; k < 5; k++) if ((bit >> 3) + k < nbytes) w |= (u64)q[k] << (8 * k); // a value spans at most 5 bytes
    const u32 mask = bw >= 32 ? 0xffffffffu : ((1u << bw) - 1u);
    return (u32)(w >> (bit & 7)) & mask;
}

} // namespace cb
#endif
