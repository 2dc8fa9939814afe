// rle_test.cpp -- test-only driver of device/cb_rle.h on the host (the hybrid walk and unpack the dictionary-index and definition-level
// kernels use), built with g++ by tests/test_parquet_pages_cpu.py like delta_test.cpp.
#include "device/cb_rle.h"

// Decodes at most `want` values of the hybrid stream buf[0, n) of bit width `bw` into out[0, want).  Returns the values decoded, or
// walk_hybrid's HYB_MALFORMED (-1) / HYB_TRUNCATED (-2).
extern "C" long long cb_rle_decode(const unsigned char* buf, long long n, int bw, long long want, unsigned* out) {
    long long row = 0;
    return cb::walk_hybrid(buf, buf + n, bw, want, [&](int packed, int count, unsigned value, const unsigned char* data) {
        const long long nbytes = ((long long)count * bw + 7) / 8;
        for (int i = 0; i < count; i++) out[row + i] = packed ? cb::hybrid_unpack(data, nbytes, i, bw) : value;
        row += count;
    });
}
