// delta_test.cpp -- test-only driver of device/cb_delta.h on the host (the walk the decode kernels and the string path share), built
// with g++ by tests/test_parquet_encodings_cpu.py like host_math_test.cpp.
#include "device/cb_delta.h"

// Decodes the DELTA_BINARY_PACKED stream buf[0, n) of a `bits`-wide physical type into out[0, cap).  Returns the value count; -1 when the
// stream is malformed, -2 when its value count is not `expect` (the page's non-null count; -1 = any).  *consumed = the stream's bytes.
extern "C" long long cb_dbp_decode(const unsigned char* buf, long long n, int bits, long long expect, long long* out, long long cap, long long* consumed) {
    long long count = 0;
    const unsigned char* e = cb::dbp_decode_serial(buf, buf + n, bits, (cb::i64*)out, cap, &count);
    if (!e) return -1;
    if (expect >= 0 && count != expect) return -2;
    if (bits == 32) for (long long i = 0; i < count; i++) out[i] = (long long)(int)(unsigned)(unsigned long long)out[i];
    *consumed = e - buf;
    return count;
}
