// rangepart_test.cpp -- test-only driver of device/cb_rangepart.h on the host (the boundary search k_range_pids runs and the string
// rank of a range key), built with g++ together with sortkey_test.cpp by tests/test_range_partition_cpu.py.
#include "device/cb_rangepart.h"
#include "device/cb_sortkey.h"

#include <cstring>
#include <string>
#include <vector>

extern "C" {

// the top level k_range_pids stages for nb boundary rows of W words and a shared-memory budget: its shift and row count
int cb_rp_shift(unsigned nb, int W, unsigned budget) { return cb::rp_shift(nb, W, budget); }

// out[i] = the number of the nb boundary rows (W words each, non-decreasing) <= keys[i], searched as the kernel does: over the
// sampled top level of `shift` (built here from the bounds), then the bounds themselves.  Returns -1 unless 1 <= W <= 4.
int cb_rp_pids(const unsigned long long* bounds, unsigned nb, int W, int shift, const unsigned long long* keys, long long n, unsigned* out) {
    if (W < 1 || W > 4) return -1;
    std::vector<unsigned long long> top;
    const unsigned n_top = nb >> shift;
    if (shift == 0) top.assign(bounds, bounds + (size_t)nb * W);
    else
        for (unsigned j = 0; j < n_top; j++)
            top.insert(top.end(), bounds + ((((size_t)j + 1) << shift) - 1) * W, bounds + (((size_t)j + 1) << shift) * W);
    for (long long i = 0; i < n; i++) {
        const unsigned long long* k = keys + i * W;
        out[i] = W == 1 ? cb::rp_pid<1>(top.data(), n_top, shift, bounds, nb, k) : W == 2 ? cb::rp_pid<2>(top.data(), n_top, shift, bounds, nb, k)
               : W == 3 ? cb::rp_pid<3>(top.data(), n_top, shift, bounds, nb, k) : cb::rp_pid<4>(top.data(), n_top, shift, bounds, nb, k);
    }
    return 0;
}

// cb_sk_encode (sortkey_test.cpp) through sk_row_reg, the register form k_range_pids packs keys with: the same arguments, every key with
// a validity bitmap (a range key's field always has a null bit).  Returns -1 unless 1 <= words <= 4, else the rows whose code was out
// of range.
long long cb_rp_encode(int n_keys, const int* kind, const int* bits, const int* desc, const int* nulls_first, const void* const* data,
                       const unsigned char* const* validity, const unsigned* const* rank, const int* n_rank, long long n, int words,
                       unsigned long long* out) {
    if (words < 1 || words > 4) return -1;
    cb::SortKeyCols kc;
    memset(&kc, 0, sizeof(kc));
    kc.n = n_keys;
    kc.words = words;
    int off = 0;
    for (int k = n_keys - 1; k >= 0; k--) {
        cb::SortKeyCol& f = kc.col[k];
        f = {kind[k], bits[k], off, desc[k], nulls_first[k], 1, data[k], validity[k], rank[k], n_rank[k]};
        off += f.bits + 1;
    }
    long long bad = 0;
    for (long long i = 0; i < n; i++) {
        unsigned long long* w = out + i * words;
        bool ok = true;
        switch (words) {
        case 1: { cb::u64 r[1] = {}; ok = cb::sk_row_reg<1>(kc, i, r); memcpy(w, r, sizeof(r)); break; }
        case 2: { cb::u64 r[2] = {}; ok = cb::sk_row_reg<2>(kc, i, r); memcpy(w, r, sizeof(r)); break; }
        case 3: { cb::u64 r[3] = {}; ok = cb::sk_row_reg<3>(kc, i, r); memcpy(w, r, sizeof(r)); break; }
        default: { cb::u64 r[4] = {}; ok = cb::sk_row_reg<4>(kc, i, r); memcpy(w, r, sizeof(r)); break; }
        }
        if (!ok) bad++;
    }
    return bad;
}

// rank[i] of dictionary entry i (values: offsets[n + 1] + chars) against the sorted distinct boundary strings (b_off[nb + 1] + b_chars)
void cb_rp_string_ranks(const int* offsets, const char* chars, long long n, const int* b_off, const char* b_chars, long long nb, unsigned* rank) {
    std::vector<std::string> v, b;
    for (long long i = 0; i < n; i++) v.emplace_back(chars + offsets[i], (size_t)(offsets[i + 1] - offsets[i]));
    for (long long i = 0; i < nb; i++) b.emplace_back(b_chars + b_off[i], (size_t)(b_off[i + 1] - b_off[i]));
    const std::vector<unsigned> r = cb::rp_string_ranks(v, b);
    for (long long i = 0; i < n; i++) rank[i] = r[(size_t)i];
}

} // extern "C"
