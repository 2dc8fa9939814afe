// sortkey_test.cpp -- test-only driver of device/cb_sortkey.h on the host (the row-key encoder the key kernel k_sort_keys runs), built
// with g++ by tests/test_sort_cpu.py like strpred_test.cpp.
#include "device/cb_sortkey.h"

#include <cstring>

extern "C" {

// the HK_* layout constants, so the test does not restate them
int cb_sk_kind(const char* name) {
    static const struct { const char* name; int kind; } kinds[] = {
        {"bool", HK_BOOL}, {"bool8", HK_BOOL8}, {"i8", HK_I8}, {"i16", HK_I16}, {"i32", HK_I32}, {"i64", HK_I64}, {"f32", HK_F32},
        {"f64", HK_F64}, {"dec_small_32", HK_DEC_SMALL_32}, {"dec_small_64", HK_DEC_SMALL_64}, {"dec_small_128", HK_DEC_SMALL_128},
        {"dec_large_64", HK_DEC_LARGE_64}, {"dec_large_128", HK_DEC_LARGE_128}, {"dict8", HK_DICT8}, {"dict16", HK_DICT16},
        {"dict32", HK_DICT32}};
    for (auto& k : kinds)
        if (!strcmp(k.name, name)) return k.kind;
    return -1;
}

// Row keys of n rows over up to 8 key columns (arrays indexed by key, the first key most significant), `words` words per row into out.
// Field offsets are laid out as the executor lays them out: bits + has_null per key, the last key at bit 0.  Returns the number of rows
// whose dictionary code was outside its rank table.
long long cb_sk_encode(int n_keys, const int* kind, const int* bits, const int* desc, const int* nulls_first, const void* const* data,
                       const unsigned char* const* validity, const unsigned* const* rank, const int* n_rank, long long n, int words,
                       unsigned long long* out) {
    cb::SortKeyCols kc;
    memset(&kc, 0, sizeof(kc));
    kc.n = n_keys;
    kc.words = words;
    int off = 0;
    for (int k = n_keys - 1; k >= 0; k--) {
        cb::SortKeyCol& f = kc.col[k];
        f.kind = kind[k];
        f.bits = bits[k];
        f.desc = desc[k];
        f.nulls_first = nulls_first[k];
        f.has_null = validity[k] != nullptr;
        f.data = data[k];
        f.validity = validity[k];
        f.rank = rank[k];
        f.n_rank = n_rank[k];
        f.off = off;
        off += f.bits + f.has_null;
    }
    long long bad = 0;
    for (long long i = 0; i < n; i++) {
        unsigned long long* w = out + i * words;
        for (int j = 0; j < words; j++) w[j] = 0;
        if (!cb::sk_row(kc, i, w)) bad++;
    }
    return bad;
}

} // extern "C"
