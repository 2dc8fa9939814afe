// cb_sortkey.h -- the packed row key of a Sort: key values turned into unsigned bits whose lexicographic order is the reference's
// order, shared by the key kernel k_sort_keys (aot_kernels.cu) and the host test driver sortkey_test.cpp; and the hash join's hash of
// that key.
//
// Value order is arrow-rs's (arrow-ord, which DataFusion's SortExec uses): signed integers, dates, timestamps and decimals (their
// unscaled value, any precision) numerically; booleans false < true; strings by unsigned bytes (here the dense byte-order rank of the
// dictionary entry, computed on the host); floats by IEEE totalOrder, -NaN < -Inf < ... < -0.0 < +0.0 < ... < +Inf < +NaN with NaN
// sign and payload counted (f32::total_cmp).  DESC inverts the value bits.  A NULL's place is its own bit above the value, set by
// nulls_first alone (arrow SortOptions: the null placement does not depend on the direction), and a NULL's value bits are 0.
//
// The row key is the concatenation of its fields, the first sort key most significant, as `words` 64-bit words per row with word 0 the
// most significant: comparing rows is comparing their words in order.  Field k's value occupies bits [off, off + bits) counted from the
// least significant bit of the whole key, its null bit (if any) bit off + bits.
#ifndef CB_SORTKEY_H
#define CB_SORTKEY_H
#include "cb_math.h"

// The layout of a key column, as the sources store it (rows.cpp key_kind): shared by hash partitioning, the sort and the join.
// HK_BOOL reads an Arrow bitmap, HK_BOOL8 one byte per row; HK_I32 also serves INT32-backed int8 / int16; HK_DEC_SMALL_32 is a
// decimal(p <= 9) stored as INT32, HK_DEC_SMALL_64 (= HK_I64) / HK_DEC_LARGE_64 decimals stored in 8 bytes, *_128 in 16 bytes;
// HK_DICT* are dictionary codes of 1, 2 or 4 bytes, HK_UTF8 plain offsets + chars.
enum { HK_BOOL, HK_I8, HK_I16, HK_I32, HK_I64, HK_F32, HK_F64, HK_DEC_SMALL_128, HK_DEC_LARGE_128, HK_DEC_SMALL_64 = HK_I64, HK_DEC_LARGE_64 = 9,
       HK_DICT8 = 10, HK_DICT16, HK_DICT32, HK_UTF8, HK_DEC_SMALL_32, HK_BOOL8 };

#ifdef __CUDACC__
#define CB_SK_UNROLL _Pragma("unroll")
#else
#define CB_SK_UNROLL
#endif

namespace cb {

struct SortKeyCol {
    i32 kind;             // HK_* layout of data
    i32 bits;             // value bits: 1 (bool), 8 / 16 / 32 / 64 (integers, dates, timestamps, floats), 32 (string rank), 64 / 128 (decimal)
    i32 off;             // bit offset of the value in the row key
    i32 desc, nulls_first, has_null; // has_null: the field carries a null bit (the column has a validity bitmap)
    const void* data;
    const u8* validity;   // Arrow bitmap or nullptr
    const u32* rank;      // HK_DICT*: dictionary code -> dense byte-order rank
    i32 n_rank;
};
enum { SK_MAX_KEYS = 8, SK_MAX_WORDS = 4 };
struct SortKeyCols {
    i32 n, words;
    i32* err;             // bit 5 (dictionary code out of range), as the pipelines raise it
    SortKeyCol col[SK_MAX_KEYS];
};

CB_HD u64 sk_mask(int nb) { return nb >= 64 ? ~0ull : ((1ull << nb) - 1ull); }

// OR nb <= 64 bits of v into the row key w[0, words) at bit offset off
CB_HD void sk_put(u64* w, int words, int off, u64 v, int nb) {
    const int lw = off >> 6, sh = off & 63;
    w[words - 1 - lw] |= v << sh;
    if (sh && sh + nb > 64) w[words - 2 - lw] |= v >> (64 - sh);
}

// the order bits of row i of key k (before DESC), hi:lo for 128-bit fields; false for a dictionary code outside the rank table
CB_HD bool sk_value(const SortKeyCol& k, i64 i, u64& hi, u64& lo) {
    const u8* d = (const u8*)k.data;
    i64 s = 0;      // signed value of <= 64 bits
    hi = 0;
    switch (k.kind) {
    case HK_BOOL: lo = (d[i >> 3] >> (i & 7)) & 1u; return true;
    case HK_BOOL8: lo = d[i] ? 1u : 0u; return true;
    case HK_I8: s = ((const signed char*)d)[i]; break;
    case HK_I16: s = ((const short*)d)[i]; break;
    case HK_I32: case HK_DEC_SMALL_32: s = ((const i32*)d)[i]; break;
    case HK_I64: s = ((const i64*)d)[i]; break;
    case HK_F32: { const u32 u = ((const u32*)d)[i]; lo = (u & 0x80000000u) ? (u64)(~u) : (u64)(u | 0x80000000u); return true; }
    case HK_F64: { const u64 u = ((const u64*)d)[i]; lo = (u >> 63) ? ~u : (u | (1ull << 63)); return true; }
    case HK_DEC_SMALL_128: s = (i64)((const u64*)d)[2 * i]; break;
    case HK_DEC_LARGE_128: lo = ((const u64*)d)[2 * i]; hi = ((const u64*)d)[2 * i + 1] ^ (1ull << 63); return true;
    case HK_DEC_LARGE_64: { const i64 v = ((const i64*)d)[i]; lo = (u64)v; hi = (u64)(v >> 63) ^ (1ull << 63); return true; }
    case HK_DICT8: case HK_DICT16: case HK_DICT32: {
        const i32 c = k.kind == HK_DICT8 ? (i32)((const signed char*)d)[i] : k.kind == HK_DICT16 ? (i32)((const short*)d)[i] : ((const i32*)d)[i];
        if (c < 0 || c >= k.n_rank) { lo = 0; return false; }
        lo = k.rank[c];
        return true;
    }
    default: lo = 0; return false;
    }
    lo = ((u64)s ^ (1ull << (k.bits - 1))) & sk_mask(k.bits); // sign flip of a value that fits `bits`
    return true;
}

// row i's fields as put(off, v, nb) calls (OR nb <= 64 bits of v at bit offset off); false if a dictionary code was out of range
template <typename Put> CB_HD bool sk_fields(const SortKeyCols& kc, i64 i, Put put) {
    bool ok = true;
    for (int c = 0; c < kc.n; c++) {
        const SortKeyCol& k = kc.col[c];
        const bool valid = !k.validity || ((k.validity[i >> 3] >> (i & 7)) & 1);
        if (k.has_null) put(k.off + k.bits, (valid == (bool)k.nulls_first) ? 1u : 0u, 1); // valid rows after NULLs iff nulls_first
        if (!valid) continue;
        u64 hi, lo;
        if (!sk_value(k, i, hi, lo)) ok = false;
        if (k.bits > 64) {
            if (k.desc) { hi = ~hi; lo = ~lo; }
            put(k.off, lo, 64);
            put(k.off + 64, hi & sk_mask(k.bits - 64), k.bits - 64);
        } else {
            if (k.desc) lo = ~lo & sk_mask(k.bits);
            put(k.off, lo, k.bits);
        }
    }
    return ok;
}

// OR row i's fields into w[0, kc.words) (zeroed by the caller); false if a dictionary code was out of range
CB_HD bool sk_row(const SortKeyCols& kc, i64 i, u64* w) {
    return sk_fields(kc, i, [&](int off, u64 v, int nb) { sk_put(w, kc.words, off, v, nb); });
}

// sk_row for a key of W words (W == kc.words) kept in registers: every word is addressed by a constant index
template <int W> CB_HD bool sk_row_reg(const SortKeyCols& kc, i64 i, u64 (&w)[W]) {
    return sk_fields(kc, i, [&](int off, u64 v, int nb) {
        const int lw = off >> 6, sh = off & 63;
        for (int j = 0; j < W; j++) {
            if (j == W - 1 - lw) w[j] |= v << sh;
            if (sh && sh + nb > 64 && j == W - 2 - lw) w[j] |= v >> (64 - sh);
        }
    });
}

// The join table's hash of a row key of W <= SK_MAX_WORDS words (k_join_insert / k_join_probe, aot_kernels.cu): each word in turn,
// word 0 first, XORed into the state and mixed by murmur3's fmix64.  A run's home slot is hash & (capacity - 1), its tag hash >> 32.
CB_HD u64 join_hash(const u64* k, int W) {
    u64 h = 0x9E3779B97F4A7C15ull;
CB_SK_UNROLL
    for (int j = 0; j < SK_MAX_WORDS; j++) {
        if (j >= W) break;
        h ^= k[j];
        h ^= h >> 33; h *= 0xff51afd7ed558ccdull; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 33; // murmur3 fmix64
    }
    return h;
}

// a join key has no NULL field: every field's null bit (nullmask, set on a valid value) is set
CB_HD bool join_no_null(const u64* k, const u64* nullmask, int W) {
    bool ok = true;
CB_SK_UNROLL
    for (int j = 0; j < SK_MAX_WORDS; j++)
        if (j < W) ok &= (k[j] & nullmask[j]) == nullmask[j];
    return ok;
}

} // namespace cb
#endif
