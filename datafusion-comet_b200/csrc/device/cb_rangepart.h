// cb_rangepart.h -- the partition id of a row under range partitioning: the number of boundary rows less than or equal to the row,
// both as packed row keys (device/cb_sortkey.h), shared by the kernel k_range_pids (aot_kernels.cu), the planner's check of the
// boundary order and the host test driver rangepart_test.cpp.
//
// Boundary rows are `W` 64-bit words each, word 0 the most significant, in non-decreasing order.  When all of them fit in a CTA's shared
// memory the search runs there.  Otherwise the kernel stages a sampled top level: sample t is boundary row ((t + 1) << shift) - 1.  The
// count c of samples <= the row says that boundary rows [0, c << shift) are <= it and rows from ((c + 1) << shift) - 1 on are not, so
// the search ends in the 2^shift - 1 rows between, read from global memory.
#ifndef CB_RANGEPART_H
#define CB_RANGEPART_H
#include "cb_math.h"

namespace cb {

// a <= b over W words, word 0 first (W a constant: a key in registers stays there)
template <int W> CB_HD bool rp_le(const u64* a, const u64* b) {
    for (int j = 0; j < W; j++)
        if (a[j] != b[j]) return a[j] < b[j];
    return true;
}

// the number of rows of rows[0, n) (W words each, non-decreasing) that are <= key
template <int W> CB_HD u32 rp_upper(const u64* rows, u32 n, const u64* key) {
    u32 lo = 0, len = n;
    while (len > 0) {
        const u32 half = len >> 1;
        if (rp_le<W>(rows + (u64)(lo + half) * W, key)) { lo += half + 1; len -= half + 1; }
        else len = half;
    }
    return lo;
}

// the number of the nb boundary rows that are <= key.  top: shift == 0: the boundary rows themselves (n_top = nb); else the n_top =
// nb >> shift samples of them.  bounds: all boundary rows (read only when shift > 0).
template <int W> CB_HD u32 rp_pid(const u64* top, u32 n_top, int shift, const u64* bounds, u32 nb, const u64* key) {
    const u32 c = rp_upper<W>(top, n_top, key);
    if (shift == 0) return c;
    const u32 lo = c << shift, hi = lo + (1u << shift) - 1u < nb ? lo + (1u << shift) - 1u : nb;
    return lo + rp_upper<W>(bounds + (u64)lo * W, hi - lo, key);
}

// the shift of the sampled top level for nb boundary rows of W words when `budget` bytes of shared memory hold the top level
CB_HD int rp_shift(u32 nb, int W, u32 budget) {
    int s = 0;
    while ((u64)(nb >> s) * W * 8 > budget) s++;
    return s;
}

} // namespace cb

#ifndef __CUDA_ARCH__
#include <algorithm>
#include <string>
#include <vector>
namespace cb {
// The string field of a range key is a rank against the distinct boundary strings of that key, sorted by unsigned bytes as
// b_0 < b_1 < ...: b_j packs as 2j + 1, any other string s as 2 * #{b_j < s}, so it lands between the bounds it falls between and a
// string equal to a bound packs as the bound does.  rank[code] for the dictionary `values` (one entry more, unused).
inline std::vector<u32> rp_string_ranks(const std::vector<std::string>& values, const std::vector<std::string>& sorted_bounds) {
    std::vector<u32> rank(values.size() + 1, 0);
    for (size_t i = 0; i < values.size(); i++) {
        const auto it = std::lower_bound(sorted_bounds.begin(), sorted_bounds.end(), values[i]); // std::string: unsigned byte order
        const u32 below = (u32)(it - sorted_bounds.begin());
        rank[i] = 2 * below + (it != sorted_bounds.end() && *it == values[i] ? 1u : 0u);
    }
    return rank;
}
} // namespace cb
#endif
#endif
