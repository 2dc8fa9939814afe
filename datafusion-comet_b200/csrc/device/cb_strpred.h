// cb_strpred.h -- one string predicate over one UTF-8 value (ptr, len), shared by the mask kernel k_str_pred (aot_kernels.cu), the
// planner, which compiles LIKE patterns with sp_like_compile (plan.cpp), and the host test driver strpred_test.cpp.
//
// Order is unsigned byte-lexicographic, a shorter prefix first (arrow-ord over Utf8; Spark UTF8String.compareTo).  LIKE follows the
// reference's LikeExpr (native/core/src/execution/expressions/strings.rs:36-50, arrow-string `like`): `%` matches any run of characters
// and `_` exactly one code point, both including '\n'; `\` escapes `%`, `_` and `\` only.
#ifndef CB_STRPRED_H
#define CB_STRPRED_H
#include "cb_math.h"

namespace cb {

enum StrOp { SP_EQ = 0, SP_NEQ, SP_LT, SP_LTEQ, SP_GT, SP_GTEQ, SP_IN, SP_LIKE, SP_STARTS, SP_ENDS, SP_CONTAINS };

// compiled LIKE pattern: one u16 per item, a literal byte (0..255), one code point (SP_ANY1) or a run of any length (SP_ANYN)
constexpr u16 SP_ANY1 = 256, SP_ANYN = 257;

// one predicate as the mask kernel reads it: literal i is lit[lit_off[i], lit_off[i + 1]) (IN: every member; the others: one)
struct StrPredDev {
    i32 op;
    i32 n_lits;
    const i32* lit_off;
    const u8* lit;
    const u16* pat;  // SP_LIKE: the compiled pattern
    i32 pat_len;
};

// LIKE pattern text -> items; returns the item count (<= n), or -1 for a `\` before anything but `%`, `_`, `\`, or at the end.
// Runs of `%` collapse into one SP_ANYN.
CB_HD int sp_like_compile(const u8* p, int n, u16* out) {
    int k = 0;
    for (int i = 0; i < n; i++) {
        const u8 c = p[i];
        if (c == '\\') {
            if (i + 1 >= n) return -1;
            const u8 e = p[++i];
            if (e != '%' && e != '_' && e != '\\') return -1;
            out[k++] = e;
        } else if (c == '%') {
            if (k == 0 || out[k - 1] != SP_ANYN) out[k++] = SP_ANYN;
        } else if (c == '_') out[k++] = SP_ANY1;
        else out[k++] = c;
    }
    return k;
}

// memcmp order, then length: <0, 0, >0
CB_HD int sp_compare(const u8* a, int na, const u8* b, int nb) {
    const int m = na < nb ? na : nb;
    for (int i = 0; i < m; i++)
        if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return na < nb ? -1 : na > nb ? 1 : 0;
}
CB_HD bool sp_bytes_at(const u8* s, const u8* b, int nb) {
    for (int i = 0; i < nb; i++)
        if (s[i] != b[i]) return false;
    return true;
}
CB_HD bool sp_contains(const u8* s, int n, const u8* b, int nb) {
    for (int i = 0; i + nb <= n; i++)
        if (sp_bytes_at(s + i, b, nb)) return true;
    return false;
}

// one code point forward from p (p < end) / back from q (q > lo): a lead byte and its continuation bytes 10xxxxxx
CB_HD int sp_next_cp(const u8* s, int p, int end) {
    p++;
    while (p < end && (s[p] & 0xc0) == 0x80) p++;
    return p;
}
CB_HD int sp_prev_cp(const u8* s, int q, int lo) {
    q--;
    while (q > lo && (s[q] & 0xc0) == 0x80) q--;
    return q;
}
// items pat[a, b) matched forward from p, never past end: the end of the match, or -1
CB_HD int sp_seg_fwd(const u8* s, int p, int end, const u16* pat, int a, int b) {
    for (int k = a; k < b; k++) {
        if (p >= end) return -1;
        if (pat[k] == SP_ANY1) p = sp_next_cp(s, p, end);
        else if (s[p] != pat[k]) return -1;
        else p++;
    }
    return p;
}
// items pat[a, b) matched backward so that they end at q, never before lo: the start of the match, or -1
CB_HD int sp_seg_back(const u8* s, int lo, int q, const u16* pat, int a, int b) {
    for (int k = b - 1; k >= a; k--) {
        if (q <= lo) return -1;
        if (pat[k] == SP_ANY1) q = sp_prev_cp(s, q, lo);
        else if (s[q - 1] != pat[k]) return -1;
        else q--;
    }
    return q;
}

// LIKE: the segments between SP_ANYN items.  The first is anchored at the start, the last at the end (matched backwards, so `_` steps
// over whole code points from the end); each middle one takes its leftmost match.  A segment matches a fixed number of code points,
// so the leftmost start also gives the earliest end, and greedy placement finds a match whenever one exists.
CB_HD bool sp_like(const u8* s, int n, const u16* pat, int np) {
    int first = 0;
    while (first < np && pat[first] != SP_ANYN) first++;
    if (first == np) return sp_seg_fwd(s, 0, n, pat, 0, np) == n;
    int p = sp_seg_fwd(s, 0, n, pat, 0, first);
    if (p < 0) return false;
    int last = np - 1;
    while (pat[last] != SP_ANYN) last--;
    const int q = sp_seg_back(s, p, n, pat, last + 1, np);
    if (q < 0) return false;
    int a = first + 1;
    while (a < last) {
        int b = a;
        while (pat[b] != SP_ANYN) b++;
        int e = -1;
        for (int start = p; start <= q; start = sp_next_cp(s, start, q)) {
            e = sp_seg_fwd(s, start, q, pat, a, b);
            if (e >= 0 || start == q) break;
        }
        if (e < 0) return false;
        p = e;
        a = b + 1;
    }
    return true;
}

// the predicate's value for a non-NULL string (IN: whether some member equals it; negation and the NULL rule are the caller's)
CB_HD bool sp_eval(const StrPredDev& d, const u8* s, int n) {
    if (d.op == SP_LIKE) return sp_like(s, n, d.pat, d.pat_len);
    if (d.op == SP_IN) {
        for (int i = 0; i < d.n_lits; i++) {
            const int nb = d.lit_off[i + 1] - d.lit_off[i];
            if (nb == n && sp_bytes_at(s, d.lit + d.lit_off[i], nb)) return true;
        }
        return false;
    }
    const u8* b = d.lit + d.lit_off[0];
    const int nb = d.lit_off[1] - d.lit_off[0];
    switch (d.op) {
    case SP_STARTS: return nb <= n && sp_bytes_at(s, b, nb);
    case SP_ENDS: return nb <= n && sp_bytes_at(s + (n - nb), b, nb);
    case SP_CONTAINS: return sp_contains(s, n, b, nb);
    default: break;
    }
    const int c = sp_compare(s, n, b, nb);
    switch (d.op) {
    case SP_EQ: return c == 0;
    case SP_NEQ: return c != 0;
    case SP_LT: return c < 0;
    case SP_LTEQ: return c <= 0;
    case SP_GT: return c > 0;
    default: return c >= 0;
    }
}

} // namespace cb
#endif
