// ranges.h -- magnitude bounds of decimal expressions.
//
// Given |column c| <= col_maxabs[c] this computes a bound B(e) with |e| <= B(e) for every row, following
// the exact arithmetic the kernels perform.  Used twice:
//   * codegen.cpp: with ASSUMED (and in-kernel validated) column bounds, to pick 64-bit arithmetic and
//     drop checks that provably never fire (CheckOverflow, i128 overflow, wide-decimal bound);
//   * agg.cpp: with OBSERVED column bounds (OR-masks the kernels accumulate over every valid input
//     value), to certify that a parallel decimal SUM cannot overflow for any row order, which is what
//     makes it bit-identical to the reference's row-by-row accumulation
//     (native/spark-expr/src/agg_funcs/sum_decimal.rs:418-439).
#pragma once
#include "plan.h"

namespace cb200 {

typedef unsigned __int128 u128r;
static const u128r RSAT = (u128r)1 << 127; // "unbounded"

inline u128r r_mul(u128r a, u128r b) {
    if (a == 0 || b == 0) return 0;
    if (a >= RSAT || b >= RSAT || a > RSAT / b) return RSAT;
    u128r p = a * b;
    return p >= RSAT ? RSAT : p;
}
inline u128r r_add(u128r a, u128r b) {
    if (a >= RSAT || b >= RSAT || a + b >= RSAT) return RSAT;
    return a + b;
}
inline u128r r_pow10(int e) {
    u128r r = 1;
    for (int i = 0; i < e; i++) r = r_mul(r, 10);
    return r;
}
inline u128r r_prec_max(int precision) { return r_pow10(precision) - 1; } // 10^p - 1
inline u128r r_rescale(u128r b, int scale_diff) { // scale_diff > 0: divide by 10^d (HALF_UP), < 0: multiply
    if (b >= RSAT) return RSAT;
    if (scale_diff > 0) return b / r_pow10(scale_diff) + 1;
    if (scale_diff < 0) return r_mul(b, r_pow10(-scale_diff));
    return b;
}
inline int r_bitlen(u128r v) { int n = 0; while (v) { n++; v >>= 1; } return n; }

// raw (pre-check) bound of a decimal binary op
inline u128r r_binary_raw(const Expr& e, u128r L, u128r R) {
    const DType &lt = e.children[0]->type, &rt = e.children[1]->type;
    if (e.kind == ExprKind::Mul) return r_mul(L, R);
    int ms = std::max(lt.scale, rt.scale);
    return r_add(r_mul(L, r_pow10(ms - lt.scale)), r_mul(R, r_pow10(ms - rt.scale)));
}

inline u128r expr_maxabs(const Expr& e, const std::vector<u128r>& col_maxabs) {
    auto child = [&](int i) { return expr_maxabs(*e.children[(size_t)i], col_maxabs); };
    if (!e.type.is_decimal()) return RSAT;
    switch (e.kind) {
    case ExprKind::Literal: {
        if (e.lit_null) return 0;
        __int128 v = (__int128)e.lit_dec;
        return (u128r)(v < 0 ? -v : v);
    }
    case ExprKind::Bound: return e.index >= 0 && e.index < (int)col_maxabs.size() ? col_maxabs[(size_t)e.index] : RSAT;
    case ExprKind::Add: case ExprKind::Sub: case ExprKind::Mul: {
        if (!e.children[0]->type.is_decimal() || !e.children[1]->type.is_decimal()) return RSAT;
        u128r raw = r_binary_raw(e, child(0), child(1));
        if (!e.wide_decimal) return raw;
        const DType &lt = e.children[0]->type, &rt = e.children[1]->type;
        int natural = e.kind == ExprKind::Mul ? lt.scale + rt.scale : std::max(lt.scale, rt.scale);
        return std::min(r_rescale(raw, natural - e.type.scale), r_prec_max(e.type.precision)); // overflow -> NULL
    }
    case ExprKind::CheckOverflow: return std::min(child(0), r_prec_max(e.type.precision));
    case ExprKind::Cast:
        if (e.children[0]->type.is_decimal())
            return std::min(r_rescale(child(0), e.children[0]->type.scale - e.type.scale), r_prec_max(e.type.precision));
        return r_prec_max(e.type.precision);
    case ExprKind::UnaryMinus: return child(0);
    case ExprKind::If: return std::max(child(1), child(2));
    default: return RSAT;
    }
}

} // namespace cb200
