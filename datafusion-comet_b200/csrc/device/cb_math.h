// cb_math.h -- integer / decimal / hash arithmetic shared by every comet_b200 kernel.
//
// Plain C++ with no includes so that the same text compiles three ways:
//   * under NVRTC as part of a JIT-specialised pipeline kernel (sm_90a),
//   * under nvcc for the ahead-of-time kernels (parquet decode, partition, hash table),
//   * under g++ (CB_HOST_TEST) so tests/ can check every function against the oracle on CPU.
//
// Semantics follow the reference (apache/datafusion-comet); each block cites the file:line of the
// Rust it replaces (paths relative to native/).
#ifndef CB_MATH_H
#define CB_MATH_H

#if defined(__CUDACC__) || defined(__CUDACC_RTC__)
#define CB_HD __host__ __device__ __forceinline__
#define CB_D __device__ __forceinline__
#else
#define CB_HD inline
#define CB_D inline
#endif

namespace cb {

typedef unsigned long long u64;
typedef long long i64;
typedef unsigned int u32;
typedef int i32;
typedef unsigned char u8;
typedef unsigned short u16;

// ------------------------------------------------------------------------------------------------
// 64x64 -> 128 primitives
// ------------------------------------------------------------------------------------------------
CB_HD u64 umulhi64(u64 a, u64 b) {
#if defined(__CUDA_ARCH__)
    return __umul64hi(a, b);
#else
    return (u64)(((unsigned __int128)a * b) >> 64);
#endif
}

// 128-bit two's-complement integer, Arrow Decimal128 layout (little-endian lo, hi).
struct
#if defined(__CUDACC__) || defined(__CUDACC_RTC__)
    __align__(16)
#endif
        i128 {
    u64 lo;
    i64 hi;
};

struct u128 {
    u64 lo, hi;
};
struct u256 {
    u64 w[4];
};

CB_HD i128 mk128(u64 lo, i64 hi) { i128 r; r.lo = lo; r.hi = hi; return r; }
CB_HD i128 i128_from_i64(i64 v) { return mk128((u64)v, v >> 63); }
CB_HD bool i128_is_neg(i128 a) { return a.hi < 0; }
CB_HD bool i128_eq(i128 a, i128 b) { return a.lo == b.lo && a.hi == b.hi; }
CB_HD bool i128_lt(i128 a, i128 b) { return a.hi < b.hi || (a.hi == b.hi && a.lo < b.lo); }
CB_HD bool i128_le(i128 a, i128 b) { return a.hi < b.hi || (a.hi == b.hi && a.lo <= b.lo); }
CB_HD i128 i128_add(i128 a, i128 b) { // wrapping
    i128 r; r.lo = a.lo + b.lo; r.hi = (i64)((u64)a.hi + (u64)b.hi + (r.lo < a.lo ? 1ull : 0ull)); return r;
}
CB_HD i128 i128_sub(i128 a, i128 b) { // wrapping
    i128 r; r.lo = a.lo - b.lo; r.hi = (i64)((u64)a.hi - (u64)b.hi - (a.lo < b.lo ? 1ull : 0ull)); return r;
}
CB_HD i128 i128_neg(i128 a) { return i128_sub(mk128(0, 0), a); }
// overflowing_add: returns true when the signed addition overflowed
CB_HD bool i128_add_overflow(i128 a, i128 b, i128& r) {
    r = i128_add(a, b);
    return ((a.hi ^ r.hi) & (b.hi ^ r.hi)) < 0;
}
CB_HD bool i128_sub_overflow(i128 a, i128 b, i128& r) {
    r = i128_sub(a, b);
    return ((a.hi ^ b.hi) & (a.hi ^ r.hi)) < 0;
}
CB_HD u128 i128_abs_u(i128 a) { // |a| as unsigned (|i128::MIN| = 2^127 is representable)
    if (a.hi < 0) a = i128_neg(a);
    u128 r; r.lo = a.lo; r.hi = (u64)a.hi; return r;
}
CB_HD bool i128_fits_i64(i128 a) { return a.hi == ((i64)a.lo >> 63); }

// full signed 64x64 -> 128 product
CB_HD i128 mul_i64_i64(i64 a, i64 b) {
    u64 lo = (u64)a * (u64)b;
    u64 hi = umulhi64((u64)a, (u64)b);
    if (a < 0) hi -= (u64)b;
    if (b < 0) hi -= (u64)a;
    return mk128(lo, (i64)hi);
}

CB_HD u256 umul_128x128(u128 a, u128 b) {
    u256 r;
    u64 p0l = a.lo * b.lo, p0h = umulhi64(a.lo, b.lo);
    u64 p1l = a.lo * b.hi, p1h = umulhi64(a.lo, b.hi);
    u64 p2l = a.hi * b.lo, p2h = umulhi64(a.hi, b.lo);
    u64 p3l = a.hi * b.hi, p3h = umulhi64(a.hi, b.hi);
    r.w[0] = p0l;
    u64 s = p0h + p1l; u64 c = s < p0h;
    u64 s2 = s + p2l; c += s2 < s;
    r.w[1] = s2;
    u64 t = p1h + p2h; u64 c2 = t < p1h;
    u64 t2 = t + p3l; c2 += t2 < t;
    u64 t3 = t2 + c; c2 += t3 < t2;
    r.w[2] = t3;
    r.w[3] = p3h + c2;
    return r;
}
CB_HD int u256_cmp(const u256& a, const u256& b) {
    for (int i = 3; i >= 0; i--) {
        if (a.w[i] != b.w[i]) return a.w[i] < b.w[i] ? -1 : 1;
    }
    return 0;
}
CB_HD bool u256_add(u256& a, const u256& b) { // returns carry out
    u64 c = 0;
    for (int i = 0; i < 4; i++) {
        u64 s = a.w[i] + b.w[i]; u64 c1 = s < a.w[i];
        u64 s2 = s + c; c1 += s2 < s;
        a.w[i] = s2; c = c1;
    }
    return c != 0;
}
CB_HD void u256_sub(u256& a, const u256& b) { // a >= b assumed
    u64 br = 0;
    for (int i = 0; i < 4; i++) {
        u64 d = a.w[i] - b.w[i]; u64 b1 = a.w[i] < b.w[i];
        u64 d2 = d - br; b1 += d < br;
        a.w[i] = d2; br = b1;
    }
}
// a *= m (m < 2^64); returns true on overflow past 256 bits
CB_HD bool u256_mul_small(u256& a, u64 m) {
    u64 carry = 0;
    for (int i = 0; i < 4; i++) {
        u64 lo = a.w[i] * m, hi = umulhi64(a.w[i], m);
        u64 s = lo + carry; hi += s < lo;
        a.w[i] = s; carry = hi;
    }
    return carry != 0;
}
// a /= d (d < 2^32), schoolbook over 32-bit digits; returns remainder
CB_HD u32 u256_div_small(u256& a, u32 d) {
    u64 rem = 0;
    for (int i = 3; i >= 0; i--) {
        u64 hi32 = a.w[i] >> 32, lo32 = a.w[i] & 0xffffffffull;
        u64 cur = (rem << 32) | hi32; u64 qh = cur / d; rem = cur % d;
        cur = (rem << 32) | lo32; u64 ql = cur / d; rem = cur % d;
        a.w[i] = (qh << 32) | ql;
    }
    return (u32)rem;
}
CB_HD u64 pow10_u64(int e) { u64 r = 1; for (int i = 0; i < e; i++) r *= 10; return r; }
CB_HD bool u256_mul_pow10(u256& a, int e) { // returns overflow
    bool o = false;
    while (e >= 19) { o |= u256_mul_small(a, 10000000000000000000ull); e -= 19; }
    if (e > 0) o |= u256_mul_small(a, pow10_u64(e));
    return o;
}
CB_HD void u256_div_pow10(u256& a, int e) { // truncating
    while (e >= 9) { u256_div_small(a, 1000000000u); e -= 9; }
    if (e > 0) u256_div_small(a, (u32)pow10_u64(e));
}
CB_HD u256 u256_pow10(int e) { u256 r; r.w[0] = 1; r.w[1] = r.w[2] = r.w[3] = 0; u256_mul_pow10(r, e); return r; }
CB_HD u256 u256_from_u128(u128 a) { u256 r; r.w[0] = a.lo; r.w[1] = a.hi; r.w[2] = r.w[3] = 0; return r; }

// ------------------------------------------------------------------------------------------------
// decimal precision bound:  |v| <= 10^p - 1      (spark-expr/src/utils.rs:332-336)
// ------------------------------------------------------------------------------------------------
CB_HD u128 pow10_u128(int p) { // p in [0,38]
    u128 r; r.lo = 1; r.hi = 0;
    for (int i = 0; i < p; i++) {
        u64 lo = r.lo * 10ull, hi = umulhi64(r.lo, 10ull) + r.hi * 10ull;
        r.lo = lo; r.hi = hi;
    }
    return r;
}
// bound = 10^p as (lo,hi); valid iff |v| < 10^p
CB_HD bool dec_fits(i128 v, u64 bound_lo, u64 bound_hi) {
    u128 a = i128_abs_u(v);
    return a.hi < bound_hi || (a.hi == bound_hi && a.lo < bound_lo);
}
CB_HD bool dec_fits_p(i128 v, int p) { u128 b = pow10_u128(p); return dec_fits(v, b.lo, b.hi); }

// ------------------------------------------------------------------------------------------------
// plain decimal arithmetic (arrow-arith 58.4.0 `decimal_op`, reached from planner.rs:1126):
// checked i128 operations; `err` is set when the i128 result overflows (arrow raises
// "Overflow happened on ...", which fails the query).
// ------------------------------------------------------------------------------------------------
CB_HD i128 i128_mul_checked(i128 a, i128 b, bool& err) {
    bool neg = (a.hi < 0) != (b.hi < 0);
    u256 p = umul_128x128(i128_abs_u(a), i128_abs_u(b));
    // magnitude must be <= 2^127-1 (or == 2^127 when negative)
    bool big = (p.w[2] | p.w[3]) != 0 || (p.w[1] >> 63) != 0;
    if (big) {
        bool is_min = neg && p.w[2] == 0 && p.w[3] == 0 && p.w[1] == 0x8000000000000000ull && p.w[0] == 0;
        if (!is_min) err = true;
    }
    i128 r = mk128(p.w[0], (i64)p.w[1]);
    return neg ? i128_neg(r) : r;
}
CB_HD i128 i128_mul_pow10_checked(i128 a, int e, bool& err) {
    if (e == 0) return a;
    u128 m = pow10_u128(e);
    return i128_mul_checked(a, mk128(m.lo, (i64)m.hi), err);
}
CB_HD i128 dec_add_plain(i128 l, int lup, i128 r, int rup, bool& err) {
    i128 a = i128_mul_pow10_checked(l, lup, err), b = i128_mul_pow10_checked(r, rup, err), o;
    if (i128_add_overflow(a, b, o)) err = true;
    return o;
}
CB_HD i128 dec_sub_plain(i128 l, int lup, i128 r, int rup, bool& err) {
    i128 a = i128_mul_pow10_checked(l, lup, err), b = i128_mul_pow10_checked(r, rup, err), o;
    if (i128_sub_overflow(a, b, o)) err = true;
    return o;
}

// ------------------------------------------------------------------------------------------------
// wide decimal arithmetic  (spark-expr/src/math_funcs/wide_decimal_binary_expr.rs:179-291,
// div_round_half_up :121-144, check_overflow_and_convert :335-350).  Sign-magnitude restatement of
// the i256 computation: |raw| < 2^254 for any Decimal128 inputs, so magnitudes never wrap.
// Returns false when the result is out of the output precision (NULL in Legacy/Try, error in ANSI).
//   scale_diff = natural_scale - s_out (>0: divide by 10^d HALF_UP, <0: multiply by 10^-d)
// ------------------------------------------------------------------------------------------------
CB_HD bool wide_finish(u256 mag, bool neg, int scale_diff, int p_out, i128& out) {
    if (scale_diff > 0) {
        // q = floor((|raw| + 10^d/2) / 10^d)  ==  truncated quotient rounded away from zero at >= half
        u256 half = u256_pow10(scale_diff - 1);
        u256_mul_small(half, 5);
        u256_add(mag, half);
        u256_div_pow10(mag, scale_diff);
    } else if (scale_diff < 0) {
        if (u256_mul_pow10(mag, -scale_diff)) return false; // astronomically out of range
    }
    u128 b = pow10_u128(p_out);
    if ((mag.w[2] | mag.w[3]) != 0) return false;
    if (!(mag.w[1] < b.hi || (mag.w[1] == b.hi && mag.w[0] < b.lo))) return false;
    i128 r = mk128(mag.w[0], (i64)mag.w[1]);
    out = neg ? i128_neg(r) : r;
    return true;
}
CB_HD bool wide_mul(i128 l, i128 r, int scale_diff, int p_out, i128& out) {
    bool neg = (l.hi < 0) != (r.hi < 0);
    u256 mag = umul_128x128(i128_abs_u(l), i128_abs_u(r));
    return wide_finish(mag, neg, scale_diff, p_out, out);
}
// l*10^lup (+/-) r*10^rup, then rescale by scale_diff
CB_HD bool wide_addsub(i128 l, int lup, i128 r, int rup, bool subtract, int scale_diff, int p_out, i128& out) {
    u256 a = u256_from_u128(i128_abs_u(l)), b = u256_from_u128(i128_abs_u(r));
    u256_mul_pow10(a, lup);
    u256_mul_pow10(b, rup);
    bool na = l.hi < 0, nb = (r.hi < 0) != subtract;
    bool neg;
    if (na == nb) { u256_add(a, b); neg = na; }
    else {
        int c = u256_cmp(a, b);
        if (c >= 0) { u256_sub(a, b); neg = na; }
        else { u256_sub(b, a); a = b; neg = nb; }
    }
    if ((a.w[0] | a.w[1] | a.w[2] | a.w[3]) == 0) neg = false;
    return wide_finish(a, neg, scale_diff, p_out, out);
}

// DecimalRescaleCheckOverflow (math_funcs/internal/decimal_rescale_check.rs:111-150):
// delta = s_out - s_in;  >0 multiply (checked), <0 divide HALF_UP via (v + sign*half)/divisor.
CB_HD bool dec_rescale_check(i128 v, int delta, int p_out, i128& out) {
    bool neg = v.hi < 0;
    u256 mag = u256_from_u128(i128_abs_u(v));
    return wide_finish(mag, neg, -delta, p_out, out);
}

// 128 / 64 signed division used by AVG(decimal).evaluate (agg_funcs/avg_decimal.rs:670-689):
//   value = sum*scaler (checked); (div, rem) = value.div_rem(count); half = div_ceil(count,2);
//   value>=0 && rem>=half -> div+1 ; value<0 && rem<=-half -> div-1.  NULL if out of target range.
CB_HD bool avg_decimal_eval(i128 sum, i64 count, int scaler_exp, int target_p, i128& out) {
    bool err = false;
    i128 value = i128_mul_pow10_checked(sum, scaler_exp, err);
    if (err) return false;
    bool neg = value.hi < 0;
    u128 mag = i128_abs_u(value);
    // divide 128-bit magnitude by count (count > 0) with 32-bit digits when count < 2^32, else bitwise
    u64 c = (u64)count;
    u128 q; u64 rem;
    if (c <= 0xffffffffull) {
        u32 d = (u32)c; u64 r = 0; u64 limbs[2] = {mag.lo, mag.hi};
        for (int i = 1; i >= 0; i--) {
            u64 hi32 = limbs[i] >> 32, lo32 = limbs[i] & 0xffffffffull;
            u64 cur = (r << 32) | hi32; u64 qh = cur / d; r = cur % d;
            cur = (r << 32) | lo32; u64 ql = cur / d; r = cur % d;
            limbs[i] = (qh << 32) | ql;
        }
        q.lo = limbs[0]; q.hi = limbs[1]; rem = r;
    } else {
        q.lo = q.hi = 0; u64 r = 0;
        for (int bit = 127; bit >= 0; bit--) {
            u64 top = r >> 63;
            r = (r << 1) | ((bit >= 64 ? (mag.hi >> (bit - 64)) : (mag.lo >> bit)) & 1ull);
            if (top || r >= c) { r -= c; if (bit >= 64) q.hi |= 1ull << (bit - 64); else q.lo |= 1ull << bit; }
        }
        rem = r;
    }
    u64 half = c / 2 + (c & 1ull);
    if (rem >= half) { q.lo += 1; if (q.lo == 0) q.hi += 1; } // symmetric for negative values
    i128 r128 = mk128(q.lo, (i64)q.hi);
    if (neg) r128 = i128_neg(r128);
    if (!dec_fits_p(r128, target_p)) return false;
    out = r128;
    return true;
}


// ---- fast paths: both operands fit in 64 bits (every d(p<=18) value does) ----------------------------
CB_HD i128 dec_mul_plain(i128 a, i128 b, bool& err) {
    if (i128_fits_i64(a) && i128_fits_i64(b)) return mul_i64_i64((i64)a.lo, (i64)b.lo); // cannot overflow i128
    return i128_mul_checked(a, b, err);
}
CB_HD bool wide_mul_fast(i128 l, i128 r, int scale_diff, int p_out, i128& out) {
    if (scale_diff == 0 && i128_fits_i64(l) && i128_fits_i64(r)) {
        i128 p = mul_i64_i64((i64)l.lo, (i64)r.lo);
        if (!dec_fits_p(p, p_out)) return false;
        out = p;
        return true;
    }
    return wide_mul(l, r, scale_diff, p_out, out);
}
// wrapping 128-bit products: exact whenever the true product is known to fit (range-proved by codegen)
CB_HD i128 mul_i128_i64(i128 a, i64 b) {
    u64 ub = (u64)b;
    u64 lo = a.lo * ub;
    u64 hi = umulhi64(a.lo, ub) + (u64)a.hi * ub;
    if (b < 0) hi -= a.lo; // signed correction for the multiplier
    return mk128(lo, (i64)hi);
}
CB_HD i128 mul_i128_wrap(i128 a, i128 b) {
    u64 lo = a.lo * b.lo;
    u64 hi = umulhi64(a.lo, b.lo) + a.lo * (u64)b.hi + (u64)a.hi * b.lo;
    return mk128(lo, (i64)hi);
}
CB_HD bool i64_add_overflow(i64 a, i64 b, i64& r) { r = (i64)((u64)a + (u64)b); return ((a ^ r) & (b ^ r)) < 0; }
CB_HD bool i64_sub_overflow(i64 a, i64 b, i64& r) { r = (i64)((u64)a - (u64)b); return ((a ^ b) & (a ^ r)) < 0; }
CB_HD bool i64_mul_overflow(i64 a, i64 b, i64& r) { i128 p = mul_i64_i64(a, b); r = (i64)p.lo; return !i128_fits_i64(p); }


// ------------------------------------------------------------------------------------------------
// decimal division (spark-expr/src/math_funcs/div.rs:75-190 spark_decimal_div_internal)
//   Decimal(p1,s1) / Decimal(p2,s2) -> Decimal(p3,s3):  q = trunc((l * 10^l_exp) / (r * 10^r_exp)) with
//   l_exp = max(0, s2+s3+1-s1), r_exp = max(0, s1-(s2+s3+1)), i.e. one digit more than the result keeps, then
//   HALF_UP on that digit: (q +- 5) / 10 (integral division keeps q).  The reference switches to BigInt when
//   the scaled operands leave 38 digits; here ONE multi-limb routine covers both (numerator up to 384 bits).
// ------------------------------------------------------------------------------------------------
#define CB_DIV_NN 12 // 32-bit limbs of the numerator:  |l| < 2^127 times 10^77 < 2^256
#define CB_DIV_ND 8  //                   the divisor:  |r| < 2^127 times 10^38 < 2^127
CB_HD int limbs_len(const u32* a, int n) { while (n > 0 && a[n - 1] == 0) n--; return n; }
CB_HD void limbs_mul_small(u32* a, int n, u32 m) {
    u64 carry = 0;
    for (int i = 0; i < n; i++) { u64 t = (u64)a[i] * m + carry; a[i] = (u32)t; carry = t >> 32; }
}
CB_HD void limbs_mul_pow10(u32* a, int n, int e) {
    while (e >= 9) { limbs_mul_small(a, n, 1000000000u); e -= 9; }
    if (e > 0) limbs_mul_small(a, n, (u32)pow10_u64(e));
}
CB_HD u32 limbs_div_small(u32* a, int n, u32 d) { // in place, returns the remainder
    u64 rem = 0;
    for (int i = n - 1; i >= 0; i--) { u64 cur = (rem << 32) | a[i]; a[i] = (u32)(cur / d); rem = cur % d; }
    return (u32)rem;
}
CB_HD int clz32(u32 x) {
#if defined(__CUDA_ARCH__)
    return __clz((int)x);
#else
    return x ? __builtin_clz(x) : 32;
#endif
}
// q = n / d (truncating), Knuth TAOCP vol. 2 algorithm D in base 2^32.  n: CB_DIV_NN limbs, d: CB_DIV_ND limbs, d != 0.
CB_HD void limbs_div(const u32* n, const u32* d, u32* q) {
    for (int i = 0; i < CB_DIV_NN; i++) q[i] = 0;
    const int m = limbs_len(d, CB_DIV_ND), ln = limbs_len(n, CB_DIV_NN);
    if (ln < m) return;
    if (m == 1) {
        for (int i = 0; i < CB_DIV_NN; i++) q[i] = n[i];
        limbs_div_small(q, CB_DIV_NN, d[0]);
        return;
    }
    const int s = clz32(d[m - 1]);
    u32 dn[CB_DIV_ND], un[CB_DIV_NN + 1];
    for (int i = m - 1; i > 0; i--) dn[i] = s ? (d[i] << s) | (d[i - 1] >> (32 - s)) : d[i];
    dn[0] = d[0] << s;
    un[ln] = s ? n[ln - 1] >> (32 - s) : 0;
    for (int i = ln - 1; i > 0; i--) un[i] = s ? (n[i] << s) | (n[i - 1] >> (32 - s)) : n[i];
    un[0] = n[0] << s;
    for (int j = ln - m; j >= 0; j--) {
        const u64 num = ((u64)un[j + m] << 32) | un[j + m - 1];
        u64 qhat = num / dn[m - 1], rhat = num % dn[m - 1];
        while (qhat >= (1ull << 32) || qhat * dn[m - 2] > ((rhat << 32) | un[j + m - 2])) {
            qhat--;
            rhat += dn[m - 1];
            if (rhat >= (1ull << 32)) break;
        }
        i64 borrow = 0;
        u64 carry = 0;
        for (int i = 0; i < m; i++) { // un[j..j+m] -= qhat * dn
            const u64 p = qhat * dn[i] + carry;
            carry = p >> 32;
            const i64 t = (i64)un[i + j] - borrow - (i64)(p & 0xffffffffull);
            un[i + j] = (u32)t;
            borrow = t < 0 ? 1 : 0;
        }
        const i64 t = (i64)un[j + m] - borrow - (i64)carry;
        un[j + m] = (u32)t;
        if (t < 0) { // qhat was one too large: add the divisor back
            qhat--;
            u64 c = 0;
            for (int i = 0; i < m; i++) { const u64 sum = (u64)un[i + j] + dn[i] + c; un[i + j] = (u32)sum; c = sum >> 32; }
            un[j + m] += (u32)c;
        }
        q[j] = (u32)qhat;
    }
}
// returns false when r == 0 (`out` = 0: the reference's unreachable fallback; ANSI callers raise DIVIDE_BY_ZERO).
// fits_i64: the result fits a LONG (MathExpr.check_divide_overflow of integral division).
CB_HD bool dec_div(i128 l, i128 r, int l_exp, int r_exp, bool integral, i128& out, bool& fits_i64) {
    out = mk128(0, 0);
    fits_i64 = true;
    if (r.lo == 0 && r.hi == 0) return false;
    const bool neg = (l.hi < 0) != (r.hi < 0);
    const u128 la = i128_abs_u(l), ra = i128_abs_u(r);
    u32 n[CB_DIV_NN], d[CB_DIV_ND], q[CB_DIV_NN];
    for (int i = 0; i < CB_DIV_NN; i++) n[i] = 0;
    for (int i = 0; i < CB_DIV_ND; i++) d[i] = 0;
    n[0] = (u32)la.lo; n[1] = (u32)(la.lo >> 32); n[2] = (u32)la.hi; n[3] = (u32)(la.hi >> 32);
    d[0] = (u32)ra.lo; d[1] = (u32)(ra.lo >> 32); d[2] = (u32)ra.hi; d[3] = (u32)(ra.hi >> 32);
    limbs_mul_pow10(n, CB_DIV_NN, l_exp);
    limbs_mul_pow10(d, CB_DIV_ND, r_exp);
    limbs_div(n, d, q);
    if (!integral) { // (div + 5) / 10 on the magnitude == (div -+ 5) / 10 truncating toward zero
        u64 c = 5;
        for (int i = 0; i < CB_DIV_NN && c; i++) { const u64 t = (u64)q[i] + c; q[i] = (u32)t; c = t >> 32; }
        limbs_div_small(q, CB_DIV_NN, 10u);
    }
    // BigInt::to_i128().unwrap_or(i128::MAX): magnitudes past 2^127 - 1 (2^127 when negative) become the positive sentinel
    bool big = false;
    for (int i = 4; i < CB_DIV_NN; i++) big = big || q[i] != 0;
    const u64 qlo = ((u64)q[1] << 32) | q[0], qhi = ((u64)q[3] << 32) | q[2];
    if (!big && (qhi >> 63) != 0) big = !(neg && qhi == 0x8000000000000000ull && qlo == 0);
    if (big) { out = mk128(~0ull, 0x7fffffffffffffffll); fits_i64 = false; return true; }
    out = mk128(qlo, (i64)qhi);
    if (neg) out = i128_neg(out);
    fits_i64 = i128_fits_i64(out);
    return true;
}
// integer division, truncating (Rust `/`): err = 1 divide by zero, 2 overflow (MIN / -1)
CB_HD i64 i64_div_checked(i64 a, i64 b, int bits, int& err) {
    err = 0;
    if (b == 0) { err = 1; return 0; }
    const i64 mn = bits == 64 ? (i64)0x8000000000000000ll : -((i64)1 << (bits - 1));
    if (a == mn && b == -1) { err = 2; return mn; }
    return a / b;
}

// ---- overflow certificate for decimal sums ------------------------------------------------------
// The reference adds row by row and nulls the sum as soon as a running prefix leaves the precision
// (agg_funcs/sum_decimal.rs:418-439).  A parallel sum reproduces that exactly whenever no ordering
// of the addends can overflow: n * max|v| <= 10^p - 1.
// host certificate h (agg.cpp AggNode::certificate, from the observed input ranges):
//   0: n * max|v| <= 10^p - 1          -> no ordering can overflow, the exact total is the answer
//   1: n * max|v| <  2^127             -> the 128-bit total is exact; if IT is out of range every ordering
//                                         overflows (the last prefix is the total), otherwise order-dependent
//   2: the 128-bit total may have wrapped
// returns 0 fits, 1 overflows (NULL / ANSI error), 2 order-dependent (cannot be decided without row order)
CB_HD i128 i128_abs_of_i64(i64 v) { i128 m = i128_from_i64(v); return m.hi < 0 ? i128_neg(m) : m; } // |v| as 128 bits (|i64::MIN| fits)
// the host certificate, per GROUP: n = addends of this group, B = bound on the magnitude of any addend (lo, hi; hi = ~0: none)
CB_HD int cert_level(i64 n, u64 blo, u64 bhi, int p) {
    if (n <= 0) return 0;
    if (bhi == ~0ull) return 2;
    const bool twos = (bhi >> 63) != 0;   // flag set by the host when B comes straight from a column's value mask (see below)
    bhi &= ~(1ull << 63);
    const u64 m = (u64)n;
    const u64 p0 = blo * m, c0 = umulhi64(blo, m);
    const u64 q = bhi * m, p1 = q + c0;
    const u64 p2 = umulhi64(bhi, m) + (p1 < q ? 1ull : 0ull);
    // n * B >= 2^127: the 128-bit total may have wrapped.  When B = 2^bits is the two's-complement bound of a column's value mask,
    // every addend lies in [-B, B - 1], the total in [-n*B, n*B - n], and n * B == 2^127 exactly is still exact.
    if (p2 != 0 || ((p1 >> 63) != 0 && !(twos && p1 == (1ull << 63) && p0 == 0))) return 2;
    const u128 mx = pow10_u128(p);
    return (p1 < mx.hi || (p1 == mx.hi && p0 < mx.lo)) ? 0 : 1;   // n * B <= 10^p - 1 ?
}
CB_HD int sum_cert(int h, bool total_fits) {
    if (h == 0) return total_fits ? 0 : 1;
    if (h == 1 && !total_fits) return 1;
    return 2;
}

// ------------------------------------------------------------------------------------------------
// Spark murmur3  (spark-expr/src/hash_funcs/murmur3.rs:73-137; per-type rules hash_funcs/utils.rs)
// ------------------------------------------------------------------------------------------------
CB_HD u32 rotl32(u32 x, int r) { return (x << r) | (x >> (32 - r)); }
CB_HD u32 mm3_mix_k1(u32 k1) { k1 *= 0xcc9e2d51u; k1 = rotl32(k1, 15); k1 *= 0x1b873593u; return k1; }
CB_HD u32 mm3_mix_h1(u32 h1, u32 k1) { h1 ^= k1; h1 = rotl32(h1, 13); return h1 * 5u + 0xe6546b64u; }
CB_HD u32 mm3_fmix(u32 h1, u32 len) {
    h1 ^= len; h1 ^= h1 >> 16; h1 *= 0x85ebca6bu; h1 ^= h1 >> 13; h1 *= 0xc2b2ae35u; h1 ^= h1 >> 16;
    return h1;
}
CB_HD u32 mm3_i32(i32 v, u32 seed) { return mm3_fmix(mm3_mix_h1(seed, mm3_mix_k1((u32)v)), 4u); }
CB_HD u32 mm3_i64(i64 v, u32 seed) {
    u32 h = mm3_mix_h1(seed, mm3_mix_k1((u32)(u64)v));
    h = mm3_mix_h1(h, mm3_mix_k1((u32)((u64)v >> 32)));
    return mm3_fmix(h, 8u);
}
CB_HD u32 mm3_i128(i128 v, u32 seed) { // d(p>18): 16 little-endian bytes (utils.rs:199-226)
    u32 h = mm3_mix_h1(seed, mm3_mix_k1((u32)v.lo));
    h = mm3_mix_h1(h, mm3_mix_k1((u32)(v.lo >> 32)));
    h = mm3_mix_h1(h, mm3_mix_k1((u32)(u64)v.hi));
    h = mm3_mix_h1(h, mm3_mix_k1((u32)((u64)v.hi >> 32)));
    return mm3_fmix(h, 16u);
}
CB_HD u32 mm3_bytes(const u8* data, i32 len, u32 seed) {
    i32 aligned = len - len % 4;
    u32 h1 = seed;
    for (i32 i = 0; i < aligned; i += 4) {
        u32 w = (u32)data[i] | ((u32)data[i + 1] << 8) | ((u32)data[i + 2] << 16) | ((u32)data[i + 3] << 24);
        h1 = mm3_mix_h1(h1, mm3_mix_k1(w));
    }
    for (i32 i = aligned; i < len; i++) h1 = mm3_mix_h1(h1, mm3_mix_k1((u32)(i32)(signed char)data[i]));
    return mm3_fmix(h1, (u32)len);
}
CB_HD u32 pmod_u32(u32 hash, u32 n) { // shuffle/src/comet_partitioning.rs:51-57
    i32 h = (i32)hash, m = (i32)n;
    i32 r = h % m;
    return (u32)(r < 0 ? (r + m) % m : r);
}

// ------------------------------------------------------------------------------------------------
// IEEE-754 totalOrder keys: arrow-ord 58.4.0 `cmp` compares floats by totalOrder
// (reached from planner/macros.rs:96-98 via DataFusion BinaryExpr).
// ------------------------------------------------------------------------------------------------
CB_HD i64 f64_total_key(u64 bits) { i64 b = (i64)bits; return b ^ (i64)(((u64)(b >> 63)) >> 1); }
CB_HD i32 f32_total_key(u32 bits) { i32 b = (i32)bits; return b ^ (i32)(((u32)(b >> 31)) >> 1); }

// Float negation = sign-bit flip, exact for NaN (sign and payload) like Rust's `-x` / arrow-arith `neg`.
// On the device a plain `-x` (and any xor the optimiser can recognise as fneg) becomes neg.f64, which the
// hardware executes as an add that returns the canonical +qNaN for NaN inputs -- so the
// flip is done in opaque integer PTX.
CB_HD double f64_neg(double x) {
#if defined(__CUDA_ARCH__)
    unsigned long long b = (unsigned long long)__double_as_longlong(x), r;
    asm("xor.b64 %0, %1, 0x8000000000000000;" : "=l"(r) : "l"(b));
    return __longlong_as_double((long long)r);
#else
    u64 b; __builtin_memcpy(&b, &x, 8); b ^= 0x8000000000000000ull; __builtin_memcpy(&x, &b, 8); return x;
#endif
}
CB_HD float f32_neg(float x) {
#if defined(__CUDA_ARCH__)
    unsigned int b = (unsigned int)__float_as_int(x), r;
    asm("xor.b32 %0, %1, 0x80000000;" : "=r"(r) : "r"(b));
    return __int_as_float((int)r);
#else
    u32 b; __builtin_memcpy(&b, &x, 4); b ^= 0x80000000u; __builtin_memcpy(&x, &b, 4); return x;
#endif
}

// Two's-complement wrap of v to a `bits`-wide integer (8, 16 or 32), sign-extended, by masking and
// re-biasing: arrow-arith's wrapping add / sub / mul / neg of Int8 / Int16 / Int32.
CB_HD i64 wrap_int(i64 v, int bits) {
    const u64 m = (1ull << bits) - 1, s = 1ull << (bits - 1);
    return (i64)((((u64)v & m) ^ s) - s);
}

// NaN bits of Float32 arithmetic.  The reference runs on x86 (SSE), where a NaN result is the first
// NaN operand made quiet (payload and sign kept) and an invalid operation without a NaN operand
// (Inf - Inf, 0 * Inf, 0 / 0) returns the default NaN 0xFFC00000.  The H100's .f32 add / sub / mul /
// div return the canonical NaN 0x7FFFFFFF in all those cases (its .f64 arithmetic and the f32 -> f64
// conversion already give the x86 bits), so the emitter passes every Float32 result `r` of `a op b`
// through this rule.  Non-NaN results are returned unchanged.
CB_HD float f32_x86_nan(float a, float b, float r) {
#if defined(__CUDA_ARCH__)
    const u32 rb = __float_as_uint(r), ab = __float_as_uint(a), bb = __float_as_uint(b);
#else
    u32 rb, ab, bb; __builtin_memcpy(&rb, &r, 4); __builtin_memcpy(&ab, &a, 4); __builtin_memcpy(&bb, &b, 4);
#endif
    if ((rb & 0x7FFFFFFFu) <= 0x7F800000u) return r;
    const u32 out = (ab & 0x7FFFFFFFu) > 0x7F800000u ? ab | 0x00400000u : (bb & 0x7FFFFFFFu) > 0x7F800000u ? bb | 0x00400000u : 0xFFC00000u;
#if defined(__CUDA_ARCH__)
    return __uint_as_float(out);
#else
    float f; __builtin_memcpy(&f, &out, 4); return f;
#endif
}

// ------------------------------------------------------------------------------------------------
// double-double accumulation (float aggregates: result within 1 ULP of the exact sum)
// ------------------------------------------------------------------------------------------------
struct dd { double hi, lo; };
CB_HD void dd_add_double(dd& a, double x) { // Knuth TwoSum + renormalise
    double s = a.hi + x;
    if (s - s != 0.0) { a.hi = s; a.lo = 0.0; return; } // inf / NaN: plain IEEE propagation
    double bb = s - a.hi;
    double e = (a.hi - (s - bb)) + (x - bb);
    e += a.lo;
    double hi = s + e;
    a.lo = e - (hi - s);
    a.hi = hi;
}
CB_HD void dd_add_dd(dd& a, dd b) {
    double s = a.hi + b.hi;
    if (s - s != 0.0) { a.hi = s; a.lo = 0.0; return; }
    double bb = s - a.hi;
    double e = (a.hi - (s - bb)) + (b.hi - bb);
    e += a.lo + b.lo;
    double hi = s + e;
    a.lo = e - (hi - s);
    a.hi = hi;
}

} // namespace cb
#endif // CB_MATH_H
