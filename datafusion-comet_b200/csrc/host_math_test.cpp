// host_math_test.cpp -- compiles device/cb_math.h for the HOST so tests/test_cb_math_host.py can
// check every arithmetic routine against the oracle on CPU.  Test-only; not part of libcomet_b200.so.
#define CB_HOST_TEST 1
#include "device/cb_math.h"
#include "device/cb_snappy.h"
#include <cstdint>
using namespace cb;
extern "C" {
// op: 0 add 1 sub 2 mul ; returns valid bytes
void hm_wide(int op, int64_t n, const i128* l, int s1, const i128* r, int s2, int p_out, int s_out, i128* out,
             uint8_t* outv) {
    for (int64_t i = 0; i < n; i++) {
        i128 o = mk128(0, 0);
        bool ok;
        if (op == 2) ok = wide_mul(l[i], r[i], (s1 + s2) - s_out, p_out, o);
        else {
            int ms = s1 > s2 ? s1 : s2;
            ok = wide_addsub(l[i], ms - s1, r[i], ms - s2, op == 1, ms - s_out, p_out, o);
        }
        out[i] = ok ? o : mk128(0, 0);
        outv[i] = ok;
    }
}
int hm_plain(int op, int64_t n, const i128* l, int s1, const i128* r, int s2, i128* out) {
    bool err = false;
    int rs = s1 > s2 ? s1 : s2;
    for (int64_t i = 0; i < n; i++) {
        if (op == 2) out[i] = i128_mul_checked(l[i], r[i], err);
        else if (op == 0) out[i] = dec_add_plain(l[i], rs - s1, r[i], rs - s2, err);
        else out[i] = dec_sub_plain(l[i], rs - s1, r[i], rs - s2, err);
    }
    return err;
}
void hm_fits(int64_t n, const i128* v, int p, uint8_t* out) {
    for (int64_t i = 0; i < n; i++) out[i] = dec_fits_p(v[i], p);
}
void hm_rescale(int64_t n, const i128* v, int s_in, int p_out, int s_out, i128* out, uint8_t* outv) {
    for (int64_t i = 0; i < n; i++) {
        i128 o = mk128(0, 0);
        bool ok = dec_rescale_check(v[i], s_out - s_in, p_out, o);
        out[i] = ok ? o : mk128(0, 0);
        outv[i] = ok;
    }
}
void hm_avg(int64_t n, const i128* sum, const int64_t* count, int scaler_exp, int tp, i128* out, uint8_t* outv) {
    for (int64_t i = 0; i < n; i++) {
        i128 o = mk128(0, 0);
        bool ok = avg_decimal_eval(sum[i], count[i], scaler_exp, tp, o);
        out[i] = ok ? o : mk128(0, 0);
        outv[i] = ok;
    }
}
// decimal_div: returns 0 ok, 1 divide by zero; fits = result fits i64
void hm_dec_div(int64_t n, const i128* l, const i128* r, int l_exp, int r_exp, int integral, i128* out, uint8_t* zero, uint8_t* fits) {
    for (int64_t i = 0; i < n; i++) {
        bool f = true;
        zero[i] = dec_div(l[i], r[i], l_exp, r_exp, integral != 0, out[i], f) ? 0 : 1;
        fits[i] = f;
    }
}
void hm_mm3_i32(int64_t n, const int32_t* v, uint32_t* h) { for (int64_t i = 0; i < n; i++) h[i] = mm3_i32(v[i], h[i]); }
void hm_mm3_i64(int64_t n, const int64_t* v, uint32_t* h) { for (int64_t i = 0; i < n; i++) h[i] = mm3_i64(v[i], h[i]); }
void hm_mm3_i128(int64_t n, const i128* v, uint32_t* h) { for (int64_t i = 0; i < n; i++) h[i] = mm3_i128(v[i], h[i]); }
uint32_t hm_mm3_bytes(const uint8_t* d, int32_t len, uint32_t seed) { return mm3_bytes(d, len, seed); }
uint32_t hm_pmod(uint32_t h, uint32_t n) { return pmod_u32(h, n); }
void hm_mul_i64(int64_t n, const int64_t* a, const int64_t* b, i128* out) {
    for (int64_t i = 0; i < n; i++) out[i] = mul_i64_i64(a[i], b[i]);
}
void hm_mul_i128_i64(int64_t n, const i128* a, const int64_t* b, i128* out) {
    for (int64_t i = 0; i < n; i++) out[i] = mul_i128_i64(a[i], b[i]);
}
void hm_mul_i128_wrap(int64_t n, const i128* a, const i128* b, i128* out) {
    for (int64_t i = 0; i < n; i++) out[i] = mul_i128_wrap(a[i], b[i]);
}
void hm_f64_total_lt(int64_t n, const uint64_t* a, const uint64_t* b, uint8_t* out) {
    for (int64_t i = 0; i < n; i++) out[i] = f64_total_key(a[i]) < f64_total_key(b[i]);
}
// Float32 a op b (0 add 1 sub 2 mul 3 div) as the device computes it: the host's IEEE result with every NaN replaced by the
// device's canonical 0x7FFFFFFF, then f32_x86_nan
void hm_f32_arith(int op, int64_t n, const float* a, const float* b, float* out) {
    for (int64_t i = 0; i < n; i++) {
        volatile float x = a[i], y = b[i];
        float r = op == 0 ? x + y : op == 1 ? x - y : op == 2 ? x * y : x / y;
        if (r != r) { const u32 canon = 0x7FFFFFFFu; __builtin_memcpy(&r, &canon, 4); }
        out[i] = f32_x86_nan(a[i], b[i], r);
    }
}
void hm_dd_sum(int64_t n, const double* v, double* out) {
    dd a = {0.0, 0.0};
    for (int64_t i = 0; i < n; i++) dd_add_double(a, v[i]);
    *out = a.hi;
}
void hm_dd_sum_tree(int64_t n, const double* v, int lanes, double* out) { // lanes partials merged like the kernels do
    dd acc[64];
    for (int k = 0; k < lanes; k++) acc[k] = dd{0.0, 0.0};
    for (int64_t i = 0; i < n; i++) dd_add_double(acc[i % lanes], v[i]);
    dd t = {0.0, 0.0};
    for (int k = 0; k < lanes; k++) dd_add_dd(t, acc[k]);
    *out = t.hi;
}
long long hm_snappy(const uint8_t* in, long long n, uint8_t* out, long long cap) { return snappy_decode_serial(in, n, out, cap); }
// the per-group overflow certificate of decimal SUM / AVG (cb_finalize): 0 fits, 1 overflows in every row order, 2 order-dependent
int hm_sum_cert(int64_t n, uint64_t blo, uint64_t bhi, int p, const i128* total) { return sum_cert(cert_level(n, blo, bhi, p), dec_fits_p(*total, p)); }
int hm_cert_level(int64_t n, uint64_t blo, uint64_t bhi, int p) { return cert_level(n, blo, bhi, p); }
}
