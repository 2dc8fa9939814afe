"""device/cb_math.h compiled for the host, checked against the oracle (CPU-only)."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "datafusion-comet_b200", "csrc")


@pytest.fixture(scope="module")
def hm():
    so = os.path.join(CSRC, "libcb200_hostmath.so")
    src = [os.path.join(CSRC, "host_math_test.cpp"), os.path.join(CSRC, "device", "cb_math.h"), os.path.join(CSRC, "device", "cb_snappy.h")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in src):
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, src[0]])
    lib = C.CDLL(so)
    lib.hm_mm3_bytes.restype = C.c_uint32
    lib.hm_pmod.restype = C.c_uint32
    lib.hm_snappy.restype = C.c_longlong
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def rand_dec(rng, n, digits):
    """random signed ints with up to `digits` decimal digits, mixed magnitudes"""
    out = []
    for _ in range(n):
        d = int(rng.integers(0, digits + 1))
        v = int(rng.integers(0, 10**18)) * 10**18 * 10**2 + int(rng.integers(0, 10**18)) * 10**2 + int(rng.integers(0, 100))
        v %= 10**d if d > 0 else 1
        out.append(-v if rng.integers(0, 2) else v)
    return out


@pytest.mark.parametrize("op", [0, 1, 2])
@pytest.mark.parametrize("cfg", [(38, 6, 38, 4, 38, 6), (26, 4, 13, 2, 38, 6), (38, 10, 38, 10, 38, 10), (20, 5, 20, 5, 38, 6),
                                 (38, 0, 38, 0, 38, 0), (10, 2, 10, 2, 38, 4), (38, 18, 38, 18, 38, 6)])
def test_wide_vs_oracle(hm, oracle, op, cfg):
    p1, s1, p2, s2, po, so = cfg
    rng = np.random.default_rng(op * 100 + p1 + s1)
    n = 2000
    l = rand_dec(rng, n, p1) + [10**38 - 1, -(10**38 - 1), 0, 1, -1, 5, -5]
    r = rand_dec(rng, n, p2) + [10**38 - 1, 10**38 - 1, 0, 1, -1, 5, 5]
    n = len(l)
    L, R = oracle.dec_from_ints(l), oracle.dec_from_ints(r)
    eo, ev = oracle.wide_decimal(op, L, None, s1, R, None, s2, po, so)
    out = np.zeros((n, 2), dtype=np.uint64)
    outv = np.zeros(n, dtype=np.uint8)
    hm.hm_wide(C.c_int(op), C.c_int64(n), _p(L), C.c_int(s1), _p(R), C.c_int(s2), C.c_int(po), C.c_int(so), _p(out), _p(outv))
    assert (outv == ev).all()
    assert (out == eo).all()


@pytest.mark.parametrize("op", [0, 1, 2])
def test_plain_vs_oracle(hm, oracle, op):
    rng = np.random.default_rng(5 + op)
    n = 3000
    l, r = rand_dec(rng, n, 18), rand_dec(rng, n, 18)
    L, R = oracle.dec_from_ints(l), oracle.dec_from_ints(r)
    eo, ev, _, _ = oracle.plain_decimal(op, L, None, 18, 4, R, None, 18, 2)
    out = np.zeros((n, 2), dtype=np.uint64)
    err = hm.hm_plain(C.c_int(op), C.c_int64(n), _p(L), C.c_int(4), _p(R), C.c_int(2), _p(out))
    assert err == 0 and (out == eo).all()


def test_plain_mul_overflow_flag(hm, oracle):
    L, R = oracle.dec_from_ints([10**30]), oracle.dec_from_ints([10**30])
    out = np.zeros((1, 2), dtype=np.uint64)
    assert hm.hm_plain(C.c_int(2), C.c_int64(1), _p(L), C.c_int(0), _p(R), C.c_int(0), _p(out)) == 1
    with pytest.raises(oracle.OracleError):
        oracle.plain_decimal(2, L, None, 38, 0, R, None, 38, 0)


def test_fits_vs_oracle(hm, oracle):
    for p in (1, 3, 13, 18, 19, 22, 26, 36, 38):
        vals = [10**p - 1, 10**p, -(10**p - 1), -(10**p), 0, 10**p + 1]
        V = oracle.dec_from_ints(vals)
        out = np.zeros(len(vals), dtype=np.uint8)
        hm.hm_fits(C.c_int64(len(vals)), _p(V), C.c_int(p), _p(out))
        assert list(out) == [1, 0, 1, 0, 1, 0]


@pytest.mark.parametrize("cfg", [(4, 10, 2), (2, 10, 4), (0, 3, 0), (0, 3, 2), (2, 4, 2), (10, 38, 0), (0, 38, 20)])
def test_rescale_vs_oracle(hm, oracle, cfg):
    s_in, p_out, s_out = cfg
    rng = np.random.default_rng(11)
    vals = rand_dec(rng, 2000, 30) + [12350, 12349, -12350, 5, -5, 15, -15, 999, 1000]
    V = oracle.dec_from_ints(vals)
    eo, ev = oracle.decimal_rescale_check(V, None, s_in, p_out, s_out)
    n = len(vals)
    out = np.zeros((n, 2), dtype=np.uint64)
    outv = np.zeros(n, dtype=np.uint8)
    hm.hm_rescale(C.c_int64(n), _p(V), C.c_int(s_in), C.c_int(p_out), C.c_int(s_out), _p(out), _p(outv))
    assert (outv == ev).all() and (out == eo).all()


def test_avg_vs_oracle(hm, oracle):
    rng = np.random.default_rng(13)
    sums = rand_dec(rng, 3000, 22) + [100, -100, 500, -500, 1, -1, 0]
    counts = [int(c) for c in rng.integers(1, 10**6, 3000)] + [3, 3, 3, 3, 2, 2, 7]
    counts[5] = 2**40 + 12345  # > 32-bit divisor path
    counts[6] = 2**62
    S = oracle.dec_from_ints(sums)
    Cn = np.array(counts, dtype=np.int64)
    n = len(sums)
    acc = oracle.AvgDecimalGroups(n, 22, 2, 16, 6)
    acc.sums[:] = S
    acc.counts[:] = Cn
    eo, ev = acc.evaluate()
    out = np.zeros((n, 2), dtype=np.uint64)
    outv = np.zeros(n, dtype=np.uint8)
    hm.hm_avg(C.c_int64(n), _p(S), _p(Cn), C.c_int(4), C.c_int(16), _p(out), _p(outv))
    assert (outv == ev).all() and (out == eo).all()


def test_murmur3_vs_oracle(hm, oracle):
    rng = np.random.default_rng(17)
    v32 = rng.integers(-2**31, 2**31, 1000).astype(np.int32)
    v64 = rng.integers(-2**63, 2**63, 1000).astype(np.int64)
    h = np.full(1000, 42, dtype=np.uint32)
    hm.hm_mm3_i32(C.c_int64(1000), _p(v32), _p(h))
    assert (h == oracle.murmur3_column("i32", v32)).all()
    hm.hm_mm3_i64(C.c_int64(1000), _p(v64), _p(h))  # chained
    assert (h == oracle.murmur3_column("i64", v64, hashes=oracle.murmur3_column("i32", v32))).all()
    d = oracle.dec_from_ints([int(x) * 10**20 for x in v64[:100]])
    h = np.full(100, 42, dtype=np.uint32)
    hm.hm_mm3_i128(C.c_int64(100), _p(d), _p(h))
    assert (h == oracle.murmur3_column("dec_large", d)).all()
    for s in [b"", b"a", b"ab", b"abc", b"abcd", b"abcde", "😁".encode(), bytes(range(250, 256)) * 3]:
        buf = (C.c_uint8 * max(1, len(s))).from_buffer_copy(s or b"\0")
        assert hm.hm_mm3_bytes(buf, len(s), 42) == oracle.murmur3_bytes(s)
    for hv in [0x99F0149D, 0x9C67B85D, 0xC8008529, 0, 1, 0xFFFFFFFF, 0x80000000]:
        for n in (1, 2, 7, 8, 200):
            assert hm.hm_pmod(C.c_uint32(hv), C.c_uint32(n)) == oracle.pmod(hv, n)


def test_mul_i64(hm, oracle):
    rng = np.random.default_rng(19)
    a = rng.integers(-2**63, 2**63, 1000).astype(np.int64)
    b = rng.integers(-2**63, 2**63, 1000).astype(np.int64)
    out = np.zeros((1000, 2), dtype=np.uint64)
    hm.hm_mul_i64(C.c_int64(1000), _p(a), _p(b), _p(out))
    assert oracle.dec_to_ints(out) == [int(x) * int(y) for x, y in zip(a, b)]


def test_f64_total_order(hm):
    vals = np.array([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, np.nan, -np.nan, 1e-320, -1e-320])
    a = np.repeat(vals, len(vals)).view(np.uint64).copy()
    b = np.tile(vals, len(vals)).view(np.uint64).copy()
    out = np.zeros(a.shape[0], dtype=np.uint8)
    hm.hm_f64_total_lt(C.c_int64(a.shape[0]), _p(a), _p(b), _p(out))

    def key(bits):
        bits = int(bits)
        return (bits ^ 0x7FFFFFFFFFFFFFFF) - 2**64 if bits >> 63 else bits  # totalOrder as signed key

    exp = [key(x) < key(y) for x, y in zip(a, b)]
    assert list(out.astype(bool)) == exp


def test_dd_sum_within_1ulp_of_exact(hm, oracle):
    rng = np.random.default_rng(23)
    for scale in (1.0, 1e10):
        v = (rng.random(200000) * 2100.0 * scale).astype(np.float64)
        v[::7] *= -0.3
        exact = math.fsum(v)
        for fn, args in ((hm.hm_dd_sum, ()), (hm.hm_dd_sum_tree, (C.c_int(37),))):
            out = C.c_double(0)
            fn(C.c_int64(v.shape[0]), _p(v), *args, C.byref(out))
            assert abs(out.value - exact) <= math.ulp(exact)


def test_wrapping_products(hm, oracle):
    rng = np.random.default_rng(31)
    a = rand_dec(rng, 2000, 30)
    b64 = [int(x) for x in rng.integers(-2**63, 2**63, 2000)]
    b = rand_dec(rng, 2000, 30)
    A, B = oracle.dec_from_ints(a), oracle.dec_from_ints(b)
    B64 = np.array(b64, dtype=np.int64)
    out = np.zeros((2000, 2), dtype=np.uint64)
    hm.hm_mul_i128_i64(C.c_int64(2000), _p(A), _p(B64), _p(out))
    wrap = lambda v: ((v + (1 << 127)) % (1 << 128)) - (1 << 127)
    assert oracle.dec_to_ints(out) == [wrap(x * y) for x, y in zip(a, b64)]
    hm.hm_mul_i128_wrap(C.c_int64(2000), _p(A), _p(B), _p(out))
    assert oracle.dec_to_ints(out) == [wrap(x * y) for x, y in zip(a, b)]


def test_snappy_decoder_vs_pyarrow(hm):
    """device/cb_snappy.h (the element parser the warp decompressor shares) against pyarrow's Snappy on page-like payloads"""
    import pyarrow as pa
    rng = np.random.default_rng(7)
    payloads = [b"", b"a", b"abcd" * 1000, bytes(rng.integers(0, 256, 100_000, dtype=np.uint8)),                    # empty, tiny, overlapping copies, incompressible
                rng.integers(0, 50, 200_000).astype(np.int64).tobytes(), (rng.integers(90000, 210000, 150_000) * 7).astype(np.int64).tobytes(),
                np.repeat(rng.integers(0, 3, 5000).astype(np.int32), 40).tobytes(), b"x" * 70 + b"y" * 3 + b"x" * 100_000]
    for raw in payloads:
        comp = pa.compress(raw, codec="snappy", asbytes=True)
        out = np.zeros(len(raw) + 8, dtype=np.uint8)
        src = np.frombuffer(comp, dtype=np.uint8).copy()
        n = hm.hm_snappy(_p(src), C.c_longlong(len(comp)), _p(out), C.c_longlong(len(raw)))
        assert n == len(raw)
        assert out[:n].tobytes() == raw
    # malformed inputs are rejected, never over-read / over-written
    comp = np.frombuffer(pa.compress(b"abcd" * 1000, codec="snappy", asbytes=True), dtype=np.uint8).copy()
    out = np.zeros(4008, dtype=np.uint8)
    assert hm.hm_snappy(_p(comp), C.c_longlong(len(comp) - 3), _p(out), C.c_longlong(4000)) == -1      # truncated
    assert hm.hm_snappy(_p(comp), C.c_longlong(len(comp)), _p(out), C.c_longlong(100)) == -1            # declared length exceeds the page size
    bad = comp.copy()
    bad[2] = 0x01 | (7 << 2)   # a copy with offset beyond the start of the output
    bad[3] = 0xff
    assert hm.hm_snappy(_p(bad), C.c_longlong(len(bad)), _p(out), C.c_longlong(4000)) == -1


def test_decimal_div_matches_the_oracle(hm, oracle):
    """cb::dec_div (multi-limb Knuth division on the device) vs the oracle's restatement of spark_decimal_div_internal
    (div.rs:75-190) with Python integers: every scale combination incl. the BigInt-sized ones, zero divisors, the i128::MAX
    sentinel, integral division."""
    rng = np.random.default_rng(12)
    n = 96
    for trial in range(120):
        p1, p2 = int(rng.integers(1, 39)), int(rng.integers(1, 39))
        s1, s2, s3 = int(rng.integers(0, p1 + 1)), int(rng.integers(0, p2 + 1)), int(rng.integers(0, 39))
        integral = bool(rng.integers(0, 4) == 0)
        ls = [v % 10**p1 * (1 if v >= 0 else -1) for v in rand_dec(rng, n, 38)]
        rs = [v % 10**p2 * (1 if v >= 0 else -1) for v in rand_dec(rng, n, 38)]
        ls[:3], rs[:4] = [10**p1 - 1, -(10**p1 - 1), 0], [1, -1, 0, 3]
        la, ra = oracle.dec_from_ints(ls), oracle.dec_from_ints(rs)
        out, zero, fits = np.zeros((n, 2), dtype=np.uint64), np.zeros(n, dtype=np.uint8), np.zeros(n, dtype=np.uint8)
        l_exp, r_exp = max(0, s2 + s3 + 1 - s1), max(0, s1 - (s2 + s3 + 1))
        hm.hm_dec_div(C.c_int64(n), _p(la), _p(ra), l_exp, r_exp, int(integral), _p(out), _p(zero), _p(fits))
        exp, _ = oracle.decimal_div(la, None, s1, ra, None, s2, s3, integral)
        assert (zero.astype(bool) == np.array([r == 0 for r in rs])).all()
        assert oracle.dec_to_ints(out) == oracle.dec_to_ints(exp), (p1, s1, p2, s2, s3, integral)
        got = oracle.dec_to_ints(out)
        assert [bool(f) for f in fits] == [-(1 << 63) <= g < (1 << 63) for g in got]


def test_overflow_certificate_against_every_row_order(hm, oracle):
    """cb::cert_level / cb::sum_cert decide from (n, bound B on |addend|, exact total) what the reference's row-by-row sum
    (sum_decimal.rs:418-439: NULL as soon as a prefix leaves the precision) returns in EVERY row order.  Brute force over all
    permutations of small groups: verdict 0 => no order overflows and the total fits; 1 => every order overflows; 2 => undecided
    (the engine refuses those).  B is what the host derives from the value masks: the smallest 2^bits with -B <= v <= B - 1."""
    import itertools
    hm.hm_sum_cert.restype = C.c_int
    p = 3                                            # decimal(3, 0): |sum| <= 999
    lim = 10**p - 1
    rng = np.random.default_rng(0)
    seen = set()
    for _ in range(4000):
        n = int(rng.integers(1, 6))
        vals = [int(v) for v in rng.integers(-lim, lim + 1, n)]
        bits = max(((v ^ (v >> 63)).bit_length()) for v in vals)          # value-mask bit length, as the kernels record it
        B = 1 << bits
        total = sum(vals)
        t = oracle.dec_from_ints([total])
        verdict = hm.hm_sum_cert(C.c_int64(n), C.c_uint64(B & (2**64 - 1)), C.c_uint64((B >> 64) | (1 << 63)), C.c_int(p), _p(t))
        outcomes = set()
        for perm in set(itertools.permutations(vals)):
            s, ovf = 0, False
            for v in perm:
                s += v
                if abs(s) > lim:
                    ovf = True
                    break
            outcomes.add(ovf)
        seen.add(verdict)
        if verdict == 0:
            assert outcomes == {False} and abs(total) <= lim, (vals, verdict)
        elif verdict == 1:
            assert outcomes == {True}, (vals, verdict)
        else:
            assert verdict == 2
    assert seen == {0, 1, 2}
    # the edge the Final merge of two 8e37 partial sums hits (decimal(38, 0)): n * B == 2^127 exactly is still an exact total
    hm.hm_cert_level.restype = C.c_int
    B = 1 << 126
    assert hm.hm_cert_level(C.c_int64(2), C.c_uint64(0), C.c_uint64((B >> 64) | (1 << 63)), C.c_int(38)) == 1     # two's-complement bound: exact
    assert hm.hm_cert_level(C.c_int64(2), C.c_uint64(0), C.c_uint64(B >> 64), C.c_int(38)) == 2                    # magnitude bound: may have wrapped
    assert hm.hm_cert_level(C.c_int64(3), C.c_uint64(0), C.c_uint64((B >> 64) | (1 << 63)), C.c_int(38)) == 2


F32_NAN_EDGES = np.array([0x7FC00000, 0xFFC00000, 0x7FC0BEEF, 0x7F800001, 0xFF800123, 0x7F800000, 0xFF800000, 0x00000000, 0x80000000,
                          0x00000001, 0x807FFFFF, 0x7F7FFFFF, 0x3F800000, 0xC0400000], dtype=np.uint32)   # NaNs (quiet, signalling,
                                                                                                          # payloads, signs), +-Inf, +-0, subnormals


@pytest.mark.parametrize("op", [0, 1, 2, 3])
def test_f32_x86_nan_rule(hm, op):
    """cb::f32_x86_nan turns the device's canonical NaN back into the bits numpy (x86 SSE, like the reference) returns: the first NaN
    operand made quiet, else the default NaN 0xFFC00000 for an invalid operation.  Every pair of edge values, both operand orders."""
    n = len(F32_NAN_EDGES)
    a = np.repeat(F32_NAN_EDGES, n).view(np.float32).copy()
    b = np.tile(F32_NAN_EDGES, n).view(np.float32).copy()
    out = np.zeros(n * n, dtype=np.float32)
    hm.hm_f32_arith(C.c_int(op), C.c_int64(n * n), _p(a), _p(b), _p(out))
    with np.errstate(all="ignore"):
        want = [a + b, a - b, a * b, a / b][op]
    assert np.isnan(want).sum() > n       # the pairs reach NaN operands and invalid operations
    bad = np.nonzero(out.view(np.uint32) != want.view(np.uint32))[0]
    assert bad.size == 0, [(hex(a.view(np.uint32)[i]), hex(b.view(np.uint32)[i]), hex(out.view(np.uint32)[i]), hex(want.view(np.uint32)[i])) for i in bad[:4]]
