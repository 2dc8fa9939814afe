"""The decimal range machinery on the CPU: the value-mask -> bound rule, the soundness of expr_maxabs (ranges.h, compiled for the host
with the plan decoder) against exact evaluation by the expression interpreter, and the code generator's choice on each side of every
threshold the range-specialised kernels depend on (tests/test_gpu_range_levels.py runs the same thresholds on the device)."""
import ctypes as C
import itertools
import os
import re
import subprocess

import numpy as np
import pytest

import exprs as E

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "datafusion-comet_b200", "csrc")
RSAT = 1 << 127
R63 = 1 << 63


@pytest.fixture(scope="module")
def rt(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("ranges") / "libcb200_ranges.so")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-fPIC", "-shared", f"-I{cuda}/include", "-o", so,
                           os.path.join(CSRC, "ranges_test.cpp"), os.path.join(CSRC, "plan.cpp"), "-Wl,--no-undefined"])
    lib = C.CDLL(so)
    lib.rt_maxabs.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t]
    return lib


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def maxabs(rt, cb, node, col_types, bounds):
    """expr_maxabs of `node` over columns with |c| <= bounds[c]"""
    plan = cb.proto.projection(cb.proto.scan(col_types), [node.proto()])
    flat = []
    for b in bounds:
        b = min(b, RSAT)
        flat += [b & (2**64 - 1), b >> 64]
    arr = (C.c_uint64 * len(flat))(*flat)
    out = (C.c_uint64 * 2)()
    err = C.create_string_buffer(512)
    assert rt.rt_maxabs(plan, len(plan), len(bounds), arr, out, err, 512) == 0, err.value
    return out[0] | out[1] << 64


# ---- the value mask: kernels OR (v ^ sign) over the valid rows; the host assumes |v| <= 2^bitlen -----------------------------------
def mask_of(v):
    """cb_kernels.cuh vm_or on a two's-complement i128: each 64-bit word XORed with the sign word"""
    u = v & (2**128 - 1)
    s = 2**128 - 1 if v < 0 else 0
    return u ^ s


def test_mask_bound_rule_exhaustive_small_k():
    """(v ^ sign) < 2^k  =>  |v| <= 2^k, and -2^k reaches it: the bound cannot be 2^k - 1"""
    for k in range(0, 17):
        vs = range(-(1 << (k + 1)), 1 << (k + 1))
        inside = [v for v in vs if mask_of(v) < (1 << k)]
        assert inside == list(range(-(1 << k), 1 << k))
        assert max(abs(v) for v in inside) == 1 << k
        assert (int(mask_of(-(1 << k))).bit_length(), int(mask_of((1 << k) - 1)).bit_length()) == (k, k)


@pytest.mark.parametrize("k", [46, 48, 49, 62, 63, 64, 126])
def test_mask_bound_rule_at_large_k(k):
    for v in ((1 << k) - 1, -(1 << k)):
        assert mask_of(v) < (1 << k) and abs(v) <= 1 << k
        assert mask_of(v).bit_length() == k
    for v in (1 << k, -(1 << k) - 1):                      # one step out: the mask has k + 1 bits
        assert mask_of(v).bit_length() == k + 1
    # 8-byte storage (vm_or64): INT64_MIN has a 63-bit mask and magnitude 2^63
    if k == 63:
        m = (-(1 << 63) & (2**64 - 1)) ^ (2**64 - 1)
        assert m.bit_length() == 63


# ---- soundness of expr_maxabs ------------------------------------------------------------------------------------------------------
def _dec(rng, lo_p=1):
    p = int(rng.integers(lo_p, 39))
    return E.P.DECIMAL(p, int(rng.integers(0, min(p, 12) + 1)))


def _tree(rng, cols, depth):
    P = E.P
    if depth == 0 or rng.random() < 0.2:
        if rng.random() < 0.75:
            i = int(rng.integers(0, len(cols)))
            return E.Col(i, cols[i])
        dt = _dec(rng)
        lim = 10**dt.precision - 1
        v = int(rng.choice([lim, -lim, 0, 1, -1, int(rng.integers(-min(lim, 2**62), min(lim, 2**62) + 1))]))
        return E.Lit(v, dt)
    kind = rng.choice(["add", "subtract", "multiply", "cast", "check", "neg", "if"], p=[.2, .15, .2, .15, .1, .1, .1])
    if kind in ("add", "subtract", "multiply"):
        l, r = _tree(rng, cols, depth - 1), _tree(rng, cols, depth - 1)
        probe = E.Arith(kind, l, r, P.DECIMAL(38, 0))
        ret = P.DECIMAL(38, int(rng.integers(0, 13))) if probe.wide else probe.dt
        return E.Arith(kind, l, r, ret)
    c = _tree(rng, cols, depth - 1)
    if kind == "cast":
        return E.Cast(c, _dec(rng))
    if kind == "check":
        return E.CheckOverflow(c, P.DECIMAL(int(rng.integers(max(c.dt.scale, 1), 39)), c.dt.scale), bool(rng.random() < 0.3))
    if kind == "neg":
        return E.Neg(c)
    other = _tree(rng, cols, depth - 1)
    i = int(rng.integers(0, len(cols)))
    cond = E.Cmp("gt", E.Col(i, cols[i]), E.Lit(0, cols[i]))
    return E.If(cond, c, E.Cast(other, c.dt))


def _corners(b, bits):
    """inputs at the corners of |v| <= b: both signs, and the mask corner -2^k / 2^k - 1 when b is a power of two"""
    vs = {b, -b, 0, 1, -1}
    if bits:
        vs |= {(b - 1), -b}
    return sorted(vs)


@pytest.mark.parametrize("seed", range(6))
def test_expr_maxabs_bounds_the_exact_result(rt, cb, oracle, seed):
    """For random decimal trees of Add / Sub / Mul (plain and wide), Cast, CheckOverflow, UnaryMinus and If over mixed scales: with
    every column at a corner of its bound, the exact result of every non-NULL row is within expr_maxabs."""
    from oracle import oracle as O
    rng = np.random.default_rng(seed)
    cols = [_dec(rng, 10), _dec(rng, 1), _dec(rng, 18)]
    checked = 0
    for _ in range(60):
        node = _tree(rng, cols, int(rng.integers(1, 4)))
        if node.dt.name != "DECIMAL":
            continue
        # bounds as the kernels assume them (2^k from a value mask) and as arbitrary magnitudes up to the declared precision
        ks = [int(rng.integers(0, 64)) if rng.random() < 0.5 else None for _ in cols]
        bounds = [(1 << k) if k is not None else int(rng.integers(1, 10**min(dt.precision, 18))) for k, dt in zip(ks, cols)]
        rows = list(itertools.product(*[_corners(b, k is not None) for b, k in zip(bounds, ks)]))     # python ints: exact past 2^63
        inputs = [(O.dec_from_ints([r[c] for r in rows]), np.ones(len(rows), dtype=bool)) for c in range(len(cols))]
        try:
            out, valid = node.eval(inputs)
        except E.AnsiError:
            continue                 # a plain op left i128 / an ANSI check fired: no value to bound
        bound = maxabs(rt, cb, node, [c for c in cols], bounds)
        got = [abs(v) for v, ok in zip(O.dec_to_ints(out), valid) if ok]
        assert all(v <= bound for v in got), (seed, max(got), bound)
        checked += 1
    assert checked >= 25


def test_expr_maxabs_known_answers(rt, cb):
    P = E.P
    d18, d12_2 = P.DECIMAL(18, 0), P.DECIMAL(12, 2)
    c0, c1 = E.Col(0, d18), E.Col(1, d12_2)
    assert maxabs(rt, cb, E.Neg(c0), [d18, d12_2], [R63, 1]) == R63
    assert maxabs(rt, cb, E.Arith("multiply", c0, E.Lit(-1, P.DECIMAL(1, 0)), P.DECIMAL(20, 0)), [d18, d12_2], [R63, 1]) == R63
    # scale alignment: c0 (scale 0) is multiplied by 10^2 before the add
    assert maxabs(rt, cb, E.Arith("add", c0, c1, P.DECIMAL(21, 2)), [d18, d12_2], [5, 7]) == 507
    # CheckOverflow and Cast clamp at the precision; a Cast to a smaller scale rounds HALF_UP (+1)
    assert maxabs(rt, cb, E.CheckOverflow(c0, P.DECIMAL(5, 0)), [d18, d12_2], [10**9, 1]) == 10**5 - 1
    assert maxabs(rt, cb, E.Cast(c1, P.DECIMAL(20, 0)), [d18, d12_2], [1000, 1000]) == 11
    assert maxabs(rt, cb, E.Col(0, d18), [d18, d12_2], [RSAT, 1]) == RSAT


# ---- code generation on each side of every threshold --------------------------------------------------------------------------------
def _agg_src(cb, in_types, child, bits, scale=0):
    """the row program of an ungrouped SUM(child) kernel specialised to |column i| < 2^bits[i]"""
    P = cb.proto
    plan = P.hash_agg(P.scan(in_types), [], [P.agg_sum(child, P.DECIMAL(38, scale))], P.PARTIAL)
    src = cb.native.compile_plan_assume(plan, bits, 0)
    return src[src.index("CB_D void cb_row_agg"):src.index("CB_D void cb_finalize_group")]


def test_wrap_sum_up_to_48_bits(cb):
    """64-bit per-thread partials wrap-free while 2^14 rows * 2^k < 2^63: k <= 48"""
    P = cb.proto
    d = P.DECIMAL(38, 0)
    for k, want in ((47, "wrap"), (48, "wrap"), (49, "wide"), (62, "wide"), (63, "i128")):
        body = _agg_src(cb, [d], P.bound(0, d), [k])
        got = "wrap" if re.search(r"acc\.add_i64_wrap\(g, \d+, v\d+\)", body) else "wide" if "acc.add_i64_wide(" in body else \
            "i128" if "acc.add_i128(" in body else None
        assert got == want, (k, body)
        assert ("(cb::i64)v" in body and ".lo" in body) == (k <= 62), k       # narrow load below 2^63
        assert "acc.vm_or(0" in body                                           # the assumption is validated


@pytest.mark.parametrize("ka,kb", [(31, 31), (31, 32), (40, 22), (40, 23)])
def test_i64_multiply_below_2_63(cb, ka, kb):
    P = cb.proto
    a, b = P.DECIMAL(38, 0), P.DECIMAL(38, 0)
    m = P.multiply(P.bound(0, a), P.bound(1, b), P.DECIMAL(38, 0))
    body = _agg_src(cb, [a, b], P.check_overflow(m, P.DECIMAL(38, 0)), [ka, kb])
    fits = ka + kb < 63
    assert bool(re.search(r"cb::i64 v\d+ = v\d+ \* v\d+;", body)) == fits, (ka, kb)
    assert ("cb::mul_i64_i64(" in body) == (not fits), (ka, kb)


@pytest.mark.parametrize("k,fits", [(56, True), (57, False)])
def test_i64_add_with_scale_factor(cb, k, fits):
    """decimal(18,0) + decimal(18,2): the left side is multiplied by 100 before the add; 2^k * 100 + 2^k < 2^63 iff k <= 56"""
    P = cb.proto
    a, b = P.DECIMAL(18, 0), P.DECIMAL(18, 2)
    add = P.add(P.bound(0, a), P.bound(1, b), P.DECIMAL(21, 2))
    body = _agg_src(cb, [a, b], add, [k, k], 2)
    assert (2**k * 100 + 2**k < R63) == fits
    assert bool(re.search(r"cb::i64 v\d+ = v\d+ \* \(\(cb::i64\)100ull\) \+ v\d+;", body)) == fits, body
    assert ("cb::i128_add(" in body) == (not fits)


@pytest.mark.parametrize("delta", [0, 1])
def test_check_overflow_elided_exactly_at_the_precision(cb, delta):
    """CheckOverflow(c + L, decimal(18, 0)) with |c| <= 2^40: bound 2^40 + |L|, elided iff <= 10^18 - 1"""
    P = cb.proto
    d = P.DECIMAL(18, 0)
    lit = 10**18 - 1 - 2**40 + delta
    add = P.add(P.bound(0, d), P.literal(lit, d), P.DECIMAL(19, 0))
    body = _agg_src(cb, [d], P.check_overflow(add, d, True), [40])
    assert ("dec_fits" in body) == (delta == 1)
    assert ("set_err(p, 1)" in body) == (delta == 1)


def test_literal_near_2_63(cb):
    """decimal literals are 64-bit below 2^63 and 128-bit from it on"""
    P = cb.proto
    d = P.DECIMAL(38, 0)
    for v, narrow in ((2**63 - 1, True), (-(2**63 - 1), True), (2**63, False), (-(2**63), False)):
        body = _agg_src(cb, [d], P.add(P.bound(0, d), P.literal(v, d), P.DECIMAL(38, 0)), [10])
        assert (f"((cb::i64){v & (2**64 - 1)}ull)" in body) == narrow, v
        assert bool(re.search(r"cb::mk128\(\d+ull, \(cb::i64\)\d+ull\)", body)) == (not narrow), v


def test_unary_minus_of_a_narrow_column(cb):
    """i64 negation only below 2^63; at 2^63 (a 64-bit column may hold INT64_MIN) the negation is 128-bit"""
    P = cb.proto
    d = P.DECIMAL(38, 0)
    for k, narrow in ((62, True), (63, False)):
        body = _agg_src(cb, [d], P.unary_minus(P.bound(0, d)), [k])
        assert bool(re.search(r"cb::i64 v\d+ = -v\d+;", body)) == narrow, k
        assert ("cb::i128_neg(" in body) == (not narrow), k
