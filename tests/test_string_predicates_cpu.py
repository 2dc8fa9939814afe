"""String predicates on dictionary-coded columns, without a GPU: the CPU reference (tests/strpred_ref.py) against pyarrow, the host
compile of device/cb_strpred.h against the reference, and the planner's accept / refuse rules and generated source.

pyarrow is Arrow C++, not the reference's arrow-rs / DataFusion, so the first group is a cross-check of the restated rules."""
import ctypes as C
import os
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import strpred_ref as R

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "datafusion-comet_b200", "csrc")

HAND = ["", "a", "aa", "aaa", "ab", "b", "MAIL", "SHIP", "MAILS", "mail", "AIR", "REG AIR", "TRUCK", "FOB", "RAIL",
        "a\nb", "\n", "%", "_", "\\", "50%", "a_b", "a\\b", "é", "ée", "aé", "日本", "日本語", "x日y", "😀", "a😀b", "😀😀",
        "\x7f", "\x80", "ÿ", "z", "special requests", "blithely special packages requests", "requests special", "speciaL"]
PATTERNS = ["%", "", "%%", "_%_", "%a%a%", "a%", "%a", "%a%", "_", "__", "___", "a_", "_b", "a_b", "%special%requests%", "MAIL",
            "50\\%", "a\\_b", "a\\\\b", "%\\%", "\\_%", "%\n%", "a\nb", "_\n_", "é", "_é", "__", "日_", "%本%", "😀", "_😀_", "%😀",
            "x_y", "x__y", "%é", "é%", "%_%_%", "S%P", "%S%", "_%", "%_"]
LITS = ["", "a", "aa", "b", "MAIL", "SHIP", "é", "日本", "😀", "\x80", "\x7f", "z", "special", "\n", "%", "a%"]


def rand_strings(seed, n=300):
    rng = np.random.default_rng(seed)
    alphabet = ["a", "b", "A", "%", "_", "\\", "\n", " ", "é", "ß", "日", "本", "😀", "\x7f", "\x80", "z"]
    return ["".join(rng.choice(alphabet, size=int(rng.integers(0, 7)))) for _ in range(n)]


VALUES = HAND + rand_strings(1)


# ---- the reference against pyarrow ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", R.OPS)
def test_compare_matches_pyarrow(op):
    arr = pa.array(VALUES)
    f = {"eq": pc.equal, "neq": pc.not_equal, "lt": pc.less, "lt_eq": pc.less_equal, "gt": pc.greater, "gt_eq": pc.greater_equal}[op]
    for lit in LITS + VALUES[:40]:
        want = f(arr, pa.scalar(lit)).to_pylist()
        assert [R.cmp(op, v, lit) for v in VALUES] == want, (op, lit)


def test_byte_order_puts_non_ascii_after_ascii():
    assert R.cmp("lt", "\x7f", "\x80") and R.cmp("gt", "é", "z") and R.cmp("lt", "a", "aa") and R.cmp("lt", "", "\x00")
    assert pc.less(pa.array(["\x7f", "z"]), pa.scalar("é")).to_pylist() == [True, True]


def test_like_matches_pyarrow():
    arr = pa.array(VALUES)
    for pat in PATTERNS:
        want = pc.match_like(arr, pat).to_pylist()
        assert [R.like(v, pat) for v in VALUES] == want, pat


def test_like_hand_cases():
    assert R.like("aaa", "%a%a%") and not R.like("a", "%a%a%")
    assert R.like("", "") and not R.like("a", "") and R.like("", "%") and R.like("", "%%")
    assert R.like("日本", "_本") and R.like("😀", "_") and not R.like("😀", "__") and R.like("a\nb", "a_b") and R.like("\n\n", "%")
    assert R.like("50%", "50\\%") and not R.like("500", "50\\%") and R.like("a\\b", "a\\\\b") and R.like("a_b", "a\\_b") and not R.like("axb", "a\\_b")
    for bad in ("\\a", "a\\", "\\", "%\\n"):
        with pytest.raises(R.BadPattern):
            R.like("x", bad)


@pytest.mark.parametrize("name", ["starts_with", "ends_with", "contains"])
def test_functions_match_pyarrow(name):
    arr = pa.array(VALUES)
    f = {"starts_with": pc.starts_with, "ends_with": pc.ends_with, "contains": pc.match_substring}[name]
    for lit in LITS + VALUES[:40]:
        assert [R.func(name, v, lit) for v in VALUES] == f(arr, lit).to_pylist(), (name, lit)
    assert all(R.func(name, v, "") for v in VALUES)


def test_in_matches_pyarrow():
    arr = pa.array(VALUES)
    for lits in (["MAIL", "SHIP"], ["", "é"], ["😀", "\x80", "zz"], []):
        want = pc.is_in(arr, value_set=pa.array(lits, type=pa.string())).to_pylist()
        assert [R.in_list(v, lits)[0] for v in VALUES] == want, lits
    col = R.StrCol(0)
    vals = ["MAIL", "AIR", "x", None]
    cols = [(["MAIL", "AIR", "x", ""], np.array([True, True, True, False]))]
    assert vals[3] is None
    out, ok = R.StrIn(col, ["MAIL", None]).eval(cols)
    assert list(out[:2]) == [True, False] and list(ok) == [True, False, False, False]
    out, ok = R.StrIn(col, ["MAIL", None], negated=True).eval(cols)
    assert list(out[:1]) == [False] and list(ok) == [True, False, False, False]
    out, ok = R.StrIn(col, ["MAIL"], negated=True).eval(cols)
    assert list(out[:3]) == [False, True, True] and list(ok) == [True, True, True, False]


# ---- device/cb_strpred.h on the host ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sp(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("cbstrpred") / "libcb200_strpred.so")
    subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(CSRC, "strpred_test.cpp")])
    lib = C.CDLL(so)
    f = lib.cb_sp_eval
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_char_p, C.c_int, C.c_char_p, C.POINTER(C.c_int), C.c_int]

    def ev(op, value, lits):
        bs = [l.encode() for l in lits]
        off = [0]
        for b in bs:
            off.append(off[-1] + len(b))
        offs = (C.c_int * len(off))(*off)
        v = value.encode()
        return f(R.SP[op], v, len(v), b"".join(bs) + b"\0", offs, len(bs))
    return ev


def test_header_compare_and_functions(sp):
    for lit in LITS + VALUES[:30]:
        for v in VALUES:
            for op in R.OPS:
                assert sp(op, v, [lit]) == int(R.cmp(op, v, lit)), (op, v, lit)
            for name in ("starts_with", "ends_with", "contains"):
                assert sp(name, v, [lit]) == int(R.func(name, v, lit)), (name, v, lit)


def test_header_in(sp):
    for lits in (["MAIL", "SHIP"], ["", "é"], ["😀", "\x80", "zz"], [], VALUES[:25]):
        for v in VALUES:
            assert sp("in", v, lits) == int(R.in_list(v, lits)[0]), (v, lits)


def test_header_like(sp):
    pats = PATTERNS + [p for p in rand_strings(7, 400) if "\\" not in p]
    for pat in pats:
        for v in VALUES:
            assert sp("like", v, [pat]) == int(R.like(v, pat)), (v, pat)
    for bad in ("\\a", "a\\", "\\", "%\\n"):
        assert sp("like", "x", [bad]) == -1


def test_header_like_random_escapes(sp):
    rng = np.random.default_rng(3)
    for _ in range(600):
        pat = "".join(rng.choice(["a", "%", "_", "\\%", "\\_", "\\\\", "é", "😀", "\n"], size=int(rng.integers(0, 6))))
        for v in VALUES[:120]:
            assert sp("like", v, [pat]) == int(R.like(v, pat)), (v, pat)


# ---- planner: accepted shapes, refusals, generated source --------------------------------------------------------------------------
@pytest.fixture(scope="module")
def native():
    import comet_b200
    from comet_b200 import native
    return native


def P():
    from comet_b200 import proto
    return proto


def filt(pred, fields=None):
    p = P()
    fields = fields or [p.STRING, p.INT64, p.STRING]
    return p.projection(p.filter_(p.scan(fields), pred), [p.bound(1, p.INT64)])


def col(i=0):
    return P().bound(i, P().STRING)


def slit(v):
    return P().literal(v, P().STRING)


def accepted_shapes():
    p = P()
    c, s = col(), slit
    out = [getattr(p, op)(c, s("MAIL")) for op in R.OPS] + [getattr(p, op)(s("MAIL"), c) for op in R.OPS]
    out += [p.in_(c, [s("MAIL"), s("SHIP")]), p.in_(c, [s("MAIL"), s(None)], True), p.in_(c, [s(None)]),
            p.like(c, s("%special%requests%")), p.not_(p.like(c, s("a\\%b_\\\\"))), p.like(c, s("")), p.like(c, s(None)),
            p.scalar_func("starts_with", [c, s("PROMO")]), p.scalar_func("ends_with", [c, s("")]), p.scalar_func("contains", [c, s("é")]),
            p.eq(c, s(None)), p.and_(p.like(c, s("a%")), p.like(col(2), s("b%")))]
    return out


def test_accepted_shapes_compile(native):
    p = P()
    for i, pred in enumerate(accepted_shapes()):
        # a NULL literal operand folds the predicate to a constant: keep a column in the filter, which a pipeline needs to stage
        plan = filt(p.and_(pred, p.is_not_null(p.bound(1, p.INT64))))
        ok, why = native.supports(plan)
        assert ok, (i, why)
        assert native.compile_plan(plan), i
        proj = p.projection(p.scan([p.STRING, p.INT64, p.STRING]), [pred, p.bound(1, p.INT64)])
        assert native.supports(proj)[0], i


def test_refused_shapes(native):
    p = P()
    c, s = col(), slit
    refused = {
        "column vs column": p.eq(c, col(2)),
        "non-literal pattern": p.like(c, col(2)),
        "escape of a letter": p.like(c, s("\\a")),
        "trailing escape": p.like(c, s("ab\\")),
        "unknown scalar function": p.scalar_func("upper", [c]),
        "string function over a non-literal": p.scalar_func("contains", [c, col(2)]),
        "IN with a column member": p.in_(c, [s("a"), col(2)]),
    }
    for name, pred in refused.items():
        ok, why = native.supports(filt(pred))
        assert not ok, name
        with pytest.raises(native.Unsupported):
            native.compile_plan(filt(pred))
    many = None
    for i in range(9):
        t = p.like(c, s(f"{i}%"))
        many = t if many is None else p.and_(many, t)
    assert not native.supports(filt(many))[0]
    eight = None
    for i in range(8):
        t = p.like(c, s(f"{i}%"))
        eight = t if eight is None else p.and_(eight, t)
    assert native.supports(filt(eight))[0]


def test_source_does_not_depend_on_the_literal(native):
    p = P()
    c = col()
    pairs = [(p.eq(c, slit("MAIL")), p.eq(c, slit("SHIP"))),
             (p.in_(c, [slit("MAIL"), slit("SHIP")]), p.in_(c, [slit("AIR"), slit("RAIL")])),
             (p.like(c, slit("%special%requests%")), p.like(c, slit("PROMO%"))),
             (p.scalar_func("contains", [c, slit("x")]), p.scalar_func("contains", [c, slit("yy")]))]
    for a, b in pairs:
        for plan in (filt, lambda q: p.hash_agg(p.scan([p.STRING, p.INT64]), [col()], [p.agg_count([p.bound(1, p.INT64)], q)])):
            assert all_sources(native, plan(a)) == all_sources(native, plan(b))
            assert native.compile_plan(plan(a)) == native.compile_plan(plan(b))


def all_sources(native, plan):
    return "".join(native.kernel_source(plan, i) for i in range(len(native.compile_plan(plan))))


def test_distinct_predicates_on_one_column_get_distinct_masks(native):
    p = P()
    c = col()
    two = all_sources(native, filt(p.or_(p.like(c, slit("a%")), p.like(c, slit("b%")))))
    assert "p.smask[0]" in two and "p.smask[1]" in two
    same = all_sources(native, filt(p.or_(p.like(c, slit("a%")), p.like(c, slit("a%")))))
    assert "p.smask[0]" in same and "p.smask[1]" not in same


def test_literal_never_in_source(native):
    p = P()
    src = all_sources(native, filt(p.like(col(), slit("%zqxjk%"))))
    assert "zqxjk" not in src and "p.smask[0]" in src
