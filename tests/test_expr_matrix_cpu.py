"""The expression matrix without a GPU: the interpreter of tests/exprs.py against pyarrow.compute on data without NaNs, every plan
tests/test_gpu_expr_matrix.py builds (its random trees included, with the same seeds) accepted by the planner and compiled for
sm_90a, and the expressions the planner refuses as Unsupported."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import exprs as E
import test_gpu_expr_matrix as M
from comet_b200 import native
from comet_b200 import proto as P

F32, F64 = P.FLOAT, P.DOUBLE


def _f32_cols(seed=3, n=4000):
    rng = np.random.default_rng(seed)
    a = (rng.standard_normal(n) * 10.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    b = (rng.standard_normal(n) * 10.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    a[:6] = [np.inf, -np.inf, 0.0, -0.0, 3.4e38, 1e-45]
    b[:6] = [1.0, 2.0, -0.0, 5.0, 3.4e38, 0.5]
    b[b == 0] = 1.0
    return a, b


@pytest.mark.parametrize("op", ["add", "subtract", "multiply", "divide"])
def test_float32_arithmetic_matches_pyarrow(op):
    """Float32 stays Float32 end to end: one rounding per node, bit for bit with arrow's kernels"""
    a, b = _f32_cols()
    ones = np.ones(len(a), dtype=bool)
    cols = [(a, ones), (b, ones)]
    x, y = E.Col(0, F32), E.Col(1, F32)
    got, valid = E.Arith(op, x, y, F32).eval(cols)
    assert got.dtype == np.float32 and valid.all()
    want = np.asarray(getattr(pc, op)(pa.array(a), pa.array(b)))
    assert (np.asarray(got).view(np.uint32) == want.view(np.uint32)).all()
    neg, _ = E.Neg(E.Arith(op, x, y, F32)).eval(cols)
    assert (np.asarray(neg).view(np.uint32) == (want.view(np.uint32) ^ np.uint32(0x80000000))).all()


def test_casts_to_float32_round_once():
    """int -> FLOAT rounds the integer once (i64 above 2^24, i32 above 2^24), f32 -> f64 widens exactly"""
    vals = np.array([2 ** 24 + 1, 2 ** 24 + 3, -(2 ** 31), 2 ** 31 - 1, 2 ** 63 - 1, -(2 ** 63), 2 ** 53 + 1, 123456789], dtype=np.int64)
    ok = np.ones(len(vals), dtype=bool)
    got, _ = E.Cast(E.Col(0, P.INT64), F32).eval([(vals, ok)])
    assert got.dtype == np.float32
    assert (got == np.asarray(pc.cast(pa.array(vals), pa.float32(), safe=False))).all()
    f = np.array([1.1, 3.4e38, 1e-45], dtype=np.float32)
    got, _ = E.Cast(E.Col(0, F32), F64).eval([(f, np.ones(3, dtype=bool))])
    assert (got == f.astype(np.float64)).all() and got.dtype == np.float64


@pytest.mark.parametrize("dt,np_dt", [(P.INT8, np.int8), (P.INT16, np.int16), (P.INT32, np.int32), (P.INT64, np.int64)])
@pytest.mark.parametrize("op", ["add", "subtract", "multiply"])
def test_integer_wraparound_matches_pyarrow(dt, np_dt, op):
    """LEGACY integer arithmetic wraps at every width (arrow's *_wrapping kernels); TRY turns exactly the wrapped rows into NULL"""
    info = np.iinfo(np_dt)
    rng = np.random.default_rng(7)
    a = np.concatenate([[info.min, info.max, -1, 0, info.max], rng.integers(info.min, info.max, 500, endpoint=True)]).astype(np_dt)
    b = np.concatenate([[-1, 1, info.min, info.max, info.max], rng.integers(info.min, info.max, 500, endpoint=True)]).astype(np_dt)
    ok = np.ones(len(a), dtype=bool)
    cols = [(a.astype(np.int64), ok), (b.astype(np.int64), ok)]
    got, valid = E.Arith(op, E.Col(0, dt), E.Col(1, dt), dt).eval(cols)
    want = np.asarray(getattr(pc, op)(pa.array(a), pa.array(b)))
    assert valid.all() and (np.asarray(got) == want.astype(np.int64)).all()
    exact = getattr(np, op)(a.astype(object), b.astype(object))
    fits = np.array([info.min <= int(v) <= info.max for v in exact])
    _, tvalid = E.Arith(op, E.Col(0, dt), E.Col(1, dt), dt, E.TRY).eval(cols)
    assert (np.asarray(tvalid, dtype=bool) == fits).all() and not fits.all()
    with pytest.raises(E.AnsiError):
        E.Arith(op, E.Col(0, dt), E.Col(1, dt), dt, E.ANSI).eval(cols)


def test_float_in_compares_bits():
    """IN over FLOAT / DOUBLE is totalOrder equality: NaN matches the NaN with its bits, 0.0 does not match -0.0; NULL keeps Spark's
    three-valued result"""
    for dt, np_dt in ((F32, np.float32), (F64, np.float64)):
        v = np.array([np.nan, -0.0, 0.0, 1.0, -np.nan], dtype=np_dt)
        cols = [(v, np.array([True, True, True, True, False]))]
        x = E.Col(0, dt)
        out, valid = E.In(x, [E.Lit(float("nan"), dt)]).eval(cols)
        assert list(out[:4]) == [True, False, False, False] and list(valid) == [True] * 4 + [False]
        out, _ = E.In(x, [E.Lit(-0.0, dt)]).eval(cols)
        assert list(out[:4]) == [False, True, False, False]
        out, valid = E.In(x, [E.Lit(0.0, dt), E.Lit(None, dt)]).eval(cols)
        assert list(out[:4]) == [False, False, True, False] and list(valid) == [False, False, True, False, False]


def test_if_raises_only_for_rows_that_take_the_branch():
    vals = np.array([1, 2 ** 31 - 1, 5], dtype=np.int64)
    ok = np.ones(3, dtype=bool)
    x = E.Col(0, P.INT32)
    small = E.Cmp("lt", x, E.Lit(100, P.INT32))
    out, valid = E.If(small, E.Arith("add", x, x, P.INT32, E.ANSI), E.Lit(0, P.INT32)).eval([(vals, ok)])
    assert list(out) == [2, 0, 10] and valid.all()
    with pytest.raises(E.AnsiError):
        E.If(E.Not(small), E.Arith("add", x, x, P.INT32, E.ANSI), E.Lit(0, P.INT32)).eval([(vals, ok)])


# ---- every plan of the GPU matrix compiles ------------------------------------------------------------------------------------------------
def _scan(names):
    return P.scan([M.COLUMNS[k] for k in names])


def _compiles(node):
    ok, why = native.supports(node)
    assert ok, why
    assert native.compile_plan(node)


@pytest.mark.parametrize("source", ["arrow", "parquet-int"])
def test_expression_lists_compile(source):
    names = M.source_names(source)
    c = M.Cols(names)
    for name in M.lists_for(source):
        for g in M.groups(M.LISTS[name](c)):
            _compiles(M.plan_of(_scan(names), None, g))
    for name in ("f32-legacy", "int-try", "narrow-decimals", "casts-decimal"):
        mode_outs = M.decimal_casts(c, E.ANSI) if name == "casts-decimal" else M.LISTS[name](c)
        for g in M.groups(mode_outs):
            _compiles(M.plan_of(_scan(names), E.Logic("or", E.Cmp("lt", c.f32, M.L(0.5, F32)), E.IsNull(c.i32)), g))


@pytest.mark.parametrize("k", range(M.FUZZ_PLANS))
def test_random_trees_compile(k):
    names = M.source_names(M.fuzz_source(k))
    pred, outs = M.fuzz_plan(k, names)
    _compiles(M.plan_of(_scan(names), pred, outs))


def test_random_trees_reach_every_node_kind_and_raise_sometimes():
    """the generator is not degenerate: every node class appears, ANSI plans exist and some of them raise in the interpreter"""
    kinds, raising = set(), 0
    _, cols = M.table()

    def walk(e):
        kinds.add(type(e).__name__)
        for ch in [getattr(e, a, None) for a in ("l", "r", "c", "a", "b", "v")] + list(getattr(e, "lits", [])):
            if isinstance(ch, E.Node):
                walk(ch)
    for k in range(M.FUZZ_PLANS):
        names = M.source_names(M.fuzz_source(k))
        pred, outs = M.fuzz_plan(k, names)
        for o in outs + ([pred] if pred is not None else []):
            walk(o)
        _, res = M.interp(pred, outs, cols, names)
        raising += any(isinstance(r, E.AnsiError) for r in res)
    assert {"Col", "Lit", "Arith", "Cmp", "Logic", "Not", "IsNull", "Cast", "If", "In", "Neg"} <= kinds
    assert 0 < raising < M.FUZZ_PLANS // 2


# ---- refusals -------------------------------------------------------------------------------------------------------------------------
D12 = P.DECIMAL(12, 2)
REFUSED = {
    "narrowing int cast": ([P.INT64], lambda: P.cast(P.bound(0, P.INT64), P.INT32, 0)),
    "narrowing float cast": ([F64], lambda: P.cast(P.bound(0, F64), F32, 0)),
    "float to int cast": ([F32], lambda: P.cast(P.bound(0, F32), P.INT64, 0)),
    "decimal to double": ([D12], lambda: P.cast(P.bound(0, D12), F64, 0)),
    "decimal to float": ([D12], lambda: P.cast(P.bound(0, D12), F32, 0)),
    "arithmetic with implicit result cast": ([P.INT32], lambda: P.add(P.bound(0, P.INT32), P.bound(0, P.INT32), P.INT64, 0)),
    "float arithmetic with implicit result cast": ([F32], lambda: P.multiply(P.bound(0, F32), P.bound(0, F32), F64, 0)),
    "comparison int32 / int64": ([P.INT32, P.INT64], lambda: P.lt(P.bound(0, P.INT32), P.bound(1, P.INT64))),
    "comparison float / double": ([F32, F64], lambda: P.eq(P.bound(0, F32), P.bound(1, F64))),
    "comparison decimals of different scales": ([D12, P.DECIMAL(12, 3)], lambda: P.gt(P.bound(0, D12), P.bound(1, P.DECIMAL(12, 3)))),
    "arithmetic on timestamps": ([P.TIMESTAMP], lambda: P.add(P.bound(0, P.TIMESTAMP), P.bound(0, P.TIMESTAMP), P.TIMESTAMP, 0)),
    "cast from bool": ([P.BOOL], lambda: P.cast(P.bound(0, P.BOOL), P.INT32, 0)),
}


@pytest.mark.parametrize("name", list(REFUSED))
def test_refused_as_unsupported(name):
    """refused by the planner as Unsupported -- not a PlanError, not a crash"""
    types, mk = REFUSED[name]
    node = P.projection(P.scan(types), [mk()])
    ok, why = native.supports(node)
    assert not ok and why
    with pytest.raises(native.Unsupported):
        native.compile_plan(node)
