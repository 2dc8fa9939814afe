"""CPU checks of the join scale cases (tests/joinscale.py): the vectorised reference equals the row-by-row references on slices of every
input, for every join type, build side and condition the GPU file runs; the comparison fails on each kind of wrong answer; the Python
row key words and join_hash equal a host compile of device/cb_sortkey.h; the colliding keys really collide; and every plan is accepted
and compiles."""
import ctypes as C
import os
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import condjoinref
import joinref
import joinscale as J
import partref
import smjref
from joinref import INNER, LEFT_SEMI
from smjref import FULL_OUTER, LEFT_OUTER

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "datafusion-comet_b200", "csrc")


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def sides(case):
    """(left, right) of each GPU input (the probe side is the left one); conditions use their own sides"""
    if case == "distinct":
        return J.distinct_keys()
    if case.startswith("words-"):
        return J.word_sides(case[len("words-"):])
    if case == "collide":
        return J.collision_sides(1024, "a")
    if case == "collide-2key":
        return J.collision_sides(1024, "a", second=3)
    return {"hot": J.hot_sides, "nulls": J.null_sides, "unmatched": J.unmatched_sides, "conditions": J.condition_sides,
            "batches": J.many_batch_sides, "device": J.device_sides}[case]()


def slices(left, right, seed):
    """2 000 left rows and 3 000 right rows, in input order: half of the right rows share a first key with a chosen left row"""
    rng = np.random.default_rng(seed)
    li = np.sort(rng.choice(left.num_rows, min(2000, left.num_rows), replace=False))
    ls = left.take(pa.array(li))
    near = np.flatnonzero(np.asarray(pc.is_in(right.column(0), value_set=pc.unique(ls.column(0).combine_chunks())).fill_null(False)))
    near = rng.choice(near, min(1500, len(near)), replace=False)
    far = rng.choice(right.num_rows, min(3000 - len(near), right.num_rows), replace=False)
    ri = np.unique(np.concatenate([near, far]))
    return ls, right.take(pa.array(ri))


def row_by_row(op, left, right, keys, jt, cond, build_left):
    if cond is not None:
        return condjoinref.cond_join_table(left, right, keys, keys, jt, cond, build_left)
    if op == "hash":
        return joinref.join_table(left, right, keys, keys, jt, build_left)
    return smjref.sort_merge_join_table(left, right, keys, keys, jt)


SLICED = ["distinct", "words-i32", "words-i64", "words-i64-i64", "words-dec38-i64-i32", "collide", "collide-2key", "hot", "nulls",
          "unmatched", "conditions", "batches", "device"]


@pytest.mark.parametrize("case", SLICED)
def test_reference_matches_row_by_row_on_slices(case):
    left, right = sides(case)
    keys = J.CASES[case][1]
    ls, rs = slices(left, right, len(case))
    n_match = 0
    for op, jt, build_left, cname in J.modes(case) + [("smj", jt, False, None) for jt in J.JOIN_TYPES]:
        cond = J.condition(cname, ls.num_columns)
        res = J.join(ls, rs, keys, keys, jt, cond, build_left)
        partref.assert_tables_equal(J.table(ls, rs, res), row_by_row(op, ls, rs, keys, jt, cond, build_left))
        if cond is not None:
            assert res.candidates == condjoinref.candidate_count(ls, rs, keys, keys, jt, build_left)
        if jt == INNER:
            n_match = max(n_match, res.rows)
    assert n_match > 20, n_match


def test_string_reference_matches_row_by_row():
    (pb, ptbl), (bb, btbl) = J.string_sides()
    ls, rs = slices(ptbl, btbl, 5)
    for op, jt, build_left, _ in J.modes("strings"):
        partref.assert_tables_equal(J.join_table(ls, rs, [0], [0], jt, None, build_left), row_by_row(op, ls, rs, [0], jt, None, build_left))


# ---- the comparison catches wrong answers ------------------------------------------------------------------------------------------------
def _fails(left, right, res, li, ri):
    bad = J.Result(np.asarray(li), None if ri is None else np.asarray(ri), 0, res.probe_out, res.unmatched)
    with pytest.raises(AssertionError):
        partref.assert_tables_equal(J.table(left, right, bad), J.table(left, right, res))


def test_comparison_catches_corruptions():
    left, right = slices(*J.null_sides(), 7)
    keys = [0, 1]
    inner = J.join(left, right, keys, keys, INNER)
    li, ri = inner.left.copy(), inner.right.copy()
    i = int(np.flatnonzero((li[1:] == li[:-1]) & (ri[1:] != ri[:-1]))[0])      # two build rows of one run, swapped
    ri[i], ri[i + 1] = ri[i + 1], ri[i]
    _fails(left, right, inner, li, ri)
    _fails(left, right, inner, np.delete(inner.left, 5), np.delete(inner.right, 5))               # one pair dropped
    outer = J.join(left, right, keys, keys, LEFT_OUTER)
    null_probe = np.flatnonzero(np.asarray(left.column(1).is_null()))
    pos = int(np.flatnonzero(np.isin(outer.left, null_probe))[0])
    ri = outer.right.copy()
    ri[pos] = 0                                                                    # a NULL-key probe row matched
    _fails(left, right, outer, outer.left, ri)
    lone = np.flatnonzero((outer.right == -1)[:-1] & (outer.left[1:] != outer.left[:-1]))
    p = int(lone[0])
    order = np.arange(outer.rows)
    order[p], order[p + 1] = p + 1, p                                              # a NULL-extended row after its neighbour
    _fails(left, right, outer, outer.left[order], outer.right[order])
    full = J.join(left, right, keys, keys, FULL_OUTER)
    assert full.unmatched > 0
    _fails(left, right, full, full.left[:-1], full.right[:-1])                     # one unmatched FullOuter build row missing
    semi = J.join(left, right, keys, keys, LEFT_SEMI)
    _fails(left, right, semi, np.delete(semi.left, 3), None)


def test_batch_count_of_the_reference():
    """each probe batch's output leaves in chunkRows windows; FullOuter's unmatched rows in their own"""
    left = pa.table({"k": pa.array([1, 1, 2, 3, 9]), "row": pa.array(np.arange(5))})
    right = pa.table({"k": pa.array([1, 1, 1, 2, 5, 6]), "row": pa.array(np.arange(6))})
    res = J.join(left, right, [0], [0], FULL_OUTER)
    assert list(res.probe_out) == [3, 3, 1, 1, 1] and res.unmatched == 2
    assert res.batches([2, 3], 2) == 3 + 2 + 1


# ---- row key words and join_hash against the host compile ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sk(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("cbjoinhash") / "libcb200_sortkey.so")
    subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(CSRC, "sortkey_test.cpp")])
    lib = C.CDLL(so)
    lib.cb_sk_kind.argtypes = [C.c_char_p]
    lib.cb_sk_encode.restype = C.c_longlong
    lib.cb_join_hash.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p]
    return lib


def host_words(sk, fields):
    n, nk = len(fields[0][2]), len(fields)
    kind = {"i32": b"i32", "i64": b"i64", "dec128": b"dec_large_128"}
    data, valids = [], []
    for k, v, valid in fields:
        if k == "dec128":
            d = np.empty((n, 2), np.int64)
            d[:, 0], d[:, 1] = v[0].view(np.int64), v[1]
        else:
            d = np.asarray(v, np.int32 if k == "i32" else np.int64)
        data.append(np.ascontiguousarray(d))
        valids.append(np.packbits(np.asarray(valid, bool), bitorder="little"))
    W = J.key_words(fields).shape[1]
    out = np.zeros(n * W, np.uint64)
    ints = lambda xs: (C.c_int * nk)(*xs)
    bad = sk.cb_sk_encode(nk, ints([sk.cb_sk_kind(kind[k]) for k, _, _ in fields]), ints([J.BITS[k] for k, _, _ in fields]), ints([0] * nk),
                          ints([1] * nk), (C.c_void_p * nk)(*[d.ctypes.data for d in data]), (C.c_void_p * nk)(*[v.ctypes.data for v in valids]),
                          (C.c_void_p * nk)(*([None] * nk)), ints([0] * nk), C.c_longlong(n), W, out.ctypes.data_as(C.POINTER(C.c_uint64)))
    assert bad == 0
    return out.reshape(n, W)


def host_hash(sk, words):
    words = np.ascontiguousarray(words, np.uint64)
    out = np.zeros(len(words), np.uint64)
    sk.cb_join_hash(words.ctypes.data, len(words), words.shape[1], out.ctypes.data)
    return out


def _random_fields(kinds, n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for k in kinds:
        valid = rng.random(n) > 0.1
        if k == "dec128":
            v = (rng.integers(0, 1 << 63, n).astype(np.uint64) * np.uint64(2) + rng.integers(0, 2, n).astype(np.uint64), rng.integers(-(1 << 62), 1 << 62, n))
        elif k == "i64":
            v = rng.integers(-(1 << 63), (1 << 63) - 1, n, endpoint=True)
        else:
            v = rng.integers(-(1 << 31), 1 << 31, n)
        out.append((k, v, valid))
    return out


@pytest.mark.parametrize("kinds", list(J.WORD_SETS.values()) + [["i32", "i32", "i32", "i32", "i32", "i32"]], ids=lambda k: "-".join(k))
def test_key_words_and_hash_match_the_host_compile(sk, kinds):
    """1 to 4 words, NULLs in every field"""
    fields = _random_fields(kinds, 20_000, len(kinds))
    w = J.key_words(fields)
    assert w.shape[1] == (sum(J.BITS[k] + 1 for k in kinds) + 63) // 64
    np.testing.assert_array_equal(w, host_words(sk, fields))
    np.testing.assert_array_equal(J.join_hash(w), host_hash(sk, w))


def test_single_int64_words():
    v = np.array([0, 5, -1, -(1 << 63), (1 << 63) - 1], np.int64)
    w = J.i64_words(v)
    assert (w[:, 0] == 1).all() and (w[:, 1] == (v.view(np.uint64) ^ np.uint64(1 << 63))).all()


@pytest.mark.parametrize("cap,second", [(1024, None), (16384, None), (1024, 3)])
def test_colliding_pairs_share_tag_and_home(sk, cap, second):
    """with the host compile's hash; the two-key pairs are equal in their last word, so a table comparing only that word merges them"""
    pairs = np.array(J.colliding_pairs(cap, 25 if cap > 1024 else 24, second), np.int64)
    assert len(pairs) >= (4 if cap > 1024 else 20), len(pairs)
    wx, wy = J.i64_words(pairs[:, 0], second), J.i64_words(pairs[:, 1], second)
    hx, hy = host_hash(sk, wx), host_hash(sk, wy)
    tx, homex = J.tag_home(hx, cap)
    ty, homey = J.tag_home(hy, cap)
    assert (tx == ty).all() and (homex == homey).all() and (pairs[:, 0] != pairs[:, 1]).all()
    if second is None:
        assert (wx[:, 0] == wy[:, 0]).all()                  # equal in word 0: a table comparing only word 0 merges them too
    else:
        assert (wx[:, -1] == wy[:, -1]).all()


@pytest.mark.parametrize("cap,mode,second", [(1024, "a", None), (1024, "b", None), (16384, "a", None), (16384, "b", None),
                                             (1024, "a", 3), (1024, "b", 3)])
def test_collision_sides_fill_their_capacity(cap, mode, second):
    probe, build = J.collision_sides(cap, mode, second)
    runs = len(np.unique(np.asarray(build.column(0))))
    assert J.capacity(runs) == cap
    pairs = np.array(J.colliding_pairs(cap, 25 if cap > 1024 else 24, second), np.int64)
    bk, pk = set(np.asarray(build.column(0)).tolist()), set(np.asarray(probe.column(0)).tolist())
    used = [p for p in pairs.tolist() if p[0] in bk or p[1] in bk]
    assert len(used) >= min(len(pairs), 4)
    for x, y in used:
        assert x in pk and y in pk or (mode == "a" and y in pk)
        assert (x in bk and y in bk) == (mode == "b")


@pytest.mark.parametrize("name", list(J.WORD_SETS))
def test_word_variants_differ_in_one_word(name):
    """the first half of the variants differ from their base tuple only in word 0, the second half only in the last word; every tuple
    is distinct"""
    kinds, base, var = J.word_tuples(name, n=20_000)
    ones = np.ones(20_000, bool)
    wb = J.key_words([(k, v, ones) for k, v in zip(kinds, base)])
    wv = J.key_words([(k, v, ones) for k, v in zip(kinds, var)])
    diff = wb != wv
    assert diff.any(axis=1).all()
    W = wb.shape[1]
    assert (diff.sum(axis=1) == 1).all()
    if W > 2:
        assert diff[:10_000, 0].all() and diff[10_000:, W - 1].all()
    allw = np.concatenate([wb, wv])
    assert len(np.unique(allw, axis=0)) == len(allw)


def _home_load(words, runs):
    cap = J.capacity(runs)
    _, home = J.tag_home(J.join_hash(words), cap)
    counts = np.bincount(home.astype(np.int64), minlength=cap)
    return cap, counts


def test_hash_spreads_the_scale_keys():
    """consecutive integers, multiples of 2^20 and tuples that differ in one word land on as many home slots as random hashes would
    (1 - e^-load of them occupied), with no pile-up: a hash that mixed a word poorly would fill few slots"""
    probe, build = J.distinct_keys()
    keys = np.unique(np.asarray(build.column(0)))
    sets = [J.i64_words(keys), J.i64_words(np.arange(1 << 20, dtype=np.int64) << 20), J.i64_words(np.arange(1 << 20, dtype=np.int64))]
    for name in J.WORD_SETS:
        kinds, base, var = J.word_tuples(name, n=200_000)
        ones = np.ones(200_000, bool)
        sets.append(np.concatenate([J.key_words([(k, v, ones) for k, v in zip(kinds, base)]), J.key_words([(k, v, ones) for k, v in zip(kinds, var)])]))
    for w in sets:
        cap, counts = _home_load(w, len(w))
        load = len(w) / cap
        occupied = (counts > 0).mean()
        assert abs(occupied - (1 - np.exp(-load))) < 0.01, (len(w), occupied, load)
        assert counts.max() < 16, counts.max()


# ---- plans ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(J.CASES))
def test_plans_supported_and_compile(cb, case):
    for m, plan in J.case_plans(case):
        ok, why = cb.native.supports(plan)
        assert ok, (m, why)
        assert cb.native.compile_plan(plan) is not None
