"""Inputs and a vectorised reference for the join at scale (tests/test_gpu_join_scale.py), for every join type the join node runs:
HashJoin (inner with either build side, left semi, left anti) and SortMergeJoin (inner, left / right / full outer, left semi, left anti),
with or without a join condition.  Its answers equal tests/joinref.py, tests/smjref.py and tests/condjoinref.py bit for bit and in the
same order (tests/test_join_scale_cpu.py checks that on slices of every input), but it is built from numpy sorts and searches, so it
reaches millions of rows:

- Key matching.  Each key column of both sides together is turned into integer ranks by pyarrow's dictionary encoding (strings by
  their bytes, decimals and timestamps by value); several keys are folded into one rank per tuple.  A NULL in any key gives rank -1,
  which matches nothing.  The build rows are stably sorted by rank and each probe row finds its run with searchsorted.
- Pairs.  np.repeat over the run lengths: probe rows in input order, a row's matches in build input order.
- Outer joins.  A probe row without a (passing) match gets one pair with build row -1.  FullOuter appends the build rows in no
  (passing) pair, NULL keys included, in build input order.  RightOuter probes the right side.
- Semi / anti joins keep the probe rows with a (passing) match / without one.
- Conditions are evaluated (tests/exprs.py nodes) on the candidate pairs only; their number is cb200_stats.join_cond_pairs.

The module also restates the join's row key words (device/cb_sortkey.h, every field with a null bit set on a valid value, the last
key least significant, word 0 most significant) and join_hash, and searches for INT64 keys whose hashes share their tag (hash >> 32)
and home slot (hash & (capacity - 1)): the keys on which the table must compare stored words."""
import functools

import numpy as np
import pyarrow as pa

from condjoinref import node_columns
from joinref import INNER, LEFT_ANTI, LEFT_SEMI, _array
from smjref import FULL_OUTER, LEFT_OUTER, RIGHT_OUTER

JOIN_TYPES = [INNER, LEFT_OUTER, RIGHT_OUTER, FULL_OUTER, LEFT_SEMI, LEFT_ANTI]
HASH_MODES = [(INNER, False), (INNER, True), (LEFT_SEMI, False), (LEFT_ANTI, False)]    # (join type, build left)


# ---- the reference ---------------------------------------------------------------------------------------------------------------------------
def tuple_ranks(left, right, left_keys, right_keys):
    """(left ranks, right ranks): equal key tuples get equal ranks >= 0, a tuple with a NULL gets -1"""
    n_l = left.num_rows
    rank = None
    for a, b in zip(left_keys, right_keys):
        both = pa.concat_arrays([_array(left.column(a)), _array(right.column(b))])
        r = np.asarray(both.dictionary_encode().indices.fill_null(-1), dtype=np.int64)
        if rank is None:
            rank = r
            continue
        null = (rank < 0) | (r < 0)
        folded = np.where(null, -1, rank * (int(r.max()) + 1) + r)
        rank = np.where(null, -1, np.unique(folded, return_inverse=True)[1].reshape(-1).astype(np.int64))
    if rank is None:
        raise ValueError("a keyed join needs at least one key")
    return rank[:n_l], rank[n_l:]


def expand(probe_rank, build_rank):
    """the candidate pairs (probe rows, build rows), probe rows in input order, a row's matches in build input order"""
    valid = np.flatnonzero(build_rank >= 0)
    order = valid[np.argsort(build_rank[valid], kind="stable")]
    srt = build_rank[order]
    lo = np.searchsorted(srt, probe_rank, "left")
    cnt = np.where(probe_rank >= 0, np.searchsorted(srt, probe_rank, "right") - lo, 0)
    total = int(cnt.sum())
    p = np.repeat(np.arange(len(probe_rank), dtype=np.int64), cnt)
    within = np.arange(total, dtype=np.int64) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    return p, order[np.repeat(lo, cnt) + within]


class _PairColumns:
    """the condition's columns (left ++ right) over pairs (li, ri), built on first use as condjoinref.node_columns gives them"""

    def __init__(self, left, right, li, ri):
        self.left, self.right, self.li, self.ri, self.cache = left, right, li, ri, {}

    def __getitem__(self, i):
        if i not in self.cache:
            tbl, idx = (self.left, self.li) if i < self.left.num_columns else (self.right, self.ri)
            col = _array(tbl.column(i if i < self.left.num_columns else i - self.left.num_columns)).take(pa.array(idx))
            self.cache[i] = node_columns(pa.table([col], names=["c"]))[0]
        return self.cache[i]


class Result:
    """the operator's output rows: `left` / `right` row indices per output row (-1 = NULL-extended; `right` is None for semi / anti
    joins), the candidates a condition was evaluated on, and each probe row's output rows (probe order) plus FullOuter's unmatched
    build rows, from which the emitted batches follow"""

    def __init__(self, left, right, candidates, probe_out, unmatched):
        self.left, self.right, self.candidates, self.probe_out, self.unmatched = left, right, candidates, probe_out, unmatched

    @property
    def rows(self):
        return len(self.left)

    def batches(self, probe_batch_rows, chunk):
        """batches a join without a condition emits: each probe batch's output in chunkRows windows, then FullOuter's unmatched rows"""
        out = 0
        for a, b in zip(np.cumsum([0] + list(probe_batch_rows[:-1])), np.cumsum(probe_batch_rows)):
            out += -(-int(self.probe_out[a:b].sum()) // chunk)
        return out - (-self.unmatched // chunk)


def join(left, right, left_keys, right_keys, join_type, cond=None, build_left=False):
    """the join node's output over pa.Tables left and right (HashJoin: build_left only with INNER; SortMergeJoin never builds left,
    but probes the right side for RIGHT_OUTER)"""
    if build_left and join_type != INNER:
        raise ValueError("only an inner hash join builds the left side")
    lr, rr = tuple_ranks(left, right, left_keys, right_keys)
    probe_right = build_left or join_type == RIGHT_OUTER
    pr, br = (rr, lr) if probe_right else (lr, rr)
    n_p, n_b = len(pr), len(br)
    p, b = expand(pr, br) if n_p and n_b else (np.zeros(0, np.int64), np.zeros(0, np.int64))
    ok = np.ones(len(p), bool)
    if cond is not None and len(p):
        li, ri = (b, p) if probe_right else (p, b)
        v, valid = cond.eval(_PairColumns(left, right, li, ri))
        ok = np.asarray(v, dtype=bool) & np.asarray(valid, dtype=bool)
    n_cand = len(p) if cond is not None else 0
    p, b = p[ok], b[ok]
    passed = np.bincount(p, minlength=n_p) > 0
    if join_type in (LEFT_SEMI, LEFT_ANTI):
        keep = np.flatnonzero(passed == (join_type == LEFT_SEMI))
        out = np.zeros(n_p, np.int64)
        out[keep] = 1
        return Result(keep, None, n_cand, out, 0)
    unmatched = np.zeros(0, np.int64)
    if join_type != INNER:                                   # a probe row without a passing pair: one NULL-extended row in its place
        lone = np.flatnonzero(~passed)
        p = np.concatenate([p, lone])
        b = np.concatenate([b, np.full(len(lone), -1, np.int64)])
        order = np.argsort(p, kind="stable")
        p, b = p[order], b[order]
        if join_type == FULL_OUTER:
            hit = np.zeros(n_b, bool)
            hit[b[b >= 0]] = True
            unmatched = np.flatnonzero(~hit)
    probe_out = np.bincount(p, minlength=n_p)
    p = np.concatenate([p, np.full(len(unmatched), -1, np.int64)])
    b = np.concatenate([b, unmatched])
    li, ri = (b, p) if probe_right else (p, b)
    return Result(li, ri, n_cand, probe_out, len(unmatched))


def _take(tbl, idx):
    ia = pa.array(idx, pa.int64(), mask=idx < 0)
    return [_array(tbl.column(i)).take(ia) for i in range(tbl.num_columns)]


def table(left, right, res):
    """the expected output table of a Result: the left columns, then the right ones (semi / anti: the left ones)"""
    cols = _take(left, res.left)
    names = [f"l{i}" for i in range(left.num_columns)]
    if res.right is not None:
        cols += _take(right, res.right)
        names += [f"r{i}" for i in range(right.num_columns)]
    return pa.table(cols, names=names)


def join_table(left, right, left_keys, right_keys, join_type, cond=None, build_left=False):
    return table(left, right, join(left, right, left_keys, right_keys, join_type, cond, build_left))


# ---- row key words and join_hash ---------------------------------------------------------------------------------------------------------
BITS = {"i32": 32, "i64": 64, "dec128": 128}
M64 = (1 << 64) - 1


def key_words(fields):
    """row keys (n, W) uint64 of fields [(kind, values, valid)]: kind "i32" / "i64" (integer arrays) or "dec128" ((lo uint64, hi
    int64) word arrays); the first field most significant, each field's null bit above its value and set on a valid value"""
    total = sum(BITS[k] + 1 for k, _, _ in fields)
    W = max(1, (total + 63) // 64)
    n = len(fields[0][2])
    w = np.zeros((n, W), np.uint64)

    def put(off, v, nb):
        lw, sh = off >> 6, off & 63
        w[:, W - 1 - lw] |= v << np.uint64(sh)
        if sh and sh + nb > 64:
            w[:, W - 2 - lw] |= v >> np.uint64(64 - sh)

    off = 0
    for kind, vals, valid in reversed(fields):
        valid = np.asarray(valid, bool)
        zero = np.uint64(0)
        if kind == "dec128":
            lo, hi = vals
            put(off, np.where(valid, np.asarray(lo).view(np.uint64), zero), 64)
            put(off + 64, np.where(valid, np.asarray(hi).view(np.uint64) ^ np.uint64(1 << 63), zero), 64)
        elif kind == "i64":
            put(off, np.where(valid, np.asarray(vals, np.int64).view(np.uint64) ^ np.uint64(1 << 63), zero), 64)
        else:
            v = (np.asarray(vals, np.int64).astype(np.uint64) ^ np.uint64(1 << 31)) & np.uint64(0xFFFFFFFF)
            put(off, np.where(valid, v, zero), 32)
        off += BITS[kind]
        put(off, valid.astype(np.uint64), 1)
        off += 1
    return w


def _fmix(h):
    h ^= h >> np.uint64(33)
    h *= np.uint64(0xff51afd7ed558ccd)
    h ^= h >> np.uint64(33)
    h *= np.uint64(0xc4ceb9fe1a85ec53)
    h ^= h >> np.uint64(33)
    return h


def join_hash(words):
    """join_hash (device/cb_sortkey.h) of each row of words (n, W)"""
    with np.errstate(over="ignore"):
        h = np.full(len(words), 0x9E3779B97F4A7C15, np.uint64)
        for j in range(words.shape[1]):
            h ^= words[:, j]
            h = _fmix(h)
    return h


def capacity(runs):
    """the table's slots for `runs` distinct non-NULL build keys: the smallest power of two >= max(1024, 2 x runs)"""
    cap = 1024
    while cap < 2 * runs:
        cap <<= 1
    return cap


def tag_home(h, cap):
    return h >> np.uint64(32), h & np.uint64(cap - 1)


def i64_words(v, second=None):
    """words of one INT64 key v, or of the two keys (v, second) with second a constant"""
    v = np.asarray(v, np.int64)
    ones = np.ones(len(v), bool)
    if second is None:
        return key_words([("i64", v, ones)])
    return key_words([("i64", v, ones), ("i64", np.full(len(v), second, np.int64), ones)])


SEARCH_START = 1 << 40


@functools.lru_cache(maxsize=None)
def colliding_pairs(cap, log2_n, second=None):
    """pairs (x, y) of INT64 keys among 2^log2_n consecutive values from SEARCH_START whose join_hash shares its tag and its home slot
    at `cap` slots (with `second`: of the two-key tuples (x, second), (y, second), equal in their last word), each value in at most
    one pair.  Fails when the search finds none."""
    v = np.arange(SEARCH_START, SEARCH_START + (1 << log2_n), dtype=np.int64)
    h = join_hash(i64_words(v, second))
    tag, home = tag_home(h, cap)
    key = (tag << np.uint64(cap.bit_length() - 1)) | home
    del h, tag, home
    order = np.argsort(key, kind="stable")
    ks = key[order]
    dup = np.flatnonzero(ks[1:] == ks[:-1])
    pairs, used = [], set()
    for i in dup:
        x, y = int(v[order[i]]), int(v[order[i + 1]])
        if x not in used and y not in used:
            pairs.append((x, y))
            used.update((x, y))
    assert pairs, f"no colliding INT64 keys at {cap} slots among 2^{log2_n} values"
    return tuple(pairs)


# ---- inputs ------------------------------------------------------------------------------------------------------------------------------
def dec128(lo, hi, valid=None, precision=38, scale=0):
    """a decimal128 array from its unscaled value's words"""
    n = len(lo)
    data = np.empty((n, 2), np.int64)
    data[:, 0], data[:, 1] = np.asarray(lo).view(np.int64), hi
    bufs = [None if valid is None else pa.py_buffer(np.packbits(np.asarray(valid, bool), bitorder="little")), pa.py_buffer(data.tobytes())]
    nulls = 0 if valid is None else int((~np.asarray(valid, bool)).sum())
    return pa.Array.from_buffers(pa.decimal128(precision, scale), n, bufs, null_count=nulls)


def with_rows(cols, seed=0, u=False):
    """a table of the key columns, then row (the row number) and, with u, an int32 in [0, 100) with 1 % NULLs"""
    n = len(next(iter(cols.values())))
    cols = dict(cols)
    cols["row"] = pa.array(np.arange(n, dtype=np.int64))
    if u:
        rng = np.random.default_rng(seed)
        cols["u"] = pa.array(rng.integers(0, 100, n).astype(np.int32), mask=rng.random(n) < 0.01)
    return pa.table(cols)


def distinct_keys():
    """(build, probe) of one INT64 key, sorted by it.  Build: 4 * 10^6 rows, nearly all distinct -- consecutive integers, multiples of
    2^20 and random values, 1 % of them repeated.  Probe: 8 * 10^6 rows, half of them build keys, half keys the build side lacks (more
    consecutive integers and multiples of 2^20, and random values)."""
    rng = np.random.default_rng(11)
    pool = np.concatenate([np.arange(3_000_000, dtype=np.int64), (np.arange(3_000_000, dtype=np.int64) + 5) << 20,
                           rng.integers(-(1 << 62), 1 << 62, 2_000_000)])
    pool = rng.permutation(np.unique(pool))
    build = pool[:4_000_000].copy()
    build[rng.choice(4_000_000, 40_000, replace=False)] = build[rng.choice(4_000_000, 40_000, replace=False)]
    absent = pool[4_000_000:]
    probe = np.concatenate([rng.choice(build, 4_000_000), rng.choice(absent, 4_000_000)])
    b, p = np.sort(build), np.sort(probe)
    return with_rows({"k": pa.array(p)}), with_rows({"k": pa.array(b)})


WORD_SETS = {"i32": ["i32"], "i64": ["i64"], "i64-i64": ["i64", "i64"], "dec38-i64-i32": ["dec128", "i64", "i32"]}


def word_tuples(name, n=1_000_000, seed=21):
    """(base, variant) field lists for key set `name`: n distinct base tuples and, for each, a variant the base set lacks that differs
    from it only in word 0 (the first half) or only in the last word (the second half) of the row key.  One- and two-word keys have a
    single informative word; their variants change the value's high bits (first half) or its low bit (second half)."""
    rng = np.random.default_rng(seed)
    half = n // 2
    kinds = WORD_SETS[name]
    spread = (np.arange(half, dtype=np.int64) * 2654435761) % (1 << 29)         # distinct: an odd multiplier is a bijection mod 2^29
    first = np.arange(n) < half
    if name == "i32":
        v = rng.permutation(np.concatenate([np.arange(half), spread + (1 << 20)]))
        base, var = [v], [np.where(first, v + (1 << 30), -1 - v)]
    elif name == "i64":
        v = rng.permutation(np.concatenate([np.arange(half), (spread + 1) << 20]))
        base, var = [v], [np.where(first, v ^ (1 << 61), -1 - v)]
    elif name == "i64-i64":
        a = rng.integers(0, 1 << 62, n)
        b = np.arange(n, dtype=np.int64) * 7919
        base, var = [a, b], [np.where(first, a | np.int64(-(1 << 63)), a), np.where(first, b, -1 - b)]
    else:
        lo = rng.integers(0, 1 << 63, n).astype(np.uint64)
        hi = rng.integers(-(1 << 40), 1 << 40, n)
        x = rng.integers(-(1 << 62), 1 << 62, n)
        y = np.arange(n, dtype=np.int64) * 3 - n
        base = [(lo, hi), x, y]
        var = [(lo, np.where(first, hi + (1 << 36), hi)), x, np.where(first, y, -1 - y)]  # hi + 2^36: unscaled value + 2^100
    return kinds, base, var


def _field_array(kind, vals):
    if kind == "dec128":
        return dec128(vals[0], vals[1])
    return pa.array(np.asarray(vals, np.int64).astype(np.int32 if kind == "i32" else np.int64))


def word_sides(name):
    """(probe, build): the build side holds the base tuples; the probe side every base tuple and every variant, shuffled"""
    kinds, base, var = word_tuples(name)
    n = len(base[-1]) if not isinstance(base[-1], tuple) else len(base[-1][0])
    rng = np.random.default_rng(len(name))
    perm = rng.permutation(2 * n)

    def cat(a, b):
        return (np.concatenate([a[0], b[0]]), np.concatenate([a[1], b[1]])) if isinstance(a, tuple) else np.concatenate([a, b])

    def shuffled(v):
        return (v[0][perm], v[1][perm]) if isinstance(v, tuple) else v[perm]
    build = with_rows({f"k{i}": _field_array(k, b) for i, (k, b) in enumerate(zip(kinds, base))})
    probe = with_rows({f"k{i}": _field_array(k, shuffled(cat(b, v))) for i, (k, b, v) in enumerate(zip(kinds, base, var))})
    return probe, build


def collision_sides(cap, mode, second=None):
    """(probe, build) of colliding INT64 keys (colliding_pairs) at `cap` slots, filled with other keys so that the build side's
    distinct keys need exactly `cap` slots.  mode "a": the build side holds x of each pair (two rows), the probe side y of every pair
    and x of every other pair; mode "b": the build side holds both keys, the probe side both.  With `second`, every row's second key
    is that constant."""
    pairs = np.array(colliding_pairs(cap, 25 if cap > 1024 else 24, second), np.int64)[: 120 if cap == 1024 else 64]
    x, y = pairs[:, 0], pairs[:, 1]
    build_keys = x if mode == "a" else np.concatenate([x, y])
    runs_wanted = cap // 2 - 7                                  # capacity(runs) == cap
    rng = np.random.default_rng(cap + len(mode))
    fill = rng.integers(-(1 << 60), 0, runs_wanted - len(build_keys))  # below SEARCH_START: no filler is a pair key
    build = np.repeat(np.concatenate([build_keys, fill]), 2)
    if mode == "a":
        probe = np.concatenate([y, x[::2], fill[::3]])
    else:
        probe = np.concatenate([x, y, fill[::3]])
    build, probe = np.sort(build), rng.permutation(probe)
    bcols, pcols = {"k0": pa.array(build)}, {"k0": pa.array(probe)}
    if second is not None:
        bcols["k1"], pcols["k1"] = pa.array(np.full(len(build), second, np.int64)), pa.array(np.full(len(probe), second, np.int64))
    return with_rows(pcols), with_rows(bcols)


def hot_sides(hot_on_build=True):
    """(probe, build) of one INT64 key sorted by it: 10^6 cold keys, and a hot key (-1) with 5 * 10^5 rows on one side and 40 on the other"""
    rng = np.random.default_rng(31)
    cold = rng.permutation(np.arange(2_000_000, dtype=np.int64) * 3)
    many = np.concatenate([cold[:1_000_000], np.full(500_000, -1, np.int64)])
    few = np.concatenate([cold[500_000:1_500_000], np.full(40, -1, np.int64)])
    b, p = (many, few) if hot_on_build else (few, many)
    return with_rows({"k": pa.array(np.sort(p))}), with_rows({"k": pa.array(np.sort(b))})


def null_sides():
    """(probe, build): keys (INT64, INT32), 10 % NULLs in the INT32 key on both sides, sorted by the keys (NULLs first), 2 * 10^6 rows
    each, key tuples repeated a few times"""
    def side(seed):
        rng = np.random.default_rng(seed)
        n = 2_000_000
        a, b = rng.integers(0, 400_000, n), rng.integers(0, 3, n).astype(np.int32)
        null = rng.random(n) < 0.1
        o = np.lexsort((b, ~null, a))
        return with_rows({"k0": pa.array(a[o]), "k1": pa.array(b[o], mask=null[o])})
    return side(41), side(42)


def unmatched_sides():
    """(probe, build) for FullOuter: 2 * 10^6 build runs of 1 to 4 rows, half of them hit by one probe row each; the probe side also
    has 10^6 keys the build side lacks.  Sorted by the key; u for the condition."""
    rng = np.random.default_rng(51)
    runs = np.arange(2_000_000, dtype=np.int64) * 2
    build = np.sort(np.repeat(runs, rng.integers(1, 5, len(runs))))
    probe = np.sort(np.concatenate([rng.choice(runs, 1_000_000, replace=False), rng.choice(runs + 1, 1_000_000, replace=False)]))
    return with_rows({"k": pa.array(probe)}, 52, u=True), with_rows({"k": pa.array(build)}, 53, u=True)


HOT_BUILD, HOT_PROBE = 200_000, 30


def condition_sides():
    """(left, right) for conditions at scale, sorted by the key k: a hot key (0) with HOT_PROBE left rows and HOT_BUILD right rows,
    and 2 * 10^5 cold keys of 1 or 2 rows per side.  With the condition left.u = right.u about 1 % of the hot candidates pass; left
    hot rows 10-19 have u = 1000 + j, which only one right hot row holds, near the end of the run (a later condition slice than the
    row's first candidate), and rows 20-29 u = 5000, which no right row holds."""
    rng = np.random.default_rng(61)
    cold_l = np.repeat(np.arange(1, 200_001, dtype=np.int64), rng.integers(1, 3, 200_000))
    cold_r = np.repeat(np.arange(100_001, 300_001, dtype=np.int64), rng.integers(1, 3, 200_000))
    lk = np.concatenate([np.zeros(HOT_PROBE, np.int64), cold_l])
    rk = np.concatenate([np.zeros(HOT_BUILD, np.int64), cold_r])
    lu = rng.integers(0, 100, len(lk)).astype(np.int32)
    ru = rng.integers(0, 100, len(rk)).astype(np.int32)
    lu[10:20] = 1000 + np.arange(10)
    lu[20:30] = 5000
    ru[HOT_BUILD - 1 - 7 * np.arange(10)] = 1000 + np.arange(10)
    lm, rm = rng.random(len(lk)) < 0.01, rng.random(len(rk)) < 0.01
    lm[:HOT_PROBE] = False
    rm[HOT_BUILD - 1 - 7 * np.arange(10)] = False
    left = pa.table({"k": pa.array(lk), "row": pa.array(np.arange(len(lk), dtype=np.int64)), "u": pa.array(lu, mask=lm)})
    right = pa.table({"k": pa.array(rk), "row": pa.array(np.arange(len(rk), dtype=np.int64)), "u": pa.array(ru, mask=rm)})
    return left, right


def many_batch_sides():
    """(probe, build) of keys (INT64, INT32) sorted by them: 5 * 10^5 probe rows and 3 * 10^5 build rows, some keys on one side only"""
    def side(n, seed):
        rng = np.random.default_rng(seed)
        a, b = rng.integers(0, 60_000, n), rng.integers(0, 2, n).astype(np.int32)
        o = np.lexsort((b, a))
        return with_rows({"k0": pa.array(a[o]), "k1": pa.array(b[o])})
    return side(500_000, 71), side(300_000, 72)


def device_sides():
    """(probe, build) of keys (DECIMAL(18, 0), INT64) sorted by them, 10^6 rows each, 5 % NULLs in the decimal"""
    def side(seed):
        rng = np.random.default_rng(seed)
        n = 1_000_000
        d, x = rng.integers(-300_000, 300_000, n) * 10**12 + 17, rng.integers(0, 2, n)
        null = rng.random(n) < 0.05
        o = np.lexsort((x, d, ~null))
        return with_rows({"k0": dec128(d[o], d[o] >> 63, ~null[o], 18, 0), "k1": pa.array(x[o])})
    return side(81), side(82)


STRINGS = [f"key-{i:05d}-{'x' * (i % 7)}" for i in range(3000)]


def string_batches(n_batches, per, words_of, seed):
    """(dictionary batches, plain table): batch b carries the dictionary words_of(b) and codes into it (10 % NULLs)"""
    rng = np.random.default_rng(seed)
    out, plain = [], []
    for b in range(n_batches):
        words = words_of(b)
        s = pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, len(words), per).astype(np.int32), mask=rng.random(per) < 0.1), pa.array(words))
        v = pa.array(np.arange(b * per, (b + 1) * per, dtype=np.int64))
        out.append(pa.record_batch([s, v], names=["s", "row"]))
        plain.append(pa.record_batch([s.dictionary_decode(), v], names=["s", "row"]))
    return out, pa.Table.from_batches(plain)


def string_sides():
    """((probe batches, probe table), (build batches, build table)): the probe dictionary grows batch by batch and holds strings the
    build side lacks; the build dictionary is another order of another subset, growing too"""
    extra = [f"probe-only-{i}" for i in range(200)]
    probe = string_batches(20, 20_000, lambda b: STRINGS[: 500 + 125 * b] + extra[: 10 * b], 91)
    build = string_batches(5, 10_000, lambda b: STRINGS[::-1][: 1500 + 300 * b], 92)
    return probe, build


# ---- plans -------------------------------------------------------------------------------------------------------------------------------
JT_CODE = {INNER: 0, LEFT_OUTER: 1, RIGHT_OUTER: 2, FULL_OUTER: 3, LEFT_SEMI: 4, LEFT_ANTI: 5}
SMJ_ALL = [("smj", jt, False) for jt in JOIN_TYPES]
HASH_ALL = [("hash", jt, bl) for jt, bl in HASH_MODES]


def condition(name, n_left=3):
    """the conditions of the scale cases over sides (k, row, u): left.u = right.u (about 1 % of random pairs) or left.u < right.u"""
    import comet_b200.proto as P
    import exprs as E
    if name is None:
        return None
    return E.Cmp({"eq_u": "eq", "lt_u": "lt"}[name], E.Col(2, P.INT32), E.Col(n_left + 2, P.INT32))


def types_of(names):
    import comet_b200.proto as P
    return [{"i32": P.INT32, "i64": P.INT64, "dec128": P.DECIMAL(38, 0), "dec18": P.DECIMAL(18, 0), "str": P.STRING}[n] for n in names]


def plan(op, jt, build_left, ltypes, rtypes, keys, cond=None, lchild=None, rchild=None):
    """a HashJoin or SortMergeJoin over scans of ltypes / rtypes on key columns `keys` of both sides"""
    import comet_b200.proto as P
    lchild = lchild if lchild is not None else P.scan(ltypes)
    rchild = rchild if rchild is not None else P.scan(rtypes)
    lkeys, rkeys = [P.bound(i, ltypes[i]) for i in keys], [P.bound(i, rtypes[i]) for i in keys]
    c = cond.proto() if cond is not None else None
    if op == "hash":
        return P.hash_join(lchild, rchild, lkeys, rkeys, JT_CODE[jt], P.BUILD_LEFT if build_left else P.BUILD_RIGHT, condition=c)
    return P.sort_merge_join(lchild, rchild, lkeys, rkeys, JT_CODE[jt], [P.sort_order(k) for k in lkeys], condition=c)


# every case of the GPU file: (column kinds of both sides, key columns, [(operator, join type, build left, condition name)])
CASES = {
    "distinct": (["i64", "i64"], [0], HASH_ALL + SMJ_ALL),
    "words-i32": (["i32", "i64"], [0], [("hash", INNER, False), ("hash", LEFT_ANTI, False)]),
    "words-i64": (["i64", "i64"], [0], [("hash", INNER, False), ("hash", LEFT_ANTI, False)]),
    "words-i64-i64": (["i64", "i64", "i64"], [0, 1], [("hash", INNER, False), ("hash", LEFT_ANTI, False)]),
    "words-dec38-i64-i32": (["dec128", "i64", "i32", "i64"], [0, 1, 2], [("hash", INNER, False), ("hash", LEFT_ANTI, False)]),
    "collide": (["i64", "i64"], [0], [("hash", INNER, False), ("hash", LEFT_SEMI, False), ("hash", LEFT_ANTI, False),
                                      ("smj", FULL_OUTER, False)]),
    "collide-2key": (["i64", "i64", "i64"], [0, 1], [("hash", INNER, False), ("hash", LEFT_ANTI, False), ("smj", FULL_OUTER, False)]),
    "hot": (["i64", "i64"], [0], [("hash", INNER, False), ("hash", INNER, True), ("smj", LEFT_OUTER, False)]),
    "nulls": (["i64", "i32", "i64"], [0, 1], [("hash", INNER, False), ("hash", LEFT_ANTI, False), ("smj", FULL_OUTER, False)]),
    "unmatched": (["i64", "i64", "i32"], [0], [("smj", FULL_OUTER, False, None), ("smj", FULL_OUTER, False, "lt_u")]),
    "conditions": (["i64", "i64", "i32"], [0], [m + ("eq_u",) for m in SMJ_ALL + HASH_ALL]),
    "batches": (["i64", "i32", "i64"], [0, 1], [("hash", INNER, False), ("hash", LEFT_SEMI, False), ("hash", LEFT_ANTI, False),
                                                ("smj", FULL_OUTER, False)]),
    "device": (["dec18", "i64", "i64"], [0, 1], [("hash", INNER, False), ("smj", FULL_OUTER, False)]),
    "strings": (["str", "i64"], [0], [("hash", INNER, False), ("hash", INNER, True), ("hash", LEFT_ANTI, False), ("smj", FULL_OUTER, False)]),
    "limit": (["i64", "i64"], [0], [("hash", INNER, False), ("smj", LEFT_OUTER, False), ("hash", INNER, False, "eq_u")]),
}


def modes(case):
    """the (operator, join type, build left, condition name) of a case"""
    return [m if len(m) == 4 else m + (None,) for m in CASES[case][2]]


def case_plans(case):
    kinds, keys, _ = CASES[case]
    t = types_of(kinds)
    if case == "limit":
        t = types_of(["i64", "i64", "i32"])
    return [(m, plan(m[0], m[1], m[2], t, t, keys, condition(m[3], len(t)))) for m in modes(case)]
