"""GPU: HashJoin and SortMergeJoin at scale against the vectorised reference of tests/joinscale.py.  Every case compares every output
column bit for bit and in order, and asserts cb200_stats.join_build_rows / join_probe_rows / join_out_rows (and join_cond_pairs with a
condition).  Output is read with a batch size above chunkRows, so each batch returned is one batch the join emitted; the cases whose
point is the output split (probe input batches of at least chunkRows rows) assert how many there were.

Which case fails when a mechanism is wrong:
- the table's size and long linear-probe clusters (4 * 10^6 build keys, 8 * 10^6 probe rows): test_many_distinct_keys;
- the hash's mixing of each of 1 to 4 key words: test_key_words (tuples that differ only in word 0 or only in the last word);
- the stored-word check after a tag hit (k_join_probe's join_find): test_colliding_keys, on keys whose hashes share their tag and home
  slot -- one-key pairs differ in the last word only, two-key pairs in the first words only;
- k_join_emit's windows that start and end inside a run: test_hot_key;
- NULL keys, anti joins and FullOuter's NULL-key build rows: test_null_keys;
- k_join_unmatched's search over 2 * 10^6 runs and the per-run / per-row hit bytes: test_full_outer_unmatched;
- condition slices (cond_slice): test_conditions_at_scale;
- concatenated build batches, many probe batches, DeviceTables and per-side growing dictionaries: test_many_batches,
  test_device_tables, test_string_dictionaries;
- the refusal of a probe batch with 2^32 output rows or candidates (the count scan's 32-bit offsets): test_output_of_2_32_rows_refused,
  and just below it, under an aggregate: test_just_below_2_32_rows_under_an_aggregate (about 4.3 * 10^9 joined rows, which the device
  streams through the aggregate in a few seconds, so it stays in the file)."""
import functools

import numpy as np
import pyarrow as pa
import pytest

import joinscale as J
import partref
from joinref import INNER
from smjref import LEFT_OUTER, RIGHT_OUTER
from sources import device_table

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def run(cb, plan, inputs, chunk=None):
    """-> (the batches the plan emitted, stats)"""
    cfg = {"spark.comet.b200.chunkRows": str(chunk)} if chunk else None
    with cb.native.Plan(plan, inputs, config=cfg, batch_size=1 << 26) as p:
        batches = []
        while True:
            b = p.execute()
            if b is None:
                break
            batches.append(b)
        return batches, p.stats()


def case(cb, name, left, right, linputs=None, rinputs=None, chunk=None, lbatch=1 << 20, rbatch=1 << 20, count_batches=False, only=None):
    """every mode of J.CASES[name] (or those in `only`) over (left, right), each checked against the reference"""
    kinds, keys, _ = J.CASES[name]
    t = J.types_of(kinds) if name != "limit" else J.types_of(["i64", "i64", "i32"])
    li = linputs if linputs is not None else [left.to_batches(max_chunksize=lbatch)]
    ri = rinputs if rinputs is not None else [right.to_batches(max_chunksize=rbatch)]
    for op, jt, build_left, cname in J.modes(name):
        if only is not None and (op, jt, build_left, cname) not in only:
            continue
        cond = J.condition(cname, left.num_columns)
        what = (name, op, jt, build_left, cname)
        batches, st = run(cb, J.plan(op, jt, build_left, t, t, keys, cond), li + ri, chunk)
        res = J.join(left, right, keys, keys, jt, cond, build_left)
        want = J.table(left, right, res)
        got = pa.Table.from_batches(batches) if batches else None
        if want.num_rows == 0:
            assert got is None or got.num_rows == 0, what
        else:
            assert got is not None, what
            partref.assert_tables_equal(got, want)
        probe_left = not (build_left or jt == RIGHT_OUTER)
        build, probe = (right, left) if probe_left else (left, right)
        assert (st["join_build_rows"], st["join_probe_rows"], st["join_out_rows"]) == (build.num_rows, probe.num_rows, res.rows), (what, st)
        assert st["join_cond_pairs"] == res.candidates, (what, st["join_cond_pairs"], res.candidates)
        if chunk:
            assert max((b.num_rows for b in batches), default=0) <= chunk, what
            assert len(batches) >= -(-res.rows // chunk), what
        if count_batches and cond is None:
            pin = li if probe_left else ri
            sizes = [b.num_rows for b in pin[0]]
            assert len(batches) == res.batches(sizes, chunk or (1 << 26)), (what, len(batches), res.batches(sizes, chunk or (1 << 26)))


@functools.lru_cache(maxsize=None)
def data(name, *args):
    return getattr(J, name)(*args)


# ---- the table: size, probe clusters, key words, collisions -------------------------------------------------------------------------------
def test_many_distinct_keys(cb):
    """4 * 10^6 build rows of nearly distinct INT64 keys (consecutive integers, multiples of 2^20, random values) in a table of 2^23
    slots, 8 * 10^6 probe rows of which half hit; HashJoin inner with both build sides, semi and anti, and SortMergeJoin for every
    type, on inputs sorted by the key.  chunkRows 2^18: each probe batch's output leaves in several batches."""
    probe, build = data("distinct_keys")
    assert J.capacity(len(np.unique(np.asarray(build.column(0))))) == 1 << 23
    case(cb, "distinct", probe, build, chunk=1 << 18, lbatch=1 << 21, rbatch=1 << 21, count_batches=True)


@pytest.mark.parametrize("name", list(J.WORD_SETS))
def test_key_words(cb, name):
    """10^6 distinct tuples of 1 to 4 key words on the build side; the probe side holds them all and 10^6 tuples the build side lacks,
    each differing from a build tuple in its first or its last word only"""
    probe, build = data("word_sides", name)
    case(cb, f"words-{name}", probe, build)


@pytest.mark.parametrize("cap,mode,second", [(1024, "a", None), (1024, "b", None), (16384, "a", None), (16384, "b", None),
                                             (1024, "a", 3), (1024, "b", 3)])
def test_colliding_keys(cb, cap, mode, second):
    """keys whose hashes share their tag and their home slot (joinscale.colliding_pairs) in a table of `cap` slots.  a: only one key
    of each pair on the build side -- inner and semi match only it, anti keeps the other, and in SortMergeJoin FullOuter a build row
    whose partner alone was probed stays unmatched.  b: both keys on the build side -- each probe row finds only its own run.  With
    `second`, two-key tuples (x, 3) and (y, 3), searched for the 1 024-slot table only."""
    probe, build = data("collision_sides", cap, mode, second)
    case(cb, "collide" if second is None else "collide-2key", probe, build)


# ---- emit windows, NULL keys, FullOuter ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hot_on_build", [True, False], ids=["hot-build", "hot-probe"])
def test_hot_key(cb, hot_on_build):
    """one key with 5 * 10^5 rows on one side and 40 on the other, among 10^6 cold keys; chunkRows 65 536, so one probe row's matches
    fill several batches and windows start and end inside a run"""
    probe, build = data("hot_sides", hot_on_build)
    case(cb, "hot", probe, build, chunk=65536, count_batches=True)


def test_null_keys(cb):
    """10 % NULLs in the second of two keys on both sides: inner drops them, anti keeps the NULL-key probe rows, FullOuter emits the
    NULL-key build rows after the probe side"""
    probe, build = data("null_sides")
    case(cb, "nulls", probe, build, chunk=1 << 20, count_batches=True)


def test_full_outer_unmatched(cb):
    """2 * 10^6 build runs of 1 to 4 rows, half of them never hit: without a condition (per-run hit bytes, k_join_unmatched) and with
    left.u < right.u (per-build-row hit bytes)"""
    probe, build = data("unmatched_sides")
    case(cb, "unmatched", probe, build, chunk=1 << 20, count_batches=True)


def test_conditions_at_scale(cb):
    """every join type with left.u = right.u over a hot key of 30 x 200 000 candidates (each hot probe row's candidates span four
    65 536-pair condition slices): outer probe rows with no passing pair, and rows whose only passing pair is in a later slice"""
    left, right = data("condition_sides")
    res = J.join(left, right, [0], [0], LEFT_OUTER, J.condition("eq_u"))
    first = {int(l): int(r) for l, r in zip(res.left, res.right) if 10 <= l < 30}
    assert all(first[l] == -1 for l in range(20, 30))
    assert all(first[l] >= 65536 for l in range(10, 20))        # the run starts at right row 0: the pass is past the first slice
    case(cb, "conditions", left, right, chunk=65536, lbatch=100_000, rbatch=100_000)


# ---- batches and sources ----------------------------------------------------------------------------------------------------------------
def test_many_batches(cb):
    """a build side of 15 input batches (3 * 10^5 rows, above chunkRows) and a probe side of 50 input batches, which the scan may
    combine up to chunkRows rows, so only the least number of output batches is asserted"""
    probe, build = data("many_batch_sides")
    case(cb, "batches", probe, build, chunk=65536, lbatch=10_000, rbatch=20_000)


def test_device_tables(cb):
    """DeviceTables on both sides, the DECIMAL(18, 0) key 8 bytes wide; chunkRows below the tables"""
    probe, build = data("device_sides")
    t = J.types_of(J.CASES["device"][0])
    case(cb, "device", probe, build, linputs=[device_table(cb, probe, t, dec8=["k0"])], rinputs=[device_table(cb, build, t, dec8=["k0"])],
         chunk=1 << 18)


def test_string_dictionaries(cb):
    """a dictionary string key whose dictionaries differ per side and grow batch by batch (a few thousand distinct strings)"""
    (pb, ptbl), (bb, btbl) = J.string_sides()
    case(cb, "strings", ptbl, btbl, linputs=[pb], rinputs=[bb], chunk=65536)


# ---- 2^32 output rows ----------------------------------------------------------------------------------------------------------------------
def limit_sides(n_build):
    rng = np.random.default_rng(5)
    def side(n):
        return pa.table({"k": pa.array(np.full(n, 7, np.int64)), "row": pa.array(np.arange(n, dtype=np.int64)),
                         "u": pa.array(rng.integers(0, 100, n).astype(np.int32))})
    return side(65536), side(n_build)


@pytest.mark.parametrize("mode,message", [(("hash", INNER, False, None), "inner join output has 2\\^32 rows"),
                                          (("smj", LEFT_OUTER, False, None), "outer join output has 2\\^32 rows"),
                                          (("hash", INNER, False, "eq_u"), "join condition candidates number 2\\^32")])
def test_output_of_2_32_rows_refused(cb, mode, message):
    """65 536 x 65 536 rows of one key: exactly 2^32 output rows (or candidates) in one probe batch"""
    left, right = limit_sides(65536)
    t = J.types_of(["i64", "i64", "i32"])
    plan = J.plan(mode[0], mode[1], mode[2], t, t, [0], J.condition(mode[3]))
    with pytest.raises(cb.native.Unsupported, match=message):
        run(cb, plan, [left.to_batches(), right.to_batches()])


def test_just_below_2_32_rows_under_an_aggregate(cb):
    """65 536 x 65 535 rows of one key: 2^32 - 65 536 rows, counted and summed by a Partial aggregate"""
    P = cb.proto
    left, right = limit_sides(65535)
    t = J.types_of(["i64", "i64", "i32"])
    j = J.plan("hash", INNER, False, t, t, [0])
    agg = P.hash_agg(j, [], [P.agg_count([P.bound(0, P.INT64)]), P.agg_sum(P.bound(1, P.INT64), P.INT64), P.agg_sum(P.bound(4, P.INT64), P.INT64)],
                     P.PARTIAL)
    batches, st = run(cb, agg, [left.to_batches(), right.to_batches()])
    row = list(pa.Table.from_batches(batches).to_pylist()[0].values())
    n_l, n_r = 65536, 65535
    assert row[:3] == [n_l * n_r, n_r * (n_l * (n_l - 1) // 2), n_l * (n_r * (n_r - 1) // 2)], row
    assert (st["join_build_rows"], st["join_probe_rows"], st["join_out_rows"]) == (n_r, n_l, n_l * n_r) and n_l * n_r < 2**32
