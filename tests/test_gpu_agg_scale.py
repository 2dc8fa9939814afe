"""GPU parity of the hash aggregate at high cardinality against the vectorised reference of tests/aggscale.py, group by group: keys,
values and validity of every state column and result, for the inputs where the key table grows, id ranges spill, the reserved rows
(the NULL key, the key -1) move, wide keys are re-inserted, many warps meet one new key, a DeviceTable source sizes the table from
the rows still to come, and a stream launch is discarded and repeated.

Every case asserts the strategy that ran (cb200_stats.agg_strategies) and, where it is meant to grow, that the id-addressed state
rows were regrown with groups in them (cb200_stats.agg_table_grows).  The aggregates run as the two plans of aggscale.MERGE_SETS
(a merging hash aggregate cannot stage all twelve state layouts at once); a Partial also runs all twelve in one plan."""
import functools

import pyarrow as pa
import pytest

import aggref as R
import aggscale as A
from sources import device_table

pytestmark = pytest.mark.gpu

TABLE, STREAM, DENSE, MIGRATED = 2, 4, 1, 8


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def run(cb, plan, inputs, cfg=None, chunk=None):
    """-> (output table, stats)"""
    cfg = dict(cfg or A.TABLE_CFG)
    if chunk:
        cfg["spark.comet.b200.chunkRows"] = str(chunk)
    with cb.native.Plan(plan, inputs, config=cfg) as p:
        out = p.collect()
        return out, p.stats()


def state_types(d, aggset):
    return d.key_types + A.state_types(A.aggs(len(d.keys), aggset))


def dict_keys(tbl):
    """string keys dictionary-encoded, as a shuffle carries them (a plain Utf8 key column is limited to 4096 distinct values)"""
    cols = [c.dictionary_encode() if c.type == pa.string() else c for c in tbl.columns]
    return pa.table(cols, names=tbl.column_names)


def pipeline(cb, d, aggset, inputs, cfg=None, chunk=None, bits=TABLE, merge=True, unique=True, merge_device=False):
    """Partial -> Final and (merge) Partial -> PartialMerge -> Final, each output checked and each stage's strategy asserted;
    returns every stage's stats by name"""
    ref = d.ref()
    stats = {}
    state, stats["partial"] = run(cb, d.partial_plan(aggset), inputs, cfg, chunk)
    state = dict_keys(state)
    assert stats["partial"]["agg_strategies"] == bits, f"strategy bits {stats['partial']['agg_strategies']:#x}, want {bits:#x}"
    A.check(state, ref, f"{d.name} {aggset} partial", "state", aggset, unique=unique)
    if aggset not in A.MERGE_SETS:
        return stats
    merge_chunk = 65536 if merge_device else None
    src = [device_table(cb, state, state_types(d, aggset))] if merge_device else [state]
    res, stats["final"] = run(cb, d.merge_plan(aggset, R.FINAL), src, chunk=merge_chunk)
    A.check(res, ref, f"{d.name} {aggset} partial->final", "result", aggset, fed=state)
    if merge:
        src = [device_table(cb, state, state_types(d, aggset))] if merge_device else [state]
        merged, stats["merge"] = run(cb, d.merge_plan(aggset, R.PARTIAL_MERGE), src, chunk=merge_chunk)
        A.check(merged, ref, f"{d.name} {aggset} partial->merge", "state", aggset, fed=state)
        merged = dict_keys(merged)
        res2, stats["merge-final"] = run(cb, d.merge_plan(aggset, R.FINAL), [merged])
        A.check(res2, ref, f"{d.name} {aggset} partial->merge->final", "result", aggset, fed=merged)
    for stage in ("final", "merge", "merge-final"):
        if stage in stats:
            assert stats[stage]["agg_strategies"] == TABLE, (stage, stats[stage]["agg_strategies"])
    return stats


def grows(stats, stage="partial"):
    return stats[stage]["agg_table_grows"]


def device(cb, d):
    """the input as a DeviceTable, decimals 8 bytes wide"""
    return [device_table(cb, d.table(), d.dts, dec8=[f"c{i}" for i, t in enumerate(d.dts) if t.name == "DECIMAL"])]


@functools.lru_cache(maxsize=None)
def data(name):
    """each input (and its reference) built once per session: the Arrow-stream and DeviceTable cases share them"""
    return dict(A.all_data())[name]()


# 1. growth with every accumulator kind, three chunk sizes: the smaller the chunks, the more often the rows relocate
def test_growth_every_accumulator(cb):
    d = data("growth")
    g = {}
    for chunk in (4096, 65536, None):
        for aggset in A.MERGE_SETS:
            g[chunk, aggset] = grows(pipeline(cb, d, aggset, [d.batches()], chunk=chunk, merge=chunk == 4096))
    for aggset in A.MERGE_SETS:
        assert g[4096, aggset] > g[65536, aggset] > 0 and g[65536, aggset] > g[None, aggset], g


def test_partial_all_twelve_aggregates_in_one_plan(cb):
    """the widest accumulator row (every word kind of the twelve aggregates side by side) relocated range by range"""
    d = data("growth")
    assert grows(pipeline(cb, d, "all", [d.batches()], chunk=4096)) > 0


# 2. distinct counts around 32 768, 65 536 and 131 072, new keys in every chunk: the key table doubles while the ids grow
@pytest.mark.parametrize("distinct", A.CROSSINGS)
def test_capacity_crossings(cb, distinct):
    d = A.crossing(distinct)
    for aggset in A.MERGE_SETS:
        assert grows(pipeline(cb, d, aggset, [d.batches()], chunk=8192, merge=False)) > 0


# 3. the reserved rows (NULL key, key -1) before and after growths
@pytest.mark.parametrize("early", [True, False], ids=["early-and-late", "late-only"])
def test_reserved_rows_through_growth(cb, early):
    d = data(f"reserved-{'early' if early else 'late'}")
    for aggset in A.MERGE_SETS:
        assert grows(pipeline(cb, d, aggset, [d.batches()], chunk=8192)) > 0
    k = d.ref().kuniq                                              # both reserved groups exist (and were checked with the rest)
    assert (k[:, 0] == 0).any() and ((k[:, 0] == 1) & (k[:, 1] == -1)).any()


# 4. every row a new key: 1024-row chunks have fewer warps than id ranges (their home ranges fill and spill); one chunk does not
def test_id_range_spill(cb):
    d = A.all_new()
    for aggset in A.MERGE_SETS:
        tiny = grows(pipeline(cb, d, aggset, [d.batches()], chunk=1024, merge=False))
        one = grows(pipeline(cb, d, aggset, [d.batches()], merge=False))
        assert tiny > 10 and one == 0, (tiny, one)


# 5. two- to four-word keys, NULLs in each key column, ~5 * 10^5 groups
@pytest.mark.parametrize("which", list(A.WIDE))
def test_wide_keys_at_scale(cb, which):
    d = data(f"wide-{which}")
    for aggset in A.MERGE_SETS:
        assert grows(pipeline(cb, d, aggset, [d.batches()], chunk=65536)) > 0


# 6. 10 % of the rows on 8 keys among 10^6 cold keys: many warps claim the same new key at once while the table grows
def test_hot_and_cold_keys(cb):
    d = A.hot_cold()
    for aggset in A.MERGE_SETS:
        assert grows(pipeline(cb, d, aggset, [d.batches()], chunk=65536, merge=False)) > 0


# 7. DeviceTable sources: the table is sized from the rows still to come
@pytest.mark.parametrize("name,chunk", [("growth", 65536), ("reserved-early", 8192), ("reserved-late", 8192), ("wide-i64-i64", 65536),
                                        ("wide-i64-i32-date-i8", 65536), ("wide-dec18-i64", 65536)])
def test_device_table_source(cb, name, chunk):
    d = data(name)
    for aggset in A.MERGE_SETS:
        assert grows(pipeline(cb, d, aggset, device(cb, d), chunk=chunk, merge=False)) > 0


def test_device_table_estimate_too_small_and_too_large(cb):
    """few distinct keys first: the ratio estimate is too small and the table grows again; the reverse sizes it too large at once"""
    small, large = A.skewed(True), A.skewed(False)
    for aggset in A.MERGE_SETS:
        g_small = grows(pipeline(cb, small, aggset, device(cb, small), chunk=65536, merge=False))
        g_large = grows(pipeline(cb, large, aggset, device(cb, large), chunk=65536, merge=False))
        assert g_small > g_large > 0, (g_small, g_large)


def test_merging_from_device_table_state(cb):
    """Final and PartialMerge over a DeviceTable of ~5 * 10^5-group Partial state in 65 536-row slices: a merging aggregate sizes for
    every row still to come at its first slice (most keys are new), so it never regrows; claim-first probing (CB_CAS_FIRST)"""
    d = data("wide-i64-i64")
    for aggset in A.MERGE_SETS:
        st = pipeline(cb, d, aggset, [d.batches()], chunk=65536, merge_device=True)
        assert grows(st, "final") == 0 and grows(st, "merge") == 0, (grows(st, "final"), grows(st, "merge"))
        assert d.ref().ng > 4 * 65536


# 8. the stream strategy from a DeviceTable
def test_stream_discarded_launch_from_device_table(cb):
    """one slice: the head's run estimate is far too small for the tail, so the launch is discarded (the reserved rows restored from
    their snapshot), the arrays grow and the launch is repeated.  The NULL key has rows in the head and the tail: a missing restore
    would count them twice in its SUM / COUNT / AVG / decimal words (MIN / MAX cannot tell: the repeat adds the same rows)."""
    d = data("clustered")
    for aggset in A.MERGE_SETS:
        st = pipeline(cb, d, aggset, device(cb, d), cfg=A.STREAM_CFG, bits=STREAM, unique=False, merge=False)
        assert st["partial"]["agg_stream_reruns"] == 1, st["partial"]["agg_stream_reruns"]


def test_stream_sized_from_remaining_rows(cb):
    """2^18-row slices: every slice but the last has rows still to come.  The slice whose runs first outgrow the sampled arrays
    sizes them for the rest at the ratio seen so far (StreamState, 1.25 x ratio x remaining): one regrowth and no discarded launch,
    where growing by half each time would regrow again a slice later"""
    d = data("clustered-slices")
    for aggset in A.MERGE_SETS:
        st = pipeline(cb, d, aggset, device(cb, d), cfg=A.STREAM_CFG, chunk=1 << 18, bits=STREAM, unique=False, merge=False)
        assert (grows(st), st["partial"]["agg_stream_reruns"]) == (1, 0)


# 9. dense -> key table mid-stream, then growth
def test_dense_to_hash_migration_then_growth(cb):
    d = A.migrate()
    for aggset in A.MERGE_SETS:
        assert grows(pipeline(cb, d, aggset, [d.batches()], chunk=d.batch_rows, bits=DENSE | MIGRATED | TABLE, unique=False)) > 0
