"""GPU parity: range and round-robin repartitioning (ShuffleWriter with RangePartition / RoundRobinPartition) against the CPU reference
(tests/rangeref.py), bit-exact and in order: every output batch and its partition starts.  Ends with two global sorts built on range
partitioning: one GPU (the device Sort over each partition) and 2 / 4 ranks through cb200_exchange."""
import os
import queue
import signal
import time

import numpy as np
import pyarrow as pa
import pytest

import partref
import rangeref as R
import sortref
from comet_b200 import proto as P
from rangecases import PTYPE, dec_array, pick_bounds, special_table
from sources import device_table, scan_of, write_parquet

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def with_row(cols, names):
    n = len(cols[names[0]])
    return pa.table({**{k: cols[k] for k in names}, "row": pa.array(np.arange(n, dtype=np.int64))})


def range_plan(cb, child, types, names, keys, n_parts, bounds, dup_first=False):
    """keys: (name, desc, nulls_first); dup_first sends the first key again (with the other direction) after the others"""
    orders = [P.sort_order(P.bound(names.index(c), types[names.index(c)]), d, f) for c, d, f in keys]
    if dup_first:
        c, d, f = keys[0]
        orders.append(P.sort_order(P.bound(names.index(c), types[names.index(c)]), not d, not f))
    rows = R.bound_literals(P, bounds, [types[names.index(c)] for c, _, _ in keys])
    return P.shuffle_writer(child, P.range_partitioning(orders, n_parts, rows))


def run(cb, plan, inputs, config=None):
    """every batch the plan returns, each with the partition starts that came with it"""
    out = []
    with cb.native.Plan(plan, inputs, config=config) as p:
        while True:
            b = p.execute()
            if b is None:
                break
            out.append((b, p.partition_starts()))
    return out


def check(got, tbl, expect):
    """got: [(batch, starts)] -- each batch the partitioning of its own input rows, in input order; expect(slice) -> (starts, _, table)"""
    row0 = 0
    for b, starts in got:
        want_starts, _, want = expect(tbl.slice(row0, b.num_rows))
        assert starts == want_starts
        partref.assert_tables_equal(b, want)
        row0 += b.num_rows
    assert row0 == tbl.num_rows


def check_range(cb, tbl, types, keys, n_parts, bounds, inputs=None, child=None, config=None, dup_first=False):
    plan = range_plan(cb, child or P.scan(types), types, tbl.column_names, keys, n_parts, bounds, dup_first)
    got = run(cb, plan, [tbl.to_batches(max_chunksize=8192)] if inputs is None else inputs, config)
    check(got, tbl, lambda s: R.range_partition(s, keys, bounds, n_parts))
    return got


def types_of(tbl):
    return [PTYPE.get(c, P.INT64) for c in tbl.column_names]


# ---- every key type x direction x NULL placement ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("col", list(PTYPE))
def test_single_key(cb, col):
    cols = special_table(30_000, 11)
    tbl = with_row(cols, list(PTYPE))
    types = types_of(tbl)
    for i, (desc, nf) in enumerate([(False, True), (False, False), (True, True), (True, False)]):
        keys = [(col, desc, nf)]
        for nb, n_parts in ((0, 1), (1, 2), (7, 200), (199, 200)):
            bounds = pick_bounds(tbl, keys, nb, 10 * i + nb)
            check_range(cb, tbl, types, keys, n_parts, bounds)


def test_bound_entries(cb):
    """boundary rows with NULL, NaN of both signs and payloads, -0.0 / +0.0 and type extremes, duplicated"""
    cols = special_table(20_000, 5)
    tbl = with_row(cols, ["f64", "f32", "i64", "d38"])
    types = types_of(tbl)
    f64 = np.array([0xFFF8000000000000, 0xFFF0000000000123, 0x8000000000000000, 0x0, 0x0, 0x7FF0000000000000, 0x7FF8000000000000,
                    0x7FF800000000BEEF], np.uint64).view(np.float64)
    for nf in (True, False):
        b = pa.array(f64, mask=np.zeros(len(f64), bool))
        b = pa.concat_arrays([pa.array([None], pa.float64()), b]) if nf else pa.concat_arrays([b, pa.array([None], pa.float64())])
        check_range(cb, tbl, types, [("f64", False, nf)], 16, pa.table({"k0": b}))
    f32 = pa.array(np.array([0xFF800123, 0x80000000, 0x0, 0x7FC00000, 0x7FC0BEEF], np.uint32).view(np.float32))
    check_range(cb, tbl, types, [("f32", False, True)], 8, pa.table({"k0": f32}))
    i64 = pa.array([np.iinfo(np.int64).max, np.iinfo(np.int64).max, 0, np.iinfo(np.int64).min], pa.int64())
    check_range(cb, tbl, types, [("i64", True, True)], 8, pa.table({"k0": i64}))
    m38 = 10**38 - 1
    check_range(cb, tbl, types, [("d38", False, False)], 8, pa.table({"k0": dec_array([-m38, -1, 0, m38, m38], 38, 4)}))


def test_multi_key_prefix(cb):
    """rows equal in a prefix of the keys: later keys decide; a repeated key is dropped; 4 words of key (230 bits)"""
    rng = np.random.default_rng(3)
    n = 40_000
    cols = special_table(n, 17)
    cols["g"] = pa.array(rng.integers(0, 3, n).astype(np.int32))
    tbl = with_row(cols, ["g", "s", "d38", "b", "f32"])
    types = [P.INT32] + types_of(tbl)[1:]
    for trial in range(3):
        keys = [("g", False, True)] + [(c, bool(rng.integers(2)), bool(rng.integers(2))) for c in ("s", "d38", "b", "f32")]
        for nb in (5, 150):
            bounds = pick_bounds(tbl, keys, nb, trial * 7 + nb)
            check_range(cb, tbl, types, keys, 200, bounds, dup_first=trial == 1)


@pytest.mark.parametrize("n_parts,keys", [(16384, ["i64"]), (16384, ["i32", "s", "d38"]), (3000, ["d38", "i64", "s"])])
def test_many_partitions(cb, n_parts, keys):
    """boundary sets that fit in shared memory and ones that do not (sampled top level, the search ending in L2)"""
    n = 200_000
    rng = np.random.default_rng(n_parts)
    cols = {"i64": pa.array(rng.integers(-10**6, 10**6, n)), "i32": pa.array(rng.integers(-50, 50, n).astype(np.int32)),
            "s": pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, 300, n).astype(np.int32)), pa.array([f"v{i:03d}" for i in range(300)])),
            "d38": dec_array([int(x) * 10**20 for x in rng.integers(-10**4, 10**4, n)], 38, 4)}
    tbl = with_row(cols, keys)
    types = [{"i64": P.INT64, "i32": P.INT32, "s": P.STRING, "d38": P.DECIMAL(38, 4)}[c] for c in keys] + [P.INT64]
    kk = [(c, i % 2 == 1, True) for i, c in enumerate(keys)]
    for nb in (n_parts - 1, n_parts // 3):
        bounds = pick_bounds(tbl, kk, nb, nb)
        check_range(cb, tbl, types, kk, n_parts, bounds)


def test_changing_dictionaries(cb):
    """string keys whose dictionary differs and grows between batches, values equal to a bound: the ids of one big batch"""
    rng = np.random.default_rng(9)
    batches = []
    for k, words in enumerate([["m", "c", "x"], ["a", "m", "zz", "c"], ["q", "b", "m", "mm", "", "x"]]):
        n = 3000
        d = pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, len(words), n).astype(np.int32), mask=rng.random(n) < 0.1), pa.array(words))
        batches.append(pa.record_batch([d, pa.array(np.arange(k * n, (k + 1) * n, dtype=np.int64))], names=["s", "row"]))
    whole = pa.table({"s": pa.concat_arrays([b.column(0).dictionary_decode() for b in batches]),
                      "row": pa.concat_arrays([b.column(1) for b in batches])})
    bounds = pa.table({"k0": pa.array(["b", "c", "m", "m", "n"])})
    for desc in (False, True):
        b = bounds if not desc else bounds.take(pa.array([4, 3, 2, 1, 0]))
        keys = [("s", desc, False)]
        plan = range_plan(cb, P.scan([P.STRING, P.INT64]), [P.STRING, P.INT64], ["s", "row"], keys, 8, b)
        got = run(cb, plan, [batches], config={"spark.comet.b200.chunkRows": "1024"})
        assert len(got) >= 2
        check(got, whole, lambda s: R.range_partition(s, keys, b, 8))


def test_plain_utf8_key_refused(cb):
    tbl = pa.table({"s": pa.array(["a", "b", "c"]), "row": pa.array([0, 1, 2], pa.int64())})
    plan = range_plan(cb, P.scan([P.STRING, P.INT64]), [P.STRING, P.INT64], ["s", "row"], [("s", False, True)], 4, pa.table({"k0": pa.array(["b"])}))
    with pytest.raises(cb.native.Unsupported, match="plain string"):
        run(cb, plan, [tbl.to_batches()])


def test_device_table_source(cb):
    cols = special_table(20_000, 23)
    s = cols["s"]   # device table dictionaries travel as C strings: no embedded NUL
    cols["s"] = pa.DictionaryArray.from_arrays(s.indices, pa.array([w.replace("\x00", "0") for w in s.dictionary.to_pylist()]))
    names = ["i8", "b", "d18", "s", "f32", "date"]
    tbl = with_row(cols, names)
    types = types_of(tbl)
    t = device_table(cb, tbl, types, dec8=("d18",))
    keys = [("d18", True, False), ("b", False, True), ("s", False, False)]
    bounds = pick_bounds(tbl, keys, 30, 1)
    got = run(cb, range_plan(cb, P.scan(types), types, tbl.column_names, keys, 31, bounds), [t], config={"spark.comet.b200.chunkRows": "8192"})
    assert len(got) >= 2
    check(got, tbl, lambda s: R.range_partition(s, keys, bounds, 31))


def test_native_scan_source(cb, tmp_path):
    rng = np.random.default_rng(2)
    n = 60_000
    cols = {"i16": (pa.array(rng.integers(-50, 50, n).astype(np.int16), mask=rng.random(n) < 0.1), P.INT16),
            "d7": (dec_array([int(x) for x in rng.integers(-10**6, 10**6, n)], 7, 2), P.DECIMAL(7, 2)),
            "sd": (pa.array([f"k{x}" for x in rng.integers(0, 40, n)]), P.STRING),
            "f64": (pa.array(rng.standard_normal(n)), P.DOUBLE),
            "row": (pa.array(np.arange(n, dtype=np.int64)), P.INT64)}
    path = str(tmp_path / "r.parquet")
    write_parquet(path, cols, True)
    names = list(cols)
    scan, types = scan_of(cb, cols, names, path)
    tbl = pa.table({k: cols[k][0] for k in names})
    keys = [("sd", False, True), ("d7", True, True), ("i16", False, False)]
    bounds = pick_bounds(tbl, keys, 40, 3)
    plan = range_plan(cb, scan, types, names, keys, 64, bounds)
    got = run(cb, plan, [], config={"spark.comet.b200.chunkRows": "40000"})
    assert len(got) >= 2
    check(got, tbl, lambda s: R.range_partition(s, keys, bounds, 64))


def test_partial_aggregate_state(cb):
    """ShuffleWriter(RangePartition) over HashAggregate(Partial): the map side of a sorted aggregation"""
    rng = np.random.default_rng(4)
    n = 100_000
    tbl = pa.table({"k": pa.array(rng.integers(0, 5000, n)), "v": pa.array(rng.integers(0, 100, n))})
    agg = P.hash_agg(P.scan([P.INT64, P.INT64]), [P.bound(0, P.INT64)], [P.agg_sum(P.bound(1, P.INT64), P.INT64)], P.PARTIAL)
    bounds = pa.table({"k0": pa.array([4000, 2500, 2500, 100], pa.int64())})
    keys = [("col_0", True, True)]
    plan = P.shuffle_writer(agg, P.range_partitioning([P.sort_order(P.bound(0, P.INT64), True, True)], 8,
                                                      R.bound_literals(P, bounds, [P.INT64])))
    got = run(cb, plan, [tbl.to_batches(max_chunksize=8192)])
    total = 0
    for b, starts in got:
        t = pa.table({"col_0": b.column(0), "s": b.column(1)})
        want_starts, _, _ = R.range_partition(t, keys, bounds, 8)
        assert starts == want_starts                      # each batch already in partition order: the ids are non-decreasing
        pids = R.range_pids(t, keys, bounds)
        assert (np.diff(pids) >= 0).all()
        total += b.num_rows
    assert total == len(np.unique(tbl.column("k").to_numpy()))


def test_changing_layouts(cb):
    """chunks whose validity buffers and dictionary code widths change (tests/layoutcases.py)"""
    import layoutcases as L
    n, C = 4 * 1024, 1024
    rng = np.random.default_rng(6)
    words = ["w%d" % i for i in range(20)]
    chunk = np.arange(n) // C
    xnull = np.isin(chunk, [1, 3]) & (rng.random(n) < 0.2)      # NULLs only in the chunks whose recipe holds them
    snull = np.isin(chunk, [0, 2]) & (rng.random(n) < 0.2)
    tbl = pa.table({"x": pa.array(rng.integers(-9, 9, n).astype(np.int32), mask=xnull),
                    "s": pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, 20, n).astype(np.int32), mask=snull), pa.array(words)),
                    "row": pa.array(np.arange(n, dtype=np.int64))})
    rec = [{"x": "none", "s": "nulls"}, {"x": "nulls", "s": "none"}, {"x": "zero", "s": "nulls"}, {"x": "nulls", "s": "zero"}]
    keys = [("x", False, True), ("s", True, False)]
    bounds = pick_bounds(tbl, keys, 9, 2)
    plan = range_plan(cb, P.scan([P.INT32, P.STRING, P.INT64]), [P.INT32, P.STRING, P.INT64], tbl.column_names, keys, 12, bounds)
    got = run(cb, plan, [L.source(L.chunked(tbl, C, rec))], config={"spark.comet.b200.chunkRows": str(C)})
    assert len(got) == 4
    check(got, tbl, lambda s: R.range_partition(s, keys, bounds, 12))


# ---- round-robin ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_cols", [1, 3, 8, 9, 12])
def test_round_robin(cb, oracle, n_cols):
    cols = special_table(25_000, n_cols)
    names = (list(PTYPE) * 2)[:n_cols]
    tbl = pa.table({f"c{i}": cols[c] for i, c in enumerate(names)})
    types = [PTYPE[c] for c in names]
    for m, n_parts in ((0, 200), (-1, 7), (n_cols - 1, 16384), (n_cols + 3, 2)):
        plan = P.shuffle_writer(P.scan(types), P.round_robin_partitioning(n_parts, m))
        got = run(cb, plan, [tbl.to_batches(max_chunksize=8192)])
        check(got, tbl, lambda s: R.round_robin_partition(oracle, s, n_parts, m))


# ---- global sorts ---------------------------------------------------------------------------------------------------------------------
def test_global_sort_one_gpu(cb):
    """range partitioning, then the device Sort over each partition: the concatenation is the stable sort of the whole input"""
    cols = special_table(50_000, 31)
    names = ["s", "f64", "d38", "i16"]
    tbl = with_row(cols, names)
    types = types_of(tbl)
    keys = [("s", False, False), ("f64", True, True), ("d38", False, True)]
    bounds = pick_bounds(tbl, keys, 63, 5)
    plan = range_plan(cb, P.scan(types), types, tbl.column_names, keys, 64, bounds)
    with cb.native.Plan(plan, [tbl.to_batches(max_chunksize=8192)], config={"spark.comet.b200.chunkRows": str(tbl.num_rows)}) as p:
        part = p.execute()
        starts = p.partition_starts()
    orders = [P.sort_order(P.bound(tbl.column_names.index(c), types[tbl.column_names.index(c)]), d, f) for c, d, f in keys]
    pieces = []
    for q in range(64):
        sl = part.slice(starts[q], starts[q + 1] - starts[q])
        if sl.num_rows == 0:
            continue
        sl = pa.table([sl.column(j).dictionary_encode() if pa.types.is_string(sl.column(j).type) else sl.column(j) for j in range(sl.num_columns)],
                      names=tbl.column_names)
        with cb.native.Plan(P.sort(P.scan(types), orders), [sl.to_batches()]) as p:
            pieces.append(p.collect())
    got = pa.concat_tables(pieces)
    want = sortref.sort_table(tbl, keys)
    partref.assert_tables_equal(got, want)


def _sort_rank_input(rank):
    rng = np.random.default_rng(100 + rank)
    n = 20_000 + 1000 * rank
    return pa.table({"k": pa.array(rng.integers(-1000, 1000, n), mask=rng.random(n) < 0.05),
                     "f": pa.array(rng.integers(-8, 8, n) / 4.0),
                     "row": pa.array(np.arange(n, dtype=np.int64) + rank * 10**6)})


SORT_KEYS = [("k", False, True), ("f", True, False)]


def _global_bounds(world):
    allt = pa.concat_tables([_sort_rank_input(r) for r in range(world)])
    return pick_bounds(allt, SORT_KEYS, world - 1, world)


def _sort_worker(rank, world, parent_pid, ids, results):
    """one rank on GPU `rank`: range partition its input into `world` partitions, exchange, sort what it received"""
    import ctypes as C
    C.CDLL(None).prctl(1, signal.SIGKILL)   # PR_SET_PDEATHSIG: dies with the parent
    if os.getppid() != parent_pid:
        os._exit(1)
    try:
        import comet_b200 as cb

        def bcast(b):
            if rank == 0:
                for _ in range(world - 1):
                    ids.put(b)
                return b
            return ids.get(timeout=60)
        comm = cb.native.Comm(rank, world, rank, bcast)
        tbl = _sort_rank_input(rank)
        types = [P.INT64, P.DOUBLE, P.INT64]
        plan = range_plan(cb, P.scan(types), types, tbl.column_names, SORT_KEYS, world, _global_bounds(world))
        mp_ = cb.native.Plan(plan, [tbl.to_batches(max_chunksize=8192)], config={"spark.comet.b200.chunkRows": str(1 << 20)}, device=comm.device)
        mp_.execute_device()
        recv, _ = comm.exchange(mp_)
        mp_.release()
        orders = [P.sort_order(P.bound(tbl.column_names.index(c), types[tbl.column_names.index(c)]), d, f) for c, d, f in SORT_KEYS]
        got = None
        if recv.n_rows:
            with cb.native.Plan(P.sort(P.scan(types), orders), [recv], device=comm.device) as p:
                got = p.collect()
        recv.release()
        comm.destroy()
        results.put((rank, True, got.column(2).to_numpy().tolist() if got is not None else []))
    except Exception:
        import traceback
        results.put((rank, False, traceback.format_exc()[-2000:]))
        os._exit(1)


@pytest.mark.parametrize("world", [2, 4])
def test_global_sort_across_ranks(world):
    """2 and 4 ranks through cb200_exchange: the ranks' sorted partitions, in rank order, are the stable sort of every rank's input
    (rank 0's rows first among equal keys)"""
    import multiprocessing as mp

    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"{world} ranks need {world} visible GPUs ({torch.cuda.device_count()} visible)")
    ctx = mp.get_context("spawn")
    ids, results = ctx.Queue(), ctx.Queue()
    procs = [ctx.Process(target=_sort_worker, args=(r, world, os.getpid(), ids, results), daemon=True) for r in range(world)]
    for p in procs:
        p.start()
    deadline = time.monotonic() + 180
    msgs = {}
    try:
        while len(msgs) < world and time.monotonic() < deadline:
            try:
                r, ok, payload = results.get(timeout=1)
                msgs[r] = (ok, payload)
                if not ok:
                    break
            except queue.Empty:
                if not any(p.is_alive() for p in procs):
                    break
        for p in procs:
            p.join(max(0.0, deadline - time.monotonic()))
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join(10)
    failed = [f"rank {r}: {m}" for r, (ok, m) in msgs.items() if not ok]
    assert not failed and len(msgs) == world, ("\n".join(failed), sorted(msgs))
    allt = pa.concat_tables([_sort_rank_input(r) for r in range(world)])
    want = allt.column("row").to_numpy()[sortref.order(allt, SORT_KEYS)]
    got = np.concatenate([np.array(msgs[r][1], np.int64) for r in range(world)])
    assert (got == want).all()
