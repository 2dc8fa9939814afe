"""GPU: the exchange step (cb200_exchange) and the small-payload all-gather (cb200_comm_allgather_small) against CPU references.

One GPU (world = 1, always runs): a ShuffleWriter into one partition, then the local copy, the byte-per-row validity / booleans of
the received table, their packing to bitmaps and the TableSource's 1024-row slicing, read back through a plain Scan plan.
  raw rows   every fixed-width column type, Arrow / device-table / NativeScan sources, no / some / all NULLs, 0 .. 2500 rows: the
             received table equals the reference partitioning bit for bit (floats by their bits, NULL slots by validity)
  Config 4   Partial -> ShuffleWriter -> exchange -> Final against tests/aggref.py over the whole input
  stats      rows and bytes are exact: every column moves its values and one validity byte per row, NULLs or not
  empty      a map plan that emitted no batch takes part with zero rows of its schema

Several GPUs (skipped when fewer are visible): one spawned process per GPU, the NCCL id handed over a multiprocessing queue.  Each
worker rebuilds every rank's input from (seed, rank) and checks its own result; ranks that disagree on NULLs, and ranks with no rows,
are part of the matrix."""
import ctypes as C
import os
import queue
import signal
import time
import traceback

import numpy as np
import pyarrow as pa
import pytest

import aggref as R
import exchangecases as X
import partref
from sources import device_table, write_parquet
from test_gpu_agg_matrix import check_results, check_states, rows_of

pytestmark = pytest.mark.gpu

CHUNK = 1024   # the reader's spark.comet.b200.chunkRows: a received table of more rows is handed out in 1024-row slices


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


@pytest.fixture(scope="module")
def comm(cb):
    c = cb.native.Comm(0, 1, 0)
    yield c
    c.destroy()


def read_back(cb, recv, types, device=0):
    """the received table through a plain Scan plan on the communicator's device (None when it has no rows)"""
    with cb.native.Plan(cb.proto.scan(types), [recv], config={"spark.comet.b200.chunkRows": str(CHUNK)}, device=device) as p:
        return p.collect()


def exchange_map(cb, comm, plan, inputs, mode="device", config=None):
    """run the map plan's one batch on the communicator's device, exchange it, release the map plan (as bench.py does):
    -> (map rows or None, table, stats)"""
    p = cb.native.Plan(plan, inputs, config=config, device=comm.device)
    out = p.execute_device() if mode == "device" else p.execute()
    rows = None if out is None else (out[0] if mode == "device" else out.num_rows)
    recv, st = comm.exchange(p)
    p.release()
    return rows, recv, st


def check_stats(st, sent, received, types):
    assert st["rows_sent"] == sent and st["rows_received"] == received, st
    assert st["bytes_sent"] == sent * X.row_bytes(types), (st, X.row_bytes(types))
    assert st["bytes_received"] == received * X.row_bytes(types), st


# ---- raw rows, one GPU ----------------------------------------------------------------------------------------------------------------
def raw_source(cb, tmp_path, source, n, nulls, seed):
    """(map inputs, map plan child or None, proto types, column names, expected table)"""
    if source.startswith("parquet"):
        cols, want = X.parquet_cols(n, seed, nulls)
        path = str(tmp_path / "x.parquet")
        write_parquet(path, cols, source == "parquet-int")
        fields = [(k, cols[k][1], True) for k in X.PARQUET]
        return [], cb.proto.native_scan(fields, fields, [path]), [cols[k][1] for k in X.PARQUET], X.PARQUET, want
    tbl, types = X.raw_table(n, seed, nulls)
    inputs = [device_table(cb, tbl, types, dec8=("d9", "d18"))] if source == "device" else [tbl.to_batches(max_chunksize=700)] if n else [tbl]
    return inputs, None, types, X.RAW, tbl


# zero rows only from the Arrow source: a source of no rows emits no batch whatever its layout, and the map plan that emitted none is
# what the exchange sees
RAW_GRID = [(source, nulls, n) for source in ("stream", "device", "parquet-int", "parquet-flba") for nulls in ("none", "some", "all")
            for n in ([0] if source == "stream" else []) + [1, 31, 33, 2500]]


@pytest.mark.parametrize("source,nulls,n", RAW_GRID)
def test_raw_rows(cb, oracle, comm, tmp_path, source, nulls, n):
    """a ShuffleWriter over a Scan into one partition, exchanged: the input in order, bit for bit.  2500 rows make three 1024-row
    slices of the received table, the last one not a multiple of 8 rows."""
    inputs, child, types, names, want = raw_source(cb, tmp_path, source, n, nulls, seed=n * 7 + len(source))
    keys = X.RAW_KEYS if source in ("stream", "device") else ["i32", "d12"]
    rows, recv, st = exchange_map(cb, comm, X.raw_map_plan(types, names, keys, 1, child), inputs)
    try:
        assert recv.n_rows == n and (rows or 0) == n
        check_stats(st, n, n, types)
        got = read_back(cb, recv, types)
        if n == 0:
            assert rows is None and got is None
        else:
            partref.assert_tables_equal(got, X.expected_partitions(oracle, want, keys, 1)[0])
    finally:
        recv.release()


@pytest.mark.parametrize("mode", ["device", "arrow"])
def test_exchange_after_either_execute(cb, oracle, comm, mode):
    """the exchange reads the batch cb200_execute (Arrow export) and cb200_execute_device leave behind alike"""
    tbl, types = X.raw_table(3000, 5)
    rows, recv, st = exchange_map(cb, comm, X.raw_map_plan(types, X.RAW, ["i64"], 1), [tbl.to_batches(max_chunksize=1000)], mode)
    assert rows == 3000
    check_stats(st, 3000, 3000, types)
    partref.assert_tables_equal(read_back(cb, recv, types), tbl)
    recv.release()


def test_two_exchanges_on_one_communicator(cb, oracle, comm):
    """schemas and sizes change between exchanges; the first table stays valid after the second exchange"""
    t1, ty1 = X.raw_table(40, 6, names=["b", "d38", "row"])
    t2, ty2 = X.raw_table(5000, 7, names=["f32", "i8", "date", "i64", "row"])
    _, r1, s1 = exchange_map(cb, comm, X.raw_map_plan(ty1, ["b", "d38", "row"], ["d38"], 1), [t1])
    _, r2, s2 = exchange_map(cb, comm, X.raw_map_plan(ty2, ["f32", "i8", "date", "i64", "row"], ["i8", "f32"], 1), [t2])
    check_stats(s1, 40, 40, ty1)
    check_stats(s2, 5000, 5000, ty2)
    partref.assert_tables_equal(read_back(cb, r2, ty2), t2)
    partref.assert_tables_equal(read_back(cb, r1, ty1), t1)
    r1.release()
    r2.release()


def test_table_outlives_its_communicator(cb, oracle):
    """a received table is read and released after its communicator (and the communicator's stream) are gone"""
    tbl, types = X.raw_table(2000, 8)
    c = cb.native.Comm(0, 1, 0)
    _, recv, _ = exchange_map(cb, c, X.raw_map_plan(types, X.RAW, ["date"], 1), [tbl])
    c.destroy()
    partref.assert_tables_equal(read_back(cb, recv, types), tbl)
    recv.release()


# ---- Config 4, one GPU -----------------------------------------------------------------------------------------------------------------
def run_e2e(cb, comm, case, world=1, filtered=False):
    """Partial -> ShuffleWriter -> exchange -> Final, every plan on the communicator's device: (map rows or None, received state
    table, stats, Final result)"""
    rows, recv, st = exchange_map(cb, comm, case.map_plan(world, filtered), [case.batches()], config=case.config())
    try:
        states = read_back(cb, recv, case.state_types(), comm.device)
        with cb.native.Plan(case.final_plan(), [recv], device=comm.device) as f:
            res = f.collect()
    finally:
        recv.release()
    return rows, states, st, res


def check_e2e(case, table, states, res, stage, keep=None):
    """the received states (merged by the reference) and the Final result against aggref over `table`; `keep(keys)` restricts the
    reference to the groups this rank owns"""
    exp_state = R.partial(table, case.dts, case.key_cols, case.aggs) if table.num_rows else {}
    exp = R.aggregate(table, case.dts, case.key_cols, case.aggs) if table.num_rows else {}
    if keep is not None:
        exp_state = {k: v for k, v in exp_state.items() if keep(k)}
        exp = {k: v for k, v in exp.items() if keep(k)}
    got_state = rows_of(states, case)
    check_states(got_state, exp_state, case, stage + " states")
    check_results(rows_of(res, case, state=False), exp, case, stage, R.final(got_state, case.aggs))


@pytest.mark.parametrize("aggset", ["dec", "f64"])
@pytest.mark.parametrize("nulls", ["some", "none"])
@pytest.mark.parametrize("key", list(X.E2E_KEYS))
def test_partial_exchange_final(cb, comm, key, nulls, aggset):
    case = X.e2e_case(key, seed=900 + list(X.E2E_KEYS).index(key), nulls=nulls, aggset=aggset)
    rows, states, st, res = run_e2e(cb, comm, case)
    assert rows is not None and rows > 0
    check_stats(st, rows, rows, case.state_types())
    check_e2e(case, case.table(), states, res, f"{case.name}/{nulls}")


@pytest.mark.parametrize("how", ["no rows", "filtered"])
def test_grouped_partial_with_no_rows(cb, comm, how):
    """a grouped Partial over no rows emits no batch (a filter that removes every row: a 0-row batch); its ShuffleWriter takes part
    with zero rows either way, and the Final emits nothing"""
    case = X.e2e_case("i64", seed=5, n=0 if how == "no rows" else 500)
    rows, states, st, res = run_e2e(cb, comm, case, filtered=how == "filtered")
    assert rows == (None if how == "no rows" else 0) and states is None and res is None
    check_stats(st, 0, 0, case.state_types())


def test_empty_map_plan(cb, comm):
    """A map plan that emitted no batch returns a 0-row table with the plan's schema; an ungrouped Final over it emits the one row of
    fresh accumulators (the grouped Final emits nothing: test_grouped_partial_with_no_rows).  The table outlives the map plan."""
    P = cb.proto
    aggs = X.e2e_aggs(0, "dec")
    types = R.state_schema([], aggs)
    empty = pa.table([pa.array([], type=R.arrow_type(t)) for t in types], names=[f"s{i}" for i in range(len(types))])
    p = cb.native.Plan(X.raw_map_plan(types, list(range(len(types))), [0], 1), [empty])
    assert p.execute_device() is None and p.partition_starts() == []
    recv, st = comm.exchange(p)
    p.release()
    assert recv.n_rows == 0
    check_stats(st, 0, 0, types)
    assert read_back(cb, recv, types) is None
    with cb.native.Plan(R.merge_plan([], aggs), [recv]) as f:
        res = f.collect()
    assert res is not None and res.num_rows == 1
    want = R.final([], aggs, ungrouped=True)[()]
    got = [R.pyvalues(res.column(i), a.result_type())[0] for i, a in enumerate(aggs)]
    recv.release()
    assert got == want, (got, want)


# ---- refusals ----------------------------------------------------------------------------------------------------------------------------
def exchange_error(cb, comm, plan_handle):
    from comet_b200 import native
    l = native.lib()
    l.cb200_exchange.restype = C.c_void_p
    l.cb200_exchange.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(native.ExchangeStats), C.POINTER(native._Error)]
    err = native._Error()
    h = l.cb200_exchange(comm.handle if comm else None, plan_handle, None, None, C.byref(err))
    assert not h
    return err.code, err.message.decode(errors="replace")


def test_refusals(cb, oracle, comm):
    P = cb.proto
    words = pa.DictionaryArray.from_arrays(pa.array([0, 1, 0], pa.int8()), pa.array(["x", "y"]))
    dict_tbl = pa.table({"s": words, "v": pa.array([1, 2, 3], pa.int64())})
    cases = [
        ("dictionary string column", X.raw_map_plan([P.STRING, P.INT64], ["s", "v"], ["v"], 1), [dict_tbl], 1, "string"),
        ("num_partitions != world", X.raw_map_plan([P.INT64], ["v"], ["v"], 2), [dict_tbl.select(["v"])], 4, "partitions"),
        ("not a ShuffleWriter", P.scan([P.INT64]), [dict_tbl.select(["v"])], 4, "ShuffleWriter"),
    ]
    for what, plan, inputs, code, text in cases:
        with cb.native.Plan(plan, inputs) as p:
            assert p.execute() is not None, what
            got, msg = exchange_error(cb, comm, p.handle)
            assert got == code and text in msg, (what, got, msg)
            with pytest.raises(cb.native.CometB200Error):
                comm.exchange(p)
    with cb.native.Plan(X.raw_map_plan([P.INT64], ["v"], ["v"], 1), [dict_tbl.select(["v"])]) as p:
        got, msg = exchange_error(cb, comm, p.handle)                 # never executed
        assert got == 4 and "not been executed" in msg, msg
    with cb.native.Plan(X.raw_map_plan([P.INT64], ["v"], ["v"], 1), [dict_tbl.select(["v"])], device=comm.device + 1) as p:
        got, msg = exchange_error(cb, comm, p.handle)                 # created for another device (never started: no GPU touched)
        assert got == 4 and "device" in msg, msg
        assert exchange_error(cb, None, p.handle)[0] == 4             # null communicator
    assert exchange_error(cb, comm, None)[0] == 4                     # null plan
    # the communicator is still good
    tbl, types = X.raw_table(100, 3)
    _, recv, st = exchange_map(cb, comm, X.raw_map_plan(types, X.RAW, ["i16"], 1), [tbl])
    partref.assert_tables_equal(read_back(cb, recv, types), tbl)
    recv.release()


# ---- allgather_small ---------------------------------------------------------------------------------------------------------------------
def allgather_raw(comm, payload, n_bytes, slot):
    from comet_b200 import native
    l = native.lib()
    l.cb200_comm_allgather_small.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.c_int64, C.c_char_p, C.POINTER(C.c_int64), C.POINTER(native._Error)]
    out = C.create_string_buffer(max(slot, 16) * comm.world)
    sizes = (C.c_int64 * comm.world)()
    err = native._Error()
    rc = l.cb200_comm_allgather_small(comm.handle, payload, n_bytes, slot, out, sizes, C.byref(err))
    return rc, err.code, out.raw, list(sizes)


def test_allgather_small(cb, comm):
    pattern = lambda k, seed=0: bytes((i * 31 + seed) % 256 for i in range(k))
    for slot in (16, 4096, 32, 1 << 16, 16):      # a larger slot after a smaller one reallocates; smaller ones reuse it
        for k in sorted({0, 1, slot - 8}):
            assert comm.allgather_small(pattern(k, slot), slot_bytes=slot) == [pattern(k, slot)], (slot, k)
    for slot, k in ((24, 0), (8, 0), (0, 0), (16, 9), (4096, 4089), (-16, 0)):
        rc, code, _, _ = allgather_raw(comm, b"\0" * max(k, 1), k, slot)
        assert rc != 0 and code == 4, (slot, k)
    rc, code, _, _ = allgather_raw(comm, b"", -1, 16)
    assert rc != 0 and code == 4
    assert comm.allgather_small(b"abc", slot_bytes=16) == [b"abc"]


# ---- several GPUs: one spawned process per rank ------------------------------------------------------------------------------------
DEADLINE_S = 180


def _rank_input_raw(rank, variant):
    n = 0 if variant == "empty" and rank == 1 else 1500 + 37 * rank
    nulls = "some"
    if variant == "mixed":
        nulls = "some" if rank % 2 == 0 else "none"
    elif variant == "mixed-swapped":
        nulls = "none" if rank % 2 == 0 else "some"
    return X.raw_table(n, 4000 + 10 * rank + len(variant), nulls)


def multi_raw(cb, o, comm, rank, world, variant):
    tbl, types = _rank_input_raw(rank, variant)
    inputs = [tbl.to_batches(max_chunksize=500)] if tbl.num_rows else [tbl]
    _, recv, st = exchange_map(cb, comm, X.raw_map_plan(types, X.RAW, X.RAW_KEYS, world), inputs)
    parts = [X.expected_partitions(o, _rank_input_raw(s, variant)[0], X.RAW_KEYS, world) for s in range(world)]
    counts = [parts[s][p].num_rows for s in range(world) for p in range(world)]        # the N x N matrix, row-major
    total, _, _ = cb.native.exchange_layout(counts, world, rank)
    want = pa.concat_tables([parts[s][rank] for s in range(world)])
    try:
        assert recv.n_rows == total == want.num_rows
        check_stats(st, tbl.num_rows, total, types)
        got = read_back(cb, recv, types, comm.device)
        if total:
            partref.assert_tables_equal(got, want)
        else:
            assert got is None
    finally:
        recv.release()


def _rank_case(rank, variant):
    key = "bool-dense" if variant.startswith("bool") else "i32" if variant.startswith("mixed") else "i64"
    nulls = "some"
    if variant in ("mixed", "bool-mixed"):
        nulls = "some" if rank == 0 else "none"
    elif variant in ("mixed-swapped", "bool-mixed-swapped"):
        nulls = "none" if rank == 0 else "some"
    n = 0 if variant == "empty" and rank == 1 else 1200 + 50 * rank
    return X.e2e_case(key, seed=7000 + 13 * rank + len(variant), n=n, nulls=nulls,
                      aggset="f64" if variant in ("every", "bool-mixed-swapped", "filtered") else "dec")   # one plan on every rank


def multi_e2e(cb, o, comm, rank, world, variant):
    filtered = variant == "filtered" and rank == 1
    case = _rank_case(rank, variant)
    rows, states, st, res = run_e2e(cb, comm, case, world, filtered)
    assert st["rows_sent"] == (rows or 0)
    check_stats(st, rows or 0, st["rows_received"], case.state_types())
    tables = [_rank_case(s, variant).table() for s in range(world) if not (variant == "filtered" and s == 1)]
    table = pa.concat_tables(tables)
    nk = len(case.key_cols)
    if res is not None:   # every key this rank holds is its own
        keys = pa.table([res.column(i) for i in range(nk)], names=[f"k{i}" for i in range(nk)])
        assert (X.owner(o, keys, world) == rank).all()

    def mine(key):
        kt = pa.table([R.arrow_column([v], t) for v, t in zip(key, case.key_types)], names=[f"k{i}" for i in range(nk)])
        return X.owner(o, kt, world)[0] == rank
    check_e2e(case, table, states, res, f"rank {rank} {variant}", keep=mine)


def multi_q1(cb, o, comm, rank, world, variant):
    """Q1 through cb200_comm_allgather_small as bench.py runs it, then payloads of different lengths per rank.  Both collectives come
    before any check, so a failed check leaves no peer waiting in the middle of the case."""
    from comet_b200 import tpch
    from comet_b200.dist import table_from_bytes, table_to_bytes

    def lineitem(r):
        cols = tpch.gen_lineitem(3000, seed=42 + r)
        t = tpch.lineitem_table(cols, "dec", dictionary=True)
        return t.slice(0, 0) if variant == "empty" and r == world - 1 else t

    def partial(t):
        with cb.native.Plan(tpch.q1_partial_plan("dec"), [t.to_batches(max_chunksize=1024)] if t.num_rows else [t], device=comm.device) as p:
            return p.collect()

    state = partial(lineitem(rank))
    blobs = comm.allgather_small(table_to_bytes(state) if state is not None else b"")
    lens = [0, 1, 1000, (1 << 16) - 8]      # 0 included, and a payload that fills its 64 KiB slot
    pay = lambda r: bytes((i * 7 + r) % 256 for i in range(lens[r % 4]))
    got_pay = comm.allgather_small(pay(rank), slot_bytes=1 << 16)
    assert got_pay == [pay(r) for r in range(world)]
    assert len(blobs) == world and (blobs[rank] == b"") == (state is None)
    if rank == 0:
        states = [table_from_bytes(b) for b in blobs if b]
        with cb.native.Plan(tpch.q1_final_plan("dec"), [pa.concat_tables(states)], device=comm.device) as p:
            got = p.collect()
        whole = pa.concat_tables([lineitem(r) for r in range(world)])
        with cb.native.Plan(tpch.q1_final_plan("dec"), [partial(whole)], device=comm.device) as p:
            want = p.collect()
        key = lambda r: (r["col_0"], r["col_1"])
        assert sorted(got.to_pylist(), key=key) == sorted(want.to_pylist(), key=key)


MULTI = [("raw/nulls-on-every-rank", multi_raw, "every"), ("raw/mixed", multi_raw, "mixed"), ("raw/mixed-swapped", multi_raw, "mixed-swapped"),
         ("raw/empty-rank", multi_raw, "empty"),
         ("e2e/nulls-on-every-rank", multi_e2e, "every"), ("e2e/mixed", multi_e2e, "mixed"), ("e2e/mixed-swapped", multi_e2e, "mixed-swapped"),
         ("e2e/bool-mixed", multi_e2e, "bool-mixed"), ("e2e/bool-mixed-swapped", multi_e2e, "bool-mixed-swapped"),
         ("e2e/empty-rank", multi_e2e, "empty"), ("e2e/filtered-rank", multi_e2e, "filtered"),
         ("q1/allgather", multi_q1, "every"), ("q1/allgather-empty-rank", multi_q1, "empty")]


def _worker(rank, world, parent_pid, ids, results):
    """One rank on GPU `rank`: every plan and the communicator on that device.  It dies with its parent (PR_SET_PDEATHSIG; pytest's
    timeout ends pytest with os._exit, which skips cleanup) and exits at once if the parent is already gone.  The cases run in order;
    at the first failure the rank reports it and the cases it did not run, and exits without another collective or a communicator
    teardown: its peers' later collectives would no longer match its own, and the parent kills them."""
    C.CDLL(None).prctl(1, signal.SIGKILL)   # PR_SET_PDEATHSIG
    if os.getppid() != parent_pid:          # the parent ended before the prctl took effect
        os._exit(1)

    def stop(name, done):
        results.put((rank, name, False, traceback.format_exc()[-2000:]))
        for later, _, _ in MULTI[done:]:
            results.put((rank, later, None, "not run"))
        results.close()
        results.join_thread()                # flushed before the exit
        os._exit(1)
    try:
        import comet_b200 as cb
        from oracle import oracle as o

        def bcast(b):
            if rank == 0:
                for _ in range(world - 1):
                    ids.put(b)
                return b
            return ids.get(timeout=60)
        comm = cb.native.Comm(rank, world, rank, bcast)
    except Exception:
        stop("setup", 0)
    for i, (name, fn, variant) in enumerate(MULTI):
        try:
            fn(cb, o, comm, rank, world, variant)
        except Exception:
            stop(name, i + 1)
        results.put((rank, name, True, ""))
    comm.destroy()


@pytest.mark.parametrize("world", [2, 4])
def test_multi_rank(oracle, world):
    import multiprocessing as mp

    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"{world} ranks need {world} visible GPUs ({torch.cuda.device_count()} visible)")
    ctx = mp.get_context("spawn")
    ids, results = ctx.Queue(), ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, os.getpid(), ids, results), daemon=True) for r in range(world)]
    for p in procs:
        p.start()
    deadline = time.monotonic() + DEADLINE_S
    msgs = []
    try:   # until every report is in, a rank reports a failure (its peers may be waiting on it: stop them now), or the deadline
        while len(msgs) < world * len(MULTI) and time.monotonic() < deadline and all(m[2] is not False for m in msgs):
            try:
                msgs.append(results.get(timeout=1))
            except queue.Empty:
                if not any(p.is_alive() for p in procs):
                    break
        if all(m[2] is not False for m in msgs):
            for p in procs:
                p.join(max(0.0, deadline - time.monotonic()))
    finally:
        survivors = [p for p in procs if p.is_alive()]
        for p in survivors:
            p.kill()
            p.join(10)
    failed = [f"rank {r} {name}:\n{msg}" for r, name, ok, msg in msgs if not ok]
    assert not failed, "\n".join(failed)
    assert not survivors, f"{len(survivors)} rank(s) still running after {DEADLINE_S} s (killed); finished: {sorted({m[1] for m in msgs})}"
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    assert len(msgs) == world * len(MULTI)
