"""GPU: page-index pruning in NativeScan.  The scan emits exactly the rows of the reference selection (tests/page_index_ref.py), with
their values and validity; query results over page-indexed files are bit-identical to the unpruned scan and to the same data written
without a page index; the pruning counters and the H2D bytes are the planned ones."""
import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from test_gpu_parquet_encodings import _check, _columns, _table
from test_parquet_pageindex_cpu import expected, lineitem, planner, scan  # noqa: F401  (planner: the CPU planner driver fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def run(cb, plan, inputs=(), chunk_rows=None):
    cfg = {"spark.comet.b200.chunkRows": str(chunk_rows)} if chunk_rows else None
    with cb.native.Plan(plan, list(inputs), config=cfg) as p:
        t = p.collect()
        st = p.stats()
    return t, st


def _selected(paths, fields, terms, rg_rows):
    """row numbers of each file's table the reference selection keeps, in scan order"""
    units, pages, rows = expected(paths, fields, terms)
    idx = []
    for f, g, n, ranges, _, _ in units:
        for a, b in ranges or [(0, n)]:
            idx.append((f, np.arange(g * rg_rows + a, g * rg_rows + b)))
    return idx, pages, rows


@pytest.mark.parametrize("version,compression,chunk_rows,memory", [("1.0", "NONE", 45_000, False), ("2.0", "SNAPPY", 7_000, True),
                                                                   ("1.0", "ZSTD", 1 << 22, True), ("2.0", "NONE", 7_000, False)])
def test_scan_emits_the_reference_selection(cb, planner, tmp_path, version, compression, chunk_rows, memory):
    """every physical -> output type pair, required and nullable columns (all-NULL pages too), a date range on a sorted column; chunkRows
    below and above the 20 k-row row groups; file paths and memory:// images.  Pages end every 2000 rows or 4 KB, so page boundaries
    differ between columns."""
    P = cb.proto
    n, rg = 60_000, 20_000
    tbl = _table(cb, n, seed=21)
    cols = _columns(P)
    enc = {k: v[2] for k, v in cols.items()}
    path = str(tmp_path / "p.parquet")
    pq.write_table(tbl, path, row_group_size=rg, compression=compression, use_dictionary=False, column_encoding=enc, data_page_version=version,
                   data_page_size=4096, max_rows_per_page=2_000, write_page_index=True, store_decimal_as_integer=True)
    names = tbl.column_names
    fields = [(k, cols[k][1], True) for k in names]
    date = names.index("date")
    dates = tbl.column("date").drop_null().cast(pa.int32()).to_numpy()
    lo = int(dates[len(dates) // 3])
    terms = [(date, "ge", lo), (date, "lt", lo + 60)]
    sel, pruned_pages, pruned_rows = _selected([path], fields, terms, rg)
    assert pruned_pages > 0 and pruned_rows > rg // 2
    want = tbl.take(np.concatenate([i for _, i in sel]))
    pinned = None
    files = [path]
    if memory:
        import torch
        b = open(path, "rb").read()
        pinned = torch.empty(len(b), dtype=torch.uint8, pin_memory=True)
        pinned.numpy()[:] = np.frombuffer(b, dtype=np.uint8)
        files = [cb.native.register_memory_file(f"pageindex-{version}-{compression}", pinned)]
    try:
        for part in (names[:8], names[8:]):
            idx = [names.index(k) for k in part]
            sub_fields = [fields[i] for i in idx]
            t = [(idx.index(date), op, lit) for _, op, lit in terms] if date in idx else None
            if t is None:                                     # the date column rides along so that the terms apply to every part
                sub_fields = sub_fields + [fields[date]]
                t = [(len(sub_fields) - 1, op, lit) for _, op, lit in terms]
            plan = P.projection(scan(cb, sub_fields, files, t), [P.bound(i, f[1]) for i, f in enumerate(sub_fields)])
            res, st = run(cb, plan, chunk_rows=chunk_rows)
            assert res.num_rows == want.num_rows
            _check(res.select(list(range(len(part)))), want.select(part))
            assert st["scan_pruned_pages"] == _selected([path], sub_fields, t, rg)[1]
            assert st["scan_page_pruned_rows"] == pruned_rows
            planned = planner(scan(cb, sub_fields, [path], t), chunk_rows)
            assert st["h2d_bytes"] == sum(b["upload_bytes"] for b in planned["batches"])
    finally:
        if memory:
            cb.native.register_memory_file(files[0][len("memory://"):], None)


def _q_files(cb, tmp_path, variant, n=400_000, rg=100_000):
    """the same date-sorted lineitem with and without a page index"""
    cols, a = lineitem(cb, n, str(tmp_path / f"pi_{variant}.parquet"), seed=41, variant=variant, rg=rg)
    _, b = lineitem(cb, n, str(tmp_path / f"nopi_{variant}.parquet"), seed=41, variant=variant, rg=rg, index=False)
    return cols, a, b


@pytest.mark.parametrize("variant", ["dec", "f64"])
def test_q6_over_page_indexed_files(cb, planner, tmp_path, variant, monkeypatch):
    t = cb.tpch
    P = cb.proto
    cols, a, b = _q_files(cb, tmp_path, variant)
    plan = lambda f: t.q6_partial_plan(variant, scan=t.q6_native_scan(variant, [f]))
    state, st = run(cb, plan(a), chunk_rows=60_000)
    m = t._money(variant)
    fields = list(zip(t.Q6_COLUMNS, [m, m, m, P.DATE], [True] * 4))
    lit = (lambda c: c) if variant == "dec" else (lambda c: c / 100.0)
    terms = [(3, "ge", t.DATE_1994_01_01), (3, "lt", t.DATE_1995_01_01), (2, "ge", lit(5)), (2, "le", lit(7)), (0, "lt", lit(2400))]
    _, pages, rows = expected([a], fields, terms)
    assert st["scan_pruned_pages"] == pages > 0 and st["scan_page_pruned_rows"] == rows
    planned = planner(scan(cb, fields, [a], terms), 60_000)
    assert st["h2d_bytes"] == sum(x["upload_bytes"] for x in planned["batches"])
    state_nopi, st_nopi = run(cb, plan(b), chunk_rows=60_000)
    assert st_nopi["scan_pruned_pages"] == 0 and state.equals(state_nopi)
    monkeypatch.setenv("CB200_NO_PRUNE", "1")
    state_all, st_all = run(cb, plan(a), chunk_rows=60_000)
    assert st_all["scan_pruned_pages"] == 0 and st_all["scan_pruned_row_groups"] == 0 and state.equals(state_all)
    assert st["h2d_bytes"] < st_nopi["h2d_bytes"] < st_all["h2d_bytes"]


def test_q1_over_page_indexed_files(cb, tmp_path, monkeypatch):
    t = cb.tpch
    cols, a, b = _q_files(cb, tmp_path, "dec")
    plan = lambda f: t.q1_partial_plan("dec", scan=t.q1_native_scan("dec", [f]))
    key = lambda tb: sorted(tb.to_pylist(), key=lambda r: (r["col_0"], r["col_1"]))
    state, st = run(cb, plan(a), chunk_rows=150_000)
    assert st["scan_pruned_pages"] > 0 and st["scan_page_pruned_rows"] > 0
    state_nopi, _ = run(cb, plan(b), chunk_rows=150_000)
    monkeypatch.setenv("CB200_NO_PRUNE", "1")
    state_all, st_all = run(cb, plan(a), chunk_rows=150_000)
    assert st_all["scan_pruned_pages"] == 0
    assert key(state) == key(state_nopi) == key(state_all)


def _filter_project(cb, files, cutoff):
    """Config-1 shape over NativeScan: Filter(l_shipdate < cutoff) -> Projection(l_quantity * l_extendedprice, l_shipdate)"""
    t = cb.tpch
    P = cb.proto
    sc = t.q1_native_scan("dec", files)
    ship = P.bound(6, P.DATE)
    flt = P.filter_(sc, P.lt(ship, P.literal(cutoff, P.DATE)))
    return P.projection(flt, [P.bound(0, t.D12), P.bound(1, t.D12), ship])


def test_filter_projection_rows_in_order(cb, tmp_path, monkeypatch):
    t = cb.tpch
    _, a, _ = _q_files(cb, tmp_path, "dec", n=300_000)
    plan = _filter_project(cb, [a], t.DATE_1994_01_01)
    res, st = run(cb, plan, chunk_rows=70_000)
    assert st["scan_pruned_pages"] > 0
    monkeypatch.setenv("CB200_NO_PRUNE", "1")
    res_all, _ = run(cb, plan, chunk_rows=70_000)
    assert res.num_rows > 0 and res.equals(res_all)


def test_one_week_inside_one_large_row_group(cb, tmp_path, monkeypatch):
    """a one-week l_shipdate range in a single 1 Mi-row row group: well under a tenth of the row group crosses PCIe"""
    t = cb.tpch
    P = cb.proto
    n = 1 << 20
    cols, path = lineitem(cb, n, str(tmp_path / "big.parquet"), seed=7, rg=n)
    lo = t.DATE_1995_06_17
    sc = scan(cb, list(zip(t.Q1_COLUMNS, t.q1_scan_fields("dec"), [True] * 7)), [path], [(6, "ge", lo), (6, "lt", lo + 7)])
    ship = P.bound(6, P.DATE)
    plan = P.filter_(sc, P.and_(P.gt_eq(ship, P.literal(lo, P.DATE)), P.lt(ship, P.literal(lo + 7, P.DATE))))
    res, st = run(cb, plan)
    monkeypatch.setenv("CB200_NO_PRUNE", "1")
    res_all, st_all = run(cb, plan)
    want = int(((cols["l_shipdate"] >= lo) & (cols["l_shipdate"] < lo + 7)).sum())
    assert res.num_rows == want > 0 and res.equals(res_all)
    assert st["h2d_bytes"] < 0.1 * st_all["h2d_bytes"]
