"""NativeScan over a date-sorted lineitem with and without a Parquet page index.

Writes the lineitem the way bench.py's e2e leg does -- in-memory file images in pinned host memory, INT64 decimals, dictionary flags,
PLAIN numerics -- sorted by l_shipdate, with 10^6-byte pages (a power-of-two page size would end the 4- and 8-byte columns' pages on
the same rows, which parquet-mr's row-count checks do not), in 1 Mi-row and 4 Mi-row row groups, with and without a page index; plus an unsorted copy with
a page index, where nothing can be pruned.  Per layout and query it reports H2D bytes and ms per step, the scan's pruning counters, and
(in a torch.profiler run) the time of k_pq_select with its algorithmic bandwidth: covered rows x width read + selected rows x width
written, from the page index (tests/page_index_ref.py).  Queries:
  day    SUM(l_extendedprice) WHERE l_shipdate = one day
  week   SUM(l_extendedprice) WHERE l_shipdate in one week
  q6     TPC-H Q6 partial aggregate
  q1     TPC-H Q1 partial aggregate (keeps ~98 % of the rows: the select kernel's cost when little is pruned)
Prints one JSON line.  Every query's output must be identical with and without the page index."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "datafusion-comet_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np

DAY = 9298  # 1995-06-17
HBM_TBPS = 3.35


def images(args, rg, index, sort):
    import pyarrow as pa
    import pyarrow.parquet as pq
    from comet_b200 import tpch
    cols = tpch.gen_lineitem(args.rows, seed=args.seed)
    if sort:
        order = np.argsort(cols["l_shipdate"], kind="stable")
        cols = {k: v[order] for k, v in cols.items()}
    tbl = tpch.lineitem_table(cols, "dec", dictionary=True)
    per = (args.rows + args.files - 1) // args.files
    out = []
    for i in range(args.files):
        sink = pa.BufferOutputStream()
        pq.write_table(tbl.slice(i * per, per), sink, row_group_size=rg, compression="NONE", data_page_version="1.0", use_dictionary=["l_returnflag", "l_linestatus"],
                       store_decimal_as_integer=True, write_page_index=index, data_page_size=1_000_000)
        out.append(sink.getvalue().to_pybytes())
    return out


def plans(q, files):
    from comet_b200 import proto as P, tpch
    if q == "q1":
        return tpch.q1_partial_plan("dec", scan=tpch.q1_native_scan("dec", files))
    if q == "q6":
        return tpch.q6_partial_plan("dec", scan=tpch.q6_native_scan("dec", files))
    hi = DAY + (1 if q == "day" else 7)
    fields = list(zip(tpch.Q1_COLUMNS, tpch.q1_scan_fields("dec"), [True] * 7))
    ship = P.bound(6, P.DATE)
    pred = P.and_(P.gt_eq(ship, P.literal(DAY, P.DATE)), P.lt(ship, P.literal(hi, P.DATE)))
    sc = P.native_scan(fields, fields, files, data_filters=[pred])
    return P.hash_agg(P.filter_(sc, pred), [], [P.agg_sum(P.bound(1, tpch.D12), P.DECIMAL(22, 2))], P.PARTIAL)


def terms(q):
    """the conjuncts each query pushes to the scan, as (column of the Q1 projection, op, literal, physical type)"""
    if q == "q1":
        return [(6, "le", 10493, "INT32")]
    if q == "q6":
        return [(6, "ge", 8766, "INT32"), (6, "lt", 9131, "INT32"), (2, "ge", 5, "INT64"), (2, "le", 7, "INT64"), (0, "lt", 2400, "INT64")]
    return [(6, "ge", DAY, "INT32"), (6, "lt", DAY + (1 if q == "day" else 7), "INT32")]


def select_bytes(imgs, q):
    """algorithmic bytes of k_pq_select over the columns the query reads: covered rows x width in, selected rows x width out"""
    import page_index_ref as ref
    width = [8, 8, 8, 8, 4, 4, 4]                                     # Q1 projection: decimals as INT64, flag codes, date
    read = [0, 1, 2, 6] if q == "q6" else list(range(7)) if q == "q1" else [1, 6]
    t = terms(q)
    total = 0
    for raw in imgs:
        for chunks, g in zip(ref.footer_chunks(raw), ref.page_indexes(raw)):
            if any(oi is None or ci is None for oi, ci in g):
                continue
            n = chunks[0]["num_rows"]
            ranges = ref.selection(t, g, n)
            sel = sum(b - a for a, b in ranges)
            if sel in (0, n):
                continue
            for c in read:
                _, cov, _ = ref.column_window(g[c][0], n, ranges)
                if cov != sel:
                    total += (cov + sel) * width[c]
    return total


def step(native, q, files, chunk_rows):
    with native.Plan(plans(q, files), [], config={"spark.comet.b200.chunkRows": str(chunk_rows)}) as p:
        out = p.collect()
        st = p.stats()
    return out, st


def canonical(res):
    rows = sorted(res.to_pylist(), key=lambda r: json.dumps(r, default=repr))
    return json.dumps(rows, default=repr)


def select_ms(torch, native, q, files, chunk_rows):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(native, q, files, chunk_rows)
        torch.cuda.synchronize()
    ms = 0.0
    for e in prof.key_averages():
        if "k_pq_select" in e.key:
            ms += (getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)) / 1e3
    return ms


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 25)
    ap.add_argument("--files", type=int, default=16)
    ap.add_argument("--seed", type=int, default=42)
    ap.add_argument("--chunk-rows", type=int, default=1 << 23)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--queries", default="day,week,q6,q1")
    args = ap.parse_args()
    import torch
    from comet_b200 import native
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "rows": args.rows, "files": args.files, "chunk_rows": args.chunk_rows,
           "layouts": {}}
    layouts = [("sorted_1Mi_index", 1 << 20, True, True), ("sorted_1Mi_noindex", 1 << 20, False, True),
               ("sorted_4Mi_index", 1 << 22, True, True), ("sorted_4Mi_noindex", 1 << 22, False, True), ("unsorted_1Mi_index", 1 << 20, True, False)]
    outputs = {}
    for name, rg, index, sort in layouts:
        imgs = images(args, rg, index, sort)
        pinned, files = [], []
        for i, b in enumerate(imgs):
            h = torch.empty(len(b), dtype=torch.uint8, pin_memory=True)
            h.numpy()[:] = np.frombuffer(b, dtype=np.uint8)
            pinned.append(h)
            files.append(native.register_memory_file(f"pi-{name}-{i}", h))
        lay = {"file_bytes": sum(len(b) for b in imgs), "queries": {}}
        for q in args.queries.split(","):
            for _ in range(args.warmup):
                step(native, q, files, args.chunk_rows)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            h2d = 0
            for _ in range(args.steps):
                out, st = step(native, q, files, args.chunk_rows)
                h2d += st["h2d_bytes"]
            el = time.perf_counter() - t0
            outputs[(name, q)] = canonical(out)
            r = {"h2d_bytes_per_step": h2d // args.steps, "ms_per_step": 1e3 * el / args.steps, "pruned_row_groups": st["scan_pruned_row_groups"],
                 "pruned_pages": st["scan_pruned_pages"], "page_pruned_rows": st["scan_page_pruned_rows"]}
            if index:
                ms = select_ms(torch, native, q, files, args.chunk_rows)
                nbytes = select_bytes(imgs, q)
                tbps = nbytes / (ms * 1e-3) / 1e12 if ms > 0 else None
                r["k_pq_select"] = {"ms_per_step": ms, "bytes": nbytes, "TBps": tbps, "of_hbm_peak": tbps / HBM_TBPS if tbps else None}
            lay["queries"][q] = r
        for f in files:
            native.register_memory_file(f[len("memory://"):], None)
        del pinned, imgs
        res["layouts"][name] = lay
    res["outputs_identical"] = all(outputs[(f"sorted_{s}_index", q)] == outputs[(f"sorted_{s}_noindex", q)] for s in ("1Mi", "4Mi") for q in args.queries.split(","))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
