"""String predicates on dictionary-coded columns: what they cost on the GPU.

1. `q12`: a TPC-H Q12-shaped single-table aggregate over HBM-resident lineitem (device table, default 600 M rows):
       SELECT l_shipinstruct, SUM(l_extendedprice), COUNT(*) FROM lineitem WHERE l_shipmode IN ('MAIL', 'SHIP') GROUP BY l_shipinstruct
   against the same plan with the predicate as an integer IN over the same code column (the column typed int8, codes 5 and 3).  Both
   group by the same dictionary column, so both run the dense strategy and differ only in the predicate.  Reported: pipeline kernel
   time per step (CUDA events around the fused kernels) and wall time, alternating the two plans.
2. `like`: l_comment LIKE '%special%requests%' -> COUNT / SUM over Parquet images in pinned host memory, where l_comment is
   high-cardinality and its pages fall back to PLAIN, so every batch grows the dictionary.  One profiled step (torch.profiler) gives the
   k_str_pred time per batch beside the Parquet decode kernels and the host-to-device copies.

Prints one JSON line per measurement, with the card's name and power limit.
    python bench_string_predicates.py [--rows 600000000] [--steps 10] [--warmup 2] [--comment-rows 16000000]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "datafusion-comet_b200")]
os.environ.setdefault("CB200_CACHE_DIR", tempfile.mkdtemp(prefix="cb200_jit_"))  # the tree may be read-only


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def q12(args, torch, native, tpch, P):
    n = args.rows
    g = torch.Generator(device="cuda")
    g.manual_seed(12)
    mode = torch.randint(0, len(tpch.SHIPMODES), (n,), generator=g, device="cuda", dtype=torch.int8)
    instr = torch.randint(0, len(tpch.SHIPINSTRUCTS), (n,), generator=g, device="cuda", dtype=torch.int8)
    price = torch.randint(90000, 10_500_000, (n,), generator=g, device="cuda", dtype=torch.int64)  # cents, d(12,2) stored as int64
    D12 = P.DECIMAL(12, 2)

    def table(mode_type):
        t = native.DeviceTable(n)
        if mode_type == "str":
            t.add(P.STRING, mode.data_ptr(), 1, dictionary=tpch.SHIPMODES, keep=mode)
        else:
            t.add(P.INT8, mode.data_ptr(), 1, keep=mode)
        t.add(P.STRING, instr.data_ptr(), 1, dictionary=tpch.SHIPINSTRUCTS, keep=instr)
        t.add(D12, price.data_ptr(), 8, keep=price)
        return t

    def plan(mode_type):
        if mode_type == "str":
            pred = P.in_(P.bound(0, P.STRING), [P.literal("MAIL", P.STRING), P.literal("SHIP", P.STRING)])
        else:
            pred = P.in_(P.bound(0, P.INT8), [P.literal(tpch.SHIPMODES.index("MAIL"), P.INT8), P.literal(tpch.SHIPMODES.index("SHIP"), P.INT8)])
        scan = P.scan([P.STRING if mode_type == "str" else P.INT8, P.STRING, D12])
        return P.hash_agg(P.filter_(scan, pred), [P.bound(1, P.STRING)], [P.agg_sum(P.bound(2, D12), P.DECIMAL(22, 2)), P.agg_count([P.bound(2, D12)])])

    def step(mode_type):
        t = table(mode_type)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with native.Plan(plan(mode_type), [t], config={"spark.comet.b200.chunkRows": str(1 << 30)}) as p:
            res = p.collect()
            st = p.stats()
        return (time.perf_counter() - t0) * 1e3, st["pipeline_ms"], st["agg_strategies"], sorted(res.to_pylist(), key=lambda r: r["col_0"])

    for _ in range(args.warmup):
        step("str")
        step("int")
    ms = {"str": [], "int": []}
    outs = {}
    for _ in range(args.steps):
        for m in ("str", "int"):
            wall, kern, strat, out = step(m)
            ms[m].append((wall, kern))
            outs[m] = (out, strat)
    assert outs["str"][0] == outs["int"][0], "string and integer IN disagree"
    for m in ("str", "int"):
        kern = sorted(k for _, k in ms[m])
        wall = sorted(w for w, _ in ms[m])
        print(json.dumps(dict(bench="q12_shipmode_in", predicate=m, rows=n, strategy=outs[m][1], kernel_ms_median=kern[len(kern) // 2],
                              kernel_ms_min=kern[0], kernel_ms_max=kern[-1], wall_ms_median=wall[len(wall) // 2], card=card())))


def like(args, torch, native, tpch, P):
    import pyarrow as pa
    import pyarrow.compute as pc
    import pyarrow.parquet as pq
    import numpy as np
    n, n_files = args.comment_rows, 8
    rng = np.random.default_rng(7)
    vocab = pa.array(["special", "requests", "carefully", "final", "deposits", "sleep", "quickly", "ironic", "packages", "furiously", "bold",
                      "accounts", "pending", "express", "regular", "blithely", "even", "theodolites", "asymptotes", "platelets"] +
                     [f"w{i}" for i in range(400)])
    parts = [pc.take(vocab, pa.array(rng.integers(0, len(vocab), n))) for _ in range(6)]
    comment = pc.binary_join_element_wise(*parts, " ")
    price = pa.array(rng.integers(90000, 10_500_000, n))
    cnt = int(pc.sum(pc.match_like(comment, "%special%requests%").cast(pa.int64())).as_py())
    names = []
    per = n // n_files
    for f in range(n_files):
        t = pa.table({"l_comment": comment.slice(f * per, per), "l_extendedprice": price.slice(f * per, per)})
        sink = pa.BufferOutputStream()
        pq.write_table(t, sink, row_group_size=1 << 20, compression="NONE", use_dictionary=True)
        buf = sink.getvalue()
        host = torch.empty(buf.size, dtype=torch.uint8, pin_memory=True)
        host.numpy()[:] = np.frombuffer(buf, dtype=np.uint8)
        names.append(native.register_memory_file(f"comment{f}", host))
    md = pq.ParquetFile(pa.BufferReader(buf)).metadata
    encodings = sorted(set(md.row_group(0).column(0).encodings))
    fields = [("l_comment", P.STRING, True), ("l_extendedprice", P.INT64, True)]
    pred = P.like(P.bound(0, P.STRING), P.literal("%special%requests%", P.STRING))
    plan = P.hash_agg(P.filter_(P.native_scan(fields, fields, names), pred), [], [P.agg_count([P.bound(1, P.INT64)]), P.agg_sum(P.bound(1, P.INT64), P.INT64)])
    batch_rows = 1 << 21
    cfg = {"spark.comet.b200.chunkRows": str(batch_rows)}

    def step():
        t0 = time.perf_counter()
        with native.Plan(plan, [], config=cfg) as p:
            r = p.collect().to_pylist()[0]
        assert r["col_0"] == cnt, (r, cnt)
        return (time.perf_counter() - t0) * 1e3

    for _ in range(args.warmup):
        step()
    walls = sorted(step() for _ in range(args.steps))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    tot = {"k_str_pred": [0.0, 0], "parquet_kernels": [0.0, 0], "h2d_copies": [0.0, 0], "pipeline": [0.0, 0]}
    for e in prof.events():
        name = e.name
        us = e.device_time_total
        key = "k_str_pred" if "k_str_pred" in name else "parquet_kernels" if "k_pq" in name else \
              "h2d_copies" if ("HtoD" in name or "Memcpy HtoD" in name) else "pipeline" if "cb_pipeline" in name else None
        if key:
            tot[key][0] += us / 1e3
            tot[key][1] += 1
    batches = (n + batch_rows - 1) // batch_rows
    print(json.dumps(dict(bench="comment_like", rows=n, batches=batches, matches=cnt, comment_encodings=encodings, wall_ms_median=walls[len(walls) // 2],
                          per_batch_ms={k: v[0] / batches for k, v in tot.items()}, launches={k: v[1] for k, v in tot.items()}, card=card())))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600_000_000)
    ap.add_argument("--comment-rows", type=int, default=16_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", choices=["q12", "like"], default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_string_predicates.py measures the GPU: no CUDA device")
    import comet_b200  # noqa: F401
    from comet_b200 import native, tpch, proto as P
    if args.only in (None, "q12"):
        q12(args, torch, native, tpch, P)
    if args.only in (None, "like"):
        like(args, torch, native, tpch, P)


if __name__ == "__main__":
    main()
