"""Join conditions on the GPU: the TPC-H Q21-shaped lineitem self-joins over an HBM-resident synthetic lineitem.

    SELECT COUNT(*), SUM(l1.l_suppkey) FROM lineitem l1
    WHERE [NOT] EXISTS (SELECT * FROM lineitem l2 WHERE l2.l_orderkey = l1.l_orderkey AND l2.l_suppkey <> l1.l_suppkey)

as Comet plans it over inputs sorted by l_orderkey: a SortMergeJoin (LeftSemi for EXISTS, LeftAnti for NOT EXISTS) of lineitem with
itself on l_orderkey with the condition l_suppkey <> l_suppkey, under a HashAggregate(Partial).  lineitem is one device table generated
from a seed (numpy): --rows rows of orders with 1 to 7 lines, sorted by l_orderkey, l_suppkey drawn from three suppliers per order, so
that about a fifth of the orders have one supplier only.  Every timed result is checked against the numpy answer: a row passes EXISTS
exactly when its order has two suppliers or more.

Reports, per size and join type: the step time (host clock around the plan, which ends by copying its one-row result to the host;
median over --steps after --warmup), the kernel time per stage from torch.profiler in a separate step, the join counters, and GB/s per
stage by the byte model in `model()`.  The gathers of the condition's columns and of the output rows share kernels: "gathers" holds both.
Prints one JSON line per size and join type, with the card's name and power limit.
    python bench_join_condition.py [--rows 100000000,600000000] [--steps 5] [--warmup 1]
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

LEFT_SEMI, LEFT_ANTI = 4, 5


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def lineitem(np, n, seed):
    """(l_orderkey, l_suppkey) as int64 arrays, sorted by l_orderkey, and the answers {semi: (count, sum), anti: (count, sum)}"""
    rng = np.random.default_rng(seed)
    sizes = rng.integers(1, 8, n // 3 + 16)
    sizes = sizes[:np.searchsorted(np.cumsum(sizes), n) + 1]
    okey = np.repeat(np.arange(len(sizes), dtype=np.int64), sizes)[:n]
    supp = (okey * 7919 + rng.integers(0, 3, n)) % 100_000
    starts = np.flatnonzero(np.r_[True, okey[1:] != okey[:-1]])
    multi = np.minimum.reduceat(supp, starts) != np.maximum.reduceat(supp, starts)
    row_multi = np.repeat(multi, np.diff(np.r_[starts, n]))
    answers = {LEFT_SEMI: (int(row_multi.sum()), int(supp[row_multi].sum())), LEFT_ANTI: (int((~row_multi).sum()), int(supp[~row_multi].sum()))}
    return okey, supp, answers


def device_table(native, P, torch, np, okey, supp):
    t = native.DeviceTable(len(okey))
    keep = []
    for arr in (okey, supp):
        v = torch.from_numpy(np.concatenate([arr, np.zeros(2, np.int64)])).cuda()
        keep.append(v)
        t.add(P.INT64, v.data_ptr(), 8, None, 0, keep=v)
    return t, keep


# ---- stages and the byte model ---------------------------------------------------------------------------------------------------------
STAGES = {"key_packing": ("k_sort_keys",), "join_build": ("k_sort_hist", "k_sort_scatter", "k_sort_iota", "k_join_heads", "k_join_insert"),
          "join_lookups": ("k_join_probe",), "count_scans": ("k_scan_chunks", "k_scan_totals"), "candidate_emit": ("k_join_emit",),
          "gathers": ("k_gather_rows", "k_gather_bits", "k_bytes_to_bitmap"), "condition_kernel": ("cb_select_count",),
          "resolution": ("k_join_cond_mark", "k_flags_not", "k_block_counts", "k_scan_counts", "k_compact_scatter"),
          "aggregate": ("cb_pipeline_agg", "cb_finalize")}


def stage_of(name):
    for st, pats in STAGES.items():
        if any(p in name for p in pats):
            return st
    return "other"


def model(stats, n):
    """algorithmic bytes: an emitted candidate reads its probe row's run and offsets (12 B) and writes two indices (8 B); the condition's
    gathers read two indices and two 8-byte values and write the values (32 B per candidate), the output gathers read an index and two
    8-byte columns and write them (36 B per output row); the condition kernel reads two 8-byte columns and writes a bit (16 B per
    candidate); resolution reads a bit, two indices and writes a passed byte (9 B per candidate), then compacts the probe rows (1 B read,
    4 B written each); a lookup reads its key (8 B), one slot, the run bounds and its first key (24 B) and writes a count and a run (8 B)"""
    c, out = stats["join_cond_pairs"], stats["join_out_rows"]
    return {"candidate_emit": c * 20, "gathers": c * 32 + out * 36, "condition_kernel": c * 16, "resolution": c * 9 + n * 5,
            "join_lookups": stats["join_probe_rows"] * 40}


def profile(torch, fn):
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    stages = {}
    for e in p.events():
        if e.device_time_total > 0:
            st = stage_of(e.name)
            stages[st] = stages.get(st, 0.0) + e.device_time_total / 1e3
    return stages


def plan(P, join_type):
    t = [P.INT64, P.INT64]
    cond = P.neq(P.bound(1, P.INT64), P.bound(3, P.INT64))          # l1.l_suppkey <> l2.l_suppkey over (l1 ++ l2)
    j = P.sort_merge_join(P.scan(t), P.scan(t), [P.bound(0, P.INT64)], [P.bound(0, P.INT64)], join_type, [P.sort_order(P.bound(0, P.INT64))],
                          condition=cond)
    return P.hash_agg(j, [], [P.agg_count([P.bound(0, P.INT64)]), P.agg_sum(P.bound(1, P.INT64), P.INT64)], P.PARTIAL)


def step(native, p, table):
    with native.Plan(p, [table, table]) as pl:
        return pl.collect(), pl.stats()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="100000000,600000000")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=21)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_join_condition.py measures the GPU: no CUDA device")
    import comet_b200  # noqa: F401
    from comet_b200 import native, proto as P
    for n in (int(x) for x in args.rows.split(",")):
        t0 = time.perf_counter()
        okey, supp, answers = lineitem(np, n, args.seed)
        table, keep = device_table(native, P, torch, np, okey, supp)
        del okey, supp
        gen_s = time.perf_counter() - t0
        for jt, name in ((LEFT_SEMI, "left_semi"), (LEFT_ANTI, "left_anti")):
            p = plan(P, jt)
            walls = []
            for _ in range(args.warmup + args.steps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res, stats = step(native, p, table)
                walls.append((time.perf_counter() - t0) * 1e3)
                row = list(res.to_pylist()[0].values())
                assert (row[0], row[1]) == answers[jt], (row, answers[jt])
            walls = sorted(walls[args.warmup:])
            stages = profile(torch, lambda: step(native, p, table))
            bytes_ = model(stats, n)
            print(json.dumps(dict(bench="q21_join_condition", join_type=name, rows=n,
                                  step_ms_median=round(walls[len(walls) // 2], 2), step_ms_min=round(walls[0], 2), step_ms_max=round(walls[-1], 2),
                                  checked_steps=args.warmup + args.steps, check="numpy answer: count and sum of l_suppkey",
                                  join_cond_pairs=stats["join_cond_pairs"], join_probe_rows=stats["join_probe_rows"],
                                  join_out_rows=stats["join_out_rows"], kernel_launches=stats["kernel_launches"],
                                  stage_ms={k: round(v, 3) for k, v in stages.items()}, model_gb={k: round(v / 1e9, 3) for k, v in bytes_.items()},
                                  stage_gbps={k: round(bytes_[k] / (stages[k] * 1e6), 1) for k in bytes_ if stages.get(k)},
                                  data_gen_s=round(gen_s, 1), card=card())), flush=True)
        del table, keep
        torch.cuda.empty_cache()
        native.lib().cb200_release_cached_memory(0)


if __name__ == "__main__":
    main()
