"""Nested-loop joins on the GPU: band and NOT IN joins of HBM-resident event rows against a broadcast side of ranges.

    inner band:  SELECT COUNT(*), SUM(e.t) FROM events e JOIN ranges r ON e.t >= r.lo AND e.t < r.hi
    semi band:   SELECT COUNT(*), SUM(e.t) FROM events e WHERE EXISTS (SELECT * FROM ranges r WHERE e.t >= r.lo AND e.t < r.hi)
    not in:      SELECT COUNT(*), SUM(e.t) FROM events e WHERE (e.a, e.b) NOT IN (SELECT x, y FROM ranges)

as Comet plans them: a BroadcastNestedLoopJoin (Inner, LeftSemi, LeftAnti; BuildRight) under a HashAggregate(Partial).  NOT IN over two
columns becomes a LeftAnti join with the condition (a = x OR isnull(a = x)) AND (b = y OR isnull(b = y)).  Both sides are device
tables generated from a seed (numpy): events (t int64 in [0, 1e9), a, b int32 in [0, 1000)) and ranges (lo, hi int64 with hi - lo
below 2e8 / ranges, x, y int32 in [0, 1000) with 2% NULLs).  Every timed result is checked against numpy: the band joins by searchsorted over
the sorted bounds, NOT IN by a match table over the (a, b) domain.

Reports, per size and join: the step time (host clock around the plan, which ends by copying its one-row result to the host; median
over --steps after --warmup), the kernel time per stage from torch.profiler in a separate step, the pairs evaluated per second of step
time, and bytes per pair by the byte model in `model()`.  Prints one JSON line per size and join, with the card's name and power limit.
    python bench_nested_loop_join.py [--sizes 100000000:1024,10000000:16384] [--steps 3] [--warmup 1]
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

INNER, LEFT_SEMI, LEFT_ANTI = 0, 4, 5
DOM = 1000   # a, b, x, y in [0, DOM)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def generate(np, n, m, seed):
    rng = np.random.default_rng(seed)
    ev = {"t": rng.integers(0, 10**9, n, dtype=np.int64), "a": rng.integers(0, DOM, n).astype(np.int32), "b": rng.integers(0, DOM, n).astype(np.int32)}
    lo = rng.integers(0, 10**9, m, dtype=np.int64)
    rg = {"lo": lo, "hi": lo + rng.integers(1, max(2, 2 * 10**8 // m), m), "x": rng.integers(0, DOM, m).astype(np.int32),
          "y": rng.integers(0, DOM, m).astype(np.int32), "xv": rng.random(m) >= 0.02, "yv": rng.random(m) >= 0.02}
    return ev, rg


def answers(np, ev, rg):
    """{join: (count, sum of t)} by numpy, without enumerating pairs"""
    t = ev["t"]
    cnt = np.searchsorted(np.sort(rg["lo"]), t, side="right") - np.searchsorted(np.sort(rg["hi"]), t, side="right")   # lo < hi
    hit = cnt > 0
    # NOT IN: build row (x, y) rules out probe (a, b) when each column is equal or either side is NULL (the probe has no NULLs here)
    x, y, xv, yv = rg["x"], rg["y"], rg["xv"], rg["yv"]
    match = np.zeros((DOM, DOM), bool)
    match[x[xv & yv], y[xv & yv]] = True
    match[:, y[~xv & yv]] = True
    match[x[xv & ~yv], :] = True
    match[:, :] |= bool((~xv & ~yv).any())
    keep = ~match[ev["a"], ev["b"]]
    total = lambda sel, w: (int(w.sum()), int((t * w).sum()) if sel.any() else None)   # SUM of no rows is NULL
    return {"inner_band": total(hit, cnt), "semi_band": total(hit, hit.astype(np.int64)), "not_in": total(keep, keep.astype(np.int64))}


def device_tables(native, P, torch, np, ev, rg):
    keep = []
    def col(tbl, dt, arr, width, valid=None):
        v = torch.from_numpy(np.concatenate([arr, np.zeros(2, arr.dtype)])).cuda()
        vb = torch.from_numpy(np.concatenate([valid, np.zeros(2, bool)]).astype(np.uint8)).cuda() if valid is not None else None
        keep.extend([v, vb])
        if valid is None:
            tbl.add(dt, v.data_ptr(), width, None, 0, keep=v)
        else:
            tbl.add_bytes(dt, v.data_ptr(), width, vb.data_ptr(), keep=(v, vb))
    e = native.DeviceTable(len(ev["t"]))
    col(e, P.INT64, ev["t"], 8); col(e, P.INT32, ev["a"], 4); col(e, P.INT32, ev["b"], 4)
    r = native.DeviceTable(len(rg["lo"]))
    col(r, P.INT64, rg["lo"], 8); col(r, P.INT64, rg["hi"], 8); col(r, P.INT32, rg["x"], 4, rg["xv"]); col(r, P.INT32, rg["y"], 4, rg["yv"])
    return e, r, keep


def plan(P, join):
    """events (t, a, b) ++ ranges (lo, hi, x, y): columns 0-2, 3-6"""
    band = P.and_(P.gt_eq(P.bound(0, P.INT64), P.bound(3, P.INT64)), P.lt(P.bound(0, P.INT64), P.bound(4, P.INT64)))
    eq_or_null = lambda l, r: P.or_(P.eq(l, r), P.is_null(P.eq(l, r)))
    not_in = P.and_(eq_or_null(P.bound(1, P.INT32), P.bound(5, P.INT32)), eq_or_null(P.bound(2, P.INT32), P.bound(6, P.INT32)))
    jt, cond = {"inner_band": (INNER, band), "semi_band": (LEFT_SEMI, band), "not_in": (LEFT_ANTI, not_in)}[join]
    j = P.broadcast_nested_loop_join(P.scan([P.INT64, P.INT32, P.INT32]), P.scan([P.INT64, P.INT64, P.INT32, P.INT32]), jt, P.BUILD_RIGHT,
                                     condition=cond)
    return P.hash_agg(j, [], [P.agg_count([P.bound(0, P.INT64)]), P.agg_sum(P.bound(0, P.INT64), P.INT64)], P.PARTIAL)


# ---- stages and the byte model ---------------------------------------------------------------------------------------------------------
STAGES = {"pair_enum": ("k_nlj_pairs",), "gathers": ("k_gather_rows", "k_gather_bits", "k_bytes_to_bitmap"), "condition_kernel": ("cb_select_count",),
          "resolution": ("k_join_cond_mark", "k_nlj_cond_resolve", "k_flags_not", "k_block_counts", "k_scan_counts", "k_compact_scatter"),
          "aggregate": ("cb_pipeline_agg", "cb_finalize")}
READS = {"inner_band": (8, 8, 8), "semi_band": (8, 8, 8), "not_in": (4, 4, 4, 4)}   # value bytes of each column the condition reads


def stage_of(name):
    for st, pats in STAGES.items():
        if any(p in name for p in pats):
            return st
    return "other"


def model(join, stats):
    """algorithmic bytes per stage: enumerating a pair writes two indices (8 B); gathering a column the condition reads reads an index
    and a value and writes the value (4 + 2w B per pair, plus 2 B per pair for a nullable build column's validity); the condition
    kernel reads the gathered values and writes a bit; resolution reads the bit and two indices and writes a passed byte (9 B), and an
    inner join's resolve writes the pair and a keep byte (9 B) which the compaction reads (9 B)"""
    c = stats["join_cond_pairs"]
    w = READS[join]
    nullable = 2 if join == "not_in" else 0
    out = {"pair_enum": 8 * c, "gathers": c * (sum(4 + 2 * x for x in w) + 2 * nullable), "condition_kernel": c * sum(w) + c // 8,
           "resolution": c * (9 + (18 if join == "inner_band" else 0))}
    return out


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


def step(native, p, e, r):
    with native.Plan(p, [e, r]) as pl:
        return pl.collect(), pl.stats()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100000000:1024,10000000:16384", help="events:ranges pairs")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_nested_loop_join.py measures the GPU: no CUDA device")
    import comet_b200  # noqa: F401
    from comet_b200 import native, proto as P
    for size in args.sizes.split(","):
        n, m = (int(x) for x in size.split(":"))
        t0 = time.perf_counter()
        ev, rg = generate(np, n, m, args.seed)
        want = answers(np, ev, rg)
        e, r, keep = device_tables(native, P, torch, np, ev, rg)
        del ev
        gen_s = time.perf_counter() - t0
        for join in ("inner_band", "semi_band", "not_in"):
            p = plan(P, join)
            walls = []
            for _ in range(args.warmup + args.steps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res, stats = step(native, p, e, r)
                walls.append((time.perf_counter() - t0) * 1e3)
                row = list(res.to_pylist()[0].values())
                assert (row[0], row[1]) == want[join], (join, row, want[join])
            walls = sorted(walls[args.warmup:])
            stages = profile(torch, lambda: step(native, p, e, r))
            bytes_ = model(join, stats)
            pairs = stats["join_cond_pairs"]
            assert pairs == n * m, (pairs, n * m)
            med = walls[len(walls) // 2]
            kernel_ms = sum(stages.values())
            print(json.dumps(dict(bench="nested_loop_join", join=join, events=n, ranges=m, pairs=pairs,
                                  step_ms_median=round(med, 2), step_ms_min=round(walls[0], 2), step_ms_max=round(walls[-1], 2),
                                  pairs_per_s=round(pairs / (med / 1e3), -6), checked_steps=args.warmup + args.steps,
                                  check="numpy answer: count and sum of t", join_out_rows=stats["join_out_rows"], kernel_launches=stats["kernel_launches"],
                                  stage_ms={k: round(v, 3) for k, v in stages.items()}, kernel_ms=round(kernel_ms, 2),
                                  model_bytes_per_pair={k: round(v / pairs, 2) for k, v in bytes_.items()},
                                  model_bytes_per_pair_total=round(sum(bytes_.values()) / pairs, 2),
                                  stage_gbps={k: round(bytes_[k] / (stages[k] * 1e6), 1) for k in bytes_ if stages.get(k)},
                                  data_gen_s=round(gen_s, 1), card=card())), flush=True)
        del e, r, keep
        torch.cuda.empty_cache()
        native.lib().cb200_release_cached_memory(0)


if __name__ == "__main__":
    main()
