"""Hash join on the GPU: TPC-DS Q3 over HBM-resident synthetic tables.

    SELECT d_year, i_brand_id, i_brand, SUM(ss_ext_sales_price)
    FROM date_dim, store_sales, item
    WHERE d_date_sk = ss_sold_date_sk AND ss_item_sk = i_item_sk AND i_manufact_id = 128 AND d_moy = 11
    GROUP BY d_year, i_brand, i_brand_id

as Comet plans it (BASELINE.json config 5): Scan(date_dim) -> Filter -> Projection -> BroadcastHashJoin(BuildLeft) with store_sales ->
Projection -> BroadcastHashJoin(BuildRight) with Filter(item) -> Projection -> HashAggregate(Partial); then HashAggregate(Final) over the
partial state.  All three tables are device tables generated from a seed (numpy, in chunks, copied to the device):
- date_dim: 73,049 days from 1900-01-02 (d_date_sk 2415022 ..), d_year and d_moy from the calendar;
- item: 204,000 rows (TPC-DS scale 100), i_brand_id in 1001001 .. 1001500, i_brand its dictionary-coded name, i_manufact_id in 1 .. 1000;
- store_sales: --rows rows, ss_sold_date_sk uniform over 1998-01-02 .. 2003-01-02 with 4 % NULL, ss_item_sk uniform over the items with
  0.5 % NULL, ss_ext_sales_price decimal(7, 2) stored 8 bytes wide with 1 % NULL.
Every timed result is checked against the answer numpy computes from the same chunks.

Reports, per size: the step time (host clock around both plans, which end by copying their results to the host; median over --steps
after --warmup), the kernel time per stage from torch.profiler in a separate step, the join counters, and GB/s per stage by the byte
model in `model()`.  Prints one JSON line per size, with the card's name and power limit.
    python bench_join.py [--rows 100000000,600000000] [--steps 5] [--warmup 1]
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

D0, N_DATE, N_ITEM = 2415022, 73_049, 204_000
SALES_D0, SALES_D1 = 2450816, 2452642          # 1998-01-02 .. 2003-01-02
MANUFACT, MOY = 128, 11
CHUNK = 1 << 25


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


# ---- data ---------------------------------------------------------------------------------------------------------------------------------
def dimensions(np):
    day = np.datetime64("1900-01-02") + np.arange(N_DATE)
    years = day.astype("datetime64[Y]").astype(np.int64) + 1970
    months = (day.astype("datetime64[M]").astype(np.int64) % 12 + 1)
    date_dim = {"d_date_sk": np.arange(D0, D0 + N_DATE, dtype=np.int32), "d_year": years.astype(np.int32), "d_moy": months.astype(np.int32)}
    rng = np.random.default_rng(7)
    bid = rng.integers(0, 500, N_ITEM)
    item = {"i_item_sk": np.arange(1, N_ITEM + 1, dtype=np.int32), "i_brand_id": (bid + 1001001).astype(np.int32), "i_brand": bid.astype(np.int32),
            "i_manufact_id": rng.integers(1, 1001, N_ITEM).astype(np.int32)}
    brands = [f"brand #{i + 1001001}" for i in range(500)]
    return date_dim, item, brands


def sales_chunk(np, seed, k, n):
    rng = np.random.default_rng([seed, k])
    return {"date": rng.integers(SALES_D0, SALES_D1 + 1, n).astype(np.int32), "date_ok": rng.random(n) >= 0.04,
            "item": rng.integers(1, N_ITEM + 1, n).astype(np.int32), "item_ok": rng.random(n) >= 0.005,
            "price": rng.integers(0, 10**6, n), "price_ok": rng.random(n) >= 0.01}


def build_sales(np, torch, n, seed, date_dim, item, answer):
    """store_sales on the device, and the numpy answer accumulated into `answer` {(d_year, i_brand_id): [unscaled sum, any non-NULL]}"""
    dev = {"date": torch.empty(n + 4, dtype=torch.int32, device="cuda"), "item": torch.empty(n + 4, dtype=torch.int32, device="cuda"),
           "price": torch.empty(n + 2, dtype=torch.int64, device="cuda")}
    bits = {k: torch.zeros((n + 7) // 8 + 16, dtype=torch.uint8, device="cuda") for k in ("date_ok", "item_ok", "price_ok")}
    moy_ok = date_dim["d_moy"] == MOY
    year = date_dim["d_year"]
    man_ok = np.concatenate([[False], item["i_manufact_id"] == MANUFACT])
    bid = np.concatenate([[0], item["i_brand_id"]])
    for k, r0 in enumerate(range(0, n, CHUNK)):
        m = min(CHUNK, n - r0)
        c = sales_chunk(np, seed, k, m)
        for name in ("date", "item", "price"):
            dev[name][r0:r0 + m].copy_(torch.from_numpy(c[name]))
        for name in bits:
            b = np.packbits(c[name], bitorder="little")
            bits[name][r0 // 8:r0 // 8 + len(b)].copy_(torch.from_numpy(b))
        sel = c["date_ok"] & c["item_ok"]
        sel &= moy_ok[np.where(sel, c["date"] - D0, 0)] & man_ok[np.where(sel, c["item"], 0)]
        keys = year[c["date"][sel] - D0].astype(np.int64) * 10**8 + bid[c["item"][sel]]
        price, ok = c["price"][sel], c["price_ok"][sel]
        for key, p, v in zip(keys.tolist(), price.tolist(), ok.tolist()):
            a = answer.setdefault(key, [0, False])
            if v:
                a[0] += p
                a[1] = True
    return dev, bits


def device_tables(native, P, torch, date_dim, item, brands, n, sales, bits):
    keep = []
    def put(t, dt, arr, width, validity=None, dictionary=None):
        import numpy as np
        v = arr if torch.is_tensor(arr) else torch.from_numpy(np.concatenate([arr, np.zeros(8, arr.dtype)])).cuda()
        keep.append(v)
        t.add(dt, v.data_ptr(), width, validity.data_ptr() if validity is not None else None, -1 if validity is not None else 0, dictionary=dictionary, keep=v)
    I32 = P.INT32
    dd = native.DeviceTable(N_DATE)
    for k in ("d_date_sk", "d_year", "d_moy"):
        put(dd, I32, date_dim[k], 4)
    it = native.DeviceTable(N_ITEM)
    put(it, I32, item["i_item_sk"], 4)
    put(it, I32, item["i_brand_id"], 4)
    put(it, P.STRING, item["i_brand"], 4, dictionary=brands)
    put(it, I32, item["i_manufact_id"], 4)
    ss = native.DeviceTable(n)
    put(ss, I32, sales["date"], 4, bits["date_ok"])
    put(ss, I32, sales["item"], 4, bits["item_ok"])
    put(ss, P.DECIMAL(7, 2), sales["price"], 8, bits["price_ok"])
    return [dd, ss, it], keep


# ---- stages and the byte model ---------------------------------------------------------------------------------------------------------
STAGES = {"join_keys": ("k_sort_keys",), "join_build": ("k_sort_hist", "k_sort_scatter", "k_join_heads", "k_join_insert", "k_block_counts",
                                                          "k_scan_counts", "k_compact_scatter", "k_sort_iota"),
          "join_probe": ("k_join_probe",), "scans": ("k_scan_chunks", "k_scan_totals"), "join_emit": ("k_join_emit",),
          "gathers": ("k_gather_rows", "k_gather_bits", "k_bytes_to_bitmap"), "aggregate": ("cb_pipeline_agg", "cb_finalize"),
          "filter_projection": ("cb_pipeline_select", "cb_select_count")}


def stage_of(name):
    for st, pats in STAGES.items():
        if any(p in name for p in pats):
            return st
    return "other"


def model(stats, n):
    """algorithmic bytes: keys read (4 B + a validity bit) and written (8 B) for every build and probe row; a probe reads its key, one
    8-byte slot, the run bounds (8 B) and the run's first key (8 B) and writes a count and a run (8 B); an emitted row reads its probe row's
    run and offsets (12 B) and writes two indices (8 B); the gathers of both joins read and write each output row's columns (the first
    join's 4 + 4 + 8 + 4 + 4 bytes per row of the second join's probe columns plus date columns: counted as 24 B) and an index per
    column; the aggregate and the scan's pipeline read store_sales once (16 B + 3 validity bits per row)"""
    keyed = stats["join_build_rows"] + stats["join_probe_rows"]
    out = stats["join_out_rows"]
    return {"join_keys": keyed * 12, "join_probe": stats["join_probe_rows"] * 40, "join_emit": out * 20, "gathers": out * (2 * 24 + 4 * 5)}


def profile(torch, fn):
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    kernels, stages = {}, {}
    for e in p.events():
        us = e.device_time_total
        if us <= 0:
            continue
        k = kernels.setdefault(e.name[:80], [0.0, 0])
        k[0] += us / 1e3
        k[1] += 1
        st = stage_of(e.name)
        stages[st] = stages.get(st, 0.0) + us / 1e3
    top = dict(sorted(((k, [round(v[0], 3), v[1]]) for k, v in kernels.items()), key=lambda kv: -kv[1][0])[:16])
    return stages, top


# ---- the query ----------------------------------------------------------------------------------------------------------------------------
def plans(P):
    I32, M, S = P.INT32, P.DECIMAL(7, 2), P.DECIMAL(17, 2)
    dd = P.projection(P.filter_(P.scan([I32, I32, I32]), P.eq(P.bound(2, I32), P.literal(MOY, I32))), [P.bound(0, I32), P.bound(1, I32)])
    j1 = P.hash_join(dd, P.scan([I32, I32, M]), [P.bound(0, I32)], [P.bound(0, I32)], P.INNER, P.BUILD_LEFT)
    p1 = P.projection(j1, [P.bound(1, I32), P.bound(3, I32), P.bound(4, M)])
    it = P.projection(P.filter_(P.scan([I32, I32, P.STRING, I32]), P.eq(P.bound(3, I32), P.literal(MANUFACT, I32))),
                      [P.bound(0, I32), P.bound(1, I32), P.bound(2, P.STRING)])
    j2 = P.hash_join(p1, it, [P.bound(1, I32)], [P.bound(0, I32)], P.INNER, P.BUILD_RIGHT)
    p2 = P.projection(j2, [P.bound(0, I32), P.bound(5, P.STRING), P.bound(4, I32), P.bound(2, M)])
    keys = [P.bound(0, I32), P.bound(1, P.STRING), P.bound(2, I32)]
    partial = P.hash_agg(p2, keys, [P.agg_sum(P.bound(3, M), S)], P.PARTIAL)
    final = P.hash_agg(P.scan([I32, P.STRING, I32, S, P.BOOL], source="shuffle"), keys, [P.agg_sum(P.unbound("p", M), S)], P.FINAL)
    return partial, final


def step(native, partial, final, tables):
    """(result table, partial plan's stats)"""
    with native.Plan(partial, tables) as p:
        state = p.collect()
        stats = p.stats()
    with native.Plan(final, [state]) as p:
        return p.collect(), stats


def check(res, answer, brands):
    got = {}
    for r in res.to_pylist():
        v = r["col_3"]
        assert r["col_1"] == f"brand #{r['col_2']}", r
        got[r["col_0"] * 10**8 + r["col_2"]] = None if v is None else int(v.scaleb(2))
    want = {k: (s if ok else None) for k, (s, ok) in answer.items()}
    assert got == want, (len(got), len(want))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="100000000,600000000")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=42)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_join.py measures the GPU: no CUDA device")
    import comet_b200  # noqa: F401
    from comet_b200 import native, proto as P
    date_dim, item, brands = dimensions(np)
    partial, final = plans(P)
    for n in (int(x) for x in args.rows.split(",")):
        t0 = time.perf_counter()
        answer = {}
        sales, bits = build_sales(np, torch, n, args.seed, date_dim, item, answer)
        tables, keep = device_tables(native, P, torch, date_dim, item, brands, n, sales, bits)
        gen_s = time.perf_counter() - t0
        walls = []
        for i in range(args.warmup + args.steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res, stats = step(native, partial, final, tables)
            walls.append((time.perf_counter() - t0) * 1e3)
            check(res, answer, brands)
        walls = sorted(walls[args.warmup:])
        stages, top = profile(torch, lambda: step(native, partial, final, tables))
        bytes_ = model(stats, n)
        print(json.dumps(dict(bench="q3_join", rows=n, step_ms_median=round(walls[len(walls) // 2], 2), step_ms_min=round(walls[0], 2),
                              step_ms_max=round(walls[-1], 2), groups=res.num_rows, checked_steps=args.warmup + args.steps,
                              check="numpy answer, every group", join_build_rows=stats["join_build_rows"],
                              join_probe_rows=stats["join_probe_rows"], join_out_rows=stats["join_out_rows"],
                              kernel_launches=stats["kernel_launches"], stage_ms={k: round(v, 3) for k, v in stages.items()},
                              model_gb={k: round(v / 1e9, 3) for k, v in bytes_.items()},
                              stage_gbps={k: round(bytes_[k] / (stages[k] * 1e6), 1) for k in bytes_ if stages.get(k)},
                              kernels_ms_count=top, data_gen_s=round(gen_s, 1), card=card())), flush=True)
        del tables, keep, sales, bits
        torch.cuda.empty_cache()
        native.lib().cb200_release_cached_memory(0)


if __name__ == "__main__":
    main()
