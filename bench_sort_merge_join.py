"""Sort-merge join on the GPU: a TPC-DS Q80-shaped fact-to-returns join over HBM-resident synthetic tables.

    SELECT ss_store_sk, SUM(ss_ext_sales_price), SUM(CASE WHEN sr_return_amt IS NULL THEN 0 ELSE sr_return_amt END)
    FROM store_sales LEFT OUTER JOIN store_returns ON ss_ticket_number = sr_ticket_number AND ss_item_sk = sr_item_sk
    GROUP BY ss_store_sk

as Comet plans a shuffled join: Scan -> Sort(ticket, item) on each side -> SortMergeJoin (LeftOuter; in a second run FullOuter) ->
Projection -> HashAggregate(Partial); then HashAggregate(Final) over the partial state.  Both tables are device tables generated from a
seed (numpy, in chunks, copied to the device), in no particular order:
- store_sales: --rows rows over rows / 4 tickets, four items per ticket (the (ticket, item) pair unique), ss_store_sk in 1 .. 1002,
  ss_ext_sales_price decimal(7, 2) stored 8 bytes wide;
- store_returns: about 10 % of the sales pairs plus 1 % as many pairs with no sale, sr_return_amt decimal(7, 2) with 5 % NULL.
Every timed result is checked against the answer numpy computes from the same chunks.

Reports, per size and join type: the step time (host clock around both plans, which end by copying their results to the host; median
over --steps after --warmup), the kernel time per stage from torch.profiler in a separate step, the join counters, and GB/s per stage by
the byte model in `model()`.  Prints one JSON line per size and join type, with the card's name and power limit.
    python bench_sort_merge_join.py [--rows 100000000,300000000] [--steps 5] [--warmup 1]
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

N_STORE = 1002
TICKET_MUL = 2654435761    # odd and prime to any power of two: row -> ticket is a permutation of the tickets
CHUNK = 1 << 25
LEFT_OUTER, FULL_OUTER = 1, 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


# ---- data ---------------------------------------------------------------------------------------------------------------------------------
def sales_rows(np, r0, m, n_tickets):
    """rows [r0, r0 + m) of store_sales: ticket and item.  n_tickets is a power of two; row i holds item slot i // n_tickets of ticket
    (i * TICKET_MUL) mod n_tickets"""
    i = np.arange(r0, r0 + m, dtype=np.int64)
    ticket = (i * TICKET_MUL) & (n_tickets - 1)
    item = (i // n_tickets) * 50_000 + (ticket * 7919) % 50_000 + 1
    return ticket, item.astype(np.int32)


def build(np, torch, n, seed):
    """both tables on the device, and the numpy answers {store: [sales sum, returns sum]} of LeftOuter (FullOuter adds store None)"""
    n_tickets = 1 << max(1, (n // 4 - 1).bit_length())
    rng = np.random.default_rng(seed)
    ss = {"ticket": torch.empty(n + 2, dtype=torch.int64, device="cuda"), "item": torch.empty(n + 4, dtype=torch.int32, device="cuda"),
          "store": torch.empty(n + 4, dtype=torch.int32, device="cuda"), "price": torch.empty(n + 2, dtype=torch.int64, device="cuda")}
    ret = {"ticket": [], "item": [], "amt": [], "ok": []}
    sales_sum = np.zeros(N_STORE + 1, np.int64)
    ret_sum = np.zeros(N_STORE + 1, np.int64)
    for r0 in range(0, n, CHUNK):
        m = min(CHUNK, n - r0)
        ticket, item = sales_rows(np, r0, m, n_tickets)
        store = rng.integers(1, N_STORE + 1, m).astype(np.int32)
        price = rng.integers(0, 10**6, m)
        for name, a in (("ticket", ticket), ("item", item), ("store", store), ("price", price)):
            ss[name][r0:r0 + m].copy_(torch.from_numpy(a))
        sales_sum += np.bincount(store, weights=price, minlength=N_STORE + 1).round().astype(np.int64)
        sel = rng.random(m) < 0.10
        k = int(sel.sum())
        amt, ok = rng.integers(0, 10**6, k), rng.random(k) >= 0.05
        ret_sum += np.bincount(store[sel], weights=np.where(ok, amt, 0), minlength=N_STORE + 1).round().astype(np.int64)
        for name, a in (("ticket", ticket[sel]), ("item", item[sel]), ("amt", amt), ("ok", ok)):
            ret[name].append(a)
    k = n // 100                                                    # returns of no sale: tickets past the last one
    amt, ok = rng.integers(0, 10**6, k), rng.random(k) >= 0.05
    ret["ticket"].append(n_tickets + rng.permutation(k).astype(np.int64))
    ret["item"].append(rng.integers(1, 200_000, k).astype(np.int32))
    ret["amt"].append(amt)
    ret["ok"].append(ok)
    orphan = int(np.where(ok, amt, 0).sum())
    ret = {name: np.concatenate(v) for name, v in ret.items()}
    answer = {s: [int(sales_sum[s]), int(ret_sum[s])] for s in range(1, N_STORE + 1)}
    return ss, ret, answer, orphan


def device_tables(native, P, torch, n, ss, ret):
    import numpy as np
    keep = []
    def put(t, dt, arr, width, validity=None):
        v = arr if torch.is_tensor(arr) else torch.from_numpy(np.concatenate([arr, np.zeros(8, arr.dtype)])).cuda()
        keep.append(v)
        vp = None
        if validity is not None:
            vb = torch.from_numpy(np.concatenate([np.packbits(validity, bitorder="little"), np.zeros(16, np.uint8)])).cuda()
            keep.append(vb)
            vp = vb.data_ptr()
        t.add(dt, v.data_ptr(), width, vp, -1 if vp else 0, keep=v)
    M = P.DECIMAL(7, 2)
    sales = native.DeviceTable(n)
    put(sales, P.INT64, ss["ticket"], 8)
    put(sales, P.INT32, ss["item"], 4)
    put(sales, P.INT32, ss["store"], 4)
    put(sales, M, ss["price"], 8)
    m = len(ret["ticket"])
    returns = native.DeviceTable(m)
    put(returns, P.INT64, ret["ticket"], 8)
    put(returns, P.INT32, ret["item"], 4)
    put(returns, M, ret["amt"], 8, ret["ok"])
    return [sales, returns], keep


# ---- stages and the byte model ---------------------------------------------------------------------------------------------------------
# The Sort operators' radix passes and the join build's (the returns side's keys) share kernels, so "sorts" holds both.
STAGES = {"key_packing": ("k_sort_keys",), "sorts": ("k_sort_hist", "k_sort_scatter", "k_sort_iota"),
          "join_build": ("k_join_heads", "k_join_insert", "k_block_counts", "k_scan_counts", "k_compact_scatter"),
          "join_lookups": ("k_join_probe",), "count_scans": ("k_scan_chunks", "k_scan_totals"), "pair_emit": ("k_join_emit",),
          "gathers": ("k_gather_rows", "k_gather_bits", "k_bytes_to_bitmap"), "unmatched_build": ("k_join_unmatched",),
          "aggregate": ("cb_pipeline_agg", "cb_finalize")}


def stage_of(name):
    for st, pats in STAGES.items():
        if any(p in name for p in pats):
            return st
    return "other"


def model(stats, n, m):
    """algorithmic bytes: key packing reads the key columns (12 B + a validity bit) and writes a 2-word key (16 B) per row, twice per side
    (its Sort, then the join); a radix pass reads and writes a key and an index (40 B per row moved, the Sorts' passes); a lookup reads its
    key (16 B), one 8-byte slot, the run bounds (8 B) and the run's first key (16 B) and writes a count and a run (8 B); the count scan
    reads and writes a count (8 B); an emitted pair reads its probe row's run and offsets (12 B) and writes two indices (8 B); the gathers
    read and write each output row's 7 columns (44 B each way) and read an index per column (28 B); the unmatched-build pass reads a
    sorted row, its run's hit byte and writes a flag (6 B per build row)"""
    keyed = 2 * (n + m)
    out = stats["join_out_rows"]
    return {"key_packing": keyed * 28, "sorts": stats["sort_pass_rows"] * 40, "join_lookups": stats["join_probe_rows"] * 56,
            "count_scans": stats["join_probe_rows"] * 8, "pair_emit": out * 20, "gathers": out * (2 * 44 + 28),
            "unmatched_build": stats["join_build_rows"] * 6}


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
def plans(P, join_type):
    I32, I64, M, S = P.INT32, P.INT64, P.DECIMAL(7, 2), P.DECIMAL(17, 2)
    order = [P.sort_order(P.bound(0, I64)), P.sort_order(P.bound(1, I32))]
    ss = P.sort(P.scan([I64, I32, I32, M]), order)
    sr = P.sort(P.scan([I64, I32, M]), order)
    j = P.sort_merge_join(ss, sr, [P.bound(0, I64), P.bound(1, I32)], [P.bound(0, I64), P.bound(1, I32)], join_type, order)
    amt = P.bound(6, M)                                                 # (ticket, item, store, price, sr_ticket, sr_item, sr_amt)
    proj = P.projection(j, [P.bound(2, I32), P.bound(3, M), P.case_when([P.is_null(amt)], [P.literal(0, M)], amt)])
    keys = [P.bound(0, I32)]
    partial = P.hash_agg(proj, keys, [P.agg_sum(P.bound(1, M), S), P.agg_sum(P.bound(2, M), S)], P.PARTIAL)
    final = P.hash_agg(P.scan([I32, S, P.BOOL, S, P.BOOL], source="shuffle"), keys,
                       [P.agg_sum(P.unbound("p", M), S), P.agg_sum(P.unbound("r", M), S)], P.FINAL)
    return partial, final


def step(native, partial, final, tables):
    """(result table, partial plan's stats)"""
    with native.Plan(partial, tables) as p:
        state = p.collect()
        stats = p.stats()
    with native.Plan(final, [state]) as p:
        return p.collect(), stats


def check(res, answer, orphan, join_type):
    got = {}
    for r in res.to_pylist():
        p, s = r["col_1"], r["col_2"]
        got[r["col_0"]] = [None if p is None else int(p.scaleb(2)), None if s is None else int(s.scaleb(2))]
    want = dict(answer)
    if join_type == FULL_OUTER:
        want[None] = [None, orphan]                                      # the returns of no sale: no store, no price
    assert got == want, (len(got), len(want))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="100000000,300000000")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=42)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_sort_merge_join.py measures the GPU: no CUDA device")
    import comet_b200  # noqa: F401
    from comet_b200 import native, proto as P
    for n in (int(x) for x in args.rows.split(",")):
        t0 = time.perf_counter()
        ss, ret, answer, orphan = build(np, torch, n, args.seed)
        tables, keep = device_tables(native, P, torch, n, ss, ret)
        m = len(ret["ticket"])
        gen_s = time.perf_counter() - t0
        for jt, name in ((LEFT_OUTER, "left_outer"), (FULL_OUTER, "full_outer")):
            partial, final = plans(P, jt)
            walls = []
            for i in range(args.warmup + args.steps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res, stats = step(native, partial, final, tables)
                walls.append((time.perf_counter() - t0) * 1e3)
                check(res, answer, orphan, jt)
            walls = sorted(walls[args.warmup:])
            stages, top = profile(torch, lambda: step(native, partial, final, tables))
            bytes_ = model(stats, n, m)
            print(json.dumps(dict(bench="q80_sort_merge_join", join_type=name, sales_rows=n, returns_rows=m,
                                  step_ms_median=round(walls[len(walls) // 2], 2), step_ms_min=round(walls[0], 2), step_ms_max=round(walls[-1], 2),
                                  groups=res.num_rows, checked_steps=args.warmup + args.steps, check="numpy answer, every group",
                                  join_build_rows=stats["join_build_rows"], join_probe_rows=stats["join_probe_rows"],
                                  join_out_rows=stats["join_out_rows"], sort_rows=stats["sort_rows"], kernel_launches=stats["kernel_launches"],
                                  stage_ms={k: round(v, 3) for k, v in stages.items()}, model_gb={k: round(v / 1e9, 3) for k, v in bytes_.items()},
                                  stage_gbps={k: round(bytes_[k] / (stages[k] * 1e6), 1) for k in bytes_ if stages.get(k)},
                                  kernels_ms_count=top, data_gen_s=round(gen_s, 1), card=card())), flush=True)
        del tables, keep, ss, ret
        torch.cuda.empty_cache()
        native.lib().cb200_release_cached_memory(0)


if __name__ == "__main__":
    main()
