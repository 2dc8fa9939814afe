"""A distinct aggregate on the GPU: SELECT l_shipmode, COUNT(DISTINCT l_orderkey), SUM(l_extendedprice), SUM(l_quantity) GROUP BY l_shipmode
over HBM-resident synthetic lineitem (tpch.gen_lineitem, seed 42), run as Spark's one-distinct rewrite: four HashAggregate plans.

  stage 1  group by (l_shipmode, l_orderkey)  SUM, SUM Partial                    over the device table
  stage 2  group by (l_shipmode, l_orderkey)  SUM, SUM PartialMerge               over stage 1's state
  stage 3  group by l_shipmode                SUM, SUM PartialMerge + COUNT(l_orderkey) Partial (expr_modes, offset 2)
  stage 4  group by l_shipmode                Final

--base-rows rows come from the generator and are tiled on the host up to --rows (the generator is host Python).  Each stage's output is
collected to host Arrow and handed to the next stage, as a shuffle would; the stage step time (host clock around Plan + collect, ending
in a device synchronise) includes those copies, the per-stage kernel time (torch.profiler, a separate step) does not.  Every timed
step's final result is checked against the direct answer (numpy: distinct (mode, orderkey) pairs, integer sums of the cents).

Prints one JSON line: rows, per-stage step median / min / max, per-stage kernel ms and strategy, algorithmic GB/s per stage by the byte
model in `model()`, and the card's name and power limit.
    python bench_distinct.py [--rows 100000000] [--base-rows 10000000] [--steps 3] [--warmup 1]
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

STRATEGY = {1: "dense", 2: "table", 4: "stream", 8: "migrated"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def plans(P):
    D12, D22 = P.DECIMAL(12, 2), P.DECIMAL(22, 2)
    sums = lambda merge: [P.agg_sum(P.unbound("p", D12) if merge else P.bound(2, D12), D22), P.agg_sum(P.unbound("q", D12) if merge else P.bound(3, D12), D22)]
    state2 = [P.STRING, P.INT64, D22, P.BOOL, D22, P.BOOL]
    keys2 = [P.bound(0, P.STRING), P.bound(1, P.INT64)]
    s1 = P.hash_agg(P.scan([P.STRING, P.INT64, D12, D12]), keys2, sums(False), P.PARTIAL)
    s2 = P.hash_agg(P.scan(state2, source="shuffle"), keys2, sums(True), P.PARTIAL_MERGE, initial_input_buffer_offset=2)
    s3 = P.hash_agg(P.scan(state2, source="shuffle"), [P.bound(0, P.STRING)], sums(True) + [P.agg_count([P.bound(1, P.INT64)])], P.PARTIAL,
                    expr_modes=[P.PARTIAL_MERGE, P.PARTIAL_MERGE, P.PARTIAL], initial_input_buffer_offset=2)
    state3 = [P.STRING, D22, P.BOOL, D22, P.BOOL, P.INT64]
    s4 = P.hash_agg(P.scan(state3, source="shuffle"), [P.bound(0, P.STRING)], sums(True) + [P.agg_count([P.unbound("o", P.INT64)])], P.FINAL)
    return [s1, s2, s3, s4]


def model(in_rows, out_rows):
    """algorithmic bytes per stage: every input column read once, every output column written once.  Stage 1 reads mode (1-byte code),
    orderkey (8) and two decimals (8 each, the device table's width); a state row is key (4-byte code + 8) and two (16-byte sum, 1-byte
    flag) pairs = 46 bytes; a stage 3 state row is 4 + 2 x 17 + 8 = 46 bytes; stage 4 writes 4 + 2 x 16 + 8 = 44 bytes per group."""
    row_in = [25, 46, 46, 46]
    row_out = [46, 46, 46, 44]
    return [in_rows[i] * row_in[i] + out_rows[i] * row_out[i] for i in range(4)]


def profile(torch, fn):
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    return sum(e.device_time_total for e in p.events() if e.device_time_total > 0) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--base-rows", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import numpy as np
    import torch
    from comet_b200 import native, proto as P, tpch
    if not torch.cuda.is_available():
        raise SystemExit("bench_distinct.py measures on the GPU; no CUDA device found")

    base = tpch.gen_lineitem(min(args.base_rows, args.rows), seed=42)
    reps = (args.rows + args.base_rows - 1) // args.base_rows
    host = {k: np.tile(base[k], reps)[:args.rows] for k in ("l_shipmode", "l_orderkey", "l_extendedprice", "l_quantity")}
    # the direct answer: distinct (mode, orderkey) pairs per mode, and integer sums of the cents
    pair = host["l_shipmode"].astype(np.int64) << 48 | host["l_orderkey"]
    uniq = np.unique(pair)
    exp_count = np.bincount((uniq >> 48).astype(np.int64), minlength=len(tpch.SHIPMODES))
    rows_per_mode = np.bincount(host["l_shipmode"], minlength=len(tpch.SHIPMODES))
    sums = {}
    for k in ("l_extendedprice", "l_quantity"):
        sums[k] = [int(host[k][host["l_shipmode"] == m].sum()) for m in range(len(tpch.SHIPMODES))]
    exp = {tpch.SHIPMODES[m]: (sums["l_extendedprice"][m], sums["l_quantity"][m], int(exp_count[m])) for m in range(7) if rows_per_mode[m]}
    dev = {"l_shipmode": torch.from_numpy(host["l_shipmode"].astype(np.int8)).cuda()}
    for k in ("l_orderkey", "l_extendedprice", "l_quantity"):
        dev[k] = torch.from_numpy(host[k]).cuda()
    del pair, uniq

    def table():
        t = native.DeviceTable(args.rows)
        t.add(P.STRING, dev["l_shipmode"].data_ptr(), 1, dictionary=tpch.SHIPMODES, keep=dev["l_shipmode"])
        t.add(P.INT64, dev["l_orderkey"].data_ptr(), 8, keep=dev["l_orderkey"])
        for k in ("l_extendedprice", "l_quantity"):
            t.add(P.DECIMAL(12, 2), dev[k].data_ptr(), 8, keep=dev[k])
        return t

    ps = plans(P)

    def step():
        """the four stages; -> (wall ms per stage, strategy bits per stage, input / output rows per stage, final table)"""
        walls, bits, rin, rout = [], [], [], []
        inp = [table()]
        rin.append(args.rows)
        for i, plan in enumerate(ps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with native.Plan(plan, inp) as p:
                out = p.collect()
                torch.cuda.synchronize()
                walls.append((time.perf_counter() - t0) * 1e3)
                bits.append(p.stats()["agg_strategies"])
            rout.append(out.num_rows)
            if i < 3:
                inp = [out.to_batches()]
                rin.append(out.num_rows)
        return walls, bits, rin, rout, out

    def check(res):
        got = {}
        for r in res.to_pylist():
            v = list(r.values())
            got[v[0]] = (int(v[1].scaleb(2)), int(v[2].scaleb(2)), v[3])
        assert got == exp, (got, exp)

    for _ in range(args.warmup):
        check(step()[4])
    all_walls, bits, rin, rout = [], None, None, None
    for _ in range(args.steps):
        w, bits, rin, rout, res = step()
        check(res)
        all_walls.append(w)
    # per-stage kernel time in a separate step of its own, stage by stage
    kms = []
    inp = [table()]
    for i, plan in enumerate(ps):
        box = {}

        def one():
            with native.Plan(plan, inp) as p:
                box["out"] = p.collect()
        kms.append(profile(torch, one))
        inp = [box["out"].to_batches()]
    check(box["out"])
    by = model(rin, rout)
    med = [sorted(w[i] for w in all_walls)[len(all_walls) // 2] for i in range(4)]
    print(json.dumps(dict(bench="distinct_groupby_shipmode", rows=args.rows, base_rows=args.base_rows, steps=args.steps,
                          stage_step_ms_median=[round(x, 2) for x in med],
                          stage_step_ms_min=[round(min(w[i] for w in all_walls), 2) for i in range(4)],
                          stage_step_ms_max=[round(max(w[i] for w in all_walls), 2) for i in range(4)],
                          stage_kernel_ms=[round(x, 3) for x in kms], stage_rows_in=rin, stage_rows_out=rout,
                          strategies=["+".join(n for b, n in STRATEGY.items() if bits[i] & b) for i in range(4)],
                          model_gb=[round(b / 1e9, 3) for b in by], kernel_gbps=[round(b / (k * 1e6), 1) if k > 0 else None for b, k in zip(by, kms)],
                          result_checked=True, card=card())), flush=True)


if __name__ == "__main__":
    main()
