"""Sort and TopK on the GPU: what they cost over HBM-resident synthetic lineitem (tpch.gen_lineitem, seed 42).

The base rows come from tpch.gen_lineitem(--base-rows, seed 42) and are repeated on the device up to the workload's size (the generator
is host Python; 600 M rows of it would take minutes and tens of GB of host memory).  Repeats make many ties, which the stable order
resolves by input position.

1. `full`: ORDER BY l_shipdate, l_extendedprice DESC over --full-rows rows of the Q1 DEC columns (a device table; decimals 8 bytes per row,
   flags 1-byte dictionary codes, dates 4 bytes), read back with cb200_execute_device.  The timed output is checked on the device to be in
   order; the same plan at --check-rows rows is checked column by column against numpy's stable lexsort.
2. `topk`: ORDER BY l_extendedprice DESC LIMIT 100 over --topk-rows rows of the same table, checked in full against the exact stable
   top 100 (threshold by torch.topk, then a stable sort of the rows at or above it).
3. `topk_parquet`: the same TopK end to end through NativeScan over a pinned Parquet image of the base rows, listed as many times as
   needed for --topk-rows rows.

For each: the step time (host clock around work that ends in a device synchronise; median over --steps after --warmup), per-kernel
device times from torch.profiler in a separate step, the radix passes actually run, and algorithmic GB/s per stage from the byte model in
`model()`.  Prints one JSON line per workload, with the card's name and power limit.
    python bench_sort.py [--full-rows 300000000] [--topk-rows 600000000] [--steps 5] [--warmup 1]
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

Q1 = ["l_quantity", "l_extendedprice", "l_discount", "l_tax", "l_returnflag", "l_linestatus", "l_shipdate"]
WIDTH = {"l_quantity": 8, "l_extendedprice": 8, "l_discount": 8, "l_tax": 8, "l_returnflag": 1, "l_linestatus": 1, "l_shipdate": 4}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


# ---- stages and the byte model ---------------------------------------------------------------------------------------------------------
STAGES = {"keys": ("k_sort_keys",), "passes": ("k_sort_hist", "k_scan_chunks", "k_scan_totals", "k_sort_scatter"),
          "select": ("k_sort_select", "k_block_counts", "k_scan_counts", "k_compact_scatter", "k_sort_iota"),
          "gather": ("k_gather_rows", "k_gather_bits", "k_bytes_to_bitmap"), "concat": ("k_bitmap_append", "k_remap_codes"),
          "to_arrow_layout": ("k_to_arrow_layout",), "scan": ("k_pq", "parquet")}


def stage_of(name):
    for st, pats in STAGES.items():
        if any(p in name for p in pats):
            return st
    return None


def model(stats, key_bytes, words, gathered_rows, row_bytes, n_cols):
    """algorithmic bytes per stage: key columns read + keys written; per pass 2 x (key + index) per row; per TopK select step the key read
    once; gathers read and write each column and read the index once per column"""
    return {"keys": stats["sort_rows"] * (key_bytes + 8 * words),
            "passes": stats["sort_pass_rows"] * 2 * (8 * words + 4),
            "select": stats["sort_select_rows"] * 8 * words,
            "gather": gathered_rows * (2 * row_bytes + 4 * n_cols)}


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
        if st:
            stages[st] = stages.get(st, 0.0) + us / 1e3
    top = dict(sorted(((k, [round(v[0], 3), v[1]]) for k, v in kernels.items()), key=lambda kv: -kv[1][0])[:16])
    return stages, top


def report(name, rows, walls, stats, stages, top, bytes_, extra):
    walls = sorted(walls)
    gbps = {k: round(bytes_[k] / (stages[k] * 1e6), 1) for k in bytes_ if stages.get(k)}
    print(json.dumps(dict(bench=name, rows=rows, step_ms_median=round(walls[len(walls) // 2], 2), step_ms_min=round(walls[0], 2),
                          step_ms_max=round(walls[-1], 2), radix_passes=stats["sort_passes"], pass_rows=stats["sort_pass_rows"],
                          select_rows=stats["sort_select_rows"], key_rows=stats["sort_rows"],
                          stage_ms={k: round(v, 3) for k, v in stages.items()}, model_gb={k: round(v / 1e9, 2) for k, v in bytes_.items()},
                          stage_gbps=gbps, kernels_ms_count=top, card=card(), **extra)), flush=True)


# ---- data ---------------------------------------------------------------------------------------------------------------------------------
def base_columns(torch, tpch, base_rows):
    import numpy as np
    cols = tpch.gen_lineitem(base_rows, seed=42)
    dev = {}
    for k in Q1:
        a = cols[k]
        a = a.astype(np.int8) if k in ("l_returnflag", "l_linestatus") else a
        dev[k] = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return cols, dev


def tiled(torch, dev, n):
    out = {}
    for k, t in dev.items():
        reps = (n + t.numel() - 1) // t.numel()
        out[k] = t.repeat(reps)[:n].contiguous()
    return out


def device_table(native, P, tpch, cols, n):
    D12 = P.DECIMAL(12, 2)
    t = native.DeviceTable(n)
    for k in Q1:
        if k in ("l_returnflag", "l_linestatus"):
            t.add(P.STRING, cols[k].data_ptr(), 1, dictionary=tpch.RETURNFLAGS if k == "l_returnflag" else tpch.LINESTATUS, keep=cols[k])
        elif k == "l_shipdate":
            t.add(P.DATE, cols[k].data_ptr(), 4, keep=cols[k])
        else:
            t.add(D12, cols[k].data_ptr(), 8, keep=cols[k])
    return t


def read_device(torch, p, rows, cols_out):
    """the output columns of cb200_execute_device as torch tensors (decimals: the low 8 bytes of their Arrow Decimal128 values)"""
    from comet_b200.dist import device_bytes
    out = {}
    for j, k in enumerate(Q1):
        c = cols_out[j]
        raw = device_bytes(torch, c.values, rows * c.value_width, "cuda")
        if c.value_width == 16:
            out[k] = raw.view(torch.int64).view(-1, 2)[:, 0]
        elif c.value_width == 8:
            out[k] = raw.view(torch.int64)
        elif c.value_width == 4:
            out[k] = raw.view(torch.int32)
        else:
            out[k] = raw.view(torch.int8)
    return out


def run_device(native, plan, inputs, config):
    """one step: (wall ms, stats, plan handle, rows, device columns); the caller releases the plan"""
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    p = native.Plan(plan, inputs, config=config)
    r = p.execute_device()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3
    rows, cols = r if r is not None else (0, None)
    return wall, p.stats(), p, rows, cols


# ---- workloads ----------------------------------------------------------------------------------------------------------------------------
def full(args, torch, native, tpch, P, dev):
    import numpy as np
    D12 = P.DECIMAL(12, 2)
    types = [D12] * 4 + [P.STRING, P.STRING, P.DATE]
    plan = P.sort(P.scan(types), [P.sort_order(P.bound(6, P.DATE)), P.sort_order(P.bound(1, D12), descending=True)])

    # exact check at --check-rows rows: every column against numpy's stable lexsort
    n = args.check_rows
    cols = tiled(torch, dev, n)
    _, st, p, rows, out = run_device(native, plan, [device_table(native, P, tpch, cols, n)], {"spark.comet.b200.chunkRows": str(n // 3 + 1024)})
    got = {k: v.cpu().numpy() for k, v in read_device(torch, p, rows, out).items()}
    p.release()
    host = {k: v.cpu().numpy() for k, v in cols.items()}
    order = np.lexsort((-host["l_extendedprice"], host["l_shipdate"]))
    assert rows == n
    for k in Q1:
        assert (got[k] == host[k][order]).all(), k
    del cols

    n = args.full_rows
    cols = tiled(torch, dev, n)
    table = device_table(native, P, tpch, cols, n)
    cfg = {"spark.comet.b200.chunkRows": str((n + 1023) // 1024 * 1024)}   # one slice of the table: nothing to concatenate
    walls = []
    for i in range(args.warmup + args.steps):
        wall, stats, p, rows, out = run_device(native, plan, [table], cfg)
        assert rows == n
        if i == args.warmup + args.steps - 1:   # the timed output is in order
            o = read_device(torch, p, rows, out)
            ship, price = o["l_shipdate"], o["l_extendedprice"]
            ok = (ship[:-1] < ship[1:]) | ((ship[:-1] == ship[1:]) & (price[:-1] >= price[1:]))
            assert bool(ok.all()), "full sort output out of order"
            del o, ship, price, ok
        p.release()
        if i >= args.warmup:
            walls.append(wall)
    def one():
        p = run_device(native, plan, [table], cfg)[2]
        p.release()
    stages, top = profile(torch, one)
    row_bytes = sum(WIDTH.values())
    report("full_sort", n, walls, stats, stages, top, model(stats, 4 + 8, 2, n, row_bytes, len(Q1)),
           dict(order_by="l_shipdate, l_extendedprice DESC", checked_rows=args.check_rows, check="numpy stable lexsort, every column"))


def expected_topk(torch, price, k):
    """row indices of the stable ORDER BY price DESC LIMIT k"""
    thr = torch.topk(price, k).values[-1]
    cand = torch.nonzero(price >= thr).flatten()
    order = torch.sort(price[cand], descending=True, stable=True).indices
    return cand[order][:k]


def check_topk(torch, got, cols, idx):
    for k in Q1:
        assert torch.equal(got[k], cols[k][idx]), k


def topk(args, torch, native, tpch, P, dev):
    D12 = P.DECIMAL(12, 2)
    types = [D12] * 4 + [P.STRING, P.STRING, P.DATE]
    plan = P.sort(P.scan(types), [P.sort_order(P.bound(1, D12), descending=True)], fetch=100)
    n = args.topk_rows
    cols = tiled(torch, dev, n)
    table = device_table(native, P, tpch, cols, n)
    idx = expected_topk(torch, cols["l_extendedprice"], 100)
    walls = []
    for i in range(args.warmup + args.steps):
        wall, stats, p, rows, out = run_device(native, plan, [table], None)
        assert rows == 100
        check_topk(torch, read_device(torch, p, rows, out), cols, idx)
        p.release()
        if i >= args.warmup:
            walls.append(wall)

    def one():
        _, _, p, _, _ = run_device(native, plan, [table], None)
        p.release()
    stages, top = profile(torch, one)
    report("topk", n, walls, stats, stages, top, model(stats, 8, 1, 2 * 100 * (n // (1 << 26) + 1), sum(WIDTH.values()), len(Q1)),
           dict(order_by="l_extendedprice DESC LIMIT 100", check="exact stable top 100, every column"))
    del table, cols


def topk_parquet(args, torch, native, tpch, P, dev, host_cols):
    import numpy as np
    import pyarrow as pa
    import pyarrow.parquet as pq
    tbl = tpch.lineitem_table(host_cols, "dec", dictionary=True, columns=Q1)
    sink = pa.BufferOutputStream()
    pq.write_table(tbl, sink, row_group_size=1 << 20, compression="NONE", use_dictionary=["l_returnflag", "l_linestatus"],
                   store_decimal_as_integer=True)
    buf = sink.getvalue()
    pinned = torch.empty(buf.size, dtype=torch.uint8, pin_memory=True)
    pinned.numpy()[:] = np.frombuffer(buf, dtype=np.uint8)
    name = native.register_memory_file("lineitem_sort_base", pinned)
    base = tbl.num_rows
    reps = (args.topk_rows + base - 1) // base
    n = reps * base
    fields = [(k, t, True) for k, t in zip(Q1, tpch.q1_scan_fields("dec"))]
    D12 = P.DECIMAL(12, 2)
    plan = P.sort(P.native_scan(fields, fields, [name] * reps), [P.sort_order(P.bound(1, D12), descending=True)], fetch=100)
    price = dev["l_extendedprice"].repeat(reps)
    idx = expected_topk(torch, price, 100)
    del price
    walls = []
    for i in range(args.warmup + args.steps):
        wall, stats, p, rows, out = run_device(native, plan, [], None)
        assert rows == 100
        got = read_device(torch, p, rows, out)
        for j, (k, values) in enumerate((("l_returnflag", tpch.RETURNFLAGS), ("l_linestatus", tpch.LINESTATUS))):
            col = Q1.index(k)   # the scan's dictionary has its own code order: compare the spelled-out values
            to_base = torch.tensor([values.index(v) for v in p.dict_values(col, out[col].n_dict)], dtype=torch.int8, device="cuda")
            got[k] = to_base[got[k].long()]
        p.release()
        for k in Q1:
            want = dev[k][idx % base]
            assert torch.equal(got[k], want), k
        if i >= args.warmup:
            walls.append(wall)

    def one():
        _, _, p, _, _ = run_device(native, plan, [], None)
        p.release()
    stages, top = profile(torch, one)
    report("topk_parquet", n, walls, stats, stages, top, model(stats, 8, 1, 0, sum(WIDTH.values()), len(Q1)),
           dict(order_by="l_extendedprice DESC LIMIT 100", source="NativeScan over a pinned Parquet image listed %d times" % reps,
                parquet_bytes=buf.size, check="exact stable top 100, every column"))
    native.register_memory_file("lineitem_sort_base", None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--full-rows", type=int, default=300_000_000)
    ap.add_argument("--topk-rows", type=int, default=600_000_000)
    ap.add_argument("--base-rows", type=int, default=1 << 24)
    ap.add_argument("--check-rows", type=int, default=4_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--only", choices=["full", "topk", "topk_parquet"], default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_sort.py measures the GPU: no CUDA device")
    import comet_b200  # noqa: F401
    from comet_b200 import native, tpch, proto as P
    host_cols, dev = base_columns(torch, tpch, args.base_rows)
    if args.only in (None, "full"):
        full(args, torch, native, tpch, P, dev)
        torch.cuda.empty_cache()
        native.lib().cb200_release_cached_memory(0)   # the library's recycled blocks of the full sort
    if args.only in (None, "topk"):
        topk(args, torch, native, tpch, P, dev)
        torch.cuda.empty_cache()
    if args.only in (None, "topk_parquet"):
        topk_parquet(args, torch, native, tpch, P, dev, host_cols)


if __name__ == "__main__":
    main()
