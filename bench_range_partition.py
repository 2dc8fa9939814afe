"""Repartitioning on the GPU: range, round-robin and hash partitioning of the same HBM-resident input, as a ShuffleWriter over a device
table (one batch: chunkRows covers every row).

    one key:    (k int64, row int64, p2 int32), range on k
    three keys: (a int32, s dictionary string, d decimal(38, 2), row int64), range on (a, s, d): 33 + 33 + 129 bits, 4 words of key
    (row is the input row index, a payload column)

Range bounds are Spark's: quantiles of a sorted sample of the keys (num_partitions - 1 of them).  Round-robin hashes every column
(max_hash_columns 0); hash partitioning hashes the key columns.  Every timed result is checked against numpy: the partition starts of
range partitioning by searchsorted of the rows against the bounds (the three keys combined into one int64 whose order is theirs), of
hash and round-robin partitioning by the oracle's murmur3 and a pmod.  The last step's output is read back and checked whole: every
row's partition id (from its input row's values) is the partition the starts put it in, the row indices rise inside a partition
(stable, hence a permutation), and the key columns are the input's at those rows.

Reports, per input, partition count and partitioning: the step time (host clock around the plan, median over --steps after --warmup)
and the device time of each stage -- partition ids, placement (k_pid_*: histogram, scan, stable placement) and the gather of the
columns -- from the CUDA events the ShuffleWriter records around them (cb200_stats partition_*_ms, medians), and the partition-id
kernel's bandwidth over the key bytes it reads.  Prints one JSON line each, with the card's name and power limit.
    python bench_range_partition.py [--rows 268435456] [--parts 8,200,16384] [--steps 3] [--warmup 1]
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

N_WORDS = 1000       # dictionary entries of the string key, in byte order: "s0000" ...
A_DOM = 1000         # a in [-A_DOM, A_DOM)
D_DOM = 1 << 20      # d's unscaled value in [-D_DOM, D_DOM)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def generate(np, n, shape, seed):
    rng = np.random.default_rng(seed)
    if shape == "one_key":
        return {"k": rng.integers(-2**62, 2**62, n, dtype=np.int64), "row": np.arange(n, dtype=np.int64),
                "p2": rng.integers(0, 2**31, n, dtype=np.int64).astype(np.int32)}
    return {"a": rng.integers(-A_DOM, A_DOM, n, dtype=np.int64).astype(np.int32), "s": rng.integers(0, N_WORDS, n, dtype=np.int64).astype(np.int32),
            "d": rng.integers(-D_DOM, D_DOM, n, dtype=np.int64), "row": np.arange(n, dtype=np.int64)}


def order_key(np, cols, shape):
    """one int64 per row whose order is the range keys' lexicographic order (all ascending)"""
    if shape == "one_key":
        return cols["k"]
    return ((cols["a"].astype(np.int64) + A_DOM) * N_WORDS + cols["s"]) * (2 * D_DOM) + (cols["d"] + D_DOM)


def device_table(native, P, torch, np, cols, shape):
    keep = []
    t = native.DeviceTable(len(next(iter(cols.values()))))

    def add(dt, arr, width, dictionary=None):
        v = torch.from_numpy(np.concatenate([arr.view(np.uint8).reshape(-1), np.zeros(16, np.uint8)])).cuda()
        keep.append(v)
        t.add(dt, v.data_ptr(), width, None, 0, dictionary=dictionary, keep=v)
    if shape == "one_key":
        add(P.INT64, cols["k"], 8); add(P.INT64, cols["row"], 8); add(P.INT32, cols["p2"], 4)
    else:
        add(P.INT32, cols["a"], 4)
        add(P.STRING, cols["s"], 4, dictionary=[f"s{i:04d}" for i in range(N_WORDS)])
        d = np.zeros((len(cols["d"]), 2), np.int64)
        d[:, 0] = cols["d"]
        d[:, 1] = cols["d"] >> 63
        add(P.DECIMAL(38, 2), d, 16)
        del d
        add(P.INT64, cols["row"], 8)
    return t, keep


def types_of(P, shape):
    return [P.INT64, P.INT64, P.INT32] if shape == "one_key" else [P.INT32, P.STRING, P.DECIMAL(38, 2), P.INT64]


def bounds_of(np, cols, shape, n_parts, seed):
    """num_partitions - 1 quantiles of a sorted sample of the keys, as (order keys, literal rows)"""
    rng = np.random.default_rng(seed)
    n = len(next(iter(cols.values())))
    sample = np.sort(rng.choice(n, min(n, 100 * n_parts), replace=False))
    ok = order_key(np, {k: v[sample] for k, v in cols.items()}, shape)
    srt = np.argsort(ok, kind="stable")
    pick = sample[srt[(np.arange(1, n_parts) * len(sample)) // n_parts]]
    return order_key(np, {k: v[pick] for k, v in cols.items()}, shape), pick


def plan(P, shape, how, n_parts, cols, pick):
    types = types_of(P, shape)
    if how == "hash":
        keys = [P.bound(0, types[0])] if shape == "one_key" else [P.bound(i, types[i]) for i in range(3)]
        part = P.hash_partitioning(keys, n_parts)
    elif how == "round_robin":
        part = P.round_robin_partitioning(n_parts, 0)
    else:
        if shape == "one_key":
            orders = [P.sort_order(P.bound(0, P.INT64))]
            rows = [[P.literal(int(cols["k"][i]), P.INT64)] for i in pick]
        else:
            orders = [P.sort_order(P.bound(i, types[i])) for i in range(3)]
            rows = [[P.literal(int(cols["a"][i]), P.INT32), P.literal(f"s{int(cols['s'][i]):04d}", P.STRING),
                     P.literal(int(cols["d"][i]), P.DECIMAL(38, 2))] for i in pick]
        part = P.range_partitioning(orders, n_parts, rows)
    return P.shuffle_writer(P.scan(types), part)


def expected_pids(np, cols, shape, how, n_parts, bound_keys, hashes):
    if how == "range":
        return np.searchsorted(bound_keys, order_key(np, cols, shape), side="right")
    h = hashes[how].astype(np.uint32).view(np.int32).astype(np.int64)
    return np.mod(h, n_parts)


def cudart():
    """the CUDA runtime this process already loaded (for cudaMemcpy of the plan's device output)"""
    import ctypes as C
    with open("/proc/self/maps") as f:
        paths = sorted({line.split()[-1] for line in f if "libcudart.so" in line})
    lib = C.CDLL(paths[0] if paths else "libcudart.so")
    lib.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    return lib


def to_host(np, rt, col, n, dtype, per_row=1):
    out = np.empty(n * per_row, dtype)
    assert rt.cudaMemcpy(out.ctypes.data, col.values, out.nbytes, 2) == 0   # cudaMemcpyDeviceToHost
    return out


def check_output(np, rt, out_cols, cols, shape, pids, starts):
    """the plan's output batch against the input: partition of every row, stable order, key values carried with their rows"""
    n = len(pids)
    ri = 1 if shape == "one_key" else 3
    rows = to_host(np, rt, out_cols[ri], n, np.int64)
    assert ((rows >= 0) & (rows < n)).all()
    part = np.repeat(np.arange(len(starts) - 1), np.diff(starts))
    assert (pids[rows] == part).all(), "a row in another partition than its id"
    inside = np.diff(rows) > 0
    assert (inside | (np.diff(part) > 0)).all(), "row order inside a partition is not the input order"
    if shape == "one_key":
        assert (to_host(np, rt, out_cols[0], n, np.int64) == cols["k"][rows]).all()
    else:
        assert (to_host(np, rt, out_cols[0], n, np.int32) == cols["a"][rows]).all()
        d = to_host(np, rt, out_cols[2], n, np.int64, 2).reshape(n, 2)
        assert (d[:, 0] == cols["d"][rows]).all() and (d[:, 1] == cols["d"][rows] >> 63).all()


def murmur(np, o, cols, names):
    """Spark's murmur3 (seed 42) of each row chained over the columns `names`, by the oracle"""
    import ctypes as C
    h = np.full(len(next(iter(cols.values()))), 42, dtype=np.uint32)
    for c in names:
        v = cols[c]
        if c == "s":   # the dictionary strings spelled out: 5 bytes each
            table = np.frombuffer(b"".join(f"s{i:04d}".encode() for i in range(N_WORDS)), np.uint8).reshape(N_WORDS, 5)
            chars = np.ascontiguousarray(table[v]).reshape(-1)
            offs = (np.arange(len(v) + 1, dtype=np.int64) * 5).astype(np.int32)
            valid = np.ones(len(v), np.uint8)
            p = lambda a: a.ctypes.data_as(C.c_void_p)
            o.lib().co_murmur3_strings(C.c_int64(len(v)), p(offs), p(chars), p(valid), p(h))
            del chars, offs
        elif c == "d":
            w = np.zeros((len(v), 2), np.uint64)
            w[:, 0] = v.view(np.uint64)
            w[:, 1] = (v >> 63).view(np.uint64)
            h = o.murmur3_column("dec_large", w, hashes=h)
        else:
            h = o.murmur3_column("i64" if v.dtype == np.int64 else "i32", v, hashes=h)
    return h


STAGES = ("partition_ids_ms", "partition_place_ms", "partition_gather_ms")


def step(native, p, t, n, check=None):
    """one run of the plan: (output rows, starts, stage ms); check(columns, starts) sees the device output while it is alive"""
    with native.Plan(p, [t], config={"spark.comet.b200.chunkRows": str(n)}) as pl:
        rows, out_cols = pl.execute_device()
        starts = pl.partition_starts()
        if check:
            check(out_cols, starts)
        st = pl.stats()
        return rows, starts, [st[k] for k in STAGES]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 28)
    ap.add_argument("--parts", default="8,200,16384")
    ap.add_argument("--shapes", default="one_key,three_keys")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_range_partition.py measures the GPU: no CUDA device")
    import comet_b200  # noqa: F401
    from comet_b200 import native, proto as P
    from oracle import oracle as o
    rt = cudart()
    n = args.rows
    for shape in args.shapes.split(","):
        t0 = time.perf_counter()
        cols = generate(np, n, shape, args.seed)
        t, keep = device_table(native, P, torch, np, cols, shape)
        key_names = ["k"] if shape == "one_key" else ["a", "s", "d"]
        all_names = ["k", "row", "p2"] if shape == "one_key" else ["a", "s", "d", "row"]
        hashes = {"hash": murmur(np, o, cols, key_names), "round_robin": murmur(np, o, cols, all_names)}
        gen_s = time.perf_counter() - t0
        key_bytes = n * (8 if shape == "one_key" else 4 + 4 + 16)
        for n_parts in (int(x) for x in args.parts.split(",")):
            bound_keys, pick = bounds_of(np, cols, shape, n_parts, args.seed + n_parts)
            for how in ("range", "round_robin", "hash"):
                p = plan(P, shape, how, n_parts, cols, pick)
                pids = expected_pids(np, cols, shape, how, n_parts, bound_keys, hashes)
                want = [0] + np.cumsum(np.bincount(pids, minlength=n_parts)).tolist()
                walls, stages = [], []
                for _ in range(args.warmup + args.steps):
                    torch.cuda.synchronize()
                    t1 = time.perf_counter()
                    rows, starts, st = step(native, p, t, n)
                    walls.append((time.perf_counter() - t1) * 1e3)
                    stages.append(st)
                    assert rows == n and starts == want, (shape, how, n_parts)
                step(native, p, t, n, check=lambda out, starts: check_output(np, rt, out, cols, shape, pids, starts))
                walls = sorted(walls[args.warmup:])
                med = lambda xs: sorted(xs)[len(xs) // 2]
                stage_ms = {k[len("partition_"):-len("_ms")]: round(med([s_[j] for s_ in stages[args.warmup:]]), 3) for j, k in enumerate(STAGES)}
                read = key_bytes if how != "round_robin" else n * (20 if shape == "one_key" else 32)
                print(json.dumps(dict(bench="range_partition", input=shape, rows=n, partitions=n_parts, partitioning=how,
                                      step_ms_median=round(walls[len(walls) // 2], 2), step_ms_min=round(walls[0], 2), stage_ms=stage_ms,
                                      pid_kernel_gbps_over_key_bytes=round(read / (stage_ms["ids"] * 1e6), 1),
                                      checked_steps=args.warmup + args.steps + 1,
                                      check="numpy partition starts every step; whole output (ids, stable order, key values) once",
                                      data_gen_s=round(gen_s, 1), card=card())), flush=True)
        del t, keep
        torch.cuda.empty_cache()
        native.lib().cb200_release_cached_memory(0)


if __name__ == "__main__":
    main()
