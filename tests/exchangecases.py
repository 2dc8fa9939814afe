"""Cases of the device exchange (cb200_exchange), shared by tests/test_gpu_exchange.py (one GPU, and one spawned process per GPU
for the multi-rank part) and tests/test_exchange_cpu.py (every plan compiles).

Two shapes of map plan:
  raw rows  ShuffleWriter(HashPartitioning(key, N)) over a Scan of every fixed-width column type: the received table must be the
            reference partitioning (tests/partref.py) bit for bit, in order.
  Config 4  HashAggregate(Partial) -> ShuffleWriter(HashPartitioning(keys, N)) -> exchange -> HashAggregate(Final): the results
            must equal tests/aggref.py's aggregate over all inputs, and every key must land on rank pmod(murmur3(keys, 42), N).

Every input is rebuilt from (seed, rank), so a worker of the multi-rank run can compute every rank's input and check its own result."""
import numpy as np
import pyarrow as pa

from comet_b200 import proto as P

import aggcases
import aggref as R
import exprs as E
import partref
from test_gpu_partition_layouts import make_values, parquet_table

# ---- raw rows ----------------------------------------------------------------------------------------------------------------------
RAW = ["b", "i8", "i16", "i32", "date", "i64", "ts", "f32", "f64", "d9", "d18", "d38", "row"]   # every fixed-width type, BOOL included
RAW_KEYS = ["i32", "d38", "b"]
PARQUET = ["i8", "i16", "i32", "i32w", "date", "d7", "i64", "ts", "d12", "d28", "f32", "f64", "row"]
WIDTH = {"BOOL": 1, "INT8": 1, "INT16": 2, "INT32": 4, "DATE": 4, "FLOAT": 4, "INT64": 8, "TIMESTAMP": 8, "DOUBLE": 8, "DECIMAL": 16}


def row_bytes(types):
    """bytes one row costs in an exchange: every column's values (Arrow width, BOOL one byte) plus one validity byte"""
    return sum(WIDTH[t.name] + 1 for t in types)


def with_nulls(arr, nulls):
    """arr with its own NULLs ("some"), none at all (no validity buffer), or every slot NULL"""
    arr = arr.combine_chunks() if isinstance(arr, pa.ChunkedArray) else arr
    if nulls == "some":
        return arr
    n = len(arr)
    if nulls == "none":
        bitmap = None
    else:
        bitmap = pa.py_buffer(np.zeros((n + arr.offset + 7) // 8 + 1, np.uint8).tobytes())
    return pa.Array.from_buffers(arr.type, n, [bitmap] + arr.buffers()[1:], null_count=0 if nulls == "none" else n, offset=arr.offset)


def raw_table(n, seed, nulls="some", names=RAW):
    """(table, proto types) of the raw-row columns"""
    cols = make_values(n, seed)
    tbl = pa.table({k: with_nulls(cols[k][0], nulls if k != "row" else "none") for k in names})
    return tbl, [cols[k][1] for k in names]


def parquet_cols(n, seed, nulls="some"):
    """columns for a Parquet file NativeScan reads: name -> (arrow array, requested type), expected table as the scan returns it"""
    cols = parquet_table(n, seed)
    cols = {k: (with_nulls(cols[k][0], nulls if k != "row" else "none"), cols[k][1]) for k in PARQUET}
    want = pa.table({k: (cols[k][0].cast(pa.int64()) if k == "i32w" else cols[k][0]) for k in PARQUET})
    return cols, want


def raw_map_plan(types, names, keys, world, child=None):
    return P.shuffle_writer(child if child is not None else P.scan(types),
                            P.hash_partitioning([P.bound(names.index(k), types[names.index(k)]) for k in keys], world))


def expected_partitions(o, tbl, keys, world):
    """partref's partitioning of one rank's input: [table of partition p for p in range(world)]"""
    starts, _, out = partref.partition(o, tbl, keys, world)
    return [out.slice(starts[p], starts[p + 1] - starts[p]) for p in range(world)]


# ---- Config 4: Partial -> ShuffleWriter -> exchange -> Final ------------------------------------------------------------------------
D22_2, D16_6, D28_0, D22_4 = P.DECIMAL(22, 2), P.DECIMAL(16, 6), P.DECIMAL(28, 0), P.DECIMAL(22, 4)


def e2e_aggs(nk, aggset="dec"):
    """"dec": SUM / AVG(decimal) (BOOL is_empty, DECIMAL(22 / 28) states), SUM(int) in TRY; "f64": SUM / AVG(f64), MIN / MAX,
    COUNT.  Two sets: the Final's per-thread accumulators hold only so many aggregates of a grouped merge."""
    c = lambda i: E.Col(nk + i, aggcases.VALUE_TYPES[i])
    v0, v1, v2, v5, v7 = c(0), c(1), c(2), c(5), c(7)
    A = R.Agg
    if aggset == "dec":
        return [A("sum", v2, D22_2), A("avg", v2, D16_6, sum_dt=D22_2), A("sum", v7, D28_0), A("avg", v7, D22_4, sum_dt=D28_0),
                A("sum", v5, P.INT64, mode=R.TRY)]
    return [A("sum", v1, P.DOUBLE), A("avg", v1, P.DOUBLE), A("min", v1, P.DOUBLE), A("max", v0, P.INT64), A("min", v2, aggcases.D12),
            A("count", v0)]


class E2E(aggcases.Case):
    """One Config-4 case: the aggregate matrix's input generator (tests/aggcases.py) with the exchange's aggregate set.  `nulls`
    "none" removes every NULL (validity buffers dropped) so a dense Partial flushes its state without validity."""

    def __init__(self, name, keys, n=2000, seed=0, nulls="some", aggset="dec", **kw):
        super().__init__(name, "exchange", keys, aggset, n=n, seed=seed, nullable=nulls == "some", **kw)
        self.nulls = nulls

    @property
    def aggs(self):
        return e2e_aggs(len(self.key_specs), self.aggset)

    def config(self):
        return dict(aggcases.TABLE_CFG)

    def table(self):
        t = super().table()
        if self.nulls == "none":
            t = pa.table([with_nulls(c, "none") for c in t.columns], names=t.column_names)
        return t

    def map_plan(self, world, filtered=False):
        agg = R.partial_plan(self.dts, self.key_cols, self.aggs)
        if filtered:   # a predicate no row passes: key IS NULL AND key IS NOT NULL
            k = P.bound(0, self.dts[0])
            scan = P.filter_(P.scan(self.dts), P.and_(P.is_null(k), P.is_not_null(k)))
            agg = P.hash_agg(scan, [P.bound(k, self.dts[k]) for k in self.key_cols], [a.proto() for a in self.aggs], R.PARTIAL)
        return P.shuffle_writer(agg, P.hash_partitioning([P.bound(k, t) for k, t in enumerate(self.key_types)], world))

    def state_types(self):
        return R.state_schema(self.key_types, self.aggs)

    def final_plan(self):
        return R.merge_plan(self.key_types, self.aggs, R.FINAL)


I64, I32, I8, DATE, BOOL = P.INT64, P.INT32, P.INT8, P.DATE, P.BOOL
# group keys of the Config-4 cases.  DECIMAL(p > 18) keys are refused by the aggregate's key table (csrc/agg.cpp); the raw-row cases
# partition on one.
E2E_KEYS = {"i64": [I64], "i32": [I32], "date": [DATE], "i8": [I8], "dec18": [aggcases.D18K], "bool-dense": [BOOL], "i64-i32": [I64, I32]}


def e2e_case(key, seed, n=2000, nulls="some", aggset="dec"):
    return E2E(f"e2e-{key}-{aggset}", E2E_KEYS[key], n=n, seed=seed, nulls=nulls, aggset=aggset)


def owner(o, keys_table, world):
    """rank each row of a table of key columns belongs to: pmod(murmur3(keys, 42), world)"""
    h = partref.key_hashes(o, keys_table, list(range(keys_table.num_columns)))
    return np.array([o.pmod(int(x), world) for x in h], dtype=np.int64)


def all_map_plans(world=2):
    """every map / Final / reader plan of the matrix, for the compile check"""
    plans = []
    tbl, types = raw_table(8, 1)
    plans.append(raw_map_plan(types, RAW, RAW_KEYS, world))
    plans.append(P.scan(types))
    ptypes = [parquet_table(8, 1)[k][1] for k in PARQUET]
    plans.append(P.scan(ptypes))
    for key in E2E_KEYS:
        for aggset in ("dec", "f64"):
            c = e2e_case(key, 1, n=8, aggset=aggset)
            plans += [c.map_plan(world), c.map_plan(world, filtered=True), c.final_plan(), P.scan(c.state_types())]
    return plans
