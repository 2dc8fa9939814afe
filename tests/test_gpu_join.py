"""GPU: the HashJoin operator (inner, left semi and left anti equi-joins) against the CPU reference (tests/joinref.py).  Every output
column is compared bit-exact and in order -- values, float bits, validity, strings spelled out.  Inputs cover every key type in the
layouts a source hands the operator: Arrow streams (booleans as bitmaps, dictionaries with int8 / int16 / int32 indices, growing or
replaced between batches), device tables (8-byte decimals, dictionaries that repeat a value), the Parquet scan, a filter / projection
pipeline below and above the join, and a Final hash aggregate's host-resident result."""
import numpy as np
import pyarrow as pa
import pytest

import joinref as R
import partref
from test_gpu_partition_layouts import WORDS, _dec, _words, device_table, expected_table, parquet_table, scan_of, supports, write_parquet

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


KEYS = ["b", "i8", "i16", "i32", "date", "i64", "ts", "d9", "d18", "d38", "s8", "s16", "s32"]


def key_array(name, ids, mask):
    """a key column of type `name` whose value is a function of the key id (equal ids, equal values; different ids, different values
    except for booleans and int8, which wrap)"""
    import comet_b200.proto as P
    ids = np.asarray(ids, np.int64)
    if name == "b":
        return pa.array(ids % 2 == 1, mask=mask), P.BOOL
    if name == "i8":
        return pa.array((ids % 256 - 128).astype(np.int8), mask=mask), P.INT8
    if name == "i16":
        return pa.array((ids * 37 - 20000).astype(np.int16), mask=mask), P.INT16
    if name == "i32":
        return pa.array(((ids * 2654435761) % (1 << 32) - (1 << 31)).astype(np.int32), mask=mask), P.INT32
    if name == "date":
        return pa.array((ids - 500).astype(np.int32), pa.date32(), mask=mask), P.DATE
    if name == "i64":
        return pa.array(ids * 10**15 - 2**62, mask=mask), P.INT64
    if name == "ts":
        return pa.array(ids * 10**9 - 10**11, pa.timestamp("us", tz="UTC"), mask=mask), P.TIMESTAMP
    if name == "d9":
        return _dec(ids * 12345 - 5 * 10**6, 9, 2, mask), P.DECIMAL(9, 2)
    if name == "d18":
        return _dec(ids * 10**14 - 5 * 10**16, 18, 0, mask), P.DECIMAL(18, 0)
    if name == "d38":
        return _dec(_words([(int(i) - 500) * 10**33 + int(i) for i in ids]), 38, 4, mask), P.DECIMAL(38, 4)
    width = {"s8": pa.int8(), "s16": pa.int16(), "s32": pa.int32()}[name]
    return pa.DictionaryArray.from_arrays(pa.array(ids % len(WORDS), width, mask=mask), pa.array(WORDS)), P.STRING


def side(n, keys, seed, domain, null_frac=0.08, spread=0.2):
    """a table of key columns k0.. (ids shared by a row's keys except for a `spread` fraction of them, so tuples can be equal in one key
    only) and payloads: row (the row number), pf (float64 with NULLs), ps (a dictionary string with NULLs)"""
    import comet_b200.proto as P
    rng = np.random.default_rng(seed)
    base = rng.integers(0, domain, n)
    cols, types = {}, []
    for k, name in enumerate(keys):
        ids = np.where(rng.random(n) < spread, rng.integers(0, domain, n), base)
        a, t = key_array(name, ids, rng.random(n) < null_frac)
        cols[f"k{k}"] = a
        types.append(t)
    cols["row"] = pa.array(np.arange(n, dtype=np.int64))
    cols["pf"] = pa.array(rng.standard_normal(n), mask=rng.random(n) < 0.1)
    cols["ps"] = pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, len(WORDS), n), pa.int16(), mask=rng.random(n) < 0.1), pa.array(WORDS))
    types += [P.INT64, P.DOUBLE, P.STRING]
    return pa.table(cols), types


JT = {"inner": 0, "left_semi": 4, "left_anti": 5}


def join_plan(cb, lchild, ltypes, rchild, rtypes, lk, rk, jt, build_left=False):
    P = cb.proto
    return P.hash_join(lchild, rchild, [P.bound(i, ltypes[i]) for i in lk], [P.bound(i, rtypes[i]) for i in rk], JT[jt],
                       P.BUILD_LEFT if build_left else P.BUILD_RIGHT)


def collect(cb, plan, inputs, config=None, batch_size=8192):
    with cb.native.Plan(plan, inputs, config=config, batch_size=batch_size) as p:
        got = p.collect()
        return got, p.stats()


def check(got, want):
    if want.num_rows == 0:
        assert got is None or got.num_rows == 0
        return
    assert got is not None
    partref.assert_tables_equal(got, want)


def case(cb, left, ltypes, right, rtypes, lk, rk, jt, build_left=False, lchunk=5000, rchunk=3000, config=None, linputs=None, rinputs=None):
    P = cb.proto
    plan = join_plan(cb, P.scan(ltypes), ltypes, P.scan(rtypes), rtypes, lk, rk, jt, build_left)
    li = linputs if linputs is not None else ([left.to_batches(max_chunksize=lchunk)] if left.num_rows else [left])
    ri = rinputs if rinputs is not None else ([right.to_batches(max_chunksize=rchunk)] if right.num_rows else [right])
    got, stats = collect(cb, plan, li + ri, config)
    want = R.join_table(left, right, lk, rk, jt, build_left)
    check(got, want)
    return got, want, stats


MODES = [("inner", False), ("inner", True), ("left_semi", False), ("left_anti", False)]


# ---- join types, build sides, key types ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("jt,build_left", MODES)
@pytest.mark.parametrize("key", KEYS)
def test_each_key_type(cb, key, jt, build_left):
    """one key of each type, NULLs on both sides, N:M duplicates (booleans: two values, so small sides)"""
    n_l, n_r, dom = (300, 200, 2) if key == "b" else (4000, 3000, 3000) if key in ("i8", "s8", "s16", "s32") else (12_000, 7_000, 3000)
    left, lt = side(n_l, [key], KEYS.index(key) + 1, dom)
    right, rt = side(n_r, [key], KEYS.index(key) + 101, dom)
    case(cb, left, lt, right, rt, [0], [0], jt, build_left)


def test_build_left_matches_build_right(cb):
    """the same inner join with either build side: the same rows (probe order differs), each side in its contract's order"""
    left, lt = side(9000, ["i32", "s16"], 3, 500)
    right, rt = side(6000, ["i32", "s16"], 4, 500)
    a, _, _ = case(cb, left, lt, right, rt, [0, 1], [0, 1], "inner", False)
    b, _, _ = case(cb, left, lt, right, rt, [0, 1], [0, 1], "inner", True)
    by_rows = [(a.column_names[2], "ascending"), (a.column_names[5 + 2], "ascending")]   # (left row, right row) is unique
    partref.assert_tables_equal(a.sort_by(by_rows), b.sort_by(by_rows))


@pytest.mark.parametrize("keys", ["i8+i16", "b+s8+date", "d9+d38+date", "s16+i32+date+b+d18", "b+i8+i16+date+s8+s16+i32+d9",
                                  "d38+i64+s32+i16+b"])
@pytest.mark.parametrize("jt,build_left", [("inner", False), ("left_anti", False)])
def test_key_combinations(cb, keys, jt, build_left):
    """up to 8 keys and up to 246 bits of packed key; about a third of each row's keys take another id, so tuples are often equal in some
    keys only"""
    names = keys.split("+")
    left, lt = side(6000, names, len(names), 200, spread=0.3)
    right, rt = side(4000, names, len(names) + 50, 200, spread=0.3)
    ks = list(range(len(names)))
    case(cb, left, lt, right, rt, ks, ks, jt, build_left)


@pytest.mark.parametrize("shape", ["1:1", "1:N", "N:1", "N:M"])
@pytest.mark.parametrize("jt,build_left", MODES)
def test_multiplicities(cb, shape, jt, build_left):
    """unique keys on one side or both, many duplicates on either; some keys absent from the other side"""
    P = cb.proto
    rng = np.random.default_rng(len(shape))
    def tbl(n, unique, seed):
        r = np.random.default_rng(seed)
        k = r.permutation(int(n * 1.3))[:n] if unique else r.integers(0, n // 20, n)
        return pa.table({"k": pa.array(k, pa.int64(), mask=r.random(n) < 0.05), "row": pa.array(np.arange(n, dtype=np.int64))})
    lu, ru = {"1:1": (True, True), "1:N": (True, False), "N:1": (False, True), "N:M": (False, False)}[shape]
    left, right = tbl(20_000, lu, int(rng.integers(100))), tbl(12_000, ru, 7)
    types = [P.INT64, P.INT64]
    case(cb, left, types, right, types, [0], [0], jt, build_left)


# ---- sizes ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_l,n_r", [(0, 500), (500, 0), (0, 0), (1, 500), (500, 1), (1, 1)])
@pytest.mark.parametrize("jt,build_left", MODES)
def test_empty_and_one_row(cb, n_l, n_r, jt, build_left):
    """an empty build side: inner and semi give no rows, anti every probe row; an empty probe side gives nothing"""
    left, lt = side(n_l, ["i32", "s8"], n_l + 5, 3)
    right, rt = side(n_r, ["i32", "s8"], n_r + 9, 3, spread=0.0)
    case(cb, left, lt, right, rt, [0, 1], [0, 1], jt, build_left)


@pytest.mark.parametrize("jt,build_left", MODES)
def test_batches_and_chunks(cb, jt, build_left):
    """a build side of many batches (concatenated), a probe side over several chunks, and inner-join output of a probe chunk far above
    chunkRows, which leaves in batches of at most chunkRows rows"""
    left, lt = side(20_000, ["i64", "s32"], 1, 400, spread=0.0)
    right, rt = side(8_000, ["i64", "s32"], 2, 400, spread=0.0)
    P = cb.proto
    cfg = {"spark.comet.b200.chunkRows": "16384"}
    plan = join_plan(cb, P.scan(lt), lt, P.scan(rt), rt, [0, 1], [0, 1], jt, build_left)
    sizes = []
    with cb.native.Plan(plan, [left.to_batches(max_chunksize=7000), right.to_batches(max_chunksize=3000)], config=cfg, batch_size=1 << 22) as p:
        batches = []
        while True:
            b = p.execute()
            if b is None:
                break
            batches.append(b)
            sizes.append(b.num_rows)
        stats = p.stats()
    got = pa.Table.from_batches(batches)
    want = R.join_table(left, right, [0, 1], [0, 1], jt, build_left)
    partref.assert_tables_equal(got, want)
    assert max(sizes) <= 16384
    build_n, probe_n = (20_000, 8_000) if build_left else (8_000, 20_000)
    assert stats["join_build_rows"] == build_n and stats["join_probe_rows"] == probe_n and stats["join_out_rows"] == want.num_rows
    if jt == "inner":
        assert want.num_rows > 10 * 16384 and len(sizes) > 10


# ---- strings -------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("index", [pa.int8(), pa.int16(), pa.int32()])
@pytest.mark.parametrize("mode", ["same", "growing", "replaced"])
@pytest.mark.parametrize("jt,build_left", MODES)
def test_string_dictionaries(cb, index, mode, jt, build_left):
    """the two sides carry different dictionaries; each probe batch carries the same one, one that grows, or a shuffled one that
    also holds strings the build side lacks"""
    P = cb.proto
    extra = [f"only-probe-{i}" for i in range(20)]
    def batches(k, per, words_of, seed):
        r = np.random.default_rng(seed)
        out, plain = [], []
        for b in range(k):
            words = words_of(b)
            d = pa.array(words)
            s = pa.DictionaryArray.from_arrays(pa.array(r.integers(0, len(words), per), index, mask=r.random(per) < 0.1), d)
            v = pa.array(np.arange(b * per, (b + 1) * per, dtype=np.int64))
            out.append(pa.record_batch([s, v], names=["s", "v"]))
            plain.append(pa.record_batch([s.dictionary_decode(), v], names=["s", "v"]))
        return out, pa.Table.from_batches(plain)
    build_words = lambda b: list(reversed(WORDS[:60]))
    if mode == "same":
        probe_words = lambda b: WORDS[:100]
    elif mode == "growing":
        probe_words = lambda b: WORDS[:20 + 9 * b] + extra[:b]
    else:
        probe_words = lambda b: [w for i, w in enumerate((WORDS[:100] + extra)[::-1]) if (i + b) % 3]
    pb, ptbl = batches(8, 2500, probe_words, 1)
    bb, btbl = batches(4, 1500, build_words, 2)
    types = [P.STRING, P.INT64]
    left, right, li, ri = (btbl, ptbl, bb, pb) if build_left else (ptbl, btbl, pb, bb)
    case(cb, left, types, right, types, [0], [0], jt, build_left, linputs=[li], rinputs=[ri], config={"spark.comet.b200.chunkRows": "6000"})


@pytest.mark.parametrize("jt,build_left", MODES)
def test_repeated_dictionary_values(cb, jt, build_left):
    """caller dictionaries (device tables) that hold a value more than once: each code keeps its own entry, equal strings still match"""
    P = cb.proto
    import torch
    dict_b = ["x", "y", "x", "z", "y", "", ""]
    dict_p = ["y", "y", "q", "x", "", "z", "x"]
    def table(n, d, seed):
        r = np.random.default_rng(seed)
        codes = r.integers(0, len(d), n).astype(np.int32)
        mask = r.random(n) < 0.1
        tbl = pa.table({"s": pa.DictionaryArray.from_arrays(pa.array(codes, mask=mask), pa.array(d)), "v": pa.array(np.arange(n, dtype=np.int64))})
        t = cb.native.DeviceTable(n)
        vbits = torch.from_numpy(np.concatenate([np.packbits(~mask, bitorder="little"), np.zeros(16, np.uint8)])).cuda()
        cdev = torch.from_numpy(np.concatenate([codes.view(np.uint8), np.zeros(16, np.uint8)])).cuda()
        vdev = torch.from_numpy(np.concatenate([np.arange(n, dtype=np.int64).view(np.uint8), np.zeros(16, np.uint8)])).cuda()
        t.add(P.STRING, cdev.data_ptr(), 4, vbits.data_ptr(), int(mask.sum()), dictionary=d, keep=(cdev, vbits))
        t.add(P.INT64, vdev.data_ptr(), 8, keep=vdev)
        return tbl, t
    btbl, bt = table(3000, dict_b, 1)
    ptbl, pt = table(5000, dict_p, 2)
    types = [P.STRING, P.INT64]
    left, right, li, ri = (btbl, ptbl, bt, pt) if build_left else (ptbl, btbl, pt, bt)
    case(cb, left, types, right, types, [0], [0], jt, build_left, linputs=[li], rinputs=[ri], config={"spark.comet.b200.chunkRows": "2048"})


def test_plain_utf8_refused(cb):
    P = cb.proto
    tbl = pa.table({"s": pa.array(["b", "a", None]), "v": pa.array([1, 2, 3])})
    types = [P.STRING, P.INT64]
    plan = join_plan(cb, P.scan(types), types, P.scan(types), types, [0], [0], "inner")
    assert supports(cb, plan)[0]   # a plan-time answer: the column's encoding is known only when a batch arrives
    with pytest.raises(cb.native.Unsupported, match="plain string columns"):
        collect(cb, plan, [tbl, tbl])


# ---- sources ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keys", ["b", "i8", "d9", "d18", "d38", "s8+i32", "d9+d18+s32+date"])
def test_device_tables(cb, keys):
    """device columns, decimal(9, 2) and decimal(18, 0) 8 bytes wide on the build side and 16 on the probe side; chunkRows below the
    tables: the build side's slices are concatenated"""
    names = keys.split("+")
    n_l, n_r, dom = (400, 300, 2) if keys == "b" else (20_000, 12_000, 2000)
    left, lt = side(n_l, names, 5, dom)
    right, rt = side(n_r, names, 6, dom)
    ks = list(range(len(names)))
    dl = device_table(cb, left, lt)
    dr = device_table(cb, right, rt, dec8=[f"k{i}" for i, k in enumerate(names) if k in ("d9", "d18")])
    case(cb, left, lt, right, rt, ks, ks, "inner", linputs=[dl], rinputs=[dr], config={"spark.comet.b200.chunkRows": "5120"})


@pytest.mark.parametrize("as_int", [True, False])
@pytest.mark.parametrize("keys", ["i8", "i16", "d7", "d12", "d28", "i32w+date", "sd", "sp+d7+i8"])
def test_native_scan(cb, tmp_path, as_int, keys):
    """both sides NativeScans of Parquet files: INT32-backed int8 / int16 / decimal(7, 2), INT64 or FLBA decimals, dictionary and PLAIN
    string pages; the probe file is the build file's rows shuffled, plus rows of another file"""
    n = 6000
    a, b = parquet_table(n, 31), parquet_table(n, 32)
    perm = np.random.default_rng(1).permutation(n)
    names = ["i8", "i16", "i32w", "date", "d7", "d12", "d28", "sd", "sp", "row"]
    mix = {k: (pa.concat_arrays([a[k][0].take(pa.array(perm[: n // 2])), b[k][0].slice(0, n // 2)]), a[k][1]) for k in names}
    pa_path, pb_path = str(tmp_path / "a.parquet"), str(tmp_path / "b.parquet")
    write_parquet(pa_path, {k: a[k] for k in names}, as_int)
    write_parquet(pb_path, mix, as_int)
    scan_l, types = scan_of(cb, mix, names, pb_path)
    scan_r, _ = scan_of(cb, a, names, pa_path)
    ks = [names.index(k) for k in keys.split("+")]
    for jt in ("inner", "left_anti"):
        plan = join_plan(cb, scan_l, types, scan_r, types, ks, ks, jt)
        got, _ = collect(cb, plan, [], config={"spark.comet.b200.chunkRows": "2500"})
        check(got, R.join_table(expected_table(mix, names), expected_table(a, names), ks, ks, jt))


def test_pipelines_below_and_above(cb):
    """Filter + Projection below each side (their kernels feed the join) and a Filter + Projection above it (fed by the join)"""
    P = cb.proto
    left, lt = side(30_000, ["i32", "s16"], 21, 800)
    right, rt = side(20_000, ["s16", "i32"], 22, 800)
    # left: WHERE pf > -0.5, project (row, k1, k0); right: WHERE row % ... (row >= 1000), project (k0, pf, k1, row)
    lsel = P.projection(P.filter_(P.scan(lt), P.gt(P.bound(3, P.DOUBLE), P.literal(-0.5, P.DOUBLE))),
                        [P.bound(2, P.INT64), P.bound(1, P.STRING), P.bound(0, P.INT32)])
    rsel = P.projection(P.filter_(P.scan(rt), P.gt_eq(P.bound(2, P.INT64), P.literal(1000, P.INT64))),
                        [P.bound(0, P.STRING), P.bound(3, P.DOUBLE), P.bound(1, P.INT32), P.bound(2, P.INT64)])
    ltypes, rtypes = [P.INT64, P.STRING, P.INT32], [P.STRING, P.DOUBLE, P.INT32, P.INT64]
    j = join_plan(cb, lsel, ltypes, rsel, rtypes, [2, 1], [2, 0], "inner")
    plan = P.projection(P.filter_(j, P.is_not_null(P.bound(4, P.DOUBLE))), [P.bound(0, P.INT64), P.bound(6, P.INT64), P.bound(1, P.STRING)])
    got, _ = collect(cb, plan, [left.to_batches(max_chunksize=8192), right.to_batches(max_chunksize=8192)],
                     config={"spark.comet.b200.chunkRows": "16384"})
    pf = left.column("pf").combine_chunks()
    lkept = left.filter(np.asarray(pf.fill_null(-1.0)) > -0.5).select(["row", "k1", "k0"])
    rkept = right.filter(np.asarray(right.column("row")) >= 1000).select(["k0", "pf", "k1", "row"])
    joined = R.join_table(lkept, rkept, [2, 1], [2, 0], "inner")
    want = joined.filter(np.asarray(joined.column(4).is_valid())).select([0, 6, 1])
    check(got, want)


def test_join_over_final_aggregate(cb):
    """the build side is a Final aggregate's host-resident result (TPC-H Q1's four groups), probed by a stream keyed on the same
    strings"""
    from comet_b200 import tpch
    P = cb.proto
    cols = tpch.gen_lineitem(100_000, seed=42)
    tbl = tpch.lineitem_table(cols, "dec", dictionary=True)
    with cb.native.Plan(tpch.q1_partial_plan("dec"), [tbl.to_batches(max_chunksize=8192)]) as p:
        state = p.collect()
    final = tpch.q1_final_plan("dec")
    groups, _ = collect(cb, final, [state])
    rng = np.random.default_rng(4)
    n = 20_000
    flags, status = ["A", "N", "R", "X"], ["F", "O"]
    probe = pa.table({"f": pa.array([flags[i] for i in rng.integers(0, 4, n)]).dictionary_encode(),
                      "s": pa.array([status[i] for i in rng.integers(0, 2, n)], mask=rng.random(n) < 0.05).dictionary_encode(),
                      "row": pa.array(np.arange(n, dtype=np.int64))})
    ptypes = [P.STRING, P.STRING, P.INT64]
    for jt in ("inner", "left_semi", "left_anti"):
        plan = P.hash_join(P.scan(ptypes), final, [P.bound(0, P.STRING), P.bound(1, P.STRING)], [P.bound(0, P.STRING), P.bound(1, P.STRING)],
                           JT[jt], P.BUILD_RIGHT)
        got, stats = collect(cb, plan, [probe.to_batches(max_chunksize=6000), state])
        check(got, R.join_table(probe, groups, [0, 1], [0, 1], jt))
        assert stats["join_build_rows"] == groups.num_rows


# ---- TPC-DS Q3 ------------------------------------------------------------------------------------------------------------------------------
def q3_tables(n_sales, seed):
    """store_sales (ss_sold_date_sk, ss_item_sk, ss_ext_sales_price), date_dim (d_date_sk, d_year, d_moy), item (i_item_sk, i_brand_id,
    i_brand, i_manufact_id); sales keys have NULLs and keys that match no dimension row"""
    rng = np.random.default_rng(seed)
    n_date, n_item = 73_049, 18_000
    d_sk = np.arange(2415022, 2415022 + n_date, dtype=np.int32)
    day = np.arange(n_date)
    date_dim = pa.table({"d_date_sk": pa.array(d_sk), "d_year": pa.array((1900 + day // 365).astype(np.int32)),
                         "d_moy": pa.array((1 + (day % 365) // 31).clip(1, 12).astype(np.int32))})
    brands = [f"brand#{i}" for i in range(500)]
    bid = rng.integers(0, 500, n_item)
    item = pa.table({"i_item_sk": pa.array(np.arange(1, n_item + 1, dtype=np.int32)), "i_brand_id": pa.array((bid + 1000000).astype(np.int32)),
                     "i_brand": pa.array([brands[i] for i in bid]).dictionary_encode(),
                     "i_manufact_id": pa.array(rng.integers(1, 1000, n_item).astype(np.int32))})
    sales = pa.table({"ss_sold_date_sk": pa.array(rng.integers(2415022 - 100, 2415022 + n_date, n_sales).astype(np.int32), mask=rng.random(n_sales) < 0.02),
                      "ss_item_sk": pa.array(rng.integers(1, n_item + 200, n_sales).astype(np.int32), mask=rng.random(n_sales) < 0.02),
                      "ss_ext_sales_price": _dec(rng.integers(0, 10**7, n_sales), 7, 2, rng.random(n_sales) < 0.01)})
    return date_dim, sales, item


def q3_plans(P, manufact=128, moy=11):
    """SELECT d_year, i_brand_id, i_brand, SUM(ss_ext_sales_price) FROM date_dim, store_sales, item WHERE d_date_sk = ss_sold_date_sk
    AND ss_item_sk = i_item_sk AND i_manufact_id = `manufact` AND d_moy = `moy` GROUP BY d_year, i_brand, i_brand_id, as Comet plans it:
    Scan -> Filter -> BroadcastHashJoin -> Project -> BroadcastHashJoin -> Project -> HashAggregate (Partial), then the Final aggregate"""
    I32, M, S = P.INT32, P.DECIMAL(7, 2), P.DECIMAL(17, 2)
    dd = P.projection(P.filter_(P.scan([I32, I32, I32]), P.eq(P.bound(2, I32), P.literal(moy, I32))), [P.bound(0, I32), P.bound(1, I32)])
    ss = P.scan([I32, I32, M])
    j1 = P.hash_join(dd, ss, [P.bound(0, I32)], [P.bound(0, I32)], P.INNER, P.BUILD_LEFT)        # (d_date_sk, d_year, sold_date, item, price)
    p1 = P.projection(j1, [P.bound(1, I32), P.bound(3, I32), P.bound(4, M)])                     # (d_year, ss_item_sk, price)
    it = P.projection(P.filter_(P.scan([I32, I32, P.STRING, I32]), P.eq(P.bound(3, I32), P.literal(manufact, I32))),
                      [P.bound(0, I32), P.bound(1, I32), P.bound(2, P.STRING)])
    j2 = P.hash_join(p1, it, [P.bound(1, I32)], [P.bound(0, I32)], P.INNER, P.BUILD_RIGHT)       # (d_year, item, price, i_item_sk, brand_id, brand)
    p2 = P.projection(j2, [P.bound(0, I32), P.bound(5, P.STRING), P.bound(4, I32), P.bound(2, M)])
    keys = [P.bound(0, I32), P.bound(1, P.STRING), P.bound(2, I32)]
    partial = P.hash_agg(p2, keys, [P.agg_sum(P.bound(3, M), S)], P.PARTIAL)
    final = P.hash_agg(P.scan([I32, P.STRING, I32, S, P.BOOL], source="shuffle"), keys, [P.agg_sum(P.unbound("p", M), S)], P.FINAL)
    return partial, final


def q3_answer(date_dim, sales, item, manufact=128, moy=11):
    """{(d_year, i_brand, i_brand_id): unscaled SUM} by numpy (NULL prices skipped; a group of only NULL prices sums to NULL)"""
    d = {int(k): int(y) for k, y, m in zip(*[date_dim.column(c).to_numpy() for c in ("d_date_sk", "d_year", "d_moy")]) if m == moy}
    it = item.to_pydict()
    im = {k: (b, bid) for k, b, bid, mf in zip(it["i_item_sk"], it["i_brand"], it["i_brand_id"], it["i_manufact_id"]) if mf == manufact}
    price = sales.column("ss_ext_sales_price").combine_chunks()
    raw = np.frombuffer(price.buffers()[1], np.int64)[::2][price.offset:price.offset + len(price)]
    pv = np.asarray(price.is_valid())
    out = {}
    for ds, isk, p, v in zip(sales.column("ss_sold_date_sk").to_pylist(), sales.column("ss_item_sk").to_pylist(), raw, pv):
        if ds is None or isk is None or ds not in d or isk not in im:
            continue
        k = (d[ds], im[isk][0], im[isk][1])
        cur = out.get(k)
        out[k] = (cur or 0) + int(p) if v else cur
    return out


def test_q3_shape(cb):
    """two inner joins (BuildLeft over the date dimension, BuildRight over the item dimension) -> Projection -> Partial -> Final
    aggregate, against a numpy answer"""
    P = cb.proto
    date_dim, sales, item = q3_tables(300_000, 5)
    for manufact in (128, 7):
        partial, final = q3_plans(P, manufact)
        with cb.native.Plan(partial, [date_dim.to_batches(max_chunksize=20_000), sales.to_batches(max_chunksize=65_536),
                                      item.to_batches(max_chunksize=8192)], config={"spark.comet.b200.chunkRows": "131072"}) as p:
            state = p.collect()
            stats = p.stats()
        assert stats["join_build_rows"] > 0 and stats["join_probe_rows"] >= sales.num_rows
        res, _ = collect(cb, final, [state])
        want = q3_answer(date_dim, sales, item, manufact)
        got = {}
        for r in res.to_pylist():
            v = r["col_3"]
            got[(r["col_0"], r["col_1"], r["col_2"])] = None if v is None else int(v.scaleb(2))
        assert got == want and len(want) > 10
