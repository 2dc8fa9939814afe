"""GPU: string predicates on dictionary-coded columns (comparisons, IN, LIKE, starts_with / ends_with / contains) through the C ABI, bit
for bit against the CPU reference of tests/strpred_ref.py: filters, boolean projections, CASE WHEN conditions and aggregate FILTER clauses
on the dense, key-table and stream aggregate strategies; Arrow dictionary streams (int8 / int16 / int32 indices, NULLs with garbage and
out-of-range codes under them, dictionaries that grow between launches); Parquet NativeScan (dictionary pages, PLAIN fallback pages,
page-index pruning); device tables; and a valid out-of-range code, which fails the plan instead of reading past the mask."""
import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import exprs as E
import strpred_ref as R
from test_string_predicates_cpu import HAND

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def words(rng, n):
    pool = HAND + ["MAIL", "SHIP", "AIR", "REG AIR", "DELIVER IN PERSON", "COLLECT COD", "NONE", "TAKE BACK RETURN", "PROMO BRUSHED",
                   "PROMO%", "ECONOMY ANODIZED", "x\ny", "ünïcödé", "日本語テキスト"]
    out = list(dict.fromkeys(pool))
    while len(out) < n:
        out.append("".join(rng.choice(list("abcdeMAILSHPé日😀 _%\\\n"), size=int(rng.integers(0, 9)))))
        out = list(dict.fromkeys(out))
    return out[:n]


ITYPES = {8: (pa.int8(), np.int8), 16: (pa.int16(), np.int16), 32: (pa.int32(), np.int32)}


def dict_array(rng, codes, valid, dictionary, bits=32):
    """a dictionary array whose NULL slots hold garbage codes, negative and far out of range"""
    pt, nt = ITYPES[bits]
    codes = np.asarray(codes, dtype=np.int64).copy()
    junk = rng.choice([-7, -1, np.iinfo(nt).max, len(dictionary), len(dictionary) + 1000 if bits > 8 else 120], size=len(codes))
    codes[~valid] = junk[~valid]
    vb = pa.py_buffer(np.packbits(valid, bitorder="little").tobytes())
    idx = pa.Array.from_buffers(pt, len(codes), [vb, pa.py_buffer(codes.astype(nt).tobytes())], null_count=int((~valid).sum()))
    return pa.DictionaryArray.from_arrays(idx, pa.array(dictionary, type=pa.string()), safe=False)


def predicates(c=R.StrCol(0)):
    return [R.StrCmp("eq", c, "MAIL"), R.StrCmp("lt", c, "MAIL", lit_left=True), R.StrCmp("gt_eq", c, "é"), R.StrCmp("neq", c, ""),
            R.StrCmp("lt_eq", c, "SHIP"), R.StrCmp("eq", c, None), R.StrIn(c, ["MAIL", "SHIP"]), R.StrIn(c, ["AIR", None], negated=True),
            R.StrIn(c, ["", "日本"], negated=True), R.Like(c, "%special%requests%"), R.Like(c, "_%_"), R.Like(c, "PROMO\\%"), R.Like(c, ""),
            R.Like(c, "%e%"), R.StrFunc("starts_with", c, "PROMO"), R.StrFunc("ends_with", c, "é"), R.StrFunc("contains", c, ""),
            R.StrFunc("contains", c, "\n")]


def groups(preds, k=6):
    """at most CB_MAX_STR_PREDS (8) distinct string predicates fit one pipeline"""
    return [preds[i:i + k] for i in range(0, len(preds), k)]


def run(cb, plan, inputs, config=None):
    with cb.native.Plan(plan, inputs, config=config) as p:
        t = p.collect()
        st = p.stats()
    return t, st


def check_select(cb, batches, cols, filt, outs, config=None, fields=None):
    """Filter(filt) -> Projection(outs) over the batches; cols: the reference columns of the whole input"""
    P = cb.proto
    node = P.scan(fields or [P.STRING, P.INT64])
    if filt is not None:
        node = P.filter_(node, filt.proto())
    node = P.projection(node, [o.proto() for o in outs] + [P.bound(1, P.INT64)])
    t, st = run(cb, node, [batches], config)
    n = len(cols[0][1])
    keep = np.ones(n, dtype=bool)
    if filt is not None:
        fv, fok = filt.eval(cols)
        keep = fv & fok
    got = t.to_pydict() if t is not None else {f"col_{i}": [] for i in range(len(outs) + 1)}
    assert got[f"col_{len(outs)}"] == [int(x) for x in cols[1][0][keep]]
    for i, o in enumerate(outs):
        v, ok = o.eval(cols)
        want = [bool(a) if b else None for a, b in zip(v[keep], ok[keep])]
        assert got[f"col_{i}"] == want, (i, type(o).__name__)
    return st


def stream_input(rng, n, batch, dictionary, bits=32, shared=True, null_frac=0.15):
    """batches of a (dict string, int64) stream; shared: every batch carries the same dictionary, else each its own permutation"""
    codes = rng.integers(0, len(dictionary), n)
    valid = rng.random(n) > null_frac
    ids = np.arange(n, dtype=np.int64)
    batches = []
    for a in range(0, n, batch):
        b = min(n, a + batch)
        if shared:
            d, c = dictionary, codes[a:b]
        else:
            perm = rng.permutation(len(dictionary))
            d = [dictionary[i] for i in perm]
            inv = np.argsort(perm)
            c = inv[codes[a:b]]
        batches.append(pa.record_batch([dict_array(rng, c, valid[a:b], d, bits), pa.array(ids[a:b])], names=["s", "i"]))
    cols = [([dictionary[c] if ok else "" for c, ok in zip(codes, valid)], valid), (ids, np.ones(n, dtype=bool))]
    return batches, cols


@pytest.mark.parametrize("bits,shared", [(8, True), (16, True), (32, True), (8, False), (32, False)])
def test_filter_and_projection_over_arrow_dictionaries(cb, bits, shared):
    rng = np.random.default_rng(bits + shared)
    dictionary = words(rng, 100 if bits == 8 else 700)
    batches, cols = stream_input(rng, 30_000, 4096, dictionary, bits, shared)
    preds = predicates()
    for g in groups(preds):
        check_select(cb, batches, cols, None, g)
    check_select(cb, batches, cols, R.StrIn(R.StrCol(0), ["MAIL", "SHIP", "AIR", None], negated=False), preds[:6])
    filt = R.StrFunc("contains", R.StrCol(0), "a")
    check_select(cb, batches, cols, filt, [R.Like(R.StrCol(0), "%a%"), R.StrCmp("gt", R.StrCol(0), "b")], config={"spark.comet.b200.chunkRows": "8192"})


def test_dictionary_grows_between_launches(cb):
    """each 4096-row batch is its own launch and brings new strings: the masks are extended across partial words, never left stale"""
    rng = np.random.default_rng(5)
    full = words(rng, 400)
    n, batch = 10 * 4096, 4096
    batches, sv, vv = [], [], []
    for k in range(10):
        d = full[:45 + 35 * k]          # the plan-wide dictionary grows by 35 entries per batch (not a multiple of 32)
        c = rng.integers(max(0, len(d) - 40), len(d), batch)
        valid = rng.random(batch) > 0.1
        batches.append(pa.record_batch([dict_array(rng, c, valid, d), pa.array(np.arange(k * batch, (k + 1) * batch, dtype=np.int64))], names=["s", "i"]))
        sv += [d[x] if ok else "" for x, ok in zip(c, valid)]
        vv.append(valid)
    cols = [(sv, np.concatenate(vv)), (np.arange(n, dtype=np.int64), np.ones(n, dtype=bool))]
    cfg = {"spark.comet.b200.chunkRows": "4096"}
    for g in groups(predicates()):
        check_select(cb, batches, cols, R.Like(R.StrCol(0), "%a%"), g, config=cfg)
        check_select(cb, batches, cols, None, g, config=cfg)


def test_several_predicates_on_one_column_in_one_pipeline(cb):
    rng = np.random.default_rng(9)
    batches, cols = stream_input(rng, 20_000, 8192, words(rng, 300))
    c = R.StrCol(0)
    filt = E.Logic("or", R.Like(c, "%a%"), E.Logic("and", R.StrCmp("gt", c, "M"), R.StrFunc("ends_with", c, "L")))
    outs = [R.Like(c, "%a%"), R.Like(c, "%b%"), R.StrCmp("gt", c, "M"), R.StrCmp("lt", c, "M"), R.StrIn(c, ["MAIL"]),
            R.StrFunc("starts_with", c, "a"), E.CaseWhen([R.Like(c, "a%"), R.Like(c, "b%")], [E.Lit(True, E.P.BOOL), E.Lit(False, E.P.BOOL)])]
    check_select(cb, batches, cols, filt, outs)  # pass 2 evaluates 8 distinct string predicates: the cap


# ---- aggregates ---------------------------------------------------------------------------------------------------------------------
def agg_input(rng, n, sorted_keys):
    dictionary = words(rng, 200)
    keyd = ["k0", "k1", "é", "", "日"]
    s = rng.integers(0, len(dictionary), n)
    sv = rng.random(n) > 0.1
    kd = rng.integers(0, len(keyd), n)
    kdv = rng.random(n) > 0.05
    ki = np.sort(rng.integers(0, n // 8, n)) if sorted_keys else rng.integers(0, 5000, n) * 7919
    v = rng.integers(-10**6, 10**6, n)
    vv = rng.random(n) > 0.1
    batches = []
    for a in range(0, n, 1 << 16):
        b = min(n, a + (1 << 16))
        batches.append(pa.record_batch([dict_array(rng, s[a:b], sv[a:b], dictionary), dict_array(rng, kd[a:b], kdv[a:b], keyd),
                                        pa.array(ki[a:b].astype(np.int64)), pa.array(v[a:b].astype(np.int64), mask=~vv[a:b])],
                                       names=["s", "k", "ki", "v"]))
    cols = [([dictionary[x] if ok else "" for x, ok in zip(s, sv)], sv), ([keyd[x] if ok else None for x, ok in zip(kd, kdv)], kdv),
            (ki.astype(np.int64), np.ones(n, dtype=bool)), (v.astype(np.int64), vv)]
    return batches, cols


@pytest.mark.parametrize("strategy", ["dense", "table", "stream"])
def test_aggregate_filter_clauses_and_case_when(cb, strategy):
    """Filter(str pred) -> HashAggregate Partial(COUNT(v) FILTER (WHERE like), SUM(CASE WHEN s IN (...) THEN v ELSE 0), COUNT(*))"""
    P = cb.proto
    rng = np.random.default_rng({"dense": 1, "table": 2, "stream": 3}[strategy])
    n = 300_000
    batches, cols = agg_input(rng, n, strategy == "stream")
    c = R.StrCol(0)
    filt = E.Logic("or", R.StrCmp("neq", c, "MAIL"), R.StrFunc("contains", c, "a"))
    fclause = R.Like(c, "%a%")
    cond = R.StrIn(c, ["MAIL", "SHIP", "a", "é", None])
    key = 1 if strategy == "dense" else 2
    aggs = [P.agg_count([P.bound(3, P.INT64)], fclause.proto()),
            P.agg_sum(P.if_(cond.proto(), P.bound(3, P.INT64), P.literal(0, P.INT64)), P.INT64),
            P.agg_count([P.literal(1, P.INT64)], R.StrCmp("gt_eq", c, "b").proto())]
    plan = P.hash_agg(P.filter_(P.scan([P.STRING, P.STRING, P.INT64, P.INT64]), filt.proto()), [P.bound(key, P.STRING if key == 1 else P.INT64)], aggs)
    cfg = {"spark.comet.b200.streamAgg.minRows": "0"} if strategy == "stream" else {"spark.comet.b200.streamAgg.minRows": "-1"}
    t, st = run(cb, plan, [batches], cfg)
    want_bit = {"dense": cb.native.AGG_DENSE, "table": cb.native.AGG_TABLE, "stream": cb.native.AGG_STREAM}[strategy]
    assert st["agg_strategies"] == want_bit
    fv, fok = filt.eval(cols)
    keep = fv & fok
    a1, a1ok = fclause.eval(cols)
    cv, cok = cond.eval(cols)
    g, gok = R.StrCmp("gt_eq", c, "b").eval(cols)
    v, vv = cols[3]
    keys = cols[key][0]
    exp = {}
    for i in np.nonzero(keep)[0]:
        e = exp.setdefault(keys[i], [0, 0, 0])
        e[0] += int(a1[i] and a1ok[i] and vv[i])
        e[1] += int(v[i]) if (cv[i] and cok[i] and vv[i]) else 0
        e[2] += int(g[i] and gok[i])
    got = {}
    for r in t.to_pylist():
        e = got.setdefault(r["col_0"], [0, 0, 0])
        e[0] += r["col_1"]
        e[1] += r["col_2"] or 0
        e[2] += r["col_3"]
    assert got == exp


# ---- Parquet NativeScan -------------------------------------------------------------------------------------------------------------
def parquet_case(rng, tmp_path, n, fallback):
    dictionary = words(rng, 3000 if fallback else 150)
    s = [dictionary[x] for x in rng.integers(0, len(dictionary), n)]
    sv = rng.random(n) > 0.1
    d = np.sort(rng.integers(8000, 11000, n)).astype(np.int32)
    v = rng.integers(-10**6, 10**6, n)
    tbl = pa.table([pa.array([x if ok else None for x, ok in zip(s, sv)], type=pa.string()), pa.array(d, type=pa.date32()), pa.array(v)],
                   names=["s", "d", "v"])
    path = str(tmp_path / f"s{int(fallback)}.parquet")
    kw = dict(dictionary_pagesize_limit=2048) if fallback else {}
    pq.write_table(tbl, path, row_group_size=40_000, use_dictionary=True, data_page_size=8192, write_page_index=True, **kw)
    cols = [([x if ok else "" for x, ok in zip(s, sv)], sv), (d.astype(np.int64), np.ones(n, dtype=bool)), (v.astype(np.int64), np.ones(n, dtype=bool))]
    return path, cols


@pytest.mark.parametrize("fallback", [False, True])
def test_parquet_native_scan(cb, tmp_path, fallback):
    P = cb.proto
    rng = np.random.default_rng(11 + fallback)
    n = 120_000
    path, cols = parquet_case(rng, tmp_path, n, fallback)
    if fallback:
        md = pq.ParquetFile(path).metadata
        encs = set().union(*[set(md.row_group(g).column(0).encodings) for g in range(md.num_row_groups)])
        assert "PLAIN" in encs and ("RLE_DICTIONARY" in encs or "PLAIN_DICTIONARY" in encs)
    fields = [("s", P.STRING, True), ("d", P.DATE, True), ("v", P.INT64, True)]
    c = R.StrCol(0)
    for filt in (R.Like(c, "%a%"), R.StrIn(c, ["MAIL", "SHIP", "é"]), R.StrCmp("lt", c, "M")):
        scan = P.native_scan(fields, fields, [path])
        plan = P.projection(P.filter_(scan, filt.proto()), [R.StrFunc("starts_with", c, "a").proto(), P.bound(2, P.INT64)])
        t, _ = run(cb, plan, [], {"spark.comet.b200.chunkRows": "32768"})
        fv, fok = filt.eval(cols)
        keep = fv & fok
        got = t.to_pydict() if t is not None else {"col_0": [], "col_1": []}
        assert got["col_1"] == [int(x) for x in cols[2][0][keep]]
        sw, sok = R.StrFunc("starts_with", c, "a").eval(cols)
        assert got["col_0"] == [bool(a) if b else None for a, b in zip(sw[keep], sok[keep])]


def test_parquet_page_pruning_with_string_filter(cb, tmp_path):
    P = cb.proto
    rng = np.random.default_rng(13)
    n = 120_000
    path, cols = parquet_case(rng, tmp_path, n, False)
    fields = [("s", P.STRING, True), ("d", P.DATE, True), ("v", P.INT64, True)]
    dates = cols[1][0]
    lo = int(dates[n // 3])
    c = R.StrCol(0)
    like = R.Like(c, "%A%")
    date_terms = P.and_(P.gt_eq(P.bound(1, P.DATE), P.literal(lo, P.DATE)), P.lt(P.bound(1, P.DATE), P.literal(lo + 40, P.DATE)))
    pred = P.and_(date_terms, like.proto())
    scan = P.native_scan(fields, fields, [path], data_filters=[pred])
    plan = P.hash_agg(P.filter_(scan, pred), [], [P.agg_count([P.bound(2, P.INT64)]), P.agg_sum(P.bound(2, P.INT64), P.INT64)])
    t, st = run(cb, plan, [])
    assert st["scan_pruned_pages"] > 0
    lv, lok = like.eval(cols)
    keep = (dates >= lo) & (dates < lo + 40) & lv & lok
    r = t.to_pylist()[0]
    assert r["col_0"] == int(keep.sum()) and r["col_1"] == (int(cols[2][0][keep].sum()) if keep.any() else None)


# ---- device tables and malformed codes ----------------------------------------------------------------------------------------------
def test_device_table_dictionary_column(cb):
    torch = pytest.importorskip("torch")
    P = cb.proto
    rng = np.random.default_rng(17)
    dictionary = words(rng, 90)
    n = 50_000
    codes = rng.integers(0, len(dictionary), n).astype(np.int32)
    ids = np.arange(n, dtype=np.int64)
    tc, ti = torch.from_numpy(codes).cuda(), torch.from_numpy(ids).cuda()
    tb = cb.native.DeviceTable(n).add(P.STRING, tc.data_ptr(), 4, dictionary=dictionary, keep=tc).add(P.INT64, ti.data_ptr(), 8, keep=ti)
    cols = [([dictionary[x] for x in codes], np.ones(n, dtype=bool)), (ids, np.ones(n, dtype=bool))]
    c = R.StrCol(0)
    filt = R.Like(c, "%e%")
    outs = [R.StrIn(c, ["MAIL", "SHIP"]), R.StrCmp("gt", c, "M")]
    node = P.projection(P.filter_(P.scan([P.STRING, P.INT64]), filt.proto()), [o.proto() for o in outs] + [P.bound(1, P.INT64)])
    t, _ = run(cb, node, [tb], {"spark.comet.b200.chunkRows": "16384"})
    fv, fok = filt.eval(cols)
    keep = fv & fok
    got = t.to_pydict()
    assert got["col_2"] == [int(x) for x in ids[keep]]
    for i, o in enumerate(outs):
        v, ok = o.eval(cols)
        assert got[f"col_{i}"] == [bool(a) for a in v[keep]]


@pytest.mark.parametrize("code", [-3, 12, 1 << 20])
def test_valid_out_of_range_code_fails_the_plan(cb, code):
    P = cb.proto
    rng = np.random.default_rng(19)
    dictionary = ["MAIL", "SHIP", "AIR"]
    n = 5000
    codes = rng.integers(0, 3, n)
    codes[1234] = code
    valid = np.ones(n, dtype=bool)
    batch = pa.record_batch([dict_array(rng, codes, valid, dictionary), pa.array(np.arange(n, dtype=np.int64))], names=["s", "i"])
    plan = P.projection(P.filter_(P.scan([P.STRING, P.INT64]), R.StrIn(R.StrCol(0), ["MAIL"]).proto()), [P.bound(1, P.INT64)])
    with pytest.raises(cb.native.CometB200Error, match="dictionary code out of range"):
        run(cb, plan, [[batch]])
