"""A CPU reference of Spark's one-distinct aggregate plan (AggUtils.planAggregateWithOneDistinct) as four HashAggregate stages, built
on tests/aggref.py's per-function Partial / merge / Final rules:

  stage 1  group by k, x     ordinary aggregates Partial                                       (scan rows)
  stage 2  group by k, x     ordinary aggregates PartialMerge                                  (stage 1 state)
  stage 3  group by k        ordinary aggregates PartialMerge, distinct aggregates Partial over x (stage 2 state)
  stage 4  group by k        every aggregate Final                                             (stage 3 state)

`k` are the outer keys, `x` the distinct columns (COUNT(DISTINCT x, y) is a COUNT with two children).  The native side never
deduplicates: distinctness comes from the grouping of stages 1 and 2.  Stage 3 carries per-expression modes: its merging aggregates
read their state columns consecutively from `initial_input_buffer_offset` (= the number of stage 2 group columns), the running offset
advancing over merging aggregates only (planner.rs:1265-1352), and its Partial aggregates read the distinct columns, which are stage 2
group columns.  Its output is the outer keys, then every aggregate's state columns in agg_exprs order."""
from comet_b200 import proto as P

import aggref as R
import exprs as E


class Chain:
    """One distinct query.  dts: input column types; key_cols / distinct_cols: input column indices; ordinary: aggref.Agg list over the
    input columns; distinct: [(kind, dt, sum_dt, eval_mode)] aggregates over the distinct columns (COUNT takes all of them, SUM / AVG
    the first); order: stage 3's agg_exprs as ("o", i) / ("d", i) entries (default: ordinary first, as Spark emits them)."""

    def __init__(self, dts, key_cols, distinct_cols, ordinary, distinct, order=None):
        self.dts, self.key_cols, self.distinct_cols = dts, list(key_cols), list(distinct_cols)
        self.ordinary, self.distinct_specs = list(ordinary), list(distinct)
        self.order = order or [("o", i) for i in range(len(ordinary))] + [("d", i) for i in range(len(distinct))]
        assert [i for t, i in self.order if t == "o"] == list(range(len(ordinary))), "merging aggregates keep stage 1's order"
        assert sorted(i for t, i in self.order if t == "d") == list(range(len(distinct)))

    # ---- shapes -------------------------------------------------------------------------------------------------------------------
    @property
    def key_types(self):
        return [self.dts[c] for c in self.key_cols]

    @property
    def distinct_types(self):
        return [self.dts[c] for c in self.distinct_cols]

    @property
    def inner_types(self):  # stage 1 / 2 group columns
        return self.key_types + self.distinct_types

    @property
    def stage2_schema(self):
        return R.state_schema(self.inner_types, self.ordinary)

    def distinct_aggs(self):
        """The distinct aggregates as aggref.Agg over stage 2's output (the distinct columns follow the outer keys there)."""
        nk = len(self.key_cols)
        xs = [E.Col(nk + j, t) for j, t in enumerate(self.distinct_types)]
        out = []
        for kind, dt, sum_dt, mode in self.distinct_specs:
            a = R.Agg(kind, xs[0], dt, sum_dt, mode)
            if kind == "count":
                a.args = xs
            out.append(a)
        return out

    def stage3_aggs(self):
        d = self.distinct_aggs()
        return [self.ordinary[i] if t == "o" else d[i] for t, i in self.order]

    def expr_modes(self):
        return [R.PARTIAL_MERGE if t == "o" else R.PARTIAL for t, _ in self.order]

    @property
    def mixed(self):
        return bool(self.ordinary) and bool(self.distinct_specs)

    # ---- plans --------------------------------------------------------------------------------------------------------------------
    def stage1_plan(self):
        return P.hash_agg(P.scan(self.dts), [P.bound(c, self.dts[c]) for c in self.key_cols + self.distinct_cols],
                          [a.proto() for a in self.ordinary], R.PARTIAL)

    def stage2_plan(self, with_offset=True):
        """PartialMerge over stage 1's state; with no ordinary aggregate a keys-only Partial (Comet sends no mode for it)."""
        nin = len(self.inner_types)
        scan = P.scan(self.stage2_schema, source="shuffle")
        keys = [P.bound(i, t) for i, t in enumerate(self.inner_types)]
        if not self.ordinary:
            return P.hash_agg(scan, keys, [], R.PARTIAL)
        return P.hash_agg(scan, keys, [a.proto(merge=True) for a in self.ordinary], R.PARTIAL_MERGE,
                          initial_input_buffer_offset=nin if with_offset else None)

    def stage3_plan(self):
        nk, nin = len(self.key_cols), len(self.inner_types)
        scan = P.scan(self.stage2_schema, source="shuffle")
        keys = [P.bound(i, t) for i, t in enumerate(self.key_types)]
        aggs = [self.ordinary[i].proto(merge=True) if t == "o" else agg_proto(self.distinct_aggs()[i]) for t, i in self.order]
        if not self.ordinary:   # a distinct aggregate alone: an ordinary Partial over the deduplicated rows
            return P.hash_agg(scan, keys, aggs, R.PARTIAL)
        if not self.distinct_specs:
            return P.hash_agg(scan, keys, aggs, R.PARTIAL_MERGE, initial_input_buffer_offset=nin)
        assert nk <= nin
        return P.hash_agg(scan, keys, aggs, R.PARTIAL, expr_modes=self.expr_modes(), initial_input_buffer_offset=nin)

    def stage3_schema(self):
        return R.state_schema(self.key_types, self.stage3_aggs())

    def stage4_plan(self):
        return R.merge_plan(self.key_types, self.stage3_aggs(), R.FINAL)

    # ---- the reference's answers per stage ----------------------------------------------------------------------------------------
    def stage1(self, table):
        """{(k..., x...): [ordinary state]}; keys only: every distinct (k, x)"""
        if not self.ordinary:
            groups, _, _ = R._input_rows(table, self.dts, self.key_cols + self.distinct_cols, [])
            return {k: [] for k in groups.keys}
        return R.partial(table, self.dts, self.key_cols + self.distinct_cols, self.ordinary)

    def stage2(self, stage1_rows):
        return merged_or_keys(stage1_rows, self.ordinary)

    def stage3(self, stage2_rows):
        """stage 2 rows [(k + x key, [ordinary state])] -> {k: [state per stage 3 aggregate]}"""
        nk = len(self.key_cols)
        by_k = {}
        for key, st in stage2_rows:
            by_k.setdefault(key[:nk], []).append((key, st))
        if not self.key_cols and not by_k:
            by_k[()] = []
        d_aggs = self.distinct_aggs()
        out = {}
        for k, rows in by_k.items():
            merged = R.merge([(k, st) for _, st in rows], self.ordinary)[k] if rows and self.ordinary else None
            res = []
            for t, i in self.order:
                if t == "o":
                    res.append(merged[i] if merged is not None else empty_state(self.ordinary[i]))
                    continue
                a = d_aggs[i]
                xs = [key[nk:] for key, _ in rows]
                if a.kind == "count":
                    vals = [x for x in xs if all(v is not None for v in x)]
                else:
                    vals = [x[0] for x in xs if x[0] is not None]
                if a.kind == "avg" and a.dt.name == "DECIMAL":
                    res.append(R._avg_decimal(a, [vals])[0][0])
                else:
                    res.append(R._partial_state(a, vals))
            out[k] = res
        return out

    def stage4(self, stage3_rows):
        return R.final(stage3_rows, self.stage3_aggs(), ungrouped=not self.key_cols)

    def answer(self, table):
        """The whole chain on the CPU: {k: [result per stage 3 aggregate]}."""
        s1 = self.stage1(table)
        s2 = self.stage2(list(s1.items()))
        s3 = self.stage3(list(s2.items()))
        return self.stage4(list(s3.items()))


def agg_proto(a):
    """A Partial aggregate over the distinct columns; COUNT may take several."""
    if a.kind == "count" and getattr(a, "args", None):
        return P.agg_count([x.proto() for x in a.args])
    return a.proto()


def empty_state(a):
    """The state of a fresh accumulator (an ungrouped stage over no rows)."""
    if a.kind == "avg" and a.dt.name == "DECIMAL":
        return R._avg_decimal(a, [[]])[0][0]
    return R._partial_state(a, [])


def merged_or_keys(state_rows, aggs):
    """PartialMerge of state rows; keys-only rows (no aggregates) deduplicate."""
    if not aggs:
        return {k: [] for k, _ in state_rows}
    return R.merge(state_rows, aggs)
