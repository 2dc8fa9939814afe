"""Compare the generated pipeline-kernel source of two builds, byte for byte (CPU only: code generation needs no GPU).

    python tools/compare_kernel_sources.py OTHER_TREE [THIS_TREE]

Each tree is a checkout whose libcomet_b200.so is built (`make -C datafusion-comet_b200/csrc`).  For every plan below and every
kernel index, `native.kernel_source(plan, i)` must be identical in both trees: the TPC-H Q1 partial / final (dec and f64) and Q6
plans, Config 1, the group-by map and final plans of bench.py, the string-predicate plans of tests/test_string_predicates_cpu.py and
a Sort over a pipeline.  Lists every plan whose sources or kernel count differ, and then exits 1."""
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def plans():
    from comet_b200 import proto as P, tpch
    sys.path.insert(0, os.path.join(HERE, "tests"))
    import test_string_predicates_cpu as T
    out = {}
    for v in ("dec", "f64"):
        out[f"q1_partial_{v}"] = tpch.q1_partial_plan(v)
        out[f"q1_final_{v}"] = tpch.q1_final_plan(v)
        out[f"q6_partial_{v}"] = tpch.q6_partial_plan(v)
        out[f"q6_final_{v}"] = tpch.q6_final_plan(v)
        out[f"config1_{v}"] = tpch.config1_plan(v)
    for m, sdt in ((P.DECIMAL(12, 2), P.DECIMAL(22, 2)), (P.DOUBLE, P.DOUBLE)):
        agg = P.hash_agg(P.scan([P.INT64, m]), [P.bound(0, P.INT64)], [P.agg_sum(P.bound(1, m), sdt)], P.PARTIAL)
        state = [P.INT64, sdt, P.BOOL] if sdt is not P.DOUBLE else [P.INT64, sdt]
        name = "dec" if sdt is not P.DOUBLE else "f64"
        out[f"groupby_map_{name}"] = P.shuffle_writer(agg, P.hash_partitioning([P.bound(0, P.INT64)], 8))
        out[f"groupby_final_{name}"] = P.hash_agg(P.scan(state, source="shuffle"), [P.bound(0, P.INT64)], [P.agg_sum(P.unbound("c", m), sdt)], P.FINAL)
    for i, pred in enumerate(T.accepted_shapes()):
        out[f"strpred_filter_{i}"] = T.filt(P.and_(pred, P.is_not_null(P.bound(1, P.INT64))))
        out[f"strpred_projection_{i}"] = P.projection(P.scan([P.STRING, P.INT64, P.STRING]), [pred, P.bound(1, P.INT64)])
        out[f"strpred_agg_filter_{i}"] = P.hash_agg(P.scan([P.STRING, P.INT64, P.STRING]), [T.col()], [P.agg_count([P.bound(1, P.INT64)], pred)])
    c = T.col()
    out["strpred_two_masks"] = T.filt(P.or_(P.like(c, T.slit("a%")), P.like(c, T.slit("b%"))))
    out["strpred_same_mask"] = T.filt(P.or_(P.like(c, T.slit("a%")), P.like(c, T.slit("a%"))))
    out["sort_over_filter"] = P.sort(T.filt(P.like(c, T.slit("a%"))), [P.sort_order(P.bound(0, P.INT64), descending=True)])
    return out


def dump(tree):
    """{plan name: [kernel i's source, ...]} of the build in `tree` (run in a child process, one library per process)."""
    sys.path[:0] = [os.path.join(tree, "datafusion-comet_b200")]
    from comet_b200 import native
    assert os.path.dirname(native._LIB_PATH) == os.path.join(os.path.abspath(tree), "datafusion-comet_b200"), native._LIB_PATH
    res = {}
    for name, plan in plans().items():
        srcs = []
        while True:
            try:
                srcs.append(native.kernel_source(plan, len(srcs)))
            except native.CometB200Error as e:
                if "kernel index out of range" not in str(e):
                    raise
                break
        res[name] = srcs
    return res


def main():
    if len(sys.argv) == 3 and sys.argv[1] == "--dump":
        print(json.dumps(dump(sys.argv[2])))
        return 0
    if len(sys.argv) not in (2, 3):
        print(__doc__)
        return 2
    trees = [os.path.abspath(sys.argv[1]), os.path.abspath(sys.argv[2] if len(sys.argv) == 3 else HERE)]
    dumps = [json.loads(subprocess.check_output([sys.executable, os.path.abspath(__file__), "--dump", t])) for t in trees]
    bad = [n for n in dumps[1] if dumps[0].get(n) != dumps[1][n]] + [n for n in dumps[0] if n not in dumps[1]]
    kernels = sum(len(v) for v in dumps[1].values())
    for n in bad:
        print(f"DIFFERS: {n}: {len(dumps[0].get(n, []))} vs {len(dumps[1].get(n, []))} kernels")
    print(f"{len(dumps[1])} plans, {kernels} kernels: {'identical' if not bad else f'{len(bad)} plans differ'}")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
