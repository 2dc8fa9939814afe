"""CPU-only checks of the C ABI: the library loads, exports every symbol include/comet_b200.h declares,
decodes / rejects plans, generates and NVRTC-compiles the pipeline kernels (no compute without a GPU)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def cb():
    import comet_b200
    return comet_b200


def test_library_exports_every_declared_symbol(cb):
    hdr = open(os.path.join(ROOT, "include", "comet_b200.h")).read()
    declared = set(re.findall(r"\b(cb200_[a-z_0-9]+)\s*\(", hdr))
    assert len(declared) >= 14
    lib = C.CDLL(os.path.join(ROOT, "datafusion-comet_b200", "libcomet_b200.so"))
    for sym in sorted(declared):
        assert hasattr(lib, sym), f"{sym} declared in include/comet_b200.h but not exported"
    assert set(cb.native.EXPORTED) <= declared


def test_stats_struct_matches_the_header(cb):
    """native.Stats mirrors cb200_stats field by field (the binding reads it by position), incl. agg_strategies and its bits."""
    hdr = open(os.path.join(ROOT, "include", "comet_b200.h")).read()
    body = hdr[hdr.index("typedef struct cb200_stats {"):hdr.index("} cb200_stats;")]
    fields = re.findall(r"^\s*(?:int64_t|double)\s+([a-z_0-9]+);", body, re.M)
    assert fields == [f for f, _ in cb.native.Stats._fields_]
    bits = dict(re.findall(r"#define CB200_AGG_([A-Z]+) (\d+)", hdr))
    n = cb.native
    assert {k: int(v) for k, v in bits.items()} == {"DENSE": n.AGG_DENSE, "TABLE": n.AGG_TABLE, "STREAM": n.AGG_STREAM, "MIGRATED": n.AGG_MIGRATED}
    levels = dict(re.findall(r"#define CB200_RANGE_([A-Z]+) (\d+)", hdr))
    assert {k: int(v) for k, v in levels.items()} == {"TIGHT": n.RANGE_TIGHT, "TYPE": n.RANGE_TYPE, "SAFE": n.RANGE_SAFE}


def test_version(cb):
    assert "sm_90a" in cb.native.version()


@pytest.mark.parametrize("variant", ["dec", "f64"])
def test_benchmark_plans_supported_and_compile(cb, variant):
    t = cb.tpch
    for plan in (t.q1_partial_plan(variant), t.q1_final_plan(variant), t.q6_partial_plan(variant), t.q6_final_plan(variant),
                 t.config1_plan(variant)):
        ok, why = cb.native.supports(plan)
        assert ok, why
        keys = cb.native.compile_plan(plan)  # NVRTC -> sm_90a cubin, no GPU needed
        assert len(keys) == (2 if plan is not None and plan == t.config1_plan(variant) else 1)  # filter+project: count pass + select pass


def test_generated_q1_kernel_is_fused_and_uses_tma(cb):
    src = cb.native.kernel_source(cb.tpch.q1_partial_plan("dec"))
    assert "#define CB_KERNEL_AGG 1" in src and "cb_row_agg" in src and "cb_finalize_group" in src
    # one kernel for scan+filter+project+aggregate: the filter literal and the aggregate updates are in the same row program
    body = src[src.index("CB_D void cb_row_agg"):]
    assert "10493" in body and "acc.add_" in body
    hdr = open(os.path.join(ROOT, "datafusion-comet_b200", "csrc", "device", "cb_kernels.cuh")).read()
    assert "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes" in hdr


def test_range_specialised_kernel_drops_checks(cb):
    t = cb.tpch
    generic = cb.native.kernel_source(t.q1_partial_plan("dec"))
    tight = cb.native.compile_plan_assume(t.q1_partial_plan("dec"), [15, 26, 6, 6, 0, 0, 0], 0)
    gb, tb = generic[generic.index("CB_D void cb_row_agg"):generic.index("CB_D void cb_finalize_group")], \
        tight[tight.index("CB_D void cb_row_agg"):tight.index("CB_D void cb_finalize_group")]
    assert "dec_fits" not in tb and "wide_mul" not in tb and "set_err" not in tb   # proofs removed every check
    assert "acc.vm_or" in tb                                                        # ... but inputs are still validated
    assert len(tb) < len(gb)


def test_unsupported_plans_are_rejected_not_miscomputed(cb):
    P = cb.proto
    sc = P.scan([P.STRING, P.INT64])
    # a string column REFERENCE passes through a projection as dictionary codes; string expressions are not on the fused path
    ok, why = cb.native.supports(P.projection(sc, [P.bound(0, P.STRING)]))
    assert ok, why
    ok, why = cb.native.supports(P.projection(sc, [P.if_(P.is_null(P.bound(1, P.INT64)), P.bound(0, P.STRING), P.literal("x", P.STRING))]))
    assert not ok and "string" in why
    # decimal division (decimal_div UDF) is on the path; a division that mixes types is not
    sc2 = P.scan([P.DECIMAL(12, 2), P.DECIMAL(12, 2), P.INT32])
    ok, why = cb.native.supports(P.projection(sc2, [P.divide(P.bound(0, P.DECIMAL(12, 2)), P.bound(1, P.DECIMAL(12, 2)), P.DECIMAL(27, 15))]))
    assert ok, why
    assert "cb::dec_div(" in cb.native.kernel_source(P.projection(sc2, [P.divide(P.bound(0, P.DECIMAL(12, 2)), P.bound(1, P.DECIMAL(12, 2)), P.DECIMAL(27, 15))]))
    ok, why = cb.native.supports(P.projection(sc2, [P.divide(P.bound(0, P.DECIMAL(12, 2)), P.bound(2, P.INT32), P.DECIMAL(27, 15))]))
    assert not ok
    # garbage bytes -> plan error, not a crash
    ok, why = cb.native.supports(b"\xff\xff\xff\x07garbage")
    assert not ok


def test_decimal_type_rules_follow_the_planner(cb):
    """planner.rs:998-1027: p1+p2 >= 38 -> WideDecimal (uses the proto return type), else arrow-arith result type."""
    P = cb.proto
    sc = P.scan([P.DECIMAL(26, 4), P.DECIMAL(13, 2), P.DATE])
    wide = P.multiply(P.bound(0, P.DECIMAL(26, 4)), P.bound(1, P.DECIMAL(13, 2)), P.DECIMAL(38, 6))
    plan = P.projection(P.filter_(sc, P.lt(P.bound(2, P.DATE), P.literal(5, P.DATE))), [wide])
    src = cb.native.kernel_source(plan)
    assert "wide_mul_fast" in src
    sc = P.scan([P.DECIMAL(12, 2), P.DECIMAL(12, 2), P.DATE])
    plain = P.multiply(P.bound(0, P.DECIMAL(12, 2)), P.bound(1, P.DECIMAL(12, 2)), P.DECIMAL(25, 4))
    plan = P.projection(P.filter_(sc, P.lt(P.bound(2, P.DATE), P.literal(5, P.DATE))), [plain])
    src = cb.native.kernel_source(plan)
    assert "dec_mul_plain" in src and "wide_mul" not in src


def test_create_plan_without_gpu_fails_loudly(cb):
    import pyarrow as pa
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("GPU present")
    except ImportError:
        pass
    t = cb.tpch
    tbl = t.lineitem_table(t.gen_lineitem(100), "dec", columns=["l_quantity", "l_extendedprice", "l_shipdate"])
    p = cb.native.Plan(t.config1_plan("dec"), [tbl])   # decoding the plan needs no device
    with pytest.raises(cb.native.CometB200Error):       # executing does: no CPU fallback
        p.execute()
    p.release()


def test_case_when_decodes_to_guarded_branches(cb):
    """CaseWhen (expr.proto:473) -> nested IF; ANSI errors inside a branch are raised only for rows that take it."""
    P = cb.proto
    i = P.bound(0, P.INT32)
    cw = P.case_when([P.lt(i, P.literal(0, P.INT32))], [P.add(i, i, P.INT32, P.ANSI)])          # no ELSE -> typed NULL
    src = cb.native.kernel_source(P.projection(P.scan([P.INT32]), [cw]))
    body = src[src.index("cb_row_select"):]
    assert "cb::set_err(p, 1)" in body
    guard_line = [ln for ln in body.splitlines() if "cb::set_err(p, 1)" in ln][0]
    assert "&&" in guard_line and "if (" in guard_line                                            # the overflow test is ANDed with the branch condition
    ok, why = cb.native.supports(P.projection(P.scan([P.INT32]), [P.case_when([P.lt(i, P.literal(0, P.INT32))], [i, i])]))
    assert not ok                                                                                 # mismatched when/then lists


def test_filter_project_is_two_streaming_passes(cb):
    """pass 1 stages only the predicate columns, counts per (tile, warp) and leaves a keep bit per row; pass 2 writes at scanned offsets; no look-back."""
    plan = cb.tpch.config1_plan("f64")
    keys = cb.native.compile_plan(plan)
    assert len(keys) == 2
    sel, cnt = cb.native.kernel_source(plan, 0), cb.native.kernel_source(plan, 1)
    assert "#define CB_SELECT_COUNT 1" in cnt and "#define CB_NCOLS 1\n" in cnt and "#define CB_LTILE 1024" in cnt   # only l_shipdate is staged
    # pass 2 takes pass 1's keep bits: it stages the two projected columns only, never l_shipdate again
    assert "#define CB_NCOLS 2\n" in sel and "#define CB_SEL_MASKED 1" in sel and "CB_SELECT_COUNT" not in sel
    hdr = open(os.path.join(ROOT, "datafusion-comet_b200", "csrc", "device", "cb_kernels.cuh")).read()
    assert "sel_chunk" in hdr and "tile_state" not in hdr


def test_partial_merge_and_try_sum_state_layouts(cb):
    P = cb.proto
    t = cb.tpch
    # operator-level PartialMerge: state in, state out
    sc = P.scan(t.q1_state_fields("dec"), source="shuffle")
    pm = P.hash_agg(sc, [P.bound(0, P.STRING), P.bound(1, P.STRING)], t.q1_aggs("dec", bound=False), P.PARTIAL_MERGE)
    ok, why = cb.native.supports(pm)
    assert ok, why
    # TRY sum carries (sum, has_all_nulls): a Final plan whose child lacks the flag column is a plan error
    bad = P.hash_agg(P.scan([P.INT64, P.INT64], source="shuffle"), [P.bound(0, P.INT64)], [P.agg_sum(P.unbound("s", P.INT64), P.INT64, P.TRY)], P.FINAL)
    ok, why = cb.native.supports(bad)
    assert not ok and "state" in why
    good = P.hash_agg(P.scan([P.INT64, P.INT64, P.BOOL], source="shuffle"), [P.bound(0, P.INT64)], [P.agg_sum(P.unbound("s", P.INT64), P.INT64, P.TRY)], P.FINAL)
    ok, why = cb.native.supports(good)
    assert ok, why


def test_wide_group_keys_use_tag_and_stored_key(cb):
    P = cb.proto
    one = P.hash_agg(P.scan([P.INT64, P.INT64]), [P.bound(0, P.INT64)], [P.agg_sum(P.bound(1, P.INT64), P.INT64)], P.PARTIAL)
    three = P.hash_agg(P.scan([P.INT64, P.INT64, P.DATE, P.INT64]), [P.bound(0, P.INT64), P.bound(1, P.INT64), P.bound(2, P.DATE)],
                       [P.agg_sum(P.bound(3, P.INT64), P.INT64)], P.PARTIAL)
    s1, s3 = cb.native.kernel_source(one), cb.native.kernel_source(three)
    assert "#define CB_KEY_WORDS 1" in s1 and "acc.begin(keep_" in s1 and "acc.h_add_wrap(" in s1   # warp-cooperative table update
    assert "#define CB_KEY_WORDS 4" in s3 and "acc.begin(keep_" in s3            # 64 + 64 + 33 bits + the null-flag word of the 64-bit keys
    too_wide = P.hash_agg(P.scan([P.INT64] * 6), [P.bound(k, P.INT64) for k in range(5)], [P.agg_sum(P.bound(5, P.INT64), P.INT64)], P.PARTIAL)
    ok, why = cb.native.supports(too_wide)
    assert not ok
