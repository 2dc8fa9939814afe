// join.cpp -- the join node of HashJoin (HashJoinExec with NullEquality::NullEqualsNothing, planner.rs:2192-2266: inner, left semi and
// left anti), SortMergeJoin (SortMergeJoinExec with NullEqualsNothing, planner.rs:2126-2190: those and left / right / full outer) and
// BroadcastNestedLoopJoin (NestedLoopJoinExec, planner.rs:1386-1436: inner, left / right outer, left semi and left anti, the shapes whose
// output follows the streamed side, operators.scala:2258-2266).
#include "exec_internal.h"

namespace cb200 {

// code -> canonical code of dictionary d: the code of the first entry of the build dictionary equal to it (a caller's dictionary may
// repeat values), or the build dictionary's size for a string it lacks.  On the build side d is the build dictionary itself.
static std::vector<uint32_t> canonical_codes(const Dictionary& d, const Dictionary& build) {
    const std::vector<std::string>& v = d.values();
    const uint32_t absent = (uint32_t)build.values().size();
    std::vector<uint32_t> codes(v.size());
    for (size_t i = 0; i < v.size(); i++) {
        const int32_t code = build.find(v[i]);
        codes[i] = code < 0 ? absent : (uint32_t)code;
    }
    return codes;
}

// The build side is drained before the first probe batch and concatenated on the device.  Its row keys (the sort's encoding,
// device/cb_sortkey.h) are radix-sorted, so equal keys form runs in build input order, and every run without a NULL key gets one slot of
// an open-addressing table.  A probe batch then costs one key pass and one lookup per row; an inner or outer join scans the match
// counts, writes the (probe row, build row) pairs and gathers both sides, a semi / anti join compacts the probe rows it keeps.  Output
// order: probe rows in input order, an inner / outer row's matches in build input order; output above spark.comet.b200.chunkRows rows
// leaves in several batches.
//
// Outer joins (SortMergeJoin only).  A probe row without a match counts one output row, paired with build row CB_NULL_ROW, which the
// gather turns into NULLs.  FullOuter also marks every run a lookup finds; once the probe side ends, the build rows of runs never found
// (NULL keys included) leave in build input order with NULL probe columns.  Every column of a side the join type may NULL-extend (the
// build side of every outer type, the probe side of FullOuter) has a validity bitmap in every batch.  A side with no source rows in a
// batch -- an empty build side, the probe side of the unmatched build rows -- gets all-NULL columns in the layout of that side's last batch.
//
// Equal key tuples give equal words on both sides because the field layout is fixed by the declared key types (every field has a null
// bit, whatever a batch's validity) and a string field holds a canonical code rather than the dictionary code: the code of the first
// equal entry of the build side's dictionary, or that dictionary's size (which no build key has) for a probe string it lacks.
//
// Join conditions.  A condition is evaluated on candidate pairs only -- (probe row, build row) with equal keys -- and a pair passes when
// it gives TRUE.  A probe batch with a condition is resolved in two phases, because one probe row's candidates may straddle slices:
//  1. its pairs are enumerated in slices of at most chunkRows; for each slice the columns the condition reads are gathered through the
//     pair indices (each in its stored layout), a generated predicate-only pass (count_pass_spec) leaves one pass bit per pair in the
//     batch's bit array, and launch_join_cond_mark sets the probe row's `passed` byte (and FullOuter's per-build-row hit byte);
//  2. semi / anti joins compact the probe rows by `passed`; inner and outer joins re-enumerate the pairs slice by slice and keep the
//     passing ones, plus, for a probe row that passed nothing, its first pair (an outer join's sentinel pair when it has no candidate)
//     as its NULL-extended row.  FullOuter's unmatched build rows are those whose hit byte no passing pair set.
// An outer join's sentinel pairs take part in phase 1 with NULLs on both sides and their bits cleared: the condition never sees a
// NULL-extended row, so an ANSI error comes from a candidate or from nowhere.
//
// Nested-loop joins.  A join without keys is run by the same node: every (probe row, build row) pair is a candidate.  The build side is
// drained and concatenated, with no key, sort or table.  Pairs are numbered probe-row major -- pair p of a group starting at probe row g0
// is (g0 + p / m, p % m) for m build rows -- and computed by launch_nlj_pairs, so the output order is the hash join's: probe rows in input
// order, each one's pairs in build input order.  Without a condition an inner / outer join emits all n * m pairs of a probe batch in
// chunkRows windows, and a semi / anti join passes or drops the whole batch by whether the build side is empty.  With a condition a probe
// batch is resolved in groups of max(1, chunkRows / m) whole probe rows, so that a group's pass bits and pair indices take O(chunkRows + m)
// memory however many pairs the batch has: phase 1 runs group by group (semi / anti joins run every group, then compact), and an inner
// / outer join resolves each group's pairs (launch_nlj_cond_resolve: a probe row that passed nothing keeps its pair with build row 0,
// NULL-extended) before the next group's phase 1.
//
// NULL columns of type t, n rows: the layout (and dictionary) of `like`, or without one the Arrow layout of t and an empty dictionary
static Column null_column(const DType& t, const Column* like, int64_t n, ExecContext* ctx) {
    Column o;
    o.type = t;
    if (like) { o.phys = like->phys; o.is_dict = like->is_dict; o.dict = like->dict; }
    else if (t.is_string()) { o.phys = Phys::I32; o.is_dict = true; o.dict = std::make_shared<Dictionary>(); }
    else o.phys = phys_of(t);
    const int w = phys_bytes(o.phys);
    o.data = std::make_shared<DeviceBuf>(w == 0 ? bitmap_bytes(n) : (size_t)std::max<int64_t>(n, 1) * w);
    o.validity = std::make_shared<DeviceBuf>(bitmap_bytes(n));
    cuda_check(cudaMemsetAsync(o.data->ptr, 0, o.data->bytes, ctx->stream), "memset NULL column");
    cuda_check(cudaMemsetAsync(o.validity->ptr, 0, o.validity->bytes, ctx->stream), "memset NULL validity");
    o.null_count = -1;
    return o;
}

// The condition's evaluator: a fused node over the left columns followed by the right ones, whose child produces nothing
struct JoinCondition : FusedBase {
    struct Columns : ExecNode { bool next(Batch&) override { return false; } };
    int n_left = 0;
    DeviceBufP sel_off;                      // the count pass's per-(tile, warp) counts: written, not read

    bool next(Batch&) override { return false; }
    PipelineSpec spec(const Batch* b) const { return count_pass_spec(stage_cols(b), to_slots(predicates, slot_of)); }

    // pass bits of the k pairs (probe_idx[j], build_idx[j]) into bits[0, (k + 31) / 32); or_null: a row index may be CB_NULL_ROW
    void eval(const Batch& probe, const Batch& build, bool build_left, const unsigned* probe_idx, const unsigned* build_idx, int64_t k, bool or_null,
              cb::u32* bits) {
        Batch in;
        in.n_rows = k;
        in.cols.resize(child->schema.size());
        for (int c : used_cols) {
            const bool left = c < n_left, from_probe = left != build_left;
            const Batch& side = from_probe ? probe : build;
            const unsigned* idx = from_probe ? probe_idx : build_idx;
            Batch one, g;
            one.n_rows = side.n_rows;
            one.cols = {side.cols.at((size_t)(left ? c : c - n_left))};
            if (or_null) gather_columns_or_null(one, idx, k, g, ctx);
            else gather_columns(one, idx, k, g, ctx, "joining");
            in.cols[(size_t)c] = std::move(g.cols[0]);
        }
        const PipelineSpec s = spec(&in);
        const GeneratedKernel g = generate_pipeline(s);
        auto mod = jit_get(g, true);
        cb::PipeParams p;
        fill_inputs(p, in, g.tile);
        bind_str_masks(p, s, in);
        const size_t m = (size_t)((k + 1023) / 1024) * (size_t)(g.threads / 32);
        if (!sel_off || sel_off->bytes < m * 4) sel_off = std::make_shared<DeviceBuf>(m * 4 + m / 2);
        p.sel_off = (cb::u32*)sel_off->ptr;
        p.sel_mask = bits;
        launch(mod->kernel(g.entry), dim3(std::min(ctx->num_sms, p.n_tiles)), dim3(g.threads + 32), g.dyn_smem(0), &p);
    }
};

struct JoinNode : ExecNode {
    ExecContext* ctx;
    ExecNodeP build_child, probe_child;
    std::vector<int> build_keys, probe_keys; // key columns of each side, in key order
    JoinType type = JoinType::Inner;
    bool build_left = false;
    bool nested = false;                     // a nested-loop join: no keys, every pair is a candidate
    unsigned long long nlj_inv = 0;          // nested-loop join: floor((2^64 - 1) / build rows), launch_nlj_pairs' divisor
    int bits = 0, W = 1;                     // packed key bits (fixed per plan) and words
    cb::u64 nullmask[cb::SK_MAX_WORDS] = {0, 0, 0, 0};

    bool built = false;
    Batch build;                             // the build side's rows, concatenated
    DeviceBufP keys, rows, run_start, slots; // sorted build keys and their rows, run starts (+ the end), the table
    DeviceBufP hit;                          // FullOuter: one byte per run, set when a probe row finds it
    std::shared_ptr<JoinCondition> cond;     // the join condition, or null
    DeviceBufP row_hit;                      // FullOuter with a condition: one byte per build row, set when a pair of it passes
    int64_t n_runs = 0;
    JoinTable table{};
    uint32_t h_build_rows = 0;
    std::vector<DictCodes> build_canon, probe_canon; // per key and side: dictionary code -> canonical code (canonical_codes)
    std::vector<Column> probe_like;          // the columns of the last probe batch: the layout of all-NULL probe columns
    bool probe_done = false;

    // what the rows being emitted are: (probe, build) pairs, probe rows (kept_rows), or FullOuter's unmatched build rows (kept_rows)
    // what the rows being emitted are: (probe, build) pairs, probe rows (kept_rows), FullOuter's unmatched build rows (kept_rows), or
    // the pairs a condition kept from one slice (kept_probe, kept_build)
    enum class Emit { Pairs, ProbeRows, BuildRows, KeptPairs } src = Emit::Pairs;
    Batch probe;                             // the probe batch being emitted ...
    DeviceBufP run_of, offs, chunk_off, kept_rows;
    int64_t total = 0, pos = 0;              // ... its output rows, and those emitted
    // a probe batch with a condition: the pass bit of each pair, the probe rows with a passing pair, the pairs, those resolved (phase 2)
    DeviceBufP pass_bits, passed, kept_probe, kept_build;
    int64_t cand_total = 0, cand_pos = 0;
    int64_t grp0 = 0, grp_end = 0;           // nested-loop join with a condition: the probe rows of the current group, [grp0, grp_end)

    bool outer() const { return type == JoinType::LeftOuter || type == JoinType::RightOuter || type == JoinType::FullOuter; }
    bool semi_anti() const { return type == JoinType::LeftSemi || type == JoinType::LeftAnti; }
    std::vector<ExecNodeP> children() const override { return {build_left ? build_child : probe_child, build_left ? probe_child : build_child}; }
    std::vector<PipelineSpec> build_specs() const override { return cond ? std::vector<PipelineSpec>{cond->spec(nullptr)} : std::vector<PipelineSpec>{}; }
    // pairs per condition slice: at most chunkRows, a multiple of 32 so that each slice's pass bits start on a word
    int64_t cond_slice() const { return std::max<int64_t>(32, ctx->chunk_rows / 32 * 32); }
    // nested-loop join with a condition: probe rows per group, at most chunkRows pairs (one row when m exceeds it)
    int64_t group_rows() const { return std::max<int64_t>(1, std::max<int64_t>(ctx->chunk_rows, 1) / build.n_rows); }
    // a nested-loop inner / outer join with a condition has probe rows left in the batch after the current group (with an empty build
    // side an outer join's probe rows are NULL-extended whole, without groups)
    bool more_groups() const { return nested && cond && !semi_anti() && build.n_rows > 0 && grp_end < probe.n_rows; }
    // the key layout from the declared key types: the last key is the least significant field, each with a null bit above its value
    void set_layout(const std::vector<DType>& key_types) {
        bits = 0;
        for (size_t k = key_types.size(); k-- > 0;) bits += sort_key_bits(key_types[k]) + 1;
        W = std::max(1, (bits + 63) / 64);
        int off = 0;
        for (size_t k = key_types.size(); k-- > 0;) {
            off += sort_key_bits(key_types[k]);
            cb::sk_put(nullmask, W, off, 1, 1);
            off++;
        }
    }

    cb::SortKeyCols key_cols(const Batch& b, const std::vector<int>& cols, bool build_side) {
        cb::SortKeyCols kc;
        memset(&kc, 0, sizeof(kc));
        kc.n = (int)cols.size();
        kc.words = W;
        kc.err = ctx->d_err;
        std::vector<DictCodes>& canon = build_side ? build_canon : probe_canon;
        canon.resize(cols.size());
        int off = 0;
        for (size_t k = cols.size(); k-- > 0;) {
            const Column& c = b.cols.at((size_t)cols[k]);
            cb::SortKeyCol& f = kc.col[k] = key_field(c, true, off);
            f.nulls_first = 1; // null bit set on a valid value
            if (c.is_dict) {
                const Dictionary& bd = *build.cols[(size_t)build_keys[k]].dict; // c's own when b is the build side
                f.rank = canon[k].get(c.dict, ctx, [&bd](const Dictionary& d) { return canonical_codes(d, bd); });
            }
        }
        return kc;
    }

    void build_table() {
        built = true;
        build = drain(*build_child, ctx, "joining", nested ? "nested-loop join build" : "hash join build");
        ctx->join_build_rows += build.n_rows;
        if (build.n_rows == 0) return;
        if (nested) {
            if (build.n_rows >= ((int64_t)1 << 32)) throw Unsupported("a nested-loop join build side of 2^32 rows or more");
            nlj_inv = ~0ull / (unsigned long long)build.n_rows;
            return;
        }
        TraceSpan ts("join.build");
        const int64_t n = build.n_rows;
        if (n >= ((int64_t)1 << 32)) throw Unsupported("a hash join build side of 2^32 rows or more");
        cudaStream_t st = ctx->stream;
        RowKeys rk = pack_row_keys(key_cols(build, build_keys, true), n, bits, ctx);
        rows = radix_order(ctx, rk.keys, W, n, rk.digits, &keys);
        rk.keys.reset();
        auto head = std::make_shared<DeviceBuf>((size_t)n + 16);
        launch_join_heads((const unsigned long long*)keys->ptr, W, n, (unsigned char*)head->ptr, st);
        ctx->kernel_launches++;
        const Compacted runs = compact_rows(head, n, n + 1, ctx); // run starts, then the end at [n_runs]
        n_runs = runs.n;
        run_start = runs.rows;
        h_build_rows = (uint32_t)n;
        cuda_check(cudaMemcpyAsync((uint32_t*)run_start->ptr + n_runs, &h_build_rows, 4, cudaMemcpyHostToDevice, st), "H2D run end");
        size_t cap = 1024;
        while (cap < (size_t)n_runs * 2) cap <<= 1;
        slots = std::make_shared<DeviceBuf>(cap * 8);
        cuda_check(cudaMemsetAsync(slots->ptr, 0, cap * 8, st), "memset join table");
        table.keys = (const unsigned long long*)keys->ptr;
        table.rows = (const unsigned*)rows->ptr;
        table.run_start = (const unsigned*)run_start->ptr;
        table.slots = (unsigned long long*)slots->ptr;
        table.mask = cap - 1;
        table.words = W;
        for (int j = 0; j < cb::SK_MAX_WORDS; j++) table.nullmask[j] = nullmask[j];
        launch_join_insert(table, n_runs, st);
        cuda_check(cudaGetLastError(), "k_join_insert launch");
        ctx->kernel_launches++;
        if (type == JoinType::FullOuter && cond) {
            row_hit = std::make_shared<DeviceBuf>((size_t)n + 16);
            cuda_check(cudaMemsetAsync(row_hit->ptr, 0, (size_t)n, st), "memset join row hits");
        } else if (type == JoinType::FullOuter) {
            hit = std::make_shared<DeviceBuf>((size_t)n_runs);
            cuda_check(cudaMemsetAsync(hit->ptr, 0, (size_t)n_runs, st), "memset join hits");
        }
        ctx->check_device_errors();
    }

    // the lookups of probe batch `in`: `total` output rows to emit from it
    void probe_batch(Batch& in) {
        TraceSpan ts("join.probe");
        const int64_t n = in.n_rows;
        if (n >= ((int64_t)1 << 32)) throw Unsupported("a hash join probe batch of 2^32 rows or more");
        cudaStream_t st = ctx->stream;
        pos = 0;
        if (build.n_rows == 0) { // an outer join with nothing to match: every probe row, NULL-extended
            probe = std::move(in);
            kept_rows = std::make_shared<DeviceBuf>((size_t)n * 4);
            launch_sort_iota((unsigned*)kept_rows->ptr, n, st);
            ctx->kernel_launches++;
            src = Emit::ProbeRows;
            total = n;
            return;
        }
        if (nested) {
            probe = std::move(in);
            nested_batch();
            return;
        }
        const DeviceBufP pk = pack_row_keys(key_cols(in, probe_keys, false), n, bits, ctx).keys;
        probe = std::move(in);
        if (!semi_anti() || cond) {
            const size_t n_chunks = (size_t)(n + CB_SCAN_CHUNK - 1) / CB_SCAN_CHUNK;
            run_of = std::make_shared<DeviceBuf>((size_t)n * 4);
            offs = std::make_shared<DeviceBuf>((size_t)n * 4);
            chunk_off = std::make_shared<DeviceBuf>((n_chunks + 1) * 4);
            auto tot = std::make_shared<DeviceBuf>(16);
            cuda_check(cudaMemsetAsync(tot->ptr, 0, 16, st), "memset join total");
            launch_join_probe(table, (const unsigned long long*)pk->ptr, n, outer() ? CB_JOIN_OUTER : CB_JOIN_COUNT, (unsigned*)offs->ptr,
                              (unsigned*)run_of->ptr, (unsigned long long*)tot->ptr, nullptr, hit ? (unsigned char*)hit->ptr : nullptr, st);
            launch_scan_u32((unsigned*)offs->ptr, n, CB_SCAN_CHUNK, (unsigned*)chunk_off->ptr, (long long*)tot->ptr + 1, st);
            cuda_check(cudaGetLastError(), "join probe");
            ctx->kernel_launches += 3;
            cuda_check(cudaMemcpyAsync(&total, tot->ptr, 8, cudaMemcpyDeviceToHost, st), "D2H join total");
            ctx->check_device_errors();
            // the scan's offsets are 32-bit
            if (total >= ((int64_t)1 << 32))
                throw Unsupported(std::string("a probe batch whose ") + (cond ? "join condition candidates number" : outer() ? "outer join output has" : "inner join output has") +
                                  " 2^32 rows or more (lower spark.comet.b200.chunkRows)");
            if (cond) { evaluate_condition(); return; }
            src = Emit::Pairs;
        } else {
            auto keep = std::make_shared<DeviceBuf>((size_t)n + 16);
            launch_join_probe(table, (const unsigned long long*)pk->ptr, n, type == JoinType::LeftSemi ? CB_JOIN_SEMI : CB_JOIN_ANTI, nullptr, nullptr, nullptr,
                              (unsigned char*)keep->ptr, nullptr, st);
            ctx->kernel_launches++;
            Compacted c = compact_rows(keep, n, n, ctx);
            kept_rows = c.rows;
            total = c.n;
            src = Emit::ProbeRows;
        }
    }

    // phase 1 of a probe batch with a condition (total = its pairs): the pass bits and `passed`; semi / anti joins then compact the probe
    // rows they keep, inner and outer ones resolve the pairs slice by slice (resolve_slice)
    void evaluate_condition() {
        TraceSpan ts("join.condition");
        const int64_t n = probe.n_rows;
        pass_bits = std::make_shared<DeviceBuf>((size_t)(total + 31) / 32 * 4 + 8);
        passed = std::make_shared<DeviceBuf>((size_t)n + 16);
        cuda_check(cudaMemsetAsync(passed->ptr, 0, (size_t)n, ctx->stream), "memset join passed");
        mark_pairs(total);
        pos = 0;
        if (semi_anti()) keep_passed_rows();
        else {
            cand_total = total;
            cand_pos = 0;
            total = 0;
            src = Emit::KeptPairs;
        }
    }

    // the pairs at positions [p0, p0 + k): of the probe batch (sentinels: an outer join's pair of a probe row without a match), or of
    // the current group of a nested-loop join
    void pairs_at(int64_t p0, int64_t k, bool sentinels, unsigned* pidx, unsigned* bidx) {
        if (nested) launch_nlj_pairs(p0, k, (unsigned)grp0, (unsigned)build.n_rows, nlj_inv, pidx, bidx, ctx->stream);
        else launch_join_emit(table, (const unsigned*)run_of->ptr, (const unsigned*)offs->ptr, (const unsigned*)chunk_off->ptr, probe.n_rows, p0,
                              p0 + k, sentinels, pidx, bidx, ctx->stream);
        cuda_check(cudaGetLastError(), nested ? "k_nlj_pairs launch" : "k_join_emit launch");
    }

    // phase 1 over `count` pairs (pairs_at): their pass bits from bit 0 of pass_bits, `passed`, and the candidates counted.  A hash
    // join's outer sentinel pairs take part with NULLs on both sides; a nested-loop join has none.
    void mark_pairs(int64_t count) {
        cudaStream_t st = ctx->stream;
        const int64_t S = cond_slice();
        const bool sentinels = outer() && !nested;
        auto n_cand = std::make_shared<DeviceBuf>(8);
        cuda_check(cudaMemsetAsync(n_cand->ptr, 0, 8, st), "memset join candidates");
        const size_t cap = (size_t)std::max<int64_t>(std::min(S, count), 1) * 4;
        auto pidx = std::make_shared<DeviceBuf>(cap), bidx = std::make_shared<DeviceBuf>(cap);
        for (int64_t s = 0; s < count; s += S) {
            const int64_t k = std::min(S, count - s);
            if (sentinels) { // the sentinel pairs' slots stay (CB_NULL_ROW, CB_NULL_ROW): all NULLs
                cuda_check(cudaMemsetAsync(pidx->ptr, 0xff, (size_t)k * 4, st), "memset join pairs");
                cuda_check(cudaMemsetAsync(bidx->ptr, 0xff, (size_t)k * 4, st), "memset join pairs");
            }
            pairs_at(s, k, false, (unsigned*)pidx->ptr, (unsigned*)bidx->ptr);
            cb::u32* bits = (cb::u32*)pass_bits->ptr + s / 32;
            cond->eval(probe, build, build_left, (const unsigned*)pidx->ptr, (const unsigned*)bidx->ptr, k, sentinels, bits);
            launch_join_cond_mark(bits, (const unsigned*)pidx->ptr, (const unsigned*)bidx->ptr, k, (unsigned char*)passed->ptr,
                                  row_hit ? (unsigned char*)row_hit->ptr : nullptr, (unsigned long long*)n_cand->ptr, st);
            cuda_check(cudaGetLastError(), "k_join_cond_mark launch");
            ctx->kernel_launches += 2;
        }
        int64_t* h_cand = (int64_t*)ctx->h_err + 1; // pinned scratch next to the error flag
        cuda_check(cudaMemcpyAsync(h_cand, n_cand->ptr, 8, cudaMemcpyDeviceToHost, st), "D2H join candidates");
        ctx->check_device_errors(); // also synchronises: the condition's ANSI errors are raised here
        ctx->join_cond_pairs += *h_cand;
    }

    // semi / anti joins once `passed` is final: the probe rows they keep
    void keep_passed_rows() {
        const int64_t n = probe.n_rows;
        DeviceBufP keep = passed;
        if (type == JoinType::LeftAnti) {
            keep = std::make_shared<DeviceBuf>((size_t)n + 16);
            launch_flags_not((const unsigned char*)passed->ptr, n, (unsigned char*)keep->ptr, ctx->stream);
            ctx->kernel_launches++;
        }
        Compacted c = compact_rows(keep, n, n, ctx);
        kept_rows = c.rows;
        total = c.n;
        pos = 0;
        src = Emit::ProbeRows;
        pass_bits.reset(); passed.reset(); run_of.reset(); offs.reset(); chunk_off.reset();
    }

    // a nested-loop join's probe batch, the build side not empty (semi / anti joins without a condition never get here): without a
    // condition every pair is output; with one, semi / anti joins run phase 1 over every group, inner / outer ones start the first group
    void nested_batch() {
        const int64_t n = probe.n_rows, m = build.n_rows;
        pos = 0;
        grp0 = grp_end = 0;
        if (!cond) {
            total = n * m;
            src = Emit::Pairs;
            return;
        }
        pass_bits = std::make_shared<DeviceBuf>((size_t)((std::min(n, group_rows()) * m + 31) / 32) * 4 + 8);
        passed = std::make_shared<DeviceBuf>((size_t)n + 16);
        cuda_check(cudaMemsetAsync(passed->ptr, 0, (size_t)n, ctx->stream), "memset join passed");
        if (semi_anti()) {
            while (grp_end < n) nested_group();
            keep_passed_rows();
        } else nested_group();
    }

    // phase 1 over the next group's pairs; an inner / outer join then resolves them slice by slice (resolve_slice)
    void nested_group() {
        TraceSpan ts("join.condition");
        grp0 = grp_end;
        grp_end = std::min(probe.n_rows, grp0 + group_rows());
        const int64_t count = (grp_end - grp0) * build.n_rows;
        mark_pairs(count);
        if (semi_anti()) return;
        cand_total = count;
        cand_pos = 0;
        total = 0;
        pos = 0;
        src = Emit::KeptPairs;
    }

    // phase 2, inner and outer joins: the kept pairs of the next slice (possibly none)
    void resolve_slice() {
        TraceSpan ts("join.condition.resolve");
        cudaStream_t st = ctx->stream;
        const int64_t k = std::min(cond_slice(), cand_total - cand_pos);
        auto pidx = std::make_shared<DeviceBuf>((size_t)k * 4), bidx = std::make_shared<DeviceBuf>((size_t)k * 4);
        auto keep = std::make_shared<DeviceBuf>((size_t)k + 16);
        if (nested) {
            launch_nlj_cond_resolve((const unsigned*)pass_bits->ptr, cand_pos, k, (unsigned)grp0, (unsigned)build.n_rows, nlj_inv,
                                    (const unsigned char*)passed->ptr, outer(), (unsigned*)pidx->ptr, (unsigned*)bidx->ptr, (unsigned char*)keep->ptr, st);
            ctx->kernel_launches++;
        } else {
            launch_join_emit(table, (const unsigned*)run_of->ptr, (const unsigned*)offs->ptr, (const unsigned*)chunk_off->ptr, probe.n_rows, cand_pos,
                             cand_pos + k, outer(), (unsigned*)pidx->ptr, (unsigned*)bidx->ptr, st);
            launch_join_cond_resolve((const unsigned*)pass_bits->ptr, cand_pos, (const unsigned*)pidx->ptr, (unsigned*)bidx->ptr, k, (const unsigned*)offs->ptr,
                                     (const unsigned*)chunk_off->ptr, (const unsigned char*)passed->ptr, outer(), (unsigned char*)keep->ptr, st);
            ctx->kernel_launches += 2;
        }
        cuda_check(cudaGetLastError(), "join condition resolve");
        Compacted c = compact_rows(keep, k, k, ctx, {{pidx, 4}, {bidx, 4}});
        kept_probe = c.extra_out[0];
        kept_build = c.extra_out[1];
        total = c.n;
        pos = 0;
        cand_pos += k;
    }

    // FullOuter, once the probe side has ended: the build rows no probe row matched, in build input order
    void unmatched_build_rows() {
        TraceSpan ts("join.unmatched");
        const int64_t n = build.n_rows;
        auto keep = std::make_shared<DeviceBuf>((size_t)n + 16);
        if (row_hit) launch_flags_not((const unsigned char*)row_hit->ptr, n, (unsigned char*)keep->ptr, ctx->stream);
        else launch_join_unmatched((const unsigned*)run_start->ptr, n_runs, (const unsigned*)rows->ptr, (const unsigned char*)hit->ptr, n,
                                   (unsigned char*)keep->ptr, ctx->stream);
        cuda_check(cudaGetLastError(), "k_join_unmatched launch");
        ctx->kernel_launches++;
        Compacted c = compact_rows(keep, n, n, ctx);
        kept_rows = c.rows;
        total = c.n;
        pos = 0;
        src = Emit::BuildRows;
    }

    // all-NULL columns of one side, k rows: the probe side in the layout of its last batch, the build side in the layout of its rows
    Batch null_side(bool build_side, int64_t k) {
        const std::vector<DType>& types = build_side ? build_child->schema : probe_child->schema;
        const std::vector<Column>& like = build_side ? build.cols : probe_like;
        Batch b;
        b.n_rows = k;
        for (size_t j = 0; j < types.size(); j++) b.cols.push_back(null_column(types[j], like.empty() ? nullptr : &like[j], k, ctx));
        return b;
    }

    // the next at most chunkRows output rows
    void emit(Batch& out) {
        const int64_t k = std::min<int64_t>(total - pos, std::max<int64_t>(ctx->chunk_rows, 1));
        const bool null_probe = type == JoinType::FullOuter; // the probe side may be NULL-extended
        Batch pb, bb;
        if (src == Emit::Pairs || src == Emit::KeptPairs) {
            DeviceBufP pidx, bidx;
            const unsigned *pi, *bi;
            if (src == Emit::Pairs) {
                pidx = std::make_shared<DeviceBuf>((size_t)k * 4);
                bidx = std::make_shared<DeviceBuf>((size_t)k * 4);
                pairs_at(pos, k, outer(), (unsigned*)pidx->ptr, (unsigned*)bidx->ptr);
                ctx->kernel_launches++;
                pi = (const unsigned*)pidx->ptr;
                bi = (const unsigned*)bidx->ptr;
            } else {
                pi = (const unsigned*)kept_probe->ptr + pos;
                bi = (const unsigned*)kept_build->ptr + pos;
            }
            if (null_probe) gather_columns_or_null(probe, pi, k, pb, ctx);
            else gather_columns(probe, pi, k, pb, ctx, "joining");
            if (outer()) gather_columns_or_null(build, bi, k, bb, ctx);
            else gather_columns(build, bi, k, bb, ctx, "joining");
        } else if (src == Emit::ProbeRows) {
            const unsigned* idx = (const unsigned*)kept_rows->ptr + pos;
            if (null_probe) gather_columns_or_null(probe, idx, k, pb, ctx);
            else gather_columns(probe, idx, k, pb, ctx, "joining");
            if (outer()) bb = null_side(true, k);
        } else {
            gather_columns_or_null(build, (const unsigned*)kept_rows->ptr + pos, k, bb, ctx);
            pb = null_side(false, k);
        }
        if (semi_anti()) out = std::move(pb);
        else {
            Batch& l = build_left ? bb : pb;
            Batch& r = build_left ? pb : bb;
            out.n_rows = k;
            out.cols = std::move(l.cols);
            for (auto& c : r.cols) out.cols.push_back(std::move(c));
        }
        pos += k;
        ctx->join_out_rows += k;
        ctx->check_device_errors();
        if (pos >= total && cand_pos >= cand_total && !more_groups()) {
            probe = Batch(); run_of.reset(); offs.reset(); chunk_off.reset(); kept_rows.reset();
            pass_bits.reset(); passed.reset(); kept_probe.reset(); kept_build.reset();
        }
    }

    // Empty sides: an empty build side gives no rows for inner and semi joins, every probe row for anti and outer joins; an empty probe
    // side gives no rows but FullOuter's unmatched build rows (all of them).
    bool next(Batch& out) override {
        if (!built) build_table();
        const bool empty_build = build.n_rows == 0;
        if (empty_build && (type == JoinType::Inner || type == JoinType::LeftSemi)) return false; // nothing matches
        for (;;) {
            if (pos < total) { emit(out); return true; }
            if (cand_pos < cand_total) { resolve_slice(); continue; }
            if (more_groups()) { nested_group(); continue; }
            if (probe_done) return false;
            Batch in;
            if (!probe_child->next(in)) {
                probe_done = true;
                if (type == JoinType::FullOuter && !empty_build) unmatched_build_rows();
                continue;
            }
            arrive(in, ctx, "joining");
            ctx->join_probe_rows += in.n_rows;
            if (!in.cols.empty()) { // its layout only: the batch's buffers are not kept alive
                probe_like.assign(in.cols.size(), Column());
                for (size_t j = 0; j < in.cols.size(); j++) {
                    const Column& c = in.cols[j];
                    probe_like[j].type = c.type; probe_like[j].phys = c.phys; probe_like[j].is_dict = c.is_dict; probe_like[j].dict = c.dict;
                }
            }
            if (in.n_rows == 0) continue;
            if (empty_build && type == JoinType::LeftAnti) { // every probe row
                ctx->join_out_rows += in.n_rows;
                out = std::move(in);
                return true;
            }
            if (nested && !cond && semi_anti()) { // the build side is not empty and every pair passes: LeftSemi keeps the batch, LeftAnti none of it
                if (type == JoinType::LeftAnti) continue;
                ctx->join_out_rows += in.n_rows;
                out = std::move(in);
                return true;
            }
            probe_batch(in);
        }
    }
};

ExecNodeP make_join_node(const OperatorP& op, const ExecNodeP& left, const ExecNodeP& right, ExecContext* ctx) {
    auto n = std::make_shared<JoinNode>();
    n->ctx = ctx;
    n->schema = op->schema;
    n->type = op->join_type;
    n->build_left = op->build_left;
    n->nested = op->left_keys.empty();
    std::vector<int> lk, rk;
    std::vector<DType> key_types;
    for (size_t i = 0; i < op->left_keys.size(); i++) {
        lk.push_back(op->left_keys[i]->index);
        rk.push_back(op->right_keys[i]->index);
        key_types.push_back(op->left_keys[i]->type);
    }
    n->build_child = op->build_left ? left : right;
    n->probe_child = op->build_left ? right : left;
    n->build_keys = op->build_left ? lk : rk;
    n->probe_keys = op->build_left ? rk : lk;
    n->set_layout(key_types);
    if (op->join_condition) {
        auto c = std::make_shared<JoinCondition>();
        auto cols = std::make_shared<JoinCondition::Columns>();
        cols->schema = left->schema;
        cols->schema.insert(cols->schema.end(), right->schema.begin(), right->schema.end());
        c->ctx = ctx;
        c->child = cols;
        c->n_left = (int)left->schema.size();
        c->predicates = {op->join_condition};
        c->assign_slots(c->predicates);
        if (c->used_cols.empty()) { // a condition of literals alone: the pass still needs a staged column, the first left key (without
                                    // keys, the probe side's first column)
            const int staged = lk.empty() ? (op->build_left ? c->n_left : 0) : lk[0];
            c->used_cols.push_back(staged);
            c->slot_of[staged] = 0;
        }
        n->cond = c;
    }
    return n;
}

} // namespace cb200
