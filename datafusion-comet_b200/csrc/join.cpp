// join.cpp -- hash join (HashJoinExec with NullEquality::NullEqualsNothing, planner.rs:2192-2266): inner, left semi and left anti.
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
// an open-addressing table.  A probe batch then costs one key pass and one lookup per row; an inner join scans the match counts, writes
// the (probe row, build row) pairs and gathers both sides, a semi / anti join compacts the probe rows it keeps.  Output order: probe rows
// in input order, an inner-join row's matches in build input order; an inner join's output above spark.comet.b200.chunkRows rows leaves
// in several batches.
//
// Equal key tuples give equal words on both sides because the field layout is fixed by the declared key types (every field has a null
// bit, whatever a batch's validity) and a string field holds a canonical code rather than the dictionary code: the code of the first
// equal entry of the build side's dictionary, or that dictionary's size (which no build key has) for a probe string it lacks.
struct JoinNode : ExecNode {
    ExecContext* ctx;
    ExecNodeP build_child, probe_child;
    std::vector<int> build_keys, probe_keys; // key columns of each side, in key order
    JoinType type = JoinType::Inner;
    bool build_left = false;
    int bits = 0, W = 1;                     // packed key bits (fixed per plan) and words
    cb::u64 nullmask[cb::SK_MAX_WORDS] = {0, 0, 0, 0};

    bool built = false;
    Batch build;                             // the build side's rows, concatenated
    DeviceBufP keys, rows, run_start, slots; // sorted build keys and their rows, run starts (+ the end), the table
    JoinTable table{};
    uint32_t h_build_rows = 0;
    std::vector<DictCodes> build_canon, probe_canon; // per key and side: dictionary code -> canonical code (canonical_codes)

    Batch probe;                             // the probe batch being emitted ...
    DeviceBufP run_of, offs, chunk_off, kept_rows;
    int64_t total = 0, pos = 0;              // ... its output rows, and those emitted

    std::vector<ExecNodeP> children() const override { return {build_left ? build_child : probe_child, build_left ? probe_child : build_child}; }
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
        build = drain(*build_child, ctx, "joining", "hash join build");
        ctx->join_build_rows += build.n_rows;
        if (build.n_rows == 0) return;
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
        const int64_t n_runs = runs.n;
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
        ctx->check_device_errors();
    }

    // the lookups of probe batch `in`: `total` output rows to emit from it
    void probe_batch(Batch& in) {
        TraceSpan ts("join.probe");
        const int64_t n = in.n_rows;
        if (n >= ((int64_t)1 << 32)) throw Unsupported("a hash join probe batch of 2^32 rows or more");
        cudaStream_t st = ctx->stream;
        const DeviceBufP pk = pack_row_keys(key_cols(in, probe_keys, false), n, bits, ctx).keys;
        probe = std::move(in);
        pos = 0;
        if (type == JoinType::Inner) {
            const size_t n_chunks = (size_t)(n + CB_SCAN_CHUNK - 1) / CB_SCAN_CHUNK;
            run_of = std::make_shared<DeviceBuf>((size_t)n * 4);
            offs = std::make_shared<DeviceBuf>((size_t)n * 4);
            chunk_off = std::make_shared<DeviceBuf>((n_chunks + 1) * 4);
            auto tot = std::make_shared<DeviceBuf>(16);
            cuda_check(cudaMemsetAsync(tot->ptr, 0, 16, st), "memset join total");
            launch_join_probe(table, (const unsigned long long*)pk->ptr, n, CB_JOIN_COUNT, (unsigned*)offs->ptr, (unsigned*)run_of->ptr,
                              (unsigned long long*)tot->ptr, nullptr, st);
            launch_scan_u32((unsigned*)offs->ptr, n, CB_SCAN_CHUNK, (unsigned*)chunk_off->ptr, (long long*)tot->ptr + 1, st);
            cuda_check(cudaGetLastError(), "join probe");
            ctx->kernel_launches += 3;
            cuda_check(cudaMemcpyAsync(&total, tot->ptr, 8, cudaMemcpyDeviceToHost, st), "D2H join total");
            ctx->check_device_errors();
            // the scan's offsets are 32-bit
            if (total >= ((int64_t)1 << 32)) throw Unsupported("a probe batch whose inner join output has 2^32 rows or more (lower spark.comet.b200.chunkRows)");
        } else {
            auto keep = std::make_shared<DeviceBuf>((size_t)n + 16);
            launch_join_probe(table, (const unsigned long long*)pk->ptr, n, type == JoinType::LeftSemi ? CB_JOIN_SEMI : CB_JOIN_ANTI, nullptr, nullptr, nullptr,
                              (unsigned char*)keep->ptr, st);
            ctx->kernel_launches++;
            Compacted c = compact_rows(keep, n, n, ctx);
            kept_rows = c.rows;
            total = c.n;
        }
    }

    // the next at most chunkRows output rows of the probe batch
    void emit(Batch& out) {
        const int64_t k = std::min<int64_t>(total - pos, std::max<int64_t>(ctx->chunk_rows, 1));
        if (type == JoinType::Inner) {
            auto pidx = std::make_shared<DeviceBuf>((size_t)k * 4), bidx = std::make_shared<DeviceBuf>((size_t)k * 4);
            launch_join_emit(table, (const unsigned*)run_of->ptr, (const unsigned*)offs->ptr, (const unsigned*)chunk_off->ptr, probe.n_rows, pos, pos + k,
                             (unsigned*)pidx->ptr, (unsigned*)bidx->ptr, ctx->stream);
            cuda_check(cudaGetLastError(), "k_join_emit launch");
            ctx->kernel_launches++;
            Batch pb, bb;
            gather_columns(probe, (const unsigned*)pidx->ptr, k, pb, ctx, "joining");
            gather_columns(build, (const unsigned*)bidx->ptr, k, bb, ctx, "joining");
            Batch& l = build_left ? bb : pb;
            Batch& r = build_left ? pb : bb;
            out.n_rows = k;
            out.cols = std::move(l.cols);
            for (auto& c : r.cols) out.cols.push_back(std::move(c));
        } else {
            gather_columns(probe, (const unsigned*)kept_rows->ptr + pos, k, out, ctx, "joining");
        }
        pos += k;
        ctx->join_out_rows += k;
        ctx->check_device_errors();
        if (pos >= total) { probe = Batch(); run_of.reset(); offs.reset(); chunk_off.reset(); kept_rows.reset(); }
    }

    bool next(Batch& out) override {
        if (!built) build_table();
        const bool empty_build = build.n_rows == 0;
        if (empty_build && type != JoinType::LeftAnti) return false; // nothing matches
        for (;;) {
            if (pos < total) { emit(out); return true; }
            Batch in;
            if (!probe_child->next(in)) return false;
            arrive(in, ctx, "joining");
            ctx->join_probe_rows += in.n_rows;
            if (in.n_rows == 0) continue;
            if (empty_build) { // anti: every probe row
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
    return n;
}

} // namespace cb200
