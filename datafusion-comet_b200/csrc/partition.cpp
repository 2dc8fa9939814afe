// partition.cpp -- repartitioning (ShuffleWriterExec, native/shuffle/src/partitioners/multi_partition.rs): hash, single, range and
// round-robin partitioning.
#include "exec_internal.h"

#include "device/cb_rangepart.h"

namespace cb200 {

// Output: the child's rows reordered so that partition p occupies rows [starts[p], starts[p+1]) -- what the
// reference writes as per-partition IPC blocks, kept on the device for the NVLink exchange.  A row's partition id is:
//   hash / single : pmod(murmur3 seed 42 chained over key_cols, n_parts)
//   round-robin   : the same over the first columns (multi_partition.rs:386-430); more than 8 of them chain one launch per 8 columns
//   range         : the number of boundary rows <= the row under the sort orders (multi_partition.rs:333-380), by k_range_pids over
//                   the bounds the planner packed; ids stay below n_bounds + 1, the later partitions are empty
// and every kind shares the stable placement and the gathers.
struct PartitionNode : ExecNode {
    ExecContext* ctx;
    ExecNodeP child;
    PartKind kind = PartKind::Hash;
    std::vector<int> key_cols;
    int n_parts = 1;
    // range
    std::vector<SortKey> range_keys;
    std::vector<std::vector<std::string>> range_strs;
    int words = 1;
    uint32_t n_bounds = 0, n_top = 0;
    int shift = 0;
    DeviceBufP bounds, top;             // uploaded on the first batch
    std::vector<uint64_t> h_bounds;
    std::vector<DictCodes> ranks;       // per range key: dictionary code -> rank against the boundary strings
    cudaEvent_t ev[4] = {};             // around the stages: ids, placement, gather (cb200_stats partition_*_ms)

    ~PartitionNode() override {
        for (cudaEvent_t e : ev)
            if (e) cudaEventDestroy(e);
    }
    void mark(int k) {
        if (!ev[k]) cuda_check(cudaEventCreate(&ev[k]), "event create");
        cuda_check(cudaEventRecord(ev[k], ctx->stream), "event record");
    }
    double between(int a, int b) {
        float ms = 0;
        cuda_check(cudaEventElapsedTime(&ms, ev[a], ev[b]), "event time");
        return ms;
    }
    std::vector<ExecNodeP> children() const override { return {child}; }

    // the HashKeyCol of column c (dictionaries uploaded into keep)
    static HashKeyCol hash_key(const Column& c, std::vector<DeviceBufP>& keep, ExecContext* ctx) {
        HashKeyCol k;
        memset(&k, 0, sizeof(k));
        k.data = c.data ? c.data->ptr : nullptr;
        k.validity = c.validity ? (const unsigned char*)c.validity->ptr : nullptr;
        k.kind = key_kind(c);
        switch (k.kind) {
        case HK_DICT8: case HK_DICT16: case HK_DICT32: { // the dictionary as offsets, then chars, in one upload
            std::vector<int32_t> off{0};
            for (auto& v : c.dict->values()) off.push_back(off.back() + (int32_t)v.size());
            std::string blob((const char*)off.data(), off.size() * 4);
            for (auto& v : c.dict->values()) blob += v;
            keep.push_back(host_to_device(blob.data(), blob.size(), ctx, "dict upload"));
            k.dict_offsets = (const int*)keep.back()->ptr;
            k.dict_chars = (const unsigned char*)keep.back()->ptr + off.size() * 4;
            break;
        }
        case HK_UTF8:
            if (!c.offsets || !c.chars) throw Unsupported("string partition key without offsets/chars");
            k.dict_offsets = (const int*)c.offsets->ptr;
            k.dict_chars = (const unsigned char*)c.chars->ptr;
            break;
        default: break;
        }
        return k;
    }

    // pids of a range or long round-robin partitioning
    void range_or_chain_pids(const Batch& in, unsigned* pids) {
        const int64_t n = in.n_rows;
        cudaStream_t st = ctx->stream;
        if (kind == PartKind::Range) {
            cb::SortKeyCols kc;
            memset(&kc, 0, sizeof(kc));
            kc.n = (int)range_keys.size();
            kc.words = words;
            kc.err = ctx->d_err;
            ranks.resize(range_keys.size());
            int off = 0;
            for (size_t k = range_keys.size(); k-- > 0;) { // the last key is the least significant field, as the planner packed the bounds
                const Column& c = in.cols.at((size_t)range_keys[k].expr->index);
                if (c.offsets) throw Unsupported("range partitioning plain string columns (dictionary-encode them first)");
                cb::SortKeyCol& f = kc.col[k] = key_field(c, true, off);
                f.desc = range_keys[k].descending;
                f.nulls_first = range_keys[k].nulls_first;
                const auto& strs = range_strs[k];
                if (c.is_dict) f.rank = ranks[k].get(c.dict, ctx, [&](const Dictionary& d) { return cb::rp_string_ranks(d.values(), strs); });
            }
            if (!bounds) { // uploaded once; no boundary rows: a placeholder the kernel never reads
                auto upload = [&](const std::vector<uint64_t>& v, const char* what) {
                    return v.empty() ? std::make_shared<DeviceBuf>(8) : host_to_device(v.data(), v.size() * 8, ctx, what);
                };
                bounds = upload(h_bounds, "H2D range bounds");
                std::vector<uint64_t> t;
                if (shift == 0) top = bounds;
                else {
                    for (uint32_t j = 0; j < n_top; j++)
                        t.insert(t.end(), h_bounds.begin() + (((size_t)(j + 1) << shift) - 1) * words, h_bounds.begin() + ((size_t)(j + 1) << shift) * words);
                    top = upload(t, "H2D range bound samples");
                }
                ctx->h2d_bytes += (int64_t)((h_bounds.size() + t.size()) * 8);
            }
            cuda_check(launch_range_pids(kc, n, (const unsigned long long*)top->ptr, n_top, shift, (const unsigned long long*)bounds->ptr, n_bounds, pids, st),
                       "range partition ids");
            ctx->kernel_launches++;
        } else { // round-robin over more than 8 columns: groups of 8 chained through the running hash
            std::vector<DeviceBufP> keep;
            auto hashes = std::make_shared<DeviceBuf>((size_t)n * 4 + 16);
            for (size_t g = 0; g < key_cols.size(); g += 8) {
                HashKeyCols kc;
                memset(&kc, 0, sizeof(kc));
                for (size_t j = g; j < std::min(key_cols.size(), g + 8); j++) kc.col[kc.n++] = hash_key(in.cols[(size_t)key_cols[j]], keep, ctx);
                cuda_check(launch_partition_ids_chain(kc, n, (unsigned)n_parts, g == 0, g + 8 >= key_cols.size(), (unsigned*)hashes->ptr, pids, st),
                           "round-robin partition ids");
                ctx->kernel_launches++;
            }
        }
    }

    bool next(Batch& out) override {
        Batch in;
        if (!child->next(in)) return false;
        TraceSpan ts("partition");
        columns_to_device(in, ctx);
        int64_t n = in.n_rows;
        cudaStream_t st = ctx->stream;
        const bool by_pids = kind == PartKind::Range || key_cols.size() > 8;
        HashKeyCols kc;
        memset(&kc, 0, sizeof(kc));
        std::vector<DeviceBufP> keep;
        if (!by_pids)
            for (int ci : key_cols) kc.col[kc.n++] = hash_key(in.cols[(size_t)ci], keep, ctx);
        size_t nb = (size_t)(n + 1023) / 1024 + 1;
        auto pids = std::make_shared<DeviceBuf>((size_t)n * 4 + 16);
        auto hist = std::make_shared<DeviceBuf>(nb * n_parts * 4);
        auto base = std::make_shared<DeviceBuf>(nb * n_parts * 8);
        auto starts = std::make_shared<DeviceBuf>((size_t)(n_parts + 1) * 8);
        auto row_idx = std::make_shared<DeviceBuf>((size_t)n * 8 + 16);
        cuda_check(cudaMemsetAsync(starts->ptr, 0, (size_t)(n_parts + 1) * 8, st), "memset starts");
        auto chunk_tmp = std::make_shared<DeviceBuf>((size_t)(partition_chunks(n) + 1) * n_parts * 8);
        mark(0);
        if (by_pids) range_or_chain_pids(in, (unsigned*)pids->ptr);
        else {
            cuda_check(launch_partition_ids(kc, n, (unsigned)n_parts, nullptr, (unsigned*)pids->ptr, st), "partition ids");
            ctx->kernel_launches++;
        }
        mark(1);
        cuda_check(launch_partition_place((const unsigned*)pids->ptr, n, (unsigned)n_parts, (int*)hist->ptr, (long long*)base->ptr,
                                          (long long*)chunk_tmp->ptr, (long long*)starts->ptr, (long long*)row_idx->ptr, st), "partition placement");
        ctx->kernel_launches += 5;
        mark(2);
        gather_columns(in, (const long long*)row_idx->ptr, n, out, ctx, "repartitioning");
        mark(3);
        ctx->partition_starts.assign((size_t)n_parts + 1, 0);
        cuda_check(cudaMemcpyAsync(ctx->partition_starts.data(), starts->ptr, (size_t)(n_parts + 1) * 8, cudaMemcpyDeviceToHost, st), "starts D2H"); ctx->d2h_bytes += (int64_t)((size_t)(n_parts + 1) * 8);
        ctx->check_device_errors(); // also synchronises: the events have completed
        ctx->partition_ids_ms += between(0, 1);
        ctx->partition_place_ms += between(1, 2);
        ctx->partition_gather_ms += between(2, 3);
        return true;
    }
};

ExecNodeP make_partition_node(const OperatorP& op, const ExecNodeP& child, ExecContext* ctx) {
    auto n = std::make_shared<PartitionNode>();
    n->ctx = ctx;
    n->child = child;
    n->schema = op->schema;
    n->kind = op->part_kind;
    n->n_parts = op->num_partitions;
    const char* what = op->part_kind == PartKind::Range ? "range" : op->part_kind == PartKind::RoundRobin ? "round-robin" : "hash";
    for (auto& e : op->hash_exprs) {
        if (e->kind != ExprKind::Bound) throw Unsupported("computed hash-partition keys (only plain column keys)");
        n->key_cols.push_back(e->index);
    }
    if (n->key_cols.size() > 8 && op->part_kind == PartKind::Hash) throw Unsupported("more than 8 hash-partition keys");
    if (n->n_parts > CB_MAX_HASH_PARTITIONS)
        throw Unsupported(std::string(what) + " partitioning into " + std::to_string(n->n_parts) + " partitions (at most " + std::to_string((int)CB_MAX_HASH_PARTITIONS) + ")");
    for (int ci : n->key_cols) { // refuses key types murmur3 has no rule for
        if (ci < 0 || ci >= (int)op->schema.size()) throw PlanError("hash-partition key out of range");
        Column c;
        c.type = op->schema[(size_t)ci];
        try {
            key_kind(c);
        } catch (const Unsupported&) {
            if (op->part_kind != PartKind::RoundRobin) throw;
            throw Unsupported("round-robin partitioning on column " + std::to_string(ci) + " of type " + c.type.str() + " (murmur3 has no rule for it)");
        }
    }
    if (op->part_kind == PartKind::Range) {
        n->range_keys = op->range_keys;
        n->range_strs = op->range_strs;
        n->words = op->range_words;
        n->h_bounds = op->range_bounds;
        n->n_bounds = (uint32_t)op->n_bounds;
        n->shift = cb::rp_shift(n->n_bounds, n->words, CB_RANGE_TOP_BYTES);
        n->n_top = n->n_bounds >> n->shift;
        for (auto& k : n->range_keys)
            if (k.expr->index < 0 || k.expr->index >= (int)op->schema.size()) throw PlanError("range-partition key out of range");
    }
    return n;
}

} // namespace cb200
