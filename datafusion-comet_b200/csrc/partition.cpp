// partition.cpp -- hash repartitioning (ShuffleWriterExec with HashPartition, native/shuffle/src/partitioners/multi_partition.rs).
#include "exec_internal.h"

namespace cb200 {

// Output: the child's rows reordered so that partition p occupies rows [starts[p], starts[p+1]) -- what the
// reference writes as per-partition IPC blocks, kept on the device for the NVLink exchange.
struct PartitionNode : ExecNode {
    ExecContext* ctx;
    ExecNodeP child;
    std::vector<int> key_cols;
    int n_parts = 1;

    std::vector<ExecNodeP> children() const override { return {child}; }
    bool next(Batch& out) override {
        Batch in;
        if (!child->next(in)) return false;
        TraceSpan ts("partition");
        columns_to_device(in, ctx);
        int64_t n = in.n_rows;
        cudaStream_t st = ctx->stream;
        HashKeyCols kc;
        memset(&kc, 0, sizeof(kc));
        std::vector<DeviceBufP> keep;
        for (int ci : key_cols) {
            const Column& c = in.cols[(size_t)ci];
            HashKeyCol& k = kc.col[kc.n++];
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
        }
        size_t nb = (size_t)(n + 1023) / 1024 + 1;
        auto pids = std::make_shared<DeviceBuf>((size_t)n * 4 + 16);
        auto hist = std::make_shared<DeviceBuf>(nb * n_parts * 4);
        auto base = std::make_shared<DeviceBuf>(nb * n_parts * 8);
        auto starts = std::make_shared<DeviceBuf>((size_t)(n_parts + 1) * 8);
        auto row_idx = std::make_shared<DeviceBuf>((size_t)n * 8 + 16);
        cuda_check(cudaMemsetAsync(starts->ptr, 0, (size_t)(n_parts + 1) * 8, st), "memset starts");
        auto chunk_tmp = std::make_shared<DeviceBuf>((size_t)(partition_chunks(n) + 1) * n_parts * 8);
        cuda_check(launch_partition(kc, n, (unsigned)n_parts, nullptr, (unsigned*)pids->ptr, (int*)hist->ptr, (long long*)base->ptr, (long long*)chunk_tmp->ptr,
                                    (long long*)starts->ptr, (long long*)row_idx->ptr, st), "partition launches");
        ctx->kernel_launches += 6;
        gather_columns(in, (const long long*)row_idx->ptr, n, out, ctx, "repartitioning");
        ctx->partition_starts.assign((size_t)n_parts + 1, 0);
        cuda_check(cudaMemcpyAsync(ctx->partition_starts.data(), starts->ptr, (size_t)(n_parts + 1) * 8, cudaMemcpyDeviceToHost, st), "starts D2H"); ctx->d2h_bytes += (int64_t)((size_t)(n_parts + 1) * 8);
        ctx->check_device_errors();
        return true;
    }
};

ExecNodeP make_partition_node(const OperatorP& op, const ExecNodeP& child, ExecContext* ctx) {
    auto n = std::make_shared<PartitionNode>();
    n->ctx = ctx;
    n->child = child;
    n->schema = op->schema;
    n->n_parts = op->num_partitions;
    for (auto& e : op->hash_exprs) {
        if (e->kind != ExprKind::Bound) throw Unsupported("computed hash-partition keys (only plain column keys)");
        n->key_cols.push_back(e->index);
    }
    if (n->key_cols.size() > 8) throw Unsupported("more than 8 hash-partition keys");
    if (n->n_parts > CB_MAX_HASH_PARTITIONS)
        throw Unsupported("hash partitioning into " + std::to_string(n->n_parts) + " partitions (at most " + std::to_string((int)CB_MAX_HASH_PARTITIONS) + ")");
    for (int ci : n->key_cols) { // refuses key types murmur3 has no rule for
        if (ci < 0 || ci >= (int)op->schema.size()) throw PlanError("hash-partition key out of range");
        Column c;
        c.type = op->schema[(size_t)ci];
        key_kind(c);
    }
    return n;
}

} // namespace cb200
