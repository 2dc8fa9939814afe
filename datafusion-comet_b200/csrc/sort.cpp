// sort.cpp -- Sort (SortExec(LexOrdering).with_fetch(fetch) then GlobalLimitExec(skip), planner.rs:1488-1522).
#include "exec_internal.h"

namespace cb200 {

// code -> rank of dictionary d: equal strings get equal ranks, ranks follow unsigned byte order (one entry more than the dictionary)
static std::vector<uint32_t> byte_order_ranks(const Dictionary& d) {
    const std::vector<std::string>& v = d.values();
    std::vector<uint32_t> order(v.size()), rank(v.size() + 1, 0);
    for (size_t i = 0; i < v.size(); i++) order[i] = (uint32_t)i;
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return v[a] < v[b]; }); // char_traits<char>: unsigned bytes
    uint32_t next = 0;
    for (size_t i = 0; i < order.size(); i++) {
        if (i > 0 && v[order[i]] != v[order[i - 1]]) next++;
        rank[order[i]] = next;
    }
    return rank;
}

// The output is the child's rows in a stable order of the keys (ties keep the input order: batches as they arrive, rows in order
// within a batch), rows [skip, fetch).  Without a fetch, or with one above spark.comet.b200.chunkRows, the child is drained and its
// batches concatenated on the device, sorted once and emitted as one batch.  With a smaller fetch (TopK) at most `fetch` candidate rows
// are kept between chunks: each chunk is sorted, its first `fetch` rows are sorted together with the candidates (which come first, being
// earlier input) and the first `fetch` of those become the next candidates, so device memory is bounded by fetch + one chunk.  Keys are
// built again every round from the columns: a string's rank changes as its dictionary grows.
struct SortNode : ExecNode {
    ExecContext* ctx;
    ExecNodeP child;
    std::vector<SortKey> keys; // expr: Bound child column
    int64_t fetch = -1, skip = 0;
    bool done = false;
    std::vector<DictCodes> ranks; // per key: code -> byte-order rank

    std::vector<ExecNodeP> children() const override { return {child}; }
    bool topk() const { return fetch >= 0 && fetch <= ctx->chunk_rows; }
    void count_passes(int64_t m, const std::vector<int>& digits) {
        ctx->sort_passes += (int64_t)digits.size();
        ctx->sort_pass_rows += m * (int64_t)digits.size();
    }

    bool next(Batch& out) override {
        if (done) return false;
        done = true;
        if (fetch == 0) return false;
        TraceSpan ts("sort");
        Batch all, in;
        if (topk()) {
            while (child->next(in)) {
                arrive(in, ctx, "sorting");
                if (in.n_rows == 0) continue;
                // the chunk's own first `fetch` rows, then those merged behind the candidates (earlier input: first among equal keys)
                Batch top;
                sort_rows(in, 0, std::min<int64_t>(fetch, in.n_rows), top);
                in = Batch();
                if (all.n_rows > 0) {
                    Batch u = concat_batches({all, top}, ctx, "sort");
                    sort_rows(u, 0, std::min<int64_t>(fetch, u.n_rows), all);
                } else all = std::move(top);
            }
        } else all = drain(*child, ctx, "sorting", "sort");
        const int64_t lo = std::min(skip, all.n_rows), hi = fetch >= 0 ? std::min(fetch, all.n_rows) : all.n_rows;
        if (hi <= lo) return false;
        if (topk() && lo == 0) { out = std::move(all); return true; } // the candidates are already in order
        sort_rows(all, lo, hi, out);
        return true;
    }

    // out = b's rows [lo, hi) of the stable order of the keys.  When only the first rows are wanted (lo = 0, hi < n: TopK), an MSD radix
    // select finds the key of row hi - 1 of that order, the rows up to it are compacted (the smaller keys, then the equal ones in input
    // order) and only those are sorted.
    void sort_rows(const Batch& b, int64_t lo, int64_t hi, Batch& out) {
        const int64_t n = b.n_rows;
        if (n >= ((int64_t)1 << 32)) throw Unsupported("sorting 2^32 rows or more");
        cudaStream_t st = ctx->stream;
        cb::SortKeyCols kc;
        memset(&kc, 0, sizeof(kc));
        kc.n = (int)keys.size();
        kc.err = ctx->d_err;
        ranks.resize(keys.size());
        int bits = 0;
        for (size_t k = keys.size(); k-- > 0;) { // the last key is the least significant field
            const Column& c = b.cols.at((size_t)keys[k].expr->index);
            cb::SortKeyCol& f = kc.col[k] = key_field(c, c.validity != nullptr, bits);
            f.desc = keys[k].descending;
            f.nulls_first = keys[k].nulls_first;
            if (c.is_dict) f.rank = ranks[k].get(c.dict, ctx, byte_order_ranks);
        }
        const int W = kc.words = std::max(1, (bits + 63) / 64);
        RowKeys rk = pack_row_keys(kc, n, bits, ctx);
        ctx->sort_rows += n;
        if (lo > 0 || hi >= n) {
            DeviceBufP idx = radix_order(ctx, rk.keys, W, n, rk.digits);
            count_passes(n, rk.digits);
            rk.keys.reset();
            gather_columns(b, (const unsigned*)idx->ptr + lo, hi - lo, out, ctx, "sorting");
            ctx->check_device_errors();
            return;
        }
        // select: bits equal in every row are decided already; then one histogram per differing digit, most significant first
        SortSelectKey p;
        for (int j = 0; j < W; j++) { p.mask[j] = ~(rk.and_or[j] ^ rk.and_or[W + j]); p.want[j] = rk.and_or[j] & p.mask[j]; }
        int64_t r = hi; // the selected key's rank among the rows that match p
        auto hist = std::make_shared<DeviceBuf>(256 * 4);
        std::vector<uint32_t> hh(256);
        for (size_t q = rk.digits.size(); q-- > 0;) {
            const int d = rk.digits[q], w = W - 1 - d / 8, sh = (d % 8) * 8;
            cuda_check(cudaMemsetAsync(hist->ptr, 0, 256 * 4, st), "memset select histogram");
            cuda_check(launch_sort_select_hist((const unsigned long long*)rk.keys->ptr, W, n, p, d, (unsigned*)hist->ptr, st), "select histogram");
            ctx->kernel_launches++;
            ctx->sort_select_rows += n;
            cuda_check(cudaMemcpyAsync(hh.data(), hist->ptr, 256 * 4, cudaMemcpyDeviceToHost, st), "D2H select histogram");
            cuda_check(cudaStreamSynchronize(st), "select histogram sync");
            int v = 0;
            for (; v < 255 && r > (int64_t)hh[(size_t)v]; v++) r -= hh[(size_t)v];
            p.mask[w] |= (uint64_t)0xff << sh;
            p.want[w] |= (uint64_t)v << sh;
        }
        const size_t nb = (size_t)(n + 1023) / 1024;
        auto eq = std::make_shared<DeviceBuf>((size_t)n + 16), keep = std::make_shared<DeviceBuf>((size_t)n + 16);
        auto counts = std::make_shared<DeviceBuf>(nb * 4 + 4), offsets = std::make_shared<DeviceBuf>(nb * 8 + 8), kept = std::make_shared<DeviceBuf>(8);
        cuda_check(launch_sort_select_keep((const unsigned long long*)rk.keys->ptr, W, n, p, r, (unsigned char*)eq->ptr, (int*)counts->ptr,
                                           (long long*)offsets->ptr, (long long*)kept->ptr, (unsigned char*)keep->ptr, st), "select keep");
        ctx->kernel_launches += 4;
        Compacted c = compact_rows(keep, n, hi, ctx, {{rk.keys, W * 8}});
        const int64_t m = c.n;
        if (m != hi) throw ExecError(15, "", "internal: TopK selection kept " + std::to_string(m) + " rows for a fetch of " + std::to_string(hi));
        rk.keys.reset(); eq.reset(); keep.reset();
        DeviceBufP order = radix_order(ctx, c.extra_out[0], W, m, rk.digits);
        count_passes(m, rk.digits);
        auto idx = std::make_shared<DeviceBuf>((size_t)m * 4);
        launch_gather(c.rows->ptr, 4, (const unsigned*)order->ptr, m, idx->ptr, st); // compacted position -> row of b
        ctx->kernel_launches++;
        gather_columns(b, (const unsigned*)idx->ptr, m, out, ctx, "sorting");
        ctx->check_device_errors();
    }
};

ExecNodeP make_sort_node(const OperatorP& op, const ExecNodeP& child, ExecContext* ctx) {
    auto n = std::make_shared<SortNode>();
    n->ctx = ctx;
    n->child = child;
    n->schema = op->schema;
    n->keys = op->sort_keys;
    n->fetch = op->fetch;
    n->skip = std::max<int64_t>(op->skip, 0);
    for (auto& k : n->keys)
        if (k.expr->index < 0 || k.expr->index >= (int)op->schema.size()) throw PlanError("sort key out of range");
    return n;
}

} // namespace cb200
