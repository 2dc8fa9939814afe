// agg.cpp -- the aggregate node: key preparation, range specialisation, and its three accumulation strategies.
//   dense:  group ids are mixed-radix codes of dictionary / boolean keys; thread-private accumulators, folded per launch
//   table:  a key table in HBM hands out group ids; state rows addressed by id (device/cb_kernels.cuh CB_HASH)
//   stream: Partial over clustered keys: one state row per run of equal adjacent keys, no key table (CB_STREAM)
#include "exec_internal.h"
#include "../../include/comet_b200.h"

#include "aot_kernels.h"
#include "ranges.h"

#include <algorithm>
#include <mutex>

namespace cb200 {

// value ranges seen by earlier plans, per pipeline signature (see AggNode::consume_dense)
static std::mutex g_profile_mu;
static std::map<std::string, std::vector<int>> g_range_profile;

namespace {

enum class Strategy { Undecided, Dense, Table, Stream };
enum Level { SAFE = 0, TYPE = 1, TIGHT = 2 }; // range assumptions (see ranges.h)
constexpr int DENSE_MAX_GROUPS = 64;

// ---- group ids: CB_GID_RANGES counters (device/cb_params.h); the host sees per-range counts ------------------------------------
constexpr int GK = CB_GID_RANGES;
struct HashFlags { int w[CB_HFLAG_WORDS]; };
int64_t round_ids(int64_t n) { return (n + GK - 1) / GK * GK; }

using ValueMasks = uint64_t[CB_MAX_COLS * 2];

// the value an accumulator word of this kind starts from
uint64_t identity_word(int kind) { return kind == W_MIN ? 0x7fffffffffffffffull : kind == W_MAX ? 0x8000000000000000ull : 0; }

// dense group id -> code of each key (mixed radix over the key cardinalities, the last key varying fastest)
std::vector<int> decode_gid(int g, const std::vector<int>& cards) {
    std::vector<int> code(cards.size());
    for (int k = (int)cards.size() - 1; k >= 0; k--) { code[(size_t)k] = g % cards[(size_t)k]; g /= cards[(size_t)k]; }
    return code;
}

int grid_for(const ExecContext* ctx, int n_tiles) { return std::max(1, std::min(ctx->num_sms, n_tiles)); }

struct Kernel {
    PipelineSpec spec;
    GeneratedKernel g;
    std::shared_ptr<CompiledModule> mod;
};

void launch_named(ExecContext* ctx, const Kernel& k, const char* name, dim3 grid, dim3 block, void** args) {
    cuda_check(cudaLaunchKernel((const void*)k.mod->kernel(name), grid, block, args, 0, ctx->stream), name);
    ctx->kernel_launches++;
}

// ---- dense strategy: thread-private accumulators by mixed-radix group id, folded into `totals` after every launch ----------------
struct DenseState {
    std::vector<int> cards;         // cardinality per key (incl. null slot) of the current layout
    std::vector<bool> has_null;     // per key: the layout has a null slot (always its key's last code)
    DeviceBufP totals, spill, partials;
    int groups = 0;                 // group slots in `totals`

    // cardinalities grew: move totals to the new mixed-radix layout
    void regroup(ExecContext* ctx, int n_words, const std::vector<int>& word_kinds, const std::vector<int>& new_cards) {
        int new_groups = 1;
        for (int c : new_cards) new_groups *= c;
        std::vector<uint64_t> oldt((size_t)groups * n_words * 2), newt((size_t)new_groups * n_words * 2);
        cuda_check(cudaMemcpy(oldt.data(), totals->ptr, oldt.size() * 8, cudaMemcpyDeviceToHost), "regroup D2H");
        for (size_t i = 0; i < (size_t)new_groups * n_words; i++) newt[i * 2] = identity_word(word_kinds[i % (size_t)n_words]);
        for (int g = 0; g < groups; g++) {
            const std::vector<int> code = decode_gid(g, cards);
            int ng = 0, mul = 1;
            for (int k = (int)cards.size() - 1; k >= 0; k--) {
                int cd = code[(size_t)k];
                if (has_null[(size_t)k] && cd == cards[(size_t)k] - 1) cd = new_cards[(size_t)k] - 1;
                ng += cd * mul;
                mul *= new_cards[(size_t)k];
            }
            memcpy(&newt[(size_t)ng * n_words * 2], &oldt[(size_t)g * n_words * 2], (size_t)n_words * 16);
        }
        totals = std::make_shared<DeviceBuf>(newt.size() * 8);
        cuda_check(cudaMemcpyAsync(totals->ptr, newt.data(), newt.size() * 8, cudaMemcpyHostToDevice, ctx->stream), "regroup H2D");
        cuda_check(cudaStreamSynchronize(ctx->stream), "regroup sync");
        groups = new_groups;
    }

    // dense results are tiny: finalize brings them to the host and spells the key codes out there.  `fp`: certificates filled in.
    void finalize(ExecContext* ctx, const Kernel& last, cb::FinParams fp, bool ungrouped, const std::vector<DType>& schema,
                  const std::vector<DictionaryP>& key_dicts, Batch& out) const {
        TraceSpan ts("agg.finalize");
        const GeneratedKernel& g = last.g;
        const int ng = groups;
        fp.totals = (cb::u64*)totals->ptr;
        fp.n_groups = ng;
        // all finalize outputs live in ONE device buffer so the (tiny) result comes back in a single copy
        std::vector<size_t> off_v, off_n;
        size_t total_bytes = 0;
        auto take = [&](size_t n) { size_t o = total_bytes; total_bytes += (n + 15) / 16 * 16; return o; };
        for (size_t i = 0; i < g.out_cols.size(); i++) { off_v.push_back(take((size_t)ng * g.out_bytes[i])); off_n.push_back(take((size_t)ng)); }
        size_t off_present = take((size_t)ng);
        auto dbuf = std::make_shared<DeviceBuf>(total_bytes);
        for (size_t i = 0; i < g.out_cols.size(); i++) {
            fp.out[i] = (cb::u8*)dbuf->ptr + off_v[i];
            fp.outv[i] = (cb::u8*)dbuf->ptr + off_n[i];
        }
        fp.present = (cb::u8*)dbuf->ptr + off_present;
        void* args[] = {&fp};
        cuda_check(cudaLaunchKernel((const void*)last.mod->kernel(g.finalize_entry), dim3((ng + 127) / 128), dim3(128), args, 0, ctx->stream), "finalize launch");
        ctx->kernel_launches++;
        std::vector<uint8_t> hbuf(total_bytes);
        cuda_check(cudaMemcpyAsync(hbuf.data(), dbuf->ptr, total_bytes, cudaMemcpyDeviceToHost, ctx->stream), "agg results D2H"); ctx->d2h_bytes += (int64_t)(total_bytes);
        ctx->check_device_errors(); // synchronises
        const uint8_t* pres = hbuf.data() + off_present;
        std::vector<int> rows;
        for (int gi = 0; gi < ng; gi++) if (ungrouped || pres[(size_t)gi]) rows.push_back(gi);
        out.n_rows = (int64_t)rows.size();
        out.cols.clear();
        // key columns
        for (size_t k = 0; k < key_dicts.size(); k++) {
            Column c;
            c.type = schema[k];
            c.on_host = true;
            bool any_null = false;
            std::vector<int> codes;
            for (int gi : rows) codes.push_back(decode_gid(gi, cards)[k]);
            c.h_valid.assign(rows.size(), 1);
            const bool is_bool = c.type.id == TypeId::Bool;
            if (!is_bool) c.h_offsets.push_back(0);
            for (size_t r = 0; r < rows.size(); r++) {
                const bool isnull = has_null[k] && codes[r] == cards[k] - 1;
                if (isnull) { c.h_valid[r] = 0; any_null = true; }
                if (is_bool) c.h_data.push_back(isnull ? 0 : (uint8_t)codes[r]);
                else {
                    if (!isnull) { const std::string& s = key_dicts[k]->values().at((size_t)codes[r]); c.h_data.insert(c.h_data.end(), s.begin(), s.end()); }
                    c.h_offsets.push_back((int32_t)c.h_data.size());
                }
            }
            if (!any_null) c.h_valid.clear();
            out.cols.push_back(c);
        }
        for (size_t i = 0; i < g.out_cols.size(); i++) {
            Column c;
            c.type = g.out_cols[i].type;
            c.on_host = true;
            int w = g.out_bytes[i];
            const uint8_t* all = hbuf.data() + off_v[i];
            const uint8_t* allv = hbuf.data() + off_n[i];
            c.h_data.resize(rows.size() * w);
            c.h_valid.resize(rows.size());
            bool any_null = false;
            for (size_t r = 0; r < rows.size(); r++) {
                memcpy(&c.h_data[r * w], &all[(size_t)rows[r] * w], (size_t)w);
                c.h_valid[r] = allv[(size_t)rows[r]];
                if (!c.h_valid[r]) any_null = true;
            }
            if (!any_null) c.h_valid.clear();
            out.cols.push_back(c);
        }
    }
};

// ---- state rows addressed by group id, shared by the table and stream strategies.  Ids max_groups / max_groups + 1 are reserved
//      (the key equal to the empty-slot pattern, the NULL key) and live at the tail of htotals.  The layout is the kernel's. ----------
struct IdRows {
    DeviceBufP hkey_of_gid, htotals, hflags;
    int64_t max_groups = 0;

    void ensure_flags(ExecContext* ctx) {
        if (hflags) return;
        hflags = std::make_shared<DeviceBuf>(sizeof(HashFlags));
        cuda_check(cudaMemsetAsync(hflags->ptr, 0, sizeof(HashFlags), ctx->stream), "memset hash flags");
    }
    void write_flags(ExecContext* ctx, const HashFlags& hf) {
        cuda_check(cudaMemcpyAsync(hflags->ptr, &hf, sizeof(hf), cudaMemcpyHostToDevice, ctx->stream), "write hash flags");
        cuda_check(cudaStreamSynchronize(ctx->stream), "flags sync");
    }
    // device -> host (synchronises); cnt[r] = ids handed out in range r (a counter that ran past its range is clamped); returns their sum
    int64_t read_flags(ExecContext* ctx, HashFlags& hf, int64_t cnt[GK]) {
        memset(&hf, 0, sizeof(hf));
        if (hflags) {
            cuda_check(cudaMemcpyAsync(&hf, hflags->ptr, sizeof(hf), cudaMemcpyDeviceToHost, ctx->stream), "read hash flags"); ctx->d2h_bytes += (int64_t)sizeof(hf);
            cuda_check(cudaStreamSynchronize(ctx->stream), "hash flags sync");
        }
        const int64_t R = max_groups / GK;
        int64_t total = 0;
        bool overshoot = false;
        for (int r = 0; r < GK; r++) {
            if (hf.w[CB_HFLAG_CTR + r] > R || hf.w[CB_HFLAG_CTR + r] < 0) overshoot = true;
            cnt[r] = std::min<int64_t>(std::max(hf.w[CB_HFLAG_CTR + r], 0), R);
            if (hf.w[CB_HFLAG_CTR + r] < 0) cnt[r] = R; // wrapped: it was full long ago
            total += cnt[r];
        }
        if (overshoot && hflags) { // warps that found a range full still bumped its counter: put it back to "full" so it can never wrap
            for (int r = 0; r < GK; r++) hf.w[CB_HFLAG_CTR + r] = (int)cnt[r];
            write_flags(ctx, hf);
        }
        return total;
    }
    // n rows of `totals` from row `first` on get the identity of every accumulator word
    static void init_totals(ExecContext* ctx, const Kernel& k, cb::u64* totals, int64_t first, int64_t n) {
        if (n <= 0) return;
        const int n_words = k.g.n_words;
        if (std::none_of(k.g.word_kinds.begin(), k.g.word_kinds.end(), identity_word)) {
            cuda_check(cudaMemsetAsync(totals + first * n_words * 2, 0, (size_t)n * n_words * 16, ctx->stream), "memset totals");
        } else {
            long long f = first, nn = n;
            void* a1[] = {&totals, &f, &nn};
            launch_named(ctx, k, "cb_hash_init", dim3((unsigned)((n + 255) / 256)), dim3(256), a1);
        }
    }
    // new accumulator / key arrays for nm ids (a multiple of GK): range r's rows move from r * R_old to r * R_new, the two reserved
    // groups to the new tail.  zero_fill: every other word gets its identity (the key table path updates with atomics).
    void grow(ExecContext* ctx, const Kernel& k, const int64_t cnt[GK], int64_t nm, bool zero_fill) {
        cudaStream_t st = ctx->stream;
        const int n_words = k.g.n_words, key_words = k.g.key_words;
        if (nm + 2 >= INT32_MAX) throw ExecError(16, "", "more than 2^31 groups in one partition; lower spark.comet.b200.chunkRows");
        const int64_t Ro = max_groups / GK, Rn = nm / GK;
        auto ntot = std::make_shared<DeviceBuf>((size_t)(nm + 2) * n_words * 16);
        auto nkog = std::make_shared<DeviceBuf>((size_t)nm * 8 * key_words + 16);
        cb::u64* tp = (cb::u64*)ntot->ptr;
        if (zero_fill) init_totals(ctx, k, tp, 0, nm + 2);
        else if (!htotals) init_totals(ctx, k, tp, nm, 2);
        if (htotals) {
            for (int r = 0; r < GK; r++) {
                if (cnt[r] <= 0) continue;
                cuda_check(cudaMemcpyAsync(tp + (size_t)r * Rn * n_words * 2, (cb::u64*)htotals->ptr + (size_t)r * Ro * n_words * 2, (size_t)cnt[r] * n_words * 16,
                                           cudaMemcpyDeviceToDevice, st), "copy totals");
                cuda_check(cudaMemcpyAsync((cb::u64*)nkog->ptr + (size_t)r * Rn * key_words, (cb::u64*)hkey_of_gid->ptr + (size_t)r * Ro * key_words,
                                           (size_t)cnt[r] * 8 * key_words, cudaMemcpyDeviceToDevice, st), "copy group keys");
            }
            cuda_check(cudaMemcpyAsync(tp + (size_t)nm * n_words * 2, (cb::u64*)htotals->ptr + (size_t)max_groups * n_words * 2, (size_t)2 * n_words * 16,
                                       cudaMemcpyDeviceToDevice, st), "copy reserved groups");
        }
        cuda_check(cudaStreamSynchronize(st), "table growth"); // old buffers die below
        htotals = ntot; hkey_of_gid = nkog; max_groups = nm;
    }

    // hash results: groups are dense by id, so finalize writes the output columns directly (no compaction).  `fp`: certificates filled in.
    void finalize(ExecContext* ctx, const Kernel& last, cb::FinParams fp, const std::vector<DictionaryP>& key_dicts, Batch& out) {
        TraceSpan ts("agg.finalize_hash");
        const GeneratedKernel& g = last.g;
        HashFlags hfl;
        int64_t cnt[GK];
        const int64_t ng = read_flags(ctx, hfl, cnt);
        const int* flags = hfl.w;
        const int64_t n_out = ng + ((flags[0] & CB_HF_SENTINEL) ? 1 : 0) + ((flags[0] & CB_HF_NULL_GROUP) ? 1 : 0);
        fp.totals = (cb::u64*)htotals->ptr;
        fp.hkeys = (const cb::u64*)hkey_of_gid->ptr;
        fp.sentinel_used = flags[0] & CB_HF_SENTINEL;
        fp.null_group_used = (flags[0] & CB_HF_NULL_GROUP) ? 1 : 0;
        fp.n_hash_groups = (int)ng;
        fp.max_groups = (int)max_groups;
        fp.gid_range = (int)(max_groups / GK);
        int64_t run = 0;
        for (int r = 0; r < GK; r++) { fp.gid_prefix[r] = (int)run; run += cnt[r]; }
        fp.gid_prefix[GK] = (int)run;
        fp.n_groups = (int)n_out;
        if (g.out_cols.size() > CB_MAX_OUT) throw Unsupported("too many output columns");
        out.n_rows = n_out;
        out.cols.clear();
        std::vector<DeviceBufP> vbytes;
        size_t rows_alloc = (size_t)std::max<int64_t>(n_out, 1);
        for (size_t i = 0; i < g.out_cols.size(); i++) {
            Column c;
            c.type = g.out_cols[i].type;
            c.phys = kernel_out_phys(c.type);
            c.data = std::make_shared<DeviceBuf>(rows_alloc * g.out_bytes[i]);
            vbytes.push_back(std::make_shared<DeviceBuf>(rows_alloc));
            fp.out[i] = (cb::u8*)c.data->ptr;
            fp.outv[i] = (cb::u8*)vbytes.back()->ptr;
            if ((int)i < g.n_key_cols && c.type.is_string()) { c.is_dict = true; c.dict = key_dicts[i]; }
            out.cols.push_back(c);
        }
        auto present = std::make_shared<DeviceBuf>(rows_alloc);
        fp.present = (cb::u8*)present->ptr;
        if (n_out > 0) {
            void* args[] = {&fp};
            launch_named(ctx, last, g.finalize_entry.c_str(), dim3((unsigned)((n_out + 127) / 128)), dim3(128), args);
            for (size_t i = 0; i < out.cols.size(); i++) {
                Column& c = out.cols[i];
                c.valid_bytes = vbytes[i];
                c.validity = bytes_to_bitmap(vbytes[i], n_out, ctx);
                c.null_count = -1;
                if (c.type.id == TypeId::Bool) c.bool_bytes = c.data;
            }
        }
        ctx->check_device_errors();
    }
};

// ---- table strategy: the key table over the id-addressed rows ------------------------------------------------------------------------
struct KeyTable {
    DeviceBufP hkeys;
    int64_t hcap = 0;

    // make sure `incoming` more rows (each possibly a new group) fit: dense accumulators by group id, key table at load <= 0.5.
    // remaining: rows the source will still produce (-1: unknown); merging: the input is state rows (Final / PartialMerge)
    void ensure(ExecContext* ctx, const Kernel& k, IdRows& rows, int64_t incoming, int64_t remaining, int64_t rows_scanned, bool merging) {
        cudaStream_t st = ctx->stream;
        rows.ensure_flags(ctx);
        HashFlags hf;
        int64_t cnt[GK];
        const int64_t cur = rows.read_flags(ctx, hf, cnt);
        const int64_t need = cur + incoming;
        if (need + 2 >= INT32_MAX) throw ExecError(16, "", "more than 2^31 groups in one partition; lower spark.comet.b200.chunkRows");
        bool relocated = false;
        if (need > rows.max_groups) {
            int64_t nm = std::max<int64_t>(need, rows.max_groups + rows.max_groups / 4);
            // When the source knows how many rows are still to come, size for them at the distinct ratio seen so far (+30 %) in ONE
            // step: growing means copying the totals and re-inserting every key.
            if (remaining > 0 && rows_scanned == 0 && merging) {
                // merging state rows (Final / PartialMerge): most keys are new -- size for everything that is still to come at once
                nm = std::max(nm, need + remaining);
            }
            if (remaining > 0 && rows_scanned > 0 && cur > 0) {
                const double ratio = std::min(1.0, 1.3 * (double)cur / (double)rows_scanned);
                const int64_t est = cur + incoming + (int64_t)(ratio * (double)remaining);
                nm = std::max(nm, std::min<int64_t>(est, cur + incoming + remaining));
            }
            if (nm + 2 + GK >= INT32_MAX) nm = INT32_MAX - 3 - GK;
            relocated = cur > 0;
            rows.grow(ctx, k, cnt, round_ids(nm), true);
        }
        int64_t cap = std::max<int64_t>(hcap, 1 << 16);
        while (cap < 2 * std::max(need, rows.max_groups)) cap <<= 1; // load <= 0.5 even when every reserved group id gets used
        if (cap != hcap || relocated) { // a relocation changes the ids: the slots must be rebuilt even at the same capacity
            auto nkeys = cap != hcap ? std::make_shared<DeviceBuf>((size_t)cap * 16) : hkeys;
            cuda_check(cudaMemsetAsync(nkeys->ptr, 0xff, (size_t)cap * 16, st), "memset key slots");
            if (cur > 0) {
                const cb::u64* kog = (const cb::u64*)rows.hkey_of_gid->ptr;
                int rr = (int)(rows.max_groups / GK);
                const int* ctr = (const int*)rows.hflags->ptr + CB_HFLAG_CTR;
                cb::u64* kp = (cb::u64*)nkeys->ptr;
                cb::u32 mask = (cb::u32)(cap - 1);
                void* a2[] = {&kog, &rr, &ctr, &kp, &mask};
                launch_named(ctx, k, "cb_hash_rehash", dim3((unsigned)((rows.max_groups + 255) / 256)), dim3(256), a2);
                cuda_check(cudaStreamSynchronize(st), "rehash");
            }
            hkeys = nkeys; hcap = cap;
        }
    }
};

// ---- stream strategy: the sampled decision's ratio, state-row sizing and the reserved groups' snapshot for a repeated launch ----------
struct StreamState {
    double ratio = 1.0;                // state rows per input row seen so far
    DeviceBufP reserved_snap;          // totals of the two reserved groups before a launch (restored when the launch is repeated)

    void ensure_rows(ExecContext* ctx, const Kernel& k, IdRows& rows, const int64_t cnt[GK], int64_t want_groups) {
        rows.ensure_flags(ctx);
        if (rows.htotals && want_groups <= rows.max_groups) return;
        rows.grow(ctx, k, cnt, round_ids(std::max<int64_t>(want_groups, rows.max_groups + rows.max_groups / 2)), false);
    }
    void snapshot_reserved(ExecContext* ctx, const IdRows& rows, int n_words, bool restore) {
        const size_t bytes = (size_t)2 * n_words * 16;
        if (!reserved_snap || reserved_snap->bytes < bytes) reserved_snap = std::make_shared<DeviceBuf>(bytes);
        cb::u64* tail = (cb::u64*)rows.htotals->ptr + (size_t)rows.max_groups * n_words * 2;
        if (restore) cuda_check(cudaMemcpyAsync(tail, reserved_snap->ptr, bytes, cudaMemcpyDeviceToDevice, ctx->stream), "restore reserved groups");
        else cuda_check(cudaMemcpyAsync(reserved_snap->ptr, tail, bytes, cudaMemcpyDeviceToDevice, ctx->stream), "snapshot reserved groups");
    }
};

struct AggNode : FusedBase {
    std::vector<ExprP> keys;          // over child columns; each must be a plain column reference
    std::vector<AggExpr> aggs;        // children/filter over child columns (Partial)
    std::vector<std::vector<int>> state_cols; // Final: child column index of each state column
    AggMode mode = AggMode::Partial;
    bool ungrouped = false;
    bool emitted = false;
    std::vector<Batch> outq;          // output batches (more than one only after a dense -> hash migration)
    size_t outq_pos = 0;
    std::vector<int> assume_bits;     // build time only: value-range assumption per source column (bits; <= 0: none)

    // keys
    std::vector<bool> key_has_null;               // per key: some batch so far had a validity buffer
    std::vector<DictionaryP> key_dicts;           // strings per key (dict columns); empty for bool keys
    // device string dictionaries for plain Utf8 keys
    struct DevDict { StringDictDev d; std::vector<DeviceBufP> bufs; int host_known = 0; };
    std::vector<std::shared_ptr<DevDict>> dev_dicts;

    // accumulator layout of the kernels launched so far, and the last of them (finalize runs from its module)
    int n_words = 0, key_words = 1;   // key_words: 64-bit words per packed group key (hkey_of_gid stride)
    std::vector<int> word_kinds;
    Kernel last;                      // the last kernel whose launch was kept: the node holds state once there is one
    bool have_totals() const { return last.mod != nullptr; }

    Strategy strategy = Strategy::Undecided;
    DenseState dense;
    KeyTable table;
    IdRows rows;

    // range assumptions: per child column, the max bit length of (v ^ sign) over every valid row scanned so far (-1: none)
    std::vector<int> observed_bits;
    int64_t rows_scanned = 0;
    std::string profile_key;
    DeviceBufP vmask;
    StreamState stream;

    int assume_for(int child_col, Level lv) const {
        const DType& t = child->schema[(size_t)child_col];
        if (!t.is_decimal() || lv == SAFE || mode != AggMode::Partial) return 0;
        int k = r_bitlen(r_prec_max(t.precision));
        if ((size_t)child_col < assume_bits.size() && assume_bits[(size_t)child_col] > 0) k = std::min(k, assume_bits[(size_t)child_col]);
        if (lv == TIGHT && !observed_bits.empty() && observed_bits[(size_t)child_col] >= 0) k = std::min(k, observed_bits[(size_t)child_col] + 2);
        return std::min(k, 126);
    }

    PipelineSpec make_spec(const Batch* b, Strategy st, int n_groups, Level lv = TYPE) const {
        const bool hash = st == Strategy::Table || st == Strategy::Stream;
        PipelineSpec s;
        s.cols = stage_cols(b);
        for (auto& c : s.cols) c.assume_bits = assume_for(c.src_index, lv);
        s.predicates = to_slots(predicates, slot_of);
        s.sink = SinkKind::Agg;
        s.mode = mode;
        s.ungrouped = ungrouped;
        s.hash = hash;
        s.keys = to_slots(keys, slot_of);
        for (size_t k = 0; k < keys.size(); k++) s.key_nullable.push_back(b ? key_has_null[k] : false);
        for (auto& a : aggs) {
            AggExpr c = a;
            if (mode == AggMode::Partial) {
                c.children = to_slots(a.children, slot_of);
                if (a.filter) c.filter = to_slots({a.filter}, slot_of)[0];
            }
            s.aggs.push_back(c);
        }
        for (auto& sc : state_cols) {
            std::vector<int> v;
            for (int ci : sc) v.push_back(slot_of.at(ci));
            s.state_slots.push_back(v);
        }
        if (hash) {
            // every row is a chain of dependent L2/HBM round trips (slot probe, then atomics that return a value): the kernel is
            // latency-bound and wants rows in flight, not registers -- 16+ consumer warps per SM instead of 8 (measured on Config 4:
            // 21.8 ms at 256 threads, 15.6 ms at 512)
            s.threads = ctx->hash_threads;
            s.tile = 2 * ctx->hash_threads;
            s.stream = st == Strategy::Stream;
        }
        // first pass to learn the accumulator footprint, then size the ring to the remaining smem
        GeneratedKernel probe = generate_pipeline(s);
        size_t acc = (!ungrouped && !hash) ? (size_t)std::max(n_groups, 1) * probe.n_words * s.threads * 8 : 0;
        while (acc + 2 * (size_t)probe.stage_bytes + 1024 > SMEM_BUDGET && s.threads > 32) {
            s.threads /= 2; // shrink the thread-private accumulator file (wide Final-mode merges are tiny inputs)
            acc /= 2;
        }
        if (acc + 2 * (size_t)probe.stage_bytes + 1024 > SMEM_BUDGET)
            throw Unsupported("too many groups x aggregates for the thread-private accumulators of the dense path");
        s.stages = (int)std::max<size_t>(2, std::min<size_t>(6, (SMEM_BUDGET - 1024 - acc) / (size_t)probe.stage_bytes));
        return s;
    }

    // the dense or key-table kernel, by the key types alone, and for a Partial aggregate over keys that need hashing, the
    // run-combining variant the sampled decision may pick at run time
    std::vector<PipelineSpec> build_specs() const override {
        bool hash = false;
        for (auto& k : keys) if (!k->type.is_string() && k->type.id != TypeId::Bool) hash = true;
        std::vector<PipelineSpec> out{make_spec(nullptr, hash ? Strategy::Table : Strategy::Dense, ungrouped ? 1 : 6)};
        if (hash && mode == AggMode::Partial) out.push_back(make_spec(nullptr, Strategy::Stream, 6));
        return out;
    }

    // generate and load the kernel of `spec` and adopt its accumulator layout, which must not change once state exists
    Kernel compile(const PipelineSpec& spec) {
        Kernel k{spec, generate_pipeline(spec), nullptr};
        k.mod = jit_get(k.g, true);
        if (have_totals() && (k.g.n_words != n_words || k.g.word_kinds != word_kinds)) throw ExecError(15, "", "internal: accumulator layout changed between launches");
        if (have_totals() && k.g.key_words != key_words) throw ExecError(15, "", "internal: group key packing changed between launches");
        n_words = k.g.n_words;
        word_kinds = k.g.word_kinds;
        key_words = k.g.key_words;
        return k;
    }

    // ---- value masks: per staged column, the OR of (v ^ sign) over the valid rows of one launch --------------------------------------
    void clear_vmask() {
        if (!vmask) vmask = std::make_shared<DeviceBuf>(CB_MAX_COLS * 16);
        cuda_check(cudaMemsetAsync(vmask->ptr, 0, CB_MAX_COLS * 16, ctx->stream), "memset vmask");
    }
    void copy_vmask(ValueMasks& masks) { // enqueued; complete after the next synchronisation
        cuda_check(cudaMemcpyAsync(masks, vmask->ptr, sizeof(ValueMasks), cudaMemcpyDeviceToHost, ctx->stream), "read value masks"); ctx->d2h_bytes += (int64_t)(sizeof(ValueMasks));
    }
    // bit length seen per staged decimal column (-1: not a decimal)
    static std::vector<int> mask_bits(const PipelineSpec& spec, const ValueMasks& masks) {
        std::vector<int> seen(spec.cols.size(), -1);
        for (size_t i = 0; i < spec.cols.size(); i++) {
            if (!spec.cols[i].type.is_decimal()) continue;
            uint64_t lo = masks[2 * i], hi = masks[2 * i + 1];
            seen[i] = hi ? 64 + r_bitlen(hi) : r_bitlen(lo);
        }
        return seen;
    }
    void observe(const std::vector<int>& seen) {
        for (size_t i = 0; i < seen.size(); i++)
            if (seen[i] >= 0) observed_bits[(size_t)used_cols[i]] = std::max(observed_bits[(size_t)used_cols[i]], seen[i]);
    }

    // make key column k of batch `b` a code column; returns cardinality (without null slot)
    int prepare_key(Batch& b, size_t k) {
        int ci = keys[k]->index;
        Column& c = b.cols[ci];
        if (c.type.id == TypeId::Bool) return 2;
        if (!c.type.is_string()) return -1; // integer / date / decimal keys: hash aggregation
        if (c.is_dict) {
            key_dicts[k] = c.dict;
            return (int)c.dict->values().size();
        }
        // plain Utf8 -> device dictionary builder
        if (!dev_dicts[k]) {
            auto dd = std::make_shared<DevDict>();
            const int64_t cap = 1 << 16;
            const int max_codes = 4096;
            const int64_t bytes_cap = 1 << 20;
            auto alloc = [&](size_t n) { auto bfr = std::make_shared<DeviceBuf>(n); cuda_check(cudaMemsetAsync(bfr->ptr, 0, bfr->bytes, ctx->stream), "memset dict"); dd->bufs.push_back(bfr); return bfr->ptr; };
            dd->d.tags = (unsigned long long*)alloc((size_t)cap * 8);
            dd->d.slot_code = (int*)alloc((size_t)cap * 4);
            dd->d.capacity = cap;
            dd->d.n_codes = (int*)alloc(64);
            dd->d.bytes_used = (unsigned long long*)((char*)dd->d.n_codes + 16);
            dd->d.err = (int*)((char*)dd->d.n_codes + 32);
            dd->d.max_codes = max_codes;
            dd->d.code_off = (long long*)alloc((size_t)max_codes * 8);
            dd->d.code_len = (int*)alloc((size_t)max_codes * 4);
            dd->d.bytes = (unsigned char*)alloc((size_t)bytes_cap);
            dd->d.bytes_cap = bytes_cap;
            dev_dicts[k] = dd;
            key_dicts[k] = std::make_shared<Dictionary>();
        }
        DevDict& dd = *dev_dicts[k];
        if (!c.offsets || !c.chars) throw Unsupported("string key column without offsets/chars buffers");
        auto row_slot = std::make_shared<DeviceBuf>((size_t)b.n_rows * 4);
        auto codes = std::make_shared<DeviceBuf>((size_t)b.n_rows * 4);
        launch_dict_encode(dd.d, (const int*)c.offsets->ptr, (const unsigned char*)c.chars->ptr, c.validity ? (const unsigned char*)c.validity->ptr : nullptr,
                           b.n_rows, (int*)row_slot->ptr, (int*)codes->ptr, ctx->stream);
        ctx->kernel_launches += 2;
        int hdr[12];
        cuda_check(cudaMemcpyAsync(hdr, dd.d.n_codes, sizeof(hdr), cudaMemcpyDeviceToHost, ctx->stream), "dict header");
        cuda_check(cudaStreamSynchronize(ctx->stream), "dict encode");
        int n_codes = hdr[0], derr = hdr[8];
        if (derr & CB_DICT_FULL) throw Unsupported("plain Utf8 group key with more distinct values than the device dictionary holds (dictionary-encode the column)");
        if (derr & CB_DICT_COLLISION) throw ExecError(14, "", "64-bit hash collision between distinct group key strings");
        // fetch newly added dictionary strings (metadata-sized)
        if (n_codes > dd.host_known) {
            std::vector<long long> off((size_t)n_codes);
            std::vector<int> len((size_t)n_codes);
            cuda_check(cudaMemcpy(off.data(), dd.d.code_off, (size_t)n_codes * 8, cudaMemcpyDeviceToHost), "dict offsets");
            cuda_check(cudaMemcpy(len.data(), dd.d.code_len, (size_t)n_codes * 4, cudaMemcpyDeviceToHost), "dict lengths");
            for (int i = dd.host_known; i < n_codes; i++) {
                std::string s((size_t)len[(size_t)i], '\0');
                if (len[(size_t)i]) cuda_check(cudaMemcpy(&s[0], dd.d.bytes + off[(size_t)i], (size_t)len[(size_t)i], cudaMemcpyDeviceToHost), "dict bytes");
                key_dicts[k]->append(s); // the device builder hands out codes in order: entry i is code i
            }
            dd.host_known = n_codes;
        }
        c.data = codes;
        c.phys = Phys::I32;
        c.is_dict = true;
        c.dict = key_dicts[k];
        return n_codes;
    }

    void consume(Batch& b) {
        std::vector<int> nc(keys.size());
        std::vector<bool> hn(keys.size());
        for (size_t k = 0; k < keys.size(); k++) {
            int card = prepare_key(b, k);
            const Column& c = b.cols[keys[k]->index];
            hn[k] = key_has_null[k] || c.validity != nullptr;
            nc[k] = card < 0 ? -1 : std::max(card, 1) + (hn[k] ? 1 : 0);
            if (!dense.cards.empty() && nc[k] >= 0) nc[k] = std::max(nc[k], dense.cards[k]);
        }
        bool densifiable = true;
        for (int c : nc) if (c < 0) densifiable = false;
        int n_groups = 1;
        if (densifiable) for (int c : nc) { n_groups *= c; if (n_groups > 1 << 20) break; }
        const bool needs_hash = !ungrouped && (!densifiable || n_groups > DENSE_MAX_GROUPS);
        key_has_null = hn;
        if (observed_bits.empty()) observed_bits.assign(child->schema.size(), -1);
        if (strategy == Strategy::Undecided || (strategy == Strategy::Dense && needs_hash)) {
            if (strategy == Strategy::Dense) {
                leave_dense();
                ctx->agg_strategies |= CB200_AGG_MIGRATED;
            }
            strategy = !needs_hash ? Strategy::Dense : sample_stream(b) ? Strategy::Stream : Strategy::Table;
            ctx->agg_strategies |= strategy == Strategy::Dense ? CB200_AGG_DENSE : strategy == Strategy::Stream ? CB200_AGG_STREAM : CB200_AGG_TABLE;
        }
        if (strategy == Strategy::Dense) consume_dense(b, nc, n_groups);
        else if (strategy == Strategy::Table) consume_table(b);
        else consume_stream(b);
    }

    // ---- dense strategy ----------------------------------------------------------------------------------------------------------
    void consume_dense(Batch& b, const std::vector<int>& nc, int n_groups) {
        if (have_totals() && nc != dense.cards) {
            if (n_words == 0) throw ExecError(15, "", "internal: regroup before layout");
            dense.regroup(ctx, n_words, word_kinds, nc);
        }
        dense.cards = nc;
        dense.has_null = key_has_null;
        const int64_t SAMPLE = 1 << 20;
        bool have_obs = false;
        for (int ci : used_cols) if (child->schema[(size_t)ci].is_decimal() && observed_bits[(size_t)ci] >= 0) have_obs = true;
        if (mode == AggMode::Partial && !have_obs && b.n_rows > 2 * SAMPLE) {
            // Range profile of the last plan with this very pipeline (the previous task of the same stage reads the same table):
            // start at its ranges instead of sampling again.  A profile is only a guess -- every launch validates it.
            profile_key = pipeline_signature(make_spec(&b, Strategy::Dense, n_groups, SAFE));
            std::lock_guard<std::mutex> lk(g_profile_mu);
            auto it = g_range_profile.find(profile_key);
            if (it != g_range_profile.end() && it->second.size() == observed_bits.size()) {
                observed_bits = it->second;
                for (int ci : used_cols) if (child->schema[(size_t)ci].is_decimal() && observed_bits[(size_t)ci] >= 0) have_obs = true;
            }
        }
        if (mode != AggMode::Partial) {
            run_range(b, 0, b.n_rows, n_groups, SAFE);
        } else if (!have_obs && b.n_rows > 2 * SAMPLE) {
            // sample-then-specialise: a short launch measures the value ranges, the bulk launch runs the kernel
            // specialised to them (64-bit arithmetic, unconditional accumulation); every launch validates its
            // assumptions through the value masks, so a violated guess only costs a re-run.
            run_range(b, 0, SAMPLE, n_groups, TYPE);
            run_range(b, SAMPLE, b.n_rows, n_groups, TIGHT);
        } else {
            run_range(b, 0, b.n_rows, n_groups, have_obs ? TIGHT : TYPE);
        }
        if (!profile_key.empty()) {
            std::lock_guard<std::mutex> lk(g_profile_mu);
            if (g_range_profile.size() > 256) g_range_profile.clear();
            g_range_profile[profile_key] = observed_bits;
        }
    }

    // The key cardinality outgrew the dense layout mid-stream.  A Partial / PartialMerge aggregate may emit a group more than once
    // (the Final stage merges state rows, exactly as it does for Spark's own spilling partial aggregates): flush what the dense path
    // has accumulated as one state batch and carry on with hash aggregation.
    void leave_dense() {
        if (mode == AggMode::Final) throw Unsupported("group cardinality grew past the dense path mid-stream in a Final aggregate");
        if (have_totals()) {
            Batch early;
            dense.finalize(ctx, last, certified_params(), ungrouped, schema, key_dicts, early);
            if (early.n_rows > 0) outq.push_back(std::move(early));
        }
        last = Kernel();
        dense = DenseState();
        n_words = 0; word_kinds.clear(); rows_scanned = 0;
    }

    // one (possibly split) launch over rows [row0,row1) at assumption level lv, escalating on violated assumptions
    void run_range(Batch& b, int64_t row0, int64_t row1, int n_groups, Level lv) {
        TraceSpan tsr("agg.run_range");
        while (true) {
            Kernel k;
            {
                TraceSpan ts("agg.codegen+jit");
                k = compile(make_spec(&b, Strategy::Dense, n_groups, lv));
            }
            const int64_t max_rows = (int64_t)ctx->num_sms * k.g.threads * (1ll << CB_RPT_LOG2) / 1024 * 1024;
            int64_t r0 = row0;
            while (r0 < row1 && launch_one(b, r0, std::min(row1, r0 + max_rows), n_groups, k)) r0 += max_rows;
            if (r0 >= row1) return;
            if (lv == SAFE) throw ExecError(15, "", "internal: value-mask validation failed without assumptions");
            lv = lv == TIGHT ? TYPE : SAFE; // widen: observed ranges -> declared precision -> no assumption (fully checked code)
            // sub-launches of the failed attempt before r0 validated and were folded; restart the remainder
            row0 = r0;
        }
    }

    // false: the launch broke an assumption its kernel was specialised for and was discarded
    bool launch_one(Batch& b, int64_t r0, int64_t r1, int n_groups, const Kernel& k) {
        cudaStream_t st = ctx->stream;
        size_t tot_bytes = (size_t)n_groups * n_words * 16;
        if (!have_totals()) {
            dense.totals = std::make_shared<DeviceBuf>(tot_bytes);
            dense.groups = n_groups;
        }
        if (!dense.spill || dense.spill->bytes < tot_bytes) {
            dense.spill = std::make_shared<DeviceBuf>(tot_bytes);
            cuda_check(cudaMemsetAsync(dense.spill->ptr, 0, dense.spill->bytes, st), "memset spill");
        }
        clear_vmask();
        cb::PipeParams p;
        fill_inputs(p, b, k.g.tile, r0, r1);
        bind_str_masks(p, k.spec, b);
        int grid = grid_for(ctx, p.n_tiles);
        size_t part_bytes = (size_t)grid * tot_bytes;
        if (!dense.partials || dense.partials->bytes < part_bytes) dense.partials = std::make_shared<DeviceBuf>(part_bytes);
        p.n_groups = n_groups;
        for (size_t i = 0; i < dense.cards.size() && i < CB_MAX_KEYS; i++) p.key_card[i] = dense.cards[i];
        p.partials = (cb::u8*)dense.partials->ptr;
        p.spill = (cb::u64*)dense.spill->ptr;
        p.vmask = (cb::u64*)vmask->ptr;
        launch(k.mod->kernel(k.g.entry), dim3(grid), dim3(k.g.threads + 32), k.g.dyn_smem(n_groups), &p); // + producer warp
        ctx->pipeline_rows += r1 - r0;
        ValueMasks masks;
        copy_vmask(masks);
        ctx->check_device_errors(); // synchronises
        // validate the assumptions this kernel was specialised for; either way, remember what was seen so a retry is specialised correctly
        const std::vector<int> seen = mask_bits(k.spec, masks);
        bool ok = true;
        for (size_t i = 0; i < seen.size(); i++)
            if (k.spec.cols[i].assume_bits > 0 && seen[i] > k.spec.cols[i].assume_bits) ok = false;
        observe(seen);
        if (!ok) {
            // discard this launch: partials are simply not folded; the exact-escape accumulators must be cleared
            cuda_check(cudaMemsetAsync(dense.spill->ptr, 0, dense.spill->bytes, st), "memset spill");
            return false;
        }
        rows_scanned += r1 - r0;
        cb::FinParams fp;
        memset(&fp, 0, sizeof(fp));
        fp.partials = (const cb::u64*)dense.partials->ptr;
        fp.spill = (cb::u64*)dense.spill->ptr;
        fp.totals = (cb::u64*)dense.totals->ptr;
        fp.n_ctas = grid;
        fp.n_groups = n_groups;
        fp.first = have_totals() ? 0 : 1;
        fp.err = ctx->d_err;
        int total_words = n_groups * n_words;
        void* args[] = {&fp};
        cuda_check(cudaLaunchKernel((const void*)k.mod->kernel("cb_fold"), dim3((total_words + 127) / 128), dim3(128), args, 0, st), "fold launch");
        ctx->kernel_launches++;
        last = k;
        return true;
    }

    // ---- id-addressed state rows (table and stream strategies) -------------------------------------------------------------------
    // one launch of the table or stream kernel over rows [r0, r1) of b; the stream strategy has no key table
    void launch_id_rows(Batch& b, int64_t r0, int64_t r1, const Kernel& k, bool with_table) {
        clear_vmask();
        cb::PipeParams p;
        fill_inputs(p, b, k.g.tile, r0, r1);
        bind_str_masks(p, k.spec, b);
        p.hkeys = with_table ? (cb::u64*)table.hkeys->ptr : nullptr;
        p.hkey_of_gid = (cb::u64*)rows.hkey_of_gid->ptr;
        p.htotals = (cb::u64*)rows.htotals->ptr;
        p.hmask = with_table ? (cb::u32)(table.hcap - 1) : 0;
        p.max_groups = (cb::i32)rows.max_groups;
        p.hflags = (cb::i32*)rows.hflags->ptr;
        p.vmask = (cb::u64*)vmask->ptr;
        p.n_groups = 2;
        launch(k.mod->kernel(k.g.entry), dim3(grid_for(ctx, p.n_tiles)), dim3(k.g.threads + 32), k.g.dyn_smem(0), &p);
    }

    // ---- table strategy ----------------------------------------------------------------------------------------------------------
    void consume_table(Batch& b) {
        // updates go straight into the table, so a launch cannot be discarded: no speculative assumptions here
        const Kernel k = compile(make_spec(&b, Strategy::Table, 2, SAFE));
        {
            TraceSpan ts("hash.ensure_table");
            table.ensure(ctx, k, rows, b.n_rows, child->rows_hint(), rows_scanned, mode != AggMode::Partial);
        }
        launch_id_rows(b, 0, b.n_rows, k, true);
        ctx->pipeline_rows += b.n_rows;
        ValueMasks masks;
        int flags[8];
        copy_vmask(masks);
        cuda_check(cudaMemcpyAsync(flags, rows.hflags->ptr, sizeof(flags), cudaMemcpyDeviceToHost, ctx->stream), "read hash flags"); ctx->d2h_bytes += (int64_t)(sizeof(flags));
        ctx->check_device_errors();
        if (flags[0] & CB_HF_FULL) throw ExecError(15, "", "internal: hash table full");
        if (flags[0] & CB_HF_WIDE_KEY) throw Unsupported("decimal(p > 18) group key whose value does not fit 64 bits");
        observe(mask_bits(k.spec, masks));
        rows_scanned += b.n_rows;
        last = k;
    }

    // ---- stream strategy ---------------------------------------------------------------------------------------------------------
    // one CB_STREAM launch over rows [r0, r1) of b; returns the state rows handed out so far (and the flags / per-range counts after it)
    int64_t stream_launch(Batch& b, int64_t r0, int64_t r1, const Kernel& k, HashFlags& hf, int64_t cnt[GK]) {
        launch_id_rows(b, r0, r1, k, false);
        ValueMasks masks;
        copy_vmask(masks);
        ctx->check_device_errors();
        const int64_t total = rows.read_flags(ctx, hf, cnt);
        if (hf.w[0] & CB_HF_WIDE_KEY) throw Unsupported("decimal(p > 18) group key whose value does not fit 64 bits");
        if (!(hf.w[0] & CB_HF_FULL)) observe(mask_bits(k.spec, masks));
        return total;
    }
    // On entering hash aggregation: are equal keys adjacent?  Run the stream kernel over the first rows of the first batch and look at
    // state rows per input row.  True: the stream strategy; false: the key table (whatever the sample allocated is dropped).
    bool sample_stream(Batch& b) {
        if (mode != AggMode::Partial || ctx->stream_agg_min_rows < 0) return false;
        if (b.n_rows + std::max<int64_t>(child->rows_hint(), 0) < ctx->stream_agg_min_rows || b.n_rows == 0) return false;
        const Kernel k = compile(make_spec(&b, Strategy::Stream, 2, SAFE));
        const int64_t sample = std::min<int64_t>(b.n_rows, 1 << 20);
        HashFlags hf;
        int64_t cnt[GK] = {0};
        stream.ensure_rows(ctx, k, rows, cnt, 2 * sample + 4096); // room for every row being its own run, in whichever ranges the warps draw from
        const int64_t runs = stream_launch(b, 0, sample, k, hf, cnt);
        stream.ratio = (hf.w[0] & CB_HF_FULL) ? 1.0 : (double)runs / (double)sample;
        // the sample's rows are scanned again with the rest: forget its state rows (and whatever it added to the shared NULL-key group)
        memset(&hf, 0, sizeof(hf));
        rows.write_flags(ctx, hf);
        IdRows::init_totals(ctx, k, (cb::u64*)rows.htotals->ptr, rows.max_groups, 2);
        if (stream.ratio <= ctx->stream_agg_max_ratio) return true;
        rows = IdRows();
        n_words = 0; word_kinds.clear();
        return false;
    }
    void consume_stream(Batch& b) {
        const Kernel k = compile(make_spec(&b, Strategy::Stream, 2, SAFE));
        HashFlags before, hf;
        int64_t cnt0[GK], cnt[GK];
        const int64_t cur = rows.read_flags(ctx, before, cnt0);
        // state rows this batch (and, when the source says how much is still to come, the rest) will need at the ratio seen so far
        const int64_t remaining = std::max<int64_t>(child->rows_hint(), 0);
        int64_t want = cur + std::min<int64_t>(b.n_rows, (int64_t)(1.25 * stream.ratio * (double)b.n_rows) + 65536);
        if (!rows.htotals || want > rows.max_groups) want += std::min<int64_t>(remaining, (int64_t)(1.25 * stream.ratio * (double)remaining));
        int64_t handed_out;
        while (true) {
            {
                TraceSpan ts("stream.ensure_rows");
                stream.ensure_rows(ctx, k, rows, cnt0, want);
            }
            stream.snapshot_reserved(ctx, rows, n_words, false);
            handed_out = stream_launch(b, 0, b.n_rows, k, hf, cnt);
            if (!(hf.w[0] & CB_HF_FULL)) break;
            // more runs than state rows: nothing of this launch is kept (its rows only touched ids past the old counts and the shared group)
            stream.snapshot_reserved(ctx, rows, n_words, true);
            for (int r = 0; r < GK; r++) before.w[CB_HFLAG_CTR + r] = (int)cnt0[r];
            rows.write_flags(ctx, before);
            want = cur + b.n_rows + GK; // every row its own run
        }
        ctx->pipeline_rows += b.n_rows;
        if (b.n_rows > 0) stream.ratio = std::max(stream.ratio, (double)(handed_out - cur) / (double)b.n_rows);
        rows_scanned += b.n_rows;
        last = k;
    }

    // Host side of the overflow certificate: a bound on the magnitude of any single addend of decimal SUM / AVG `ai`, from the value
    // masks observed on its input columns pushed through the same range propagation the code generator uses.  finalize multiplies
    // it by the group's own addend count (cb::cert_level): n * B <= 10^p - 1 means no row order can overflow.
    u128r certificate(size_t ai) const {
        const AggExpr& a = aggs[ai];
        if (!(a.kind == AggKind::Sum || a.kind == AggKind::Avg) || !a.datatype.is_decimal()) return 0;
        std::vector<u128r> bounds(child->schema.size(), RSAT);
        for (size_t c = 0; c < bounds.size(); c++)
            if (child->schema[c].is_decimal() && !observed_bits.empty())
                bounds[c] = observed_bits[c] < 0 ? 0 : (observed_bits[c] >= 127 ? RSAT : (u128r)1 << observed_bits[c]);
        if (mode == AggMode::Partial) return expr_maxabs(*a.children[0], bounds);
        return bounds[(size_t)state_cols[ai][0]];
    }
    // finalize parameters with every aggregate's certificate
    cb::FinParams certified_params() const {
        cb::FinParams fp;
        memset(&fp, 0, sizeof(fp));
        fp.err = ctx->d_err;
        for (size_t ai = 0; ai < aggs.size() && ai < CB_MAX_OUT; ai++) {
            const u128r b = certificate(ai);
            fp.cert_b[ai][0] = b >= RSAT ? ~0ull : (uint64_t)b;
            fp.cert_b[ai][1] = b >= RSAT ? ~0ull : (uint64_t)(b >> 64);
            // bit 63 of the high word (free: B < 2^127): B is the bound 2^bits of a value mask, i.e. addends lie in [-B, B - 1]
            const bool direct = mode != AggMode::Partial || aggs[ai].children[0]->kind == ExprKind::Bound;
            if (b < RSAT && b != 0 && direct) fp.cert_b[ai][1] |= 1ull << 63;
        }
        return fp;
    }

    bool next(Batch& out) override {
        if (!emitted) aggregate_input();
        if (outq_pos >= outq.size()) return false;
        out = std::move(outq[outq_pos++]);
        return true;
    }
    // consume every input batch, then queue the result after whatever a dense -> hash migration flushed
    void aggregate_input() {
        if (keys.size() > CB_MAX_KEYS) throw Unsupported("more than 4 group keys");
        key_has_null.assign(keys.size(), false);
        key_dicts.assign(keys.size(), nullptr);
        dev_dicts.assign(keys.size(), nullptr);
        Batch in;
        while (child->next(in)) {
            if (in.n_rows == 0) continue;
            consume(in);
            ctx->check_device_errors();
        }
        emitted = true;
        if (!have_totals()) {
            if (!ungrouped) return; // grouped aggregate over no (further) rows
            // ungrouped aggregate over an empty input still emits one row: run finalize over identities
            last = compile(make_spec(nullptr, Strategy::Dense, 1));
            std::vector<uint64_t> id((size_t)n_words * 2, 0);
            for (int w = 0; w < n_words; w++) id[(size_t)w * 2] = identity_word(word_kinds[(size_t)w]);
            dense.totals = std::make_shared<DeviceBuf>(id.size() * 8);
            cuda_check(cudaMemcpyAsync(dense.totals->ptr, id.data(), id.size() * 8, cudaMemcpyHostToDevice, ctx->stream), "identity totals");
            cuda_check(cudaStreamSynchronize(ctx->stream), "identity totals sync");
            dense.groups = 1;
        }
        Batch result;
        if (strategy == Strategy::Table || strategy == Strategy::Stream) rows.finalize(ctx, last, certified_params(), key_dicts, result);
        else dense.finalize(ctx, last, certified_params(), ungrouped, schema, key_dicts, result);
        outq.push_back(std::move(result));
    }
};

} // namespace

ExecNodeP make_agg_node(const OperatorP& agg_op, const ExecNodeP& src, const std::vector<ExprP>& preds, const std::vector<ExprP>& cols, ExecContext* ctx,
                        const std::vector<int>& assume_bits) {
    auto n = std::make_shared<AggNode>();
    n->ctx = ctx;
    n->child = src;
    n->schema = agg_op->schema;
    n->predicates = preds;
    n->mode = agg_op->mode;
    n->ungrouped = agg_op->grouping.empty();
    n->assume_bits = assume_bits;
    std::vector<ExprP> roots = preds;
    for (auto& gexp : agg_op->grouping) {
        ExprP k = substitute(gexp, cols);
        if (k->kind != ExprKind::Bound) throw Unsupported("computed group keys (only plain column keys are fused)");
        n->keys.push_back(k);
        roots.push_back(k);
    }
    size_t state_at = agg_op->grouping.size();
    for (auto& a : agg_op->aggs) {
        AggExpr c = a;
        if (agg_op->mode == AggMode::Partial) {
            for (auto& ch : c.children) { ch = substitute(ch, cols); roots.push_back(ch); }
            if (c.filter) { c.filter = substitute(c.filter, cols); roots.push_back(c.filter); }
        } else {
            std::vector<int> sc;
            for (size_t k = 0; k < agg_state_types(a).size(); k++) {
                ExprP e = cols.at(state_at++);
                if (e->kind != ExprKind::Bound) throw Unsupported("final aggregate over computed state columns");
                sc.push_back(e->index);
                roots.push_back(e);
            }
            n->state_cols.push_back(sc);
        }
        n->aggs.push_back(c);
    }
    n->assign_slots(roots);
    if (n->used_cols.empty()) {
        // COUNT(*) / COUNT(1) alone reads no column: stage the narrowest fixed-width one just to drive the row loop
        int best = -1, best_w = 1 << 30;
        for (size_t c = 0; c < src->schema.size(); c++) {
            const DType& t = src->schema[c];
            if (t.is_string()) continue;
            int w = std::max(1, phys_bytes(phys_of(t)));
            if (w < best_w) { best = (int)c; best_w = w; }
        }
        if (best < 0) throw Unsupported("COUNT(*) over a child with only string columns");
        n->used_cols.push_back(best);
        n->slot_of[best] = 0;
    }
    return n;
}

} // namespace cb200