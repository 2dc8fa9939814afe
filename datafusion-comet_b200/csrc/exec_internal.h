// exec_internal.h -- what the executor's translation units share: the fused-pipeline node base, the physical encoding of a
// logical type, the expression-slot helpers, the shared-memory budget of a pipeline kernel, the operator factories and the row
// primitives of the row operators.
#pragma once
#include "exec.h"

#include "aot_kernels.h"
#include "device/cb_params.h"

#include <algorithm>
#include <cstring>
#include <functional>
#include <map>
#include <set>

namespace cb200 {

static constexpr size_t SMEM_BUDGET = 220 * 1024;

inline Phys phys_of(const DType& t) {
    switch (t.id) {
    case TypeId::Bool: return Phys::Bitmap;
    case TypeId::Int8: return Phys::I8;
    case TypeId::Int16: return Phys::I16;
    case TypeId::Int32: case TypeId::Date: return Phys::I32;
    case TypeId::Int64: case TypeId::Timestamp: case TypeId::TimestampNtz: return Phys::I64;
    case TypeId::Float32: return Phys::F32;
    case TypeId::Float64: return Phys::F64;
    case TypeId::Decimal: return Phys::I128;
    default: return Phys::I32;
    }
}
// the layout a generated kernel writes an output column of type t in: booleans one byte per row, strings as int32 dictionary codes
inline Phys kernel_out_phys(const DType& t) { return t.id == TypeId::Bool ? Phys::I8 : t.is_string() ? Phys::I32 : phys_of(t); }

// ---- bitmaps -------------------------------------------------------------------------------------------------------
// bytes of a device bitmap of n rows: whole 32-bit words, plus 8 bytes of slack
inline size_t bitmap_bytes(int64_t n) { return (size_t)(n + 31) / 32 * 4 + 8; }
// a new device bitmap of n rows, bit r set where bytes[r] != 0 (one launch on ctx->stream, counted)
DeviceBufP bytes_to_bitmap(const DeviceBufP& bytes, int64_t n, ExecContext* ctx);
// n bytes (nonzero = set) as a host bitmap, 8 bytes of slack behind it
std::vector<uint8_t> pack_bits(const uint8_t* bytes, size_t n);

// ---- expression helpers --------------------------------------------------------------------------------------------
inline ExprP clone_expr(const ExprP& e) {
    auto c = std::make_shared<Expr>(*e);
    for (auto& ch : c->children) ch = clone_expr(ch);
    return c;
}
// replace Bound(i) by cur[i]
inline ExprP substitute(const ExprP& e, const std::vector<ExprP>& cur) {
    if (e->kind == ExprKind::Bound) {
        if (e->index < 0 || e->index >= (int)cur.size()) throw PlanError("bound reference out of range while fusing");
        return clone_expr(cur[e->index]);
    }
    auto c = std::make_shared<Expr>(*e);
    for (auto& ch : c->children) ch = substitute(ch, cur);
    return c;
}
inline void collect_bound(const ExprP& e, std::vector<int>& order, std::set<int>& seen) {
    if (e->kind == ExprKind::Bound) {
        if (!seen.count(e->index)) { seen.insert(e->index); order.push_back(e->index); }
        return;
    }
    for (auto& c : e->children) collect_bound(c, order, seen);
}
inline void rewrite_bound(const ExprP& e, const std::map<int, int>& slot_of) {
    if (e->kind == ExprKind::Bound) { e->index = slot_of.at(e->index); return; }
    for (auto& c : e->children) rewrite_bound(c, slot_of);
}

// ---- string predicate masks ----------------------------------------------------------------------------------------
// A string predicate is decided once per dictionary entry: a device bitmask over the codes of its column, read by the pipeline kernel
// (codegen.cpp emit_str_pred).  Dictionaries only grow and codes never change (Dictionary: a batch's dictionary is unified into
// the plan-wide one, the Parquet scan interns into one dictionary per column), so a mask is brought up to date before every launch
// that reads it by evaluating only the entries added since the previous one.  A column that carries another Dictionary object starts
// again from entry 0.
struct StrMask {
    DictionaryP dict;                // the dictionary `done` refers to
    int64_t done = 0;                // entries evaluated
    DeviceBufP bits;                 // mask words (capacity grows geometrically)
    DeviceBufP payload;              // the predicate's literals / LIKE items on the device
    cb::StrPredDev dev{};
    DeviceBufP off, chars;           // the tail of the dictionary being evaluated ...
    std::vector<int32_t> h_off;      // ... and its host staging (kept: the copies are asynchronous)
    std::string h_chars;
};
struct StrMasks {
    std::map<std::string, StrMask> by_key; // "<source column>@<str_pred_key>"
    // update the masks of every string predicate of `spec` for batch b and bind them to p.smask
    void bind(cb::PipeParams& p, const PipelineSpec& spec, const Batch& b, ExecContext* ctx);
};

// ---- fused pipeline nodes ------------------------------------------------------------------------------------------
struct FusedBase : ExecNode {
    ExecContext* ctx;
    ExecNodeP child;
    std::vector<ExprP> predicates;   // over child columns (Bound.index = child column)
    std::vector<int> used_cols;      // child columns staged, in slot order
    std::map<int, int> slot_of;

    std::vector<ExecNodeP> children() const override { return {child}; }

    // build the staged-column list for one batch signature
    std::vector<SourceCol> stage_cols(const Batch* b) const { return stage_cols_of(b, used_cols); }
    std::vector<SourceCol> stage_cols_of(const Batch* b, const std::vector<int>& which) const {
        std::vector<SourceCol> cols;
        for (int ci : which) {
            SourceCol sc;
            sc.src_index = ci;
            sc.type = child->schema[ci];
            if (b) {
                const Column& c = b->cols[ci];
                sc.phys = c.phys;
                sc.has_validity = c.validity != nullptr;
                if (c.is_dict) sc.phys = c.phys == Phys::I8 ? Phys::I8 : c.phys == Phys::I16 ? Phys::I16 : Phys::Dict32;
            } else {
                sc.phys = sc.type.is_string() ? Phys::Dict32 : phys_of(sc.type);
                sc.has_validity = false;
            }
            cols.push_back(sc);
        }
        return cols;
    }
    void assign_slots(const std::vector<ExprP>& roots) {
        std::set<int> seen;
        for (auto& e : roots) collect_bound(e, used_cols, seen);
        for (size_t i = 0; i < used_cols.size(); i++) slot_of[used_cols[i]] = (int)i;
    }
    static std::vector<ExprP> to_slots(const std::vector<ExprP>& es, const std::map<int, int>& slot_of) {
        std::vector<ExprP> out;
        for (auto& e : es) {
            ExprP c = clone_expr(e);
            rewrite_bound(c, slot_of);
            out.push_back(c);
        }
        return out;
    }
    void fill_inputs(cb::PipeParams& p, const Batch& b, int tile, int64_t row0 = 0, int64_t row1 = -1) const { fill_inputs_of(p, b, used_cols, tile, row0, row1); }
    void fill_inputs_of(cb::PipeParams& p, const Batch& b, const std::vector<int>& which, int tile, int64_t row0 = 0, int64_t row1 = -1) const {
        memset(&p, 0, sizeof(p));
        if (row1 < 0) row1 = b.n_rows;
        if (row0 & 1023) throw ExecError(15, "", "internal: launch range must start on a 1024-row boundary");
        for (size_t i = 0; i < which.size(); i++) {
            const Column& c = b.cols[which[i]];
            if (!c.data) throw Unsupported("column " + std::to_string(which[i]) + " (" + c.type.str() + ") has no fixed-width device representation");
            int w = phys_bytes(c.phys);
            p.col[i] = (const cb::u8*)c.data->ptr + (w == 0 ? row0 / 8 : row0 * w);
            p.val[i] = c.validity ? (const cb::u8*)c.validity->ptr + row0 / 8 : nullptr;
        }
        p.n_rows = row1 - row0;
        p.n_tiles = (int)((p.n_rows + tile - 1) / tile);
        p.err = ctx->d_err;
    }
    // the string predicate masks a launch of `spec` over b reads (after fill_inputs*, which clears p)
    StrMasks str_masks;
    void bind_str_masks(cb::PipeParams& p, const PipelineSpec& spec, const Batch& b) { str_masks.bind(p, spec, b, ctx); }
    void launch(cudaKernel_t k, dim3 grid, dim3 block, size_t smem, void* params) {
        cuda_check(cudaFuncSetAttribute((const void*)k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute(smem)");
        void* args[] = {params};
        if (ctx->ev_pending) { cuda_check(cudaStreamSynchronize(ctx->stream), "stream sync"); ctx->collect_timing(); }
        cuda_check(cudaEventRecord(ctx->ev0, ctx->stream), "event record");
        cuda_check(cudaLaunchKernel((const void*)k, grid, block, args, smem, ctx->stream), "kernel launch");
        cuda_check(cudaEventRecord(ctx->ev1, ctx->stream), "event record");
        ctx->ev_pending = true;
        ctx->kernel_launches++;
    }
};

// The predicate-only pass of a filter (SinkKind::Count) over staged columns `cols`: per (1024-row logical tile, warp) the rows every
// predicate keeps in PipeParams::sel_off, and with PipeParams::sel_mask one keep bit per row (bit r & 31 of word r >> 5, whole words up
// to the last row's).  A filter's first pass; a join condition's evaluation over its candidate pairs.
PipelineSpec count_pass_spec(std::vector<SourceCol> cols, std::vector<ExprP> predicates);

// agg.cpp: the aggregate `agg_op` over `src`, whose columns pass through the fused filters `preds` and projections `cols`.
// `assume_bits`: build-time value-range assumptions per source column (see cb200_compile_plan_assume); empty at run time.
ExecNodeP make_agg_node(const OperatorP& agg_op, const ExecNodeP& src, const std::vector<ExprP>& preds, const std::vector<ExprP>& cols, ExecContext* ctx,
                        const std::vector<int>& assume_bits);
// partition.cpp, sort.cpp, join.cpp: the row operators over their built children; each validates its operator's fields
ExecNodeP make_partition_node(const OperatorP& op, const ExecNodeP& child, ExecContext* ctx);
ExecNodeP make_sort_node(const OperatorP& op, const ExecNodeP& child, ExecContext* ctx);
ExecNodeP make_join_node(const OperatorP& op, const ExecNodeP& left, const ExecNodeP& right, ExecContext* ctx);

// ---- row primitives shared by repartitioning, Sort and the joins (rows.cpp) ------------------------------------------
// The HK_* kind of a key column (device/cb_sortkey.h).  The logical type decides how Spark hashes a value (utils.rs: i8 / i16 / i32 /
// date as i32, decimal(p <= 18) as i64, wider decimals as 16 bytes) and how many bits its sort key takes; the stored layout (DESIGN.md,
// "Data layout in HBM") decides how it is read.
int key_kind(const Column& c);
// a new device buffer holding host bytes [p, p + n), safe to use once this returns (it synchronises); not counted in h2d_bytes
DeviceBufP host_to_device(const void* p, size_t n, ExecContext* ctx, const char* what);
// small host-resident aggregate results -> device columns
void columns_to_device(Batch& b, ExecContext* ctx);
// a batch arriving at a Sort or join: columns_to_device, and plain Utf8 columns refused (`op`: "sorting", "joining")
void arrive(Batch& b, ExecContext* ctx, const char* op);
// every batch of `child`, arrived (`op` as in arrive) and concatenated (`concat_op` as in concat_batches); no rows if it has none
Batch drain(ExecNode& child, ExecContext* ctx, const char* op, const char* concat_op);
// out's columns = in's rows row_idx[0, n), in that order.  Bit-packed booleans and validity are gathered one byte per row and repacked
// (the byte forms are kept: the exchange sends them).  `op` names the operator in the refusal of plain Utf8 columns.  I: long long or
// unsigned.
template <typename I> void gather_columns(const Batch& in, const I* row_idx, int64_t n, Batch& out, ExecContext* ctx, const char* op);
// gather_columns for the columns of a join side that may be NULL-extended: row index CB_NULL_ROW gives a NULL, and every column gets a
// validity bitmap (byte form kept) whether or not a row is NULL, so its layout is the same in every batch.  Plain Utf8 never gets here
// (arrive refuses it).
void gather_columns_or_null(const Batch& in, const unsigned* row_idx, int64_t n, Batch& out, ExecContext* ctx);
// the rows of bs in one batch (`bs` non-empty, every batch on the device): values and validity appended in order; dictionary-coded strings
// that carry different Dictionary objects are recoded into one (the first batch's entries, then the others' new entries)
Batch concat_batches(const std::vector<Batch>& bs, ExecContext* ctx, const char* op);
// column c as the row-key field at bit `off` (advanced past it), with a null bit if has_null.  The caller sets desc, nulls_first and rank.
cb::SortKeyCol key_field(const Column& c, bool has_null, int& off);
// the row keys of kc (W = kc.words words each) for n rows, and_or[0, W) their AND and [W, 2W) their OR, `digits` the 8-bit digits of the
// `bits`-bit key that are not the same in every row, least significant first.  Synchronises: a dictionary code outside its dictionary
// fails here.
struct RowKeys { DeviceBufP keys; uint64_t and_or[2 * cb::SK_MAX_WORDS]; std::vector<int> digits; };
RowKeys pack_row_keys(const cb::SortKeyCols& kc, int64_t n, int bits, ExecContext* ctx);
// the stable order of m rows whose keys (`words` words each) are in keys0, by the given digits: row indices [0, m); `sorted_keys`, if
// given, receives the keys in that order
DeviceBufP radix_order(ExecContext* ctx, DeviceBufP keys0, int words, int64_t m, const std::vector<int>& digits, DeviceBufP* sorted_keys = nullptr);
// The stable compaction of n rows by their keep flags (one byte per row): the kept rows' 32-bit indices in order, in a buffer of `cap`
// rows, and their count.  Each `extra` (array, bytes per row) is compacted by the same plan into extra_out, `cap` rows each.  Reading
// the count synchronises and checks the error flags.
struct Compacted { DeviceBufP rows; int64_t n = 0; std::vector<DeviceBufP> extra_out; };
Compacted compact_rows(const DeviceBufP& keep, int64_t n, int64_t cap, ExecContext* ctx, const std::vector<std::pair<DeviceBufP, int>>& extra = {});
// A device table indexed by the codes of a column's dictionary, made on the host by `make` and counted in h2d_bytes; rebuilt when the
// column carries another dictionary or its dictionary has grown.  Holding the dictionary keeps a new one at a freed one's address apart.
struct DictCodes {
    DictionaryP dict; size_t n = 0; DeviceBufP table;
    const uint32_t* get(const DictionaryP& d, ExecContext* ctx, const std::function<std::vector<uint32_t>(const Dictionary&)>& make);
};

} // namespace cb200
