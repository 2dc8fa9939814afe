// exec_internal.h -- what the executor's translation units share: the fused-pipeline node base, the physical encoding of a
// logical type, the expression-slot helpers and the shared-memory budget of a pipeline kernel.
#pragma once
#include "exec.h"

#include "aot_kernels.h"
#include "device/cb_params.h"

#include <cstring>
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
// (codegen.cpp emit_str_pred).  Dictionaries only grow and codes never change (Dictionary::values: a batch's dictionary is unified into
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

    // build time: the pipelines this node may launch, for inputs without nulls and with dictionary-encoded strings
    virtual std::vector<PipelineSpec> build_specs() const = 0;

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
            int w = phys_bytes(c.is_dict && c.phys == Phys::I32 ? Phys::Dict32 : c.phys);
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

// agg.cpp: the aggregate `agg_op` over `src`, whose columns pass through the fused filters `preds` and projections `cols`.
// `assume_bits`: build-time value-range assumptions per source column (see cb200_compile_plan_assume); empty at run time.
ExecNodeP make_agg_node(const OperatorP& agg_op, const ExecNodeP& src, const std::vector<ExprP>& preds, const std::vector<ExprP>& cols, ExecContext* ctx,
                        const std::vector<int>& assume_bits);

} // namespace cb200
