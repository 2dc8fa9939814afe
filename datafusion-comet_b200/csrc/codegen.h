// codegen.h -- turns one fused pipeline (source columns -> filters/projections -> sink) into the CUDA
// translation unit that NVRTC compiles: generated `cb_row_*` / `cb_finalize` bodies spliced into the
// hand-written skeletons of device/cb_kernels.cuh.
#pragma once
#include "plan.h"

#include <map>
#include <string>
#include <vector>

namespace cb200 {

// physical encoding of a staged source column
enum class Phys { Bitmap, I8, I16, I32, I64, F32, F64, I128, Dict32 };
int phys_bytes(Phys p); // 0 for Bitmap

struct SourceCol {
    int src_index;   // column index in the source's schema
    DType type;      // logical type
    Phys phys;
    bool has_validity;
    int assume_bits = 0; // decimal columns: kernel may assume |v| < 2^assume_bits (validated by the value masks); 0 = no assumption
    // aggregate sinks: an earlier batch of the same aggregate carried validity for this column.  The accumulator layout keeps the
    // column's null tests apart (as if has_validity) so that it never narrows again; the null tests emitted are this batch's own.
    bool layout_nullable = false;
};

// thread-private 64-bit partial sums are exact while rows/thread <= 2^CB_RPT_LOG2 (host enforces it per launch)
#define CB_RPT_LOG2 14

enum class SinkKind { Select, Agg, Count }; // Count: pass 1 of a select pipeline (predicates only, see cb_kernels.cuh)

// accumulator word kinds (must match cb_kernels.cuh)
enum WordKind { W_SUM128 = 0, W_DD_HI = 1, W_DD_LO = 2, W_WRAP64 = 3, W_MIN = 4, W_MAX = 5 };

struct OutCol {     // one output column of the pipeline (select output or aggregate state/result column)
    DType type;
    bool nullable;
};

struct PipelineSpec {
    std::vector<SourceCol> cols;          // staged columns, position = slot in PipeParams.col[]
    std::vector<ExprP> predicates;        // keep row iff every predicate is TRUE (exprs over staged cols: Bound.index = slot)
    SinkKind sink = SinkKind::Select;
    // Select
    std::vector<ExprP> outputs;
    // Agg
    std::vector<ExprP> keys;              // each must be Bound to a Dict32 / Bitmap staged column (dense path)
    std::vector<bool> key_nullable;
    std::vector<AggExpr> aggs;            // each by its own AggExpr::mode: children/filter over staged cols (Partial), or state_slots
    std::vector<std::vector<int>> state_slots; // per agg: staged-col slot of each of its state columns (empty for a Partial agg)
    AggMode mode = AggMode::Partial;      // the operator's mode; with no aggregates (keys only) it alone says whether rows are state rows
    bool ungrouped = false;
    bool hash = false;                    // high-cardinality: global open-addressing table keyed by the packed key columns
    bool masked = false;                  // Select sink: the keep decision comes from pass 1's bit mask (PipeParams::sel_mask), not from `predicates`
    bool stream = false;                  // hash + Partial over clustered keys: one state row per run of equal adjacent keys, no key table (CB_STREAM)
    // tuning
    int tile = 512, stages = 3, threads = 256;
    int ltile = 0;                        // Count sink: rows of one logical tile of the select pass (tile is a multiple of it)
};

struct GeneratedKernel {
    std::string source;        // full translation unit
    std::string key;           // cache key (hash of source)
    std::string entry;         // cb_pipeline_agg | cb_pipeline_select
    std::string finalize_entry;// cb_finalize (agg only)
    int stage_bytes = 0;
    int n_words = 0;           // agg: accumulator words per group
    std::vector<int> word_kinds;
    // agg: the word of each accumulator role: [0] the row count (CB_W_ROWS), then per aggregate its sum, count, bits, bad, min / max
    // and abs words (-1: unused).  Two layouts of one aggregate correspond role by role (see widen_word_map).
    std::vector<int> role_words;
    std::vector<OutCol> out_cols;     // select: outputs; agg: finalize outputs (excluding key columns)
    std::vector<int> out_bytes;       // element bytes of each output column (1 for bool-as-byte)
    int threads = 256, tile = 512, stages = 3;
    bool hash = false;
    bool ungrouped = false;           // aggregate without keys: accumulators in registers (CB_G1)
    int n_key_cols = 0;               // hash: leading out_cols are the group keys
    int key_words = 1;                // hash: 64-bit words of the packed group key (1: the word is the table key; >1: tag + stored key)
    size_t dyn_smem(int n_groups) const;
};

GeneratedKernel generate_pipeline(const PipelineSpec& spec);

// For each accumulator word of layout `to`, the word of layout `from` it starts as: both are layouts of one aggregate, `to` with at
// least the nullable inputs of `from`.  Words that shared a row count in `from` and are apart in `to` both start from it, which is
// exact: every row seen so far counted toward each.  Empty when `to` does not refine `from` role by role.
std::vector<int> widen_word_map(const GeneratedKernel& from, const GeneratedKernel& to);

// The distinct string predicates (ExprKind::StrPred) of a pipeline in mask-slot order: PipeParams::smask[i] holds the mask of entry i.
// Order: predicates, outputs, group keys, then the arguments and FILTER clauses of Partial-mode aggregates, each depth first.  Throws
// Unsupported above CB_MAX_STR_PREDS.
std::vector<ExprP> str_preds_of(const PipelineSpec& spec);
// what one StrPred computes per dictionary entry: operation and literals.  Two nodes with equal keys over the same column share a mask.
std::string str_pred_key(const Expr& e);
// canonical text of a pipeline (expressions, column encodings, sink): equal specs give equal strings
std::string pipeline_signature(const PipelineSpec& spec);

} // namespace cb200
