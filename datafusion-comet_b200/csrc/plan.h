// plan.h -- in-memory form of the reference's plan IR (spark.spark_operator.Operator and friends)
// after decoding, plus the type rules the reference's planner applies
// (native/core/src/execution/planner.rs:446-1131 create_expr / create_binary_expr_with_options,
//  :2558-2917 create_agg_expr, serde.rs:71-110 to_arrow_datatype).
#pragma once
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

namespace cb200 {

struct Unsupported : std::runtime_error { // plan uses something outside the GPU hot path -> caller falls back
    using std::runtime_error::runtime_error;
};
struct PlanError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

// types.proto:43-66 DataTypeId (only the ids on the hot path are accepted)
enum class TypeId : int {
    Bool = 0, Int8 = 1, Int16 = 2, Int32 = 3, Int64 = 4, Float32 = 5, Float64 = 6, String = 7, Binary = 8,
    Timestamp = 9, Decimal = 10, TimestampNtz = 11, Date = 12, Null = 13
};

struct DType {
    TypeId id = TypeId::Null;
    int precision = 0, scale = 0;
    bool is_decimal() const { return id == TypeId::Decimal; }
    bool is_integer() const { return id == TypeId::Int8 || id == TypeId::Int16 || id == TypeId::Int32 || id == TypeId::Int64; }
    bool is_float() const { return id == TypeId::Float32 || id == TypeId::Float64; }
    bool is_string() const { return id == TypeId::String || id == TypeId::Binary; }
    bool operator==(const DType& o) const {
        return id == o.id && (id != TypeId::Decimal || (precision == o.precision && scale == o.scale));
    }
    bool operator!=(const DType& o) const { return !(*this == o); }
    std::string str() const;
    // bytes of one value in Arrow layout (0 = bitmap-packed bool, -1 = variable width)
    int arrow_width() const;
};
inline DType mk_decimal(int p, int s) { DType d; d.id = TypeId::Decimal; d.precision = p; d.scale = s; return d; }
inline DType mk_type(TypeId id) { DType d; d.id = id; return d; }

enum class EvalMode : int { Legacy = 0, Try = 1, Ansi = 2 }; // expr.proto:324

enum class ExprKind {
    Literal, Bound, Unbound,
    Add, Sub, Mul, Div,
    Eq, Neq, Gt, GtEq, Lt, LtEq,
    IsNull, IsNotNull, And, Or, Not,
    Cast, CheckOverflow, UnaryMinus, If, In,
    StrPred // a predicate on a dictionary-coded string column against literals (children[0]: the Bound column)
};

// StrPred operations (the values of cb::StrOp, device/cb_strpred.h)
enum class StrOp : int { Eq, Neq, Lt, LtEq, Gt, GtEq, In, Like, StartsWith, EndsWith, Contains };

struct Expr;
using ExprP = std::shared_ptr<Expr>;

struct Expr {
    ExprKind kind;
    std::vector<ExprP> children;
    DType type;            // resolved result type (what PhysicalExpr::data_type would return)
    // Literal
    bool lit_null = false;
    int64_t lit_i64 = 0;   // bool/int/date/timestamp
    double lit_f64 = 0;    // float/double
    uint64_t lit_bits = 0; // float/double: the value's own 32 / 64 bits as sent (NaN payloads kept)
    unsigned __int128 lit_dec = 0; // decimal unscaled (two's complement)
    std::string lit_str;
    // Bound / Unbound
    int index = -1;
    std::string name;
    // MathExpr / Cast / CheckOverflow / UnaryMinus
    DType return_type;
    EvalMode eval_mode = EvalMode::Legacy;
    bool fail_on_error = false;
    bool negated = false;  // In
    bool integral_div = false;          // Div: IntegralDivide (expr.proto:81): the quotient without the HALF_UP digit
    bool check_divide_overflow = false; // MathExpr.check_divide_overflow (expr.proto:335-340)
    // decimal arithmetic lowering chosen by the reference's rule (planner.rs:998-1027)
    bool wide_decimal = false;
    // StrPred: the literals (In: the non-NULL members; Like: the pattern text), whether an In list holds a NULL, and the compiled LIKE
    // pattern (cb_strpred.h items).  The generated kernel sees none of these: they only decide the per-code mask.
    StrOp str_op = StrOp::Eq;
    std::vector<std::string> str_lits;
    bool in_has_null = false;
    std::vector<uint16_t> like_items;
};

enum class AggKind { Count, Sum, Min, Max, Avg };
enum class AggMode : int { Partial = 0, Final = 1, PartialMerge = 2 }; // operator.proto AggregateMode

struct AggExpr {
    AggKind kind;
    std::vector<ExprP> children; // Count may have several
    DType datatype;              // result type
    DType sum_datatype;          // Avg: sum state type
    EvalMode eval_mode = EvalMode::Legacy;
    ExprP filter;                // FILTER (WHERE ...) clause, Partial mode only
    // this aggregate's own mode: the operator's, or its HashAggregate.expr_modes entry.  Partial updates from `children`;
    // PartialMerge / Final merge the state columns that start at child column `state_at` (-1 for Partial).
    AggMode mode = AggMode::Partial;
    int state_at = -1;
};

// HashJoin: both HashJoin (operator field 109) and SortMergeJoin (108) plans, which one join node runs
enum class OpKind { Scan, ShuffleScan, NativeScan, Projection, Filter, HashAgg, ShuffleWriter, Sort, HashJoin };

// operator.proto JoinType / BuildSide
enum class JoinType : int { Inner = 0, LeftOuter = 1, RightOuter = 2, FullOuter = 3, LeftSemi = 4, LeftAnti = 5 };

// ShuffleWriter partitioning (partitioning.proto Partitioning): SinglePartition runs as a hash partitioning without keys
enum class PartKind { Hash, Range, RoundRobin };

// one ORDER BY key (SortOrder expr.proto:385-389, planner.rs:927-950 create_sort_expr): arrow SortOptions{descending, nulls_first}
struct SortKey {
    ExprP expr;               // a Bound column reference of the child
    bool descending = false;  // direction == 1
    bool nulls_first = true;  // null_ordering == 0
};

struct StructField {
    std::string name;
    DType type;
    bool nullable = true;
};

struct Operator;
using OperatorP = std::shared_ptr<Operator>;

struct Operator {
    OpKind kind;
    uint32_t plan_id = 0;
    std::vector<OperatorP> children;
    std::vector<DType> schema;       // output column types (child col_i naming is positional)
    // Scan / ShuffleScan
    std::vector<DType> fields;
    std::string source;
    // NativeScan
    std::vector<StructField> required_schema, data_schema;
    std::vector<int64_t> projection_vector;
    std::vector<ExprP> data_filters;
    std::vector<std::string> files;
    std::vector<int64_t> file_start, file_length; // SparkPartitionedFile.start / length (operator.proto:103-109); 0 / 0 = the whole file
    // Projection
    std::vector<ExprP> project_list;
    // Filter
    ExprP predicate;
    // HashAgg
    std::vector<ExprP> grouping;
    std::vector<AggExpr> aggs;
    AggMode mode = AggMode::Partial; // the operator's mode (each aggregate's own: AggExpr::mode)
    // ShuffleWriter.  Hash: hash_exprs.  RoundRobin: hash_exprs are Bound columns 0 .. k-1 (max_hash_columns as the reference reads it),
    // which may be more than 8.  Range: range_keys are the sort orders with repeated columns dropped (the first occurrence kept), and
    // range_bounds the n_bounds boundary rows packed as row keys of range_words words (device/cb_sortkey.h; every field has a null bit,
    // the last key at bit 0), non-decreasing.  A string key's field is its rank against range_strs[key], that key's distinct
    // boundary strings in byte order (device/cb_rangepart.h).
    PartKind part_kind = PartKind::Hash;
    std::vector<ExprP> hash_exprs;
    int num_partitions = 0;
    int max_hash_columns = 0;
    std::vector<SortKey> range_keys;
    std::vector<uint64_t> range_bounds;
    int64_t n_bounds = 0;
    int range_words = 1;
    std::vector<std::vector<std::string>> range_strs;
    // Sort (operator.proto:641-645): the output is sorted[skip : fetch] (SortExec::with_fetch, then GlobalLimitExec(skip));
    // -1 = the field is absent
    std::vector<SortKey> sort_keys;
    int64_t fetch = -1, skip = -1;
    // HashJoin (operator.proto:754-763) and SortMergeJoin (:765-771): equi-join on Bound key columns of children[0] (left) and
    // children[1] (right).  Inner and the outer types: the output is the left columns, then the right ones; LeftSemi / LeftAnti: the
    // left columns.  A sort-merge join's build side follows from its type: the left one for RightOuter, else the right one.
    // BroadcastNestedLoopJoin (:773-777) is the same operator without keys: every (left row, right row) pair is a candidate.
    std::vector<ExprP> left_keys, right_keys;
    JoinType join_type = JoinType::Inner;
    bool build_left = false; // BuildLeft: the left child is the build side (the hash table), the right one is probed
    // the join condition (JoinFilter, planner.rs:2462-2542), or null: a boolean over the left columns followed by the right ones
    // (Bound.index = left column, or left column count + right column), whatever the build side and join type
    ExprP join_condition;
};

// Sort keys at most: 8 keys, 256 bits of packed key (value bits by declared type plus one null bit per key, sort_key_bits)
enum { MAX_SORT_KEYS = 8, MAX_SORT_KEY_BITS = 256 };
// value bits of a sort key of type t in the packed row key; throws Unsupported for types outside the sort
int sort_key_bits(const DType& t);

// Decode + resolve types.  Throws Unsupported for anything outside the GPU hot path and PlanError
// for malformed plans.
OperatorP decode_plan(const uint8_t* data, size_t len);

// state-column layout an aggregate exposes in Partial mode / consumes in Final mode
// (sum_decimal.rs:112-120, avg_decimal.rs:132-145, avg.rs:82-95, sum_int.rs:75-84)
std::vector<DType> agg_state_types(const AggExpr& a);
DType agg_result_type(const AggExpr& a);

std::string expr_str(const Expr& e);

} // namespace cb200
