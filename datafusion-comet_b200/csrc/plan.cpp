// plan.cpp -- decode the reference's protobuf plan IR and resolve expression types the way the
// reference's planner does.  Field numbers: native/proto/src/proto/{operator,expr,literal,types,
// partitioning}.proto (cited inline).  Type rules: native/core/src/execution/planner.rs.
#include "plan.h"
#include "proto_wire.h"
#include "device/cb_rangepart.h"
#include "device/cb_sortkey.h"
#include "device/cb_strpred.h"

#include <algorithm>
#include <cstring>
#include <sstream>

namespace cb200 {

std::string DType::str() const {
    switch (id) {
    case TypeId::Bool: return "bool";
    case TypeId::Int8: return "int8";
    case TypeId::Int16: return "int16";
    case TypeId::Int32: return "int32";
    case TypeId::Int64: return "int64";
    case TypeId::Float32: return "float32";
    case TypeId::Float64: return "float64";
    case TypeId::String: return "utf8";
    case TypeId::Binary: return "binary";
    case TypeId::Timestamp: return "timestamp[us,UTC]";
    case TypeId::TimestampNtz: return "timestamp[us]";
    case TypeId::Date: return "date32";
    case TypeId::Null: return "null";
    case TypeId::Decimal: {
        std::ostringstream o;
        o << "decimal128(" << precision << "," << scale << ")";
        return o.str();
    }
    }
    return "?";
}

int DType::arrow_width() const {
    switch (id) {
    case TypeId::Bool: return 0;
    case TypeId::Int8: return 1;
    case TypeId::Int16: return 2;
    case TypeId::Int32: case TypeId::Float32: case TypeId::Date: return 4;
    case TypeId::Int64: case TypeId::Float64: case TypeId::Timestamp: case TypeId::TimestampNtz: return 8;
    case TypeId::Decimal: return 16;
    default: return -1;
    }
}

// ---- DataType (types.proto:43-114) ----------------------------------------------------------------
static DType decode_dtype(PbReader r) {
    DType d;
    int id = 0;
    while (r.next()) {
        if (r.field == 1) id = (int)r.i64();
        else if (r.field == 2) { // DataTypeInfo
            PbReader info = r.sub();
            while (info.next()) {
                if (info.field == 2) { // DecimalInfo
                    PbReader di = info.sub();
                    while (di.next()) {
                        if (di.field == 1) d.precision = (int)di.i64();
                        else if (di.field == 2) d.scale = (int)di.i64();
                        else di.skip();
                    }
                } else throw Unsupported("nested data types (list/map/struct) are outside the GPU hot path");
            }
        } else r.skip();
    }
    if (id < 0 || id > 13) throw Unsupported("data type id " + std::to_string(id) + " is outside the GPU hot path");
    d.id = (TypeId)id;
    return d;
}

static ExprP decode_expr(PbReader r);

static ExprP mk(ExprKind k) {
    auto e = std::make_shared<Expr>();
    e->kind = k;
    return e;
}

// Literal (literal.proto:26-47): value is big-endian two's-complement bytes for decimals
// (planner.rs:544-548 BigInt::from_signed_bytes_be).
static ExprP decode_literal(PbReader r) {
    auto e = mk(ExprKind::Literal);
    bool have_value = false;
    std::string dec_bytes;
    while (r.next()) {
        switch (r.field) {
        case 1: case 2: case 3: case 4: case 5: e->lit_i64 = r.i64(); have_value = true; break;
        case 6: { const uint32_t u = r.fixed32(); float f; memcpy(&f, &u, 4); e->lit_f64 = (double)f; e->lit_bits = u; have_value = true; break; }
        case 7: { const uint64_t u = r.fixed64(); memcpy(&e->lit_f64, &u, 8); e->lit_bits = u; have_value = true; break; }
        case 8: case 9: e->lit_str = r.bytes(); have_value = true; break;
        case 10: dec_bytes = r.bytes(); have_value = true; break;
        case 11: throw Unsupported("list literals are outside the GPU hot path");
        case 12: e->type = decode_dtype(r.sub()); break;
        case 13: e->lit_null = r.i64() != 0; break;
        default: r.skip();
        }
    }
    if (!dec_bytes.empty() || e->type.is_decimal()) {
        if (dec_bytes.size() > 16) throw PlanError("decimal literal does not fit in i128");
        unsigned __int128 v = (!dec_bytes.empty() && ((uint8_t)dec_bytes[0] & 0x80)) ? ~(unsigned __int128)0 : 0;
        for (unsigned char c : dec_bytes) v = (v << 8) | c;
        e->lit_dec = v;
    }
    if (e->type.id == TypeId::Int8) e->lit_i64 = (int8_t)e->lit_i64;
    if (e->type.id == TypeId::Int16) e->lit_i64 = (int16_t)e->lit_i64;
    if (e->type.id == TypeId::Int32 || e->type.id == TypeId::Date) e->lit_i64 = (int32_t)e->lit_i64;
    if (!have_value && !e->lit_null && e->type.id != TypeId::Null) {
        // proto3 omits default-valued scalars: a present-but-zero literal (0, false, 0.0, "")
    }
    return e;
}

static ExprP decode_binary(ExprKind k, PbReader r, bool math) {
    auto e = mk(k);
    ExprP l, rr;
    while (r.next()) {
        if (r.field == 1) l = decode_expr(r.sub());
        else if (r.field == 2) rr = decode_expr(r.sub());
        else if (math && r.field == 4) e->return_type = decode_dtype(r.sub());
        else if (math && r.field == 5) e->eval_mode = (EvalMode)r.i64();
        else if (math && r.field == 6) e->check_divide_overflow = r.i64() != 0;
        else r.skip();
    }
    if (!l || !rr) throw PlanError("binary expression is missing an operand");
    e->children = {l, rr};
    return e;
}

static ExprP decode_unary(ExprKind k, PbReader r) {
    auto e = mk(k);
    while (r.next()) {
        if (r.field == 1) e->children.push_back(decode_expr(r.sub()));
        else if (k == ExprKind::UnaryMinus && r.field == 2) e->fail_on_error = r.i64() != 0;
        else r.skip();
    }
    if (e->children.size() != 1) throw PlanError("unary expression is missing its child");
    return e;
}

// Expr (expr.proto:30-109)
static ExprP decode_expr(PbReader r) {
    ExprP out;
    while (r.next()) {
        if (r.wire != 2) { r.skip(); continue; } // expr_id (91) etc.
        switch (r.field) {
        case 2: out = decode_literal(r.sub()); break;
        case 3: { // BoundReference expr.proto:375
            out = mk(ExprKind::Bound);
            PbReader b = r.sub();
            while (b.next()) {
                if (b.field == 1) out->index = (int)b.i64();
                else if (b.field == 2) out->type = decode_dtype(b.sub());
                else b.skip();
            }
            if (out->index < 0) out->index = 0;
            break;
        }
        case 51: { // UnboundReference
            out = mk(ExprKind::Unbound);
            PbReader b = r.sub();
            while (b.next()) {
                if (b.field == 1) out->name = b.bytes();
                else if (b.field == 2) out->type = decode_dtype(b.sub());
                else b.skip();
            }
            break;
        }
        case 4: out = decode_binary(ExprKind::Add, r.sub(), true); break;
        case 5: out = decode_binary(ExprKind::Sub, r.sub(), true); break;
        case 6: out = decode_binary(ExprKind::Mul, r.sub(), true); break;
        case 7: out = decode_binary(ExprKind::Div, r.sub(), true); break;
        case 59: out = decode_binary(ExprKind::Div, r.sub(), true); out->integral_div = true; break; // IntegralDivide
        case 8: { // Cast expr.proto:337
            out = mk(ExprKind::Cast);
            PbReader c = r.sub();
            while (c.next()) {
                if (c.field == 1) out->children.push_back(decode_expr(c.sub()));
                else if (c.field == 2) out->return_type = decode_dtype(c.sub());
                else if (c.field == 4) out->eval_mode = (EvalMode)c.i64();
                else c.skip();
            }
            if (out->children.size() != 1) throw PlanError("cast is missing its child");
            break;
        }
        case 9: out = decode_binary(ExprKind::Eq, r.sub(), false); break;
        case 10: out = decode_binary(ExprKind::Neq, r.sub(), false); break;
        case 11: out = decode_binary(ExprKind::Gt, r.sub(), false); break;
        case 12: out = decode_binary(ExprKind::GtEq, r.sub(), false); break;
        case 13: out = decode_binary(ExprKind::Lt, r.sub(), false); break;
        case 14: out = decode_binary(ExprKind::LtEq, r.sub(), false); break;
        case 15: out = decode_unary(ExprKind::IsNull, r.sub()); break;
        case 16: out = decode_unary(ExprKind::IsNotNull, r.sub()); break;
        case 17: out = decode_binary(ExprKind::And, r.sub(), false); break;
        case 18: out = decode_binary(ExprKind::Or, r.sub(), false); break;
        case 25: { // CheckOverflow
            out = mk(ExprKind::CheckOverflow);
            PbReader c = r.sub();
            while (c.next()) {
                if (c.field == 1) out->children.push_back(decode_expr(c.sub()));
                else if (c.field == 2) out->return_type = decode_dtype(c.sub());
                else if (c.field == 3) out->fail_on_error = c.i64() != 0;
                else c.skip();
            }
            if (out->children.size() != 1) throw PlanError("check_overflow is missing its child");
            break;
        }
        case 39: { // In
            out = mk(ExprKind::In);
            PbReader c = r.sub();
            while (c.next()) {
                if (c.field == 1 || c.field == 2) out->children.push_back(decode_expr(c.sub()));
                else if (c.field == 3) out->negated = c.i64() != 0;
                else c.skip();
            }
            break;
        }
        case 40: out = decode_unary(ExprKind::Not, r.sub()); break;
        case 41: out = decode_unary(ExprKind::UnaryMinus, r.sub()); break;
        case 44: { // IfExpr
            out = mk(ExprKind::If);
            PbReader c = r.sub();
            ExprP a, b, d;
            while (c.next()) {
                if (c.field == 1) a = decode_expr(c.sub());
                else if (c.field == 2) b = decode_expr(c.sub());
                else if (c.field == 3) d = decode_expr(c.sub());
                else c.skip();
            }
            if (!a || !b || !d) throw PlanError("if expression is missing an operand");
            out->children = {a, b, d};
            break;
        }
        case 38: { // CaseWhen expr.proto:473 -> nested IF chain (planner.rs:677-703 builds a CaseExpr with expr = None)
            PbReader c = r.sub();
            std::vector<ExprP> whens, thens;
            ExprP els;
            while (c.next()) {
                if (c.field == 2) whens.push_back(decode_expr(c.sub()));
                else if (c.field == 3) thens.push_back(decode_expr(c.sub()));
                else if (c.field == 4) els = decode_expr(c.sub());
                else c.skip();
            }
            if (whens.empty() || whens.size() != thens.size()) throw PlanError("CASE WHEN needs matching when/then lists");
            ExprP tail = els; // may be null: ELSE NULL, typed when types are resolved
            for (size_t i = whens.size(); i-- > 0;) {
                ExprP n = mk(ExprKind::If);
                n->children = {whens[i], thens[i]};
                if (tail) n->children.push_back(tail);
                tail = n;
            }
            out = tail;
            break;
        }
        case 26: { // Like: BinaryExpr (left, pattern); lowered in resolve
            out = decode_binary(ExprKind::StrPred, r.sub(), false);
            out->str_op = StrOp::Like;
            break;
        }
        case 31: { // ScalarFunc expr.proto:466 {func = 1, args = 2, return_type = 3, fail_on_error = 4}
            PbReader c = r.sub();
            std::string func;
            std::vector<ExprP> args;
            while (c.next()) {
                if (c.field == 1) func = c.bytes();
                else if (c.field == 2) args.push_back(decode_expr(c.sub()));
                else c.skip();
            }
            // Comet sends Spark's StartsWith / EndsWith / Contains under these names (serde/strings.scala CometScalarFunction)
            if (func != "starts_with" && func != "ends_with" && func != "contains")
                throw Unsupported("scalar function '" + func + "' is outside the GPU hot path");
            if (args.size() != 2) throw PlanError("scalar function " + func + " expects two arguments");
            out = mk(ExprKind::StrPred);
            out->str_op = func == "starts_with" ? StrOp::StartsWith : func == "ends_with" ? StrOp::EndsWith : StrOp::Contains;
            out->children = args;
            break;
        }
        case 90: r.skip(); break; // query_context
        default:
            throw Unsupported("expression field " + std::to_string(r.field) + " is outside the GPU hot path");
        }
    }
    if (!out) throw PlanError("empty expression");
    return out;
}

// ---- type resolution ------------------------------------------------------------------------------
static bool cast_supported(const DType& from, const DType& to) {
    if (from == to) return true;
    auto numeric = [](const DType& d) { return d.is_integer() || d.is_float(); };
    if (numeric(from) && numeric(to)) {
        // widening / int->float only (narrowing needs Spark's overflow rules: conversion_funcs/numeric.rs)
        auto rank = [](const DType& d) {
            switch (d.id) {
            case TypeId::Int8: return 1; case TypeId::Int16: return 2; case TypeId::Int32: return 3;
            case TypeId::Int64: return 4; case TypeId::Float32: return 5; case TypeId::Float64: return 6;
            default: return 0;
            }
        };
        return rank(to) >= rank(from);
    }
    if (from.is_integer() && to.is_decimal()) return true;
    if (from.is_decimal() && to.is_decimal()) return true;
    return false;
}

// ---- string predicates ----------------------------------------------------------------------------------------------------
static bool is_str_col(const Expr& e) { return e.kind == ExprKind::Bound && e.type.id == TypeId::String; }
static bool is_str_lit(const Expr& e) { return e.kind == ExprKind::Literal && e.type.id == TypeId::String; }
static void to_null_bool(Expr& e) { // a NULL literal operand: the predicate is NULL on every row
    e.kind = ExprKind::Literal;
    e.children.clear();
    e.lit_null = true;
    e.type = mk_type(TypeId::Bool);
}

// Lowers a comparison, IN, LIKE or starts_with / ends_with / contains whose operand is a string to StrPred over the Bound column,
// or throws Unsupported.  Only column-vs-literal shapes are evaluated: the predicate is decided once per dictionary entry.
static void lower_string_predicate(Expr& e) {
    const char* what = e.kind == ExprKind::In ? "IN" : e.kind == ExprKind::StrPred ? "string function" : "comparison";
    if (e.kind == ExprKind::In) {
        if (!is_str_col(*e.children[0])) throw Unsupported(std::string("IN over a string that is not a column reference (") + e.children[0]->type.str() + ")");
        std::vector<std::string> lits;
        bool has_null = false;
        for (size_t i = 1; i < e.children.size(); i++) {
            const Expr& m = *e.children[i];
            if (!is_str_lit(m)) throw Unsupported("IN over utf8 with a member that is not a utf8 literal");
            if (m.lit_null) has_null = true;
            else lits.push_back(m.lit_str);
        }
        if (lits.empty() && has_null) { to_null_bool(e); return; } // NULL value -> NULL, anything else -> no match, list has NULL -> NULL
        e.str_op = StrOp::In;
        e.str_lits = lits;
        e.in_has_null = has_null;
    } else {
        ExprP col = e.children[0], lit = e.children[1];
        StrOp op = e.str_op;
        if (e.kind != ExprKind::StrPred) {
            static const StrOp ops[] = {StrOp::Eq, StrOp::Neq, StrOp::Gt, StrOp::GtEq, StrOp::Lt, StrOp::LtEq};
            op = ops[(int)e.kind - (int)ExprKind::Eq];
            if (is_str_lit(*col) && is_str_col(*lit)) { // literal <op> column: mirror
                std::swap(col, lit);
                op = op == StrOp::Lt ? StrOp::Gt : op == StrOp::LtEq ? StrOp::GtEq : op == StrOp::Gt ? StrOp::Lt : op == StrOp::GtEq ? StrOp::LtEq : op;
            }
        }
        if (!is_str_col(*col)) throw Unsupported(std::string(what) + " over " + col->type.str() + " that is not a string column reference");
        if (!is_str_lit(*lit)) throw Unsupported(std::string(what) + " between " + col->type.str() + " and " + lit->type.str() + " (only a string column against a string literal)");
        if (lit->lit_null) { to_null_bool(e); return; }
        e.str_op = op;
        e.str_lits = {lit->lit_str};
        if (op == StrOp::Like) {
            std::vector<uint16_t> items(lit->lit_str.size());
            const int k = cb::sp_like_compile((const uint8_t*)lit->lit_str.data(), (int)lit->lit_str.size(), items.data());
            if (k < 0) throw Unsupported("LIKE pattern with a '\\' that escapes something other than '%', '_' or '\\', or ends the pattern");
            items.resize((size_t)k);
            e.like_items = items;
        }
        e.children = {col};
    }
    e.kind = ExprKind::StrPred;
    e.type = mk_type(TypeId::Bool);
}

static void resolve(Expr& e, const std::vector<DType>& in) {
    for (auto& c : e.children) resolve(*c, in);
    auto ct = [&](int i) -> const DType& { return e.children[i]->type; };
    switch (e.kind) {
    case ExprKind::StrPred: lower_string_predicate(e); break;
    case ExprKind::Literal: case ExprKind::Unbound: break;
    case ExprKind::Bound:
        if (e.index >= (int)in.size()) throw PlanError("bound reference index " + std::to_string(e.index) + " out of range");
        e.type = in[e.index];
        break;
    case ExprKind::Add: case ExprKind::Sub: case ExprKind::Mul: {
        const DType &l = ct(0), &r = ct(1);
        if (l.is_decimal() && r.is_decimal()) {
            // planner.rs:998-1027: wide path when the arrow-arith result could exceed precision 38
            bool wide;
            if (e.kind == ExprKind::Mul) wide = l.precision + r.precision >= 38;
            else wide = std::max(l.scale, r.scale) + std::max(l.precision - l.scale, r.precision - r.scale) >= 38;
            e.wide_decimal = wide;
            if (wide) {
                if (!e.return_type.is_decimal()) throw PlanError("Expected Decimal128 return type");
                e.type = e.return_type;
            } else if (e.kind == ExprKind::Mul) {
                e.type = mk_decimal(std::min(l.precision + r.precision + 1, 38), l.scale + r.scale);
            } else {
                int rs = std::max(l.scale, r.scale);
                e.type = mk_decimal(std::min(rs + std::max(l.precision - l.scale, r.precision - r.scale) + 1, 38), rs);
            }
        } else if ((l.is_integer() || l.is_float()) && l == r) {
            e.type = e.return_type.id == TypeId::Null ? l : e.return_type;
            if (e.type != l) throw Unsupported("arithmetic with implicit result cast " + l.str() + " -> " + e.type.str());
        } else {
            throw Unsupported("arithmetic on " + l.str() + " and " + r.str());
        }
        break;
    }
    case ExprKind::Div: {
        const DType &l = ct(0), &r = ct(1);
        if (l.is_decimal() && r.is_decimal()) { // decimal_div / decimal_integral_div UDFs (planner.rs:1028-1058): result type = the proto's
            if (!e.return_type.is_decimal()) throw PlanError("decimal division without a Decimal128 return type");
            e.type = e.return_type;
        } else if ((l.is_float() || l.is_integer()) && l == r) {
            if (e.integral_div && l.is_float()) throw Unsupported("integral division of floats");
            e.type = e.return_type.id == TypeId::Null ? l : e.return_type;
            if (e.type != l) throw Unsupported("division with implicit result cast " + l.str() + " -> " + e.type.str());
        } else throw Unsupported("division on " + l.str() + " and " + r.str());
        break;
    }
    case ExprKind::Eq: case ExprKind::Neq: case ExprKind::Gt: case ExprKind::GtEq: case ExprKind::Lt: case ExprKind::LtEq: {
        const DType &l = ct(0), &r = ct(1);
        if (l.id == TypeId::String && r.id == TypeId::String) { lower_string_predicate(e); break; }
        bool ok = l == r || (l.is_decimal() && r.is_decimal() && l.scale == r.scale);
        if (!ok || l.is_string() || l.id == TypeId::Null)
            throw Unsupported("comparison between " + l.str() + " and " + r.str());
        e.type = mk_type(TypeId::Bool);
        break;
    }
    case ExprKind::And: case ExprKind::Or:
        if (ct(0).id != TypeId::Bool || ct(1).id != TypeId::Bool) throw PlanError("AND/OR over non-boolean operands");
        e.type = mk_type(TypeId::Bool);
        break;
    case ExprKind::Not:
        if (ct(0).id != TypeId::Bool) throw PlanError("NOT over non-boolean operand");
        e.type = mk_type(TypeId::Bool);
        break;
    case ExprKind::IsNull: case ExprKind::IsNotNull: e.type = mk_type(TypeId::Bool); break;
    case ExprKind::Cast:
        if (!cast_supported(ct(0), e.return_type))
            throw Unsupported("cast " + ct(0).str() + " -> " + e.return_type.str() + " is outside the GPU hot path");
        e.type = e.return_type;
        break;
    case ExprKind::CheckOverflow:
        if (!ct(0).is_decimal() || !e.return_type.is_decimal()) throw PlanError("CheckOverflow expects only Decimal128");
        e.type = e.return_type;
        break;
    case ExprKind::UnaryMinus:
        if (ct(0).is_string() || ct(0).id == TypeId::Bool) throw Unsupported("negation of " + ct(0).str());
        e.type = ct(0);
        break;
    case ExprKind::If:
        if (e.children.size() == 2) { // CASE without ELSE: NULL of the THEN type
            auto nul = std::make_shared<Expr>();
            nul->kind = ExprKind::Literal;
            nul->lit_null = true;
            nul->type = ct(1);
            e.children.push_back(nul);
        }
        if (ct(0).id != TypeId::Bool || ct(1) != ct(2)) throw Unsupported("IF with mismatched branch types");
        e.type = ct(1);
        break;
    case ExprKind::In:
        if (ct(0).id == TypeId::String) { lower_string_predicate(e); break; }
        for (size_t i = 1; i < e.children.size(); i++) {
            if (e.children[i]->kind != ExprKind::Literal) throw Unsupported("IN list with non-literal members");
            const DType &l = ct(0), &r = ct((int)i);
            if (!(l == r || (l.is_decimal() && r.is_decimal() && l.scale == r.scale)) || l.is_string())
                throw Unsupported("IN over " + l.str() + " / " + r.str());
        }
        e.type = mk_type(TypeId::Bool);
        break;
    }
}

// ---- aggregates -----------------------------------------------------------------------------------
static AggExpr decode_agg(PbReader r) { // AggExpr expr.proto:143-176
    AggExpr a;
    bool have = false;
    while (r.next()) {
        if (r.wire != 2) { r.skip(); continue; }
        if (r.field >= 2 && r.field <= 6) {
            PbReader b = r.sub();
            have = true;
            switch (r.field) {
            case 2: a.kind = AggKind::Count; break;
            case 3: a.kind = AggKind::Sum; break;
            case 4: a.kind = AggKind::Min; break;
            case 5: a.kind = AggKind::Max; break;
            case 6: a.kind = AggKind::Avg; break;
            }
            while (b.next()) {
                if (b.field == 1) a.children.push_back(decode_expr(b.sub()));
                else if (a.kind != AggKind::Count && b.field == 2) a.datatype = decode_dtype(b.sub());
                else if (a.kind == AggKind::Sum && b.field == 3) a.eval_mode = (EvalMode)b.i64();
                else if (a.kind == AggKind::Avg && b.field == 3) a.sum_datatype = decode_dtype(b.sub());
                else if (a.kind == AggKind::Avg && b.field == 4) a.eval_mode = (EvalMode)b.i64();
                else b.skip();
            }
        } else if (r.field == 89) a.filter = decode_expr(r.sub());
        else if (r.field == 90) r.skip();
        else throw Unsupported("aggregate function field " + std::to_string(r.field) + " is outside the GPU hot path");
    }
    if (!have) throw PlanError("empty aggregate expression");
    if (a.kind == AggKind::Count) a.datatype = mk_type(TypeId::Int64);
    return a;
}

DType agg_result_type(const AggExpr& a) {
    switch (a.kind) {
    case AggKind::Count: return mk_type(TypeId::Int64);
    case AggKind::Avg: return a.datatype.is_decimal() ? a.datatype : mk_type(TypeId::Float64); // planner.rs:2656-2676
    default: return a.datatype;
    }
}

std::vector<DType> agg_state_types(const AggExpr& a) {
    switch (a.kind) {
    case AggKind::Count: return {mk_type(TypeId::Int64)};
    case AggKind::Sum:
        if (a.datatype.is_decimal()) return {a.datatype, mk_type(TypeId::Bool)}; // (sum, is_empty) sum_decimal.rs:112-120
        if (a.datatype.is_integer()) {
            if (a.eval_mode == EvalMode::Try) return {mk_type(TypeId::Int64), mk_type(TypeId::Bool)}; // sum_int.rs:75-84
            return {mk_type(TypeId::Int64)};
        }
        return {a.datatype};
    case AggKind::Avg:
        if (a.datatype.is_decimal()) return {a.sum_datatype, mk_type(TypeId::Int64)}; // avg_decimal.rs:132-145
        return {mk_type(TypeId::Float64), mk_type(TypeId::Int64)};                    // avg.rs:82-95
    case AggKind::Min: case AggKind::Max: return {a.datatype};
    }
    return {};
}

static void resolve_agg(AggExpr& a, const std::vector<DType>& in, AggMode mode) {
    if (mode == AggMode::Partial) {
        for (auto& c : a.children) resolve(*c, in);
        if (a.filter) resolve(*a.filter, in);
    }
    if (a.children.empty()) throw PlanError("aggregate without arguments");
    const DType& dt = a.datatype;
    switch (a.kind) {
    case AggKind::Count: break;
    case AggKind::Sum:
        if (!(dt.is_decimal() || dt.is_integer() || dt.id == TypeId::Float64 || dt.id == TypeId::Float32))
            throw Unsupported("SUM over " + dt.str());
        break;
    case AggKind::Avg:
        if (dt.is_decimal() && !a.sum_datatype.is_decimal()) throw PlanError("AVG(decimal) without a decimal sum type");
        if (!dt.is_decimal() && !(dt.id == TypeId::Float64)) throw Unsupported("AVG result type " + dt.str());
        break;
    case AggKind::Min: case AggKind::Max:
        if (!(dt.is_integer() || dt.id == TypeId::Date || dt.id == TypeId::Timestamp || dt.id == TypeId::TimestampNtz ||
              dt.id == TypeId::Float64 || (dt.is_decimal() && dt.precision <= 18)))
            throw Unsupported("MIN/MAX over " + dt.str());
        break;
    }
    if (mode == AggMode::Partial && a.kind != AggKind::Count) {
        const DType& ct = a.children[0]->type;
        bool ok = ct == dt || (a.kind == AggKind::Avg) ||
                  (a.kind == AggKind::Sum && ((dt.is_decimal() && ct.is_decimal() && ct.scale == dt.scale) ||
                                              (dt.is_integer() && ct.is_integer()) || (dt.is_float() && (ct.is_float() || ct.is_integer()))));
        if (!ok) throw Unsupported("aggregate input " + ct.str() + " for result " + dt.str());
        if (a.kind == AggKind::Avg) {
            if (dt.is_decimal() && !(ct.is_decimal() && ct.scale == a.sum_datatype.scale))
                throw Unsupported("AVG(decimal) over " + ct.str());
            if (!dt.is_decimal() && !(ct.is_integer() || ct.is_float())) throw Unsupported("AVG over " + ct.str());
        }
    }
}

// ---- operators ------------------------------------------------------------------------------------
static StructField decode_struct_field(PbReader r) { // SparkStructField operator.proto:97-102
    StructField f;
    while (r.next()) {
        if (r.field == 1) f.name = r.bytes();
        else if (r.field == 2) f.type = decode_dtype(r.sub());
        else if (r.field == 3) f.nullable = r.i64() != 0;
        else r.skip();
    }
    return f;
}

// one SortOrder expression (expr.proto:385-389): the Sort operator's keys and the sort-merge join's sort options
static SortKey decode_sort_order(PbReader e) {
    bool have_order = false;
    SortKey k;
    while (e.next()) {
        if (e.field != 19 || e.wire != 2) { e.skip(); continue; }
        have_order = true;
        PbReader so = e.sub();
        while (so.next()) {
            if (so.field == 1) k.expr = decode_expr(so.sub());
            else if (so.field == 2) k.descending = so.i64() == 1;
            else if (so.field == 3) k.nulls_first = so.i64() == 0;
            else so.skip();
        }
    }
    if (!have_order || !k.expr) throw PlanError("sort key is not a SortOrder with a child");
    return k;
}

// the checks HashJoin and SortMergeJoin share before their own: two children, key lists, join type (`what` names the operator)
static void decode_join(Operator& op, const std::string& what, int64_t join_type) {
    if (op.children.size() != 2) throw PlanError(what + " expects two children");
    if (op.left_keys.empty()) throw PlanError(what + " without keys");
    if (op.left_keys.size() != op.right_keys.size())
        throw PlanError(what + " with " + std::to_string(op.left_keys.size()) + " left keys and " + std::to_string(op.right_keys.size()) + " right keys");
    if (join_type < 0 || join_type > 5) throw PlanError("unknown join type " + std::to_string(join_type));
    op.join_type = (JoinType)join_type;
}

// the key pairs resolved against the children's schemas and checked (plain column keys of one type each, at most 8 keys and 256 bits
// of packed key), and the output schema: the left columns, then the right ones unless the join is a semi / anti join
static void resolve_join_keys(Operator& op, const std::string& what) {
    if (op.left_keys.size() > MAX_SORT_KEYS) throw Unsupported("more than 8 " + what + " keys");
    const auto &ls = op.children[0]->schema, &rs = op.children[1]->schema;
    int bits = 0;
    for (size_t i = 0; i < op.left_keys.size(); i++) {
        Expr &l = *op.left_keys[i], &r = *op.right_keys[i];
        resolve(l, ls);
        resolve(r, rs);
        if (l.kind != ExprKind::Bound || r.kind != ExprKind::Bound)
            throw Unsupported("computed " + what + " keys (only plain column keys: put a Projection below the join)");
        if (l.type != r.type) throw PlanError(what + " key " + std::to_string(i) + " is " + l.type.str() + " on the left and " + r.type.str() + " on the right");
        if (l.type.is_float()) throw Unsupported(what + " key of type " + l.type.str() + " (Spark normalises NaN and -0.0 in float keys)");
        if (l.type.id == TypeId::Binary) throw Unsupported(what + " key of type binary");
        bits += sort_key_bits(l.type) + 1; // the sort's key encoding: one null bit per key
    }
    if (bits > MAX_SORT_KEY_BITS) throw Unsupported(what + " keys of " + std::to_string(bits) + " bits (at most 256 bits of packed key)");
    const bool semi_anti = op.join_type == JoinType::LeftSemi || op.join_type == JoinType::LeftAnti;
    op.schema = ls;
    if (!semi_anti) op.schema.insert(op.schema.end(), rs.begin(), rs.end());
}

// the join condition resolved against the left columns followed by the right ones (operators.scala:2634-2640), for every join type.
// What the expression layer refuses stays refused, its message naming the condition.
static void resolve_join_condition(Operator& op) {
    if (!op.join_condition) return;
    std::vector<DType> both = op.children[0]->schema;
    both.insert(both.end(), op.children[1]->schema.begin(), op.children[1]->schema.end());
    try {
        resolve(*op.join_condition, both);
    } catch (const Unsupported& e) {
        throw Unsupported(std::string("join condition: ") + e.what());
    } catch (const PlanError& e) {
        throw PlanError(std::string("join condition: ") + e.what());
    }
    if (op.join_condition->type.id != TypeId::Bool) throw PlanError("join condition is " + op.join_condition->type.str() + ", not boolean");
}

// a join condition's expression (Unsupported -> a refusal naming the condition)
static ExprP decode_join_condition(PbReader r) {
    try {
        return decode_expr(r);
    } catch (const Unsupported& e) {
        throw Unsupported(std::string("join condition: ") + e.what());
    }
}

// RangePartition (planner.rs:3298-3358): the sort orders resolved against the child and deduplicated by column, as DataFusion's
// LexOrdering drops a repeated expression (the JVM sends every sort order but boundary rows of the deduplicated ones,
// CometNativeShuffleWriter.scala:263-326), and the first k entries of each boundary row, k the deduplicated key count, packed once as
// row keys.  A row's partition is then the number of packed bounds <= its packed key (multi_partition.rs:333-380 partition_point).
static void decode_range_partitioning(Operator& op, const std::vector<DType>& cs, std::vector<PbReader>& rows) {
    if (op.range_keys.empty()) throw PlanError("range partitioning without sort orders");
    std::vector<SortKey> keys;
    for (auto& k : op.range_keys) {
        resolve(*k.expr, cs);
        if (k.expr->kind != ExprKind::Bound) throw Unsupported("computed range-partition keys (only plain column keys: put a Projection below the shuffle writer)");
        bool seen = false;
        for (auto& q : keys) seen = seen || q.expr->index == k.expr->index;
        if (!seen) keys.push_back(k);
    }
    op.range_keys = keys;
    const size_t K = keys.size();
    if (K > MAX_SORT_KEYS) throw Unsupported("more than 8 range-partition keys");
    int bits = 0;
    for (auto& k : keys) {
        if (k.expr->type.id == TypeId::Binary) throw Unsupported("range-partition key of type binary");
        try {
            bits += sort_key_bits(k.expr->type) + 1; // every field carries a null bit
        } catch (const Unsupported&) {
            throw Unsupported("range-partition key of type " + k.expr->type.str());
        }
    }
    if (bits > MAX_SORT_KEY_BITS) throw Unsupported("range-partition keys of " + std::to_string(bits) + " bits (at most 256 bits of packed key)");
    if ((int64_t)rows.size() >= op.num_partitions)
        throw PlanError(std::to_string(rows.size()) + " range boundary rows for " + std::to_string(op.num_partitions) + " partitions (at most " +
                        std::to_string(op.num_partitions - 1) + ")");
    // the boundary entries: literals of their key's type
    std::vector<std::vector<ExprP>> bound(rows.size());
    for (size_t r = 0; r < rows.size(); r++) {
        PbReader br = rows[r];
        while (br.next()) {
            if (br.field == 1 && br.wire == 2) bound[r].push_back(decode_expr(br.sub()));
            else br.skip();
        }
        if (bound[r].size() < K)
            throw PlanError("range boundary row " + std::to_string(r) + " has " + std::to_string(bound[r].size()) + " entries for " + std::to_string(K) + " keys");
        for (size_t k = 0; k < K; k++) {
            const Expr& e = *bound[r][k];
            if (e.kind != ExprKind::Literal) throw PlanError("range boundary row " + std::to_string(r) + " entry " + std::to_string(k) + " is not a literal");
            if (e.type != keys[k].expr->type)
                throw PlanError("range boundary row " + std::to_string(r) + " entry " + std::to_string(k) + " is " + e.type.str() + ", its key " + keys[k].expr->type.str());
        }
    }
    op.range_strs.assign(K, {});
    for (size_t k = 0; k < K; k++) {
        if (keys[k].expr->type.id != TypeId::String) continue;
        auto& v = op.range_strs[k];
        for (auto& row : bound)
            if (!row[k]->lit_null) v.push_back(row[k]->lit_str);
        std::sort(v.begin(), v.end());
        v.erase(std::unique(v.begin(), v.end()), v.end());
    }
    // pack each row with the row-key encoder itself: a one-row column per key in the layout the encoder reads for its type
    const int W = op.range_words = std::max(1, (bits + 63) / 64);
    op.n_bounds = (int64_t)rows.size();
    op.range_bounds.assign((size_t)op.n_bounds * W, 0);
    struct Cell { uint64_t v[2]; uint8_t valid; uint32_t rank; };
    std::vector<Cell> cells(K);
    cb::SortKeyCols kc;
    memset(&kc, 0, sizeof(kc));
    kc.n = (int)K;
    kc.words = W;
    int off = 0;
    for (size_t k = K; k-- > 0;) { // the last key is the least significant field
        const DType& t = keys[k].expr->type;
        cb::SortKeyCol& f = kc.col[k];
        f.bits = sort_key_bits(t);
        switch (t.id) {
        case TypeId::Bool: f.kind = HK_BOOL8; break;
        case TypeId::Int8: f.kind = HK_I8; break;
        case TypeId::Int16: f.kind = HK_I16; break;
        case TypeId::Int32: case TypeId::Date: f.kind = HK_I32; break;
        case TypeId::Float32: f.kind = HK_F32; break;
        case TypeId::Float64: f.kind = HK_F64; break;
        case TypeId::Decimal: f.kind = t.precision <= 18 ? HK_DEC_SMALL_64 : HK_DEC_LARGE_128; break;
        case TypeId::String: f.kind = HK_DICT32; f.rank = &cells[k].rank; f.n_rank = 1; break;
        default: f.kind = HK_I64; break; // int64, timestamps
        }
        f.off = off;
        off += f.bits + 1;
        f.desc = keys[k].descending;
        f.nulls_first = keys[k].nulls_first;
        f.has_null = 1;
        f.data = cells[k].v;
        f.validity = &cells[k].valid;
    }
    for (size_t r = 0; r < rows.size(); r++) {
        for (size_t k = 0; k < K; k++) {
            const Expr& e = *bound[r][k];
            Cell& c = cells[k];
            c.v[0] = c.v[1] = 0;
            c.valid = e.lit_null ? 0 : 1;
            c.rank = 0;
            switch (e.type.id) {
            case TypeId::Bool: c.v[0] = e.lit_i64 != 0; break;
            case TypeId::Int8: { const int8_t x = (int8_t)e.lit_i64; memcpy(c.v, &x, 1); break; }
            case TypeId::Int16: { const int16_t x = (int16_t)e.lit_i64; memcpy(c.v, &x, 2); break; }
            case TypeId::Int32: case TypeId::Date: { const int32_t x = (int32_t)e.lit_i64; memcpy(c.v, &x, 4); break; }
            case TypeId::Float32: { const uint32_t x = (uint32_t)e.lit_bits; memcpy(c.v, &x, 4); break; }
            case TypeId::Float64: c.v[0] = e.lit_bits; break;
            case TypeId::Decimal: c.v[0] = (uint64_t)e.lit_dec; c.v[1] = (uint64_t)(e.lit_dec >> 64); break;
            case TypeId::String: {
                const auto& v = op.range_strs[k];
                if (!e.lit_null) c.rank = 2 * (uint32_t)(std::lower_bound(v.begin(), v.end(), e.lit_str) - v.begin()) + 1;
                break;
            }
            default: c.v[0] = (uint64_t)e.lit_i64; break;
            }
        }
        cb::u64* w = (cb::u64*)&op.range_bounds[r * (size_t)W];
        cb::sk_row(kc, 0, w);
        if (r > 0 && std::lexicographical_compare(w, w + W, w - W, w))
            throw PlanError("range boundary row " + std::to_string(r) + " sorts before row " + std::to_string(r - 1) + " (boundary rows must be in ascending order of the sort orders)");
    }
}

static OperatorP decode_operator(PbReader r) { // Operator operator.proto:32-86
    auto op = std::make_shared<Operator>();
    bool have = false;
    std::vector<PbReader> child_readers;
    // children may precede or follow the op payload; decode children first so schemas are known
    struct Pending { uint32_t field; PbReader rd; };
    std::vector<Pending> payload;
    while (r.next()) {
        if (r.field == 1) child_readers.push_back(r.sub());
        else if (r.field == 2) op->plan_id = (uint32_t)r.i64();
        else if (r.field >= 100 && r.wire == 2) payload.push_back({r.field, r.sub()});
        else r.skip();
    }
    for (auto& c : child_readers) op->children.push_back(decode_operator(c));
    if (payload.size() != 1) throw PlanError("operator must carry exactly one op_struct");
    uint32_t f = payload[0].field;
    PbReader b = payload[0].rd;
    auto child_schema = [&]() -> const std::vector<DType>& {
        if (op->children.size() != 1) throw PlanError("operator expects exactly one child");
        return op->children[0]->schema;
    };
    switch (f) {
    case 100: case 116: { // Scan operator.proto:104-107 / ShuffleScan
        op->kind = f == 100 ? OpKind::Scan : OpKind::ShuffleScan;
        while (b.next()) {
            if (b.field == 1) op->fields.push_back(decode_dtype(b.sub()));
            else if (b.field == 2) op->source = b.bytes();
            else b.skip();
        }
        op->schema = op->fields;
        have = true;
        break;
    }
    case 111: { // NativeScan operator.proto:141-185
        op->kind = OpKind::NativeScan;
        while (b.next()) {
            if (b.field == 1) { // NativeScanCommon
                PbReader c = b.sub();
                while (c.next()) {
                    if (c.field == 1) op->required_schema.push_back(decode_struct_field(c.sub()));
                    else if (c.field == 2) op->data_schema.push_back(decode_struct_field(c.sub()));
                    else if (c.field == 3) throw Unsupported("partition columns in NativeScan");
                    else if (c.field == 4) op->data_filters.push_back(decode_expr(c.sub()));
                    else if (c.field == 5) {
                        if (c.wire == 2) { PbReader pk = c.sub(); while (pk.p < pk.end) op->projection_vector.push_back((int64_t)pk.varint()); }
                        else op->projection_vector.push_back(c.i64());
                    } else if (c.field == 12) op->source = c.bytes();
                    else c.skip();
                }
            } else if (b.field == 2) { // SparkFilePartition
                PbReader fp = b.sub();
                while (fp.next()) {
                    if (fp.field == 1) {
                        PbReader pf = fp.sub();
                        int64_t start = 0, length = 0;
                        while (pf.next()) {
                            if (pf.field == 1) op->files.push_back(pf.bytes());
                            else if (pf.field == 2) start = pf.i64();
                            else if (pf.field == 3) length = pf.i64();
                            else if (pf.field == 5) throw Unsupported("partition values in NativeScan");
                            else pf.skip();
                        }
                        op->file_start.push_back(start);
                        op->file_length.push_back(length);
                    } else fp.skip();
                }
            } else b.skip();
        }
        for (auto& sf : op->required_schema) op->schema.push_back(sf.type);
        for (auto& e : op->data_filters) resolve(*e, op->schema);
        have = true;
        break;
    }
    case 101: { // Projection operator.proto:633
        op->kind = OpKind::Projection;
        while (b.next()) {
            if (b.field == 1) op->project_list.push_back(decode_expr(b.sub()));
            else b.skip();
        }
        for (auto& e : op->project_list) { resolve(*e, child_schema()); op->schema.push_back(e->type); }
        have = true;
        break;
    }
    case 102: { // Filter operator.proto:637
        op->kind = OpKind::Filter;
        while (b.next()) {
            if (b.field == 1) op->predicate = decode_expr(b.sub());
            else b.skip();
        }
        if (!op->predicate) throw PlanError("filter without predicate");
        resolve(*op->predicate, child_schema());
        if (op->predicate->type.id != TypeId::Bool) throw PlanError("filter predicate is not boolean");
        op->schema = child_schema();
        have = true;
        break;
    }
    case 104: { // HashAggregate operator.proto:647
        op->kind = OpKind::HashAgg;
        std::vector<int64_t> expr_modes;
        int64_t buffer_offset = 0; // initial_input_buffer_offset
        while (b.next()) {
            if (b.field == 1) op->grouping.push_back(decode_expr(b.sub()));
            else if (b.field == 2) op->aggs.push_back(decode_agg(b.sub()));
            else if (b.field == 5) op->mode = (AggMode)b.i64();
            else if (b.field == 6) {
                if (b.wire == 2) { PbReader pk = b.sub(); while (pk.p < pk.end) expr_modes.push_back((int64_t)pk.varint()); }
                else expr_modes.push_back(b.i64());
            } else if (b.field == 7) buffer_offset = (int32_t)b.i64();
            else b.skip();
        }
        if (op->mode != AggMode::Partial && op->mode != AggMode::Final && op->mode != AggMode::PartialMerge)
            throw PlanError("unknown aggregate mode " + std::to_string((int)op->mode));
        // Per-expression modes (the distinct rewrite, AggUtils.planAggregateWithOneDistinct): the JVM side sends them for an operator
        // whose aggregates are {Partial, PartialMerge} (operators.scala:1740-1822).  A PartialMerge aggregate there merges state
        // and emits state (MergeAsPartialUDF, merge_as_partial.rs:54-110); the output is state columns either way.
        if (!expr_modes.empty() && expr_modes.size() != op->aggs.size())
            throw PlanError("expr_modes has " + std::to_string(expr_modes.size()) + " entries for " + std::to_string(op->aggs.size()) + " aggregates");
        bool mixed = false;
        for (size_t i = 0; i < expr_modes.size(); i++) {
            const int64_t m = expr_modes[i];
            if (m != (int64_t)AggMode::Partial && m != (int64_t)AggMode::Final && m != (int64_t)AggMode::PartialMerge)
                throw PlanError("unknown aggregate mode " + std::to_string(m));
            if ((m == (int64_t)AggMode::Final) != (op->mode == AggMode::Final))
                throw Unsupported("Final mixed with Partial / PartialMerge aggregate expressions is outside the GPU hot path");
            op->aggs[i].mode = (AggMode)m;
            if (m != (int64_t)op->mode) mixed = true;
        }
        if (expr_modes.empty()) for (auto& a : op->aggs) a.mode = op->mode;
        const auto& cs = child_schema();
        for (auto& g : op->grouping) { resolve(*g, cs); op->schema.push_back(g->type); }
        for (auto& a : op->aggs) {
            resolve_agg(a, cs, a.mode); // Partial aggregates of a mixed operator may read any child column, state columns included
            if (a.mode != AggMode::Final) for (auto& t : agg_state_types(a)) op->schema.push_back(t);
            else op->schema.push_back(agg_result_type(a));
        }
        // State columns of the merging aggregates: consecutive, in agg_exprs order, from initial_input_buffer_offset; the running offset
        // advances over merging aggregates only (planner.rs:1265-1352).  A Final operator reads them right after its group columns, as
        // does a PartialMerge one that sends no offset.
        size_t at = mixed || (op->mode == AggMode::PartialMerge && buffer_offset != 0) ? (size_t)std::max<int64_t>(buffer_offset, 0) : op->grouping.size();
        if (buffer_offset < 0) throw PlanError("negative initial_input_buffer_offset");
        for (auto& a : op->aggs) {
            if (a.mode == AggMode::Partial) continue;
            a.state_at = (int)at;
            for (auto& t : agg_state_types(a)) {
                if (at >= cs.size()) throw PlanError("merging aggregate: state columns run past the child's " + std::to_string(cs.size()) + " columns");
                if (cs[at] != t) throw PlanError("merging aggregate: state column " + std::to_string(at) + " is " + cs[at].str() + ", expected " + t.str());
                at++;
            }
        }
        have = true;
        break;
    }
    case 106: { // ShuffleWriter operator.proto:688
        op->kind = OpKind::ShuffleWriter;
        std::vector<PbReader> bound_rows;
        while (b.next()) {
            if (b.field == 1) { // Partitioning
                PbReader pt = b.sub();
                while (pt.next()) {
                    if (pt.field == 1) { // HashPartition partitioning.proto:38
                        PbReader hp = pt.sub();
                        while (hp.next()) {
                            if (hp.field == 1) op->hash_exprs.push_back(decode_expr(hp.sub()));
                            else if (hp.field == 2) op->num_partitions = (int)hp.i64();
                            else hp.skip();
                        }
                    } else if (pt.field == 2) { pt.skip(); op->num_partitions = 1; }
                    else if (pt.field == 3) { // RangePartition partitioning.proto:49-53
                        op->part_kind = PartKind::Range;
                        PbReader rp = pt.sub();
                        while (rp.next()) {
                            if (rp.field == 1 && rp.wire == 2) op->range_keys.push_back(decode_sort_order(rp.sub()));
                            else if (rp.field == 2) op->num_partitions = (int32_t)rp.i64();
                            else if (rp.field == 4 && rp.wire == 2) bound_rows.push_back(rp.sub());
                            else rp.skip();
                        }
                    } else if (pt.field == 4) { // RoundRobinPartition partitioning.proto:55-59
                        op->part_kind = PartKind::RoundRobin;
                        PbReader rr = pt.sub();
                        while (rr.next()) {
                            if (rr.field == 1) op->num_partitions = (int32_t)rr.i64();
                            else if (rr.field == 2) op->max_hash_columns = (int32_t)rr.i64();
                            else rr.skip();
                        }
                    } else throw Unsupported("partitioning field " + std::to_string(pt.field) + " is outside the GPU hot path");
                }
            } else b.skip();
        }
        const auto& cs = child_schema();
        for (auto& e : op->hash_exprs) resolve(*e, cs);
        if (op->num_partitions <= 0) throw PlanError("shuffle writer without partitions");
        if (op->part_kind == PartKind::RoundRobin) { // planner.rs:3360-3370, multi_partition.rs:386-430: murmur3 over the first columns
            const size_t k = op->max_hash_columns <= 0 ? cs.size() : std::min(cs.size(), (size_t)op->max_hash_columns);
            for (size_t i = 0; i < k; i++) {
                auto e = mk(ExprKind::Bound);
                e->index = (int)i;
                e->type = cs[i];
                op->hash_exprs.push_back(e);
            }
        }
        if (op->part_kind == PartKind::Range) decode_range_partitioning(*op, cs, bound_rows);
        op->schema = cs;
        have = true;
        break;
    }
    case 103: { // Sort operator.proto:641-645 (planner.rs:1488-1522); TopK is the same message with fetch / skip (CometExecUtils.getTopKNativePlan)
        op->kind = OpKind::Sort;
        while (b.next()) {
            if (b.field == 1 && b.wire == 2) {
                op->sort_keys.push_back(decode_sort_order(b.sub()));
            } else if (b.field == 3 || b.field == 4) {
                const int32_t v = (int32_t)b.i64(); // optional int32
                if (v < 0) throw PlanError(std::string("sort ") + (b.field == 3 ? "fetch" : "skip") + " is negative");
                (b.field == 3 ? op->fetch : op->skip) = v;
            } else b.skip();
        }
        const auto& cs = child_schema();
        if (op->sort_keys.empty()) throw PlanError("sort without keys");
        if (op->sort_keys.size() > MAX_SORT_KEYS) throw Unsupported("more than 8 sort keys");
        int bits = 0;
        for (auto& k : op->sort_keys) {
            resolve(*k.expr, cs);
            if (k.expr->kind != ExprKind::Bound) throw Unsupported("computed sort keys (only plain column keys)");
            bits += sort_key_bits(k.expr->type) + 1; // every key may hold NULLs: one null bit each
        }
        if (bits > MAX_SORT_KEY_BITS) throw Unsupported("sort keys of " + std::to_string(bits) + " bits (at most 256 bits of packed key)");
        op->schema = cs;
        have = true;
        break;
    }
    case 108: { // SortMergeJoin operator.proto:765-771 (planner.rs:2126-2190: SortMergeJoinExec with NullEqualsNothing)
        // Run by the hash join's node: the side whose order the output keeps is probed, so RightOuter builds the left side and every
        // other type the right one.  The sort options must match the keys in number; the operator needs no sorted input, so their
        // directions do not change the result.
        op->kind = OpKind::HashJoin;
        int64_t join_type = 0;
        size_t n_sort_options = 0;
        while (b.next()) {
            if (b.field == 1 && b.wire == 2) op->left_keys.push_back(decode_expr(b.sub()));
            else if (b.field == 2 && b.wire == 2) op->right_keys.push_back(decode_expr(b.sub()));
            else if (b.field == 3) join_type = b.i64();
            else if (b.field == 4 && b.wire == 2) { decode_sort_order(b.sub()); n_sort_options++; }
            else if (b.field == 5 && b.wire == 2) op->join_condition = decode_join_condition(b.sub());
            else b.skip();
        }
        decode_join(*op, "sort-merge join", join_type);
        if (n_sort_options != op->left_keys.size())
            throw PlanError("sort-merge join with " + std::to_string(n_sort_options) + " sort options for " + std::to_string(op->left_keys.size()) + " keys");
        op->build_left = op->join_type == JoinType::RightOuter;
        resolve_join_keys(*op, "sort-merge join");
        resolve_join_condition(*op);
        have = true;
        break;
    }
    case 109: { // HashJoin operator.proto:754-763 (planner.rs:2192-2266: HashJoinExec with NullEqualsNothing; BuildRight swaps the inputs)
        op->kind = OpKind::HashJoin;
        bool null_aware = false;
        int64_t join_type = 0, build_side = 0;
        while (b.next()) {
            if (b.field == 1 && b.wire == 2) op->left_keys.push_back(decode_expr(b.sub()));
            else if (b.field == 2 && b.wire == 2) op->right_keys.push_back(decode_expr(b.sub()));
            else if (b.field == 3) join_type = b.i64();
            else if (b.field == 4 && b.wire == 2) op->join_condition = decode_join_condition(b.sub());
            else if (b.field == 5) build_side = b.i64();
            else if (b.field == 6) null_aware = b.i64() != 0;
            else b.skip();
        }
        decode_join(*op, "hash join", join_type);
        if (build_side != 0 && build_side != 1) throw PlanError("unknown build side " + std::to_string(build_side));
        op->build_left = build_side == 0;
        const bool semi_anti = op->join_type == JoinType::LeftSemi || op->join_type == JoinType::LeftAnti;
        if (op->join_type != JoinType::Inner && !semi_anti) throw Unsupported("outer hash joins (only inner, left semi and left anti)");
        if (semi_anti && op->build_left) throw Unsupported("left semi / anti hash join with BuildLeft (only BuildRight)");
        if (null_aware) throw Unsupported("null-aware anti join (NOT IN)");
        resolve_join_keys(*op, "hash join");
        resolve_join_condition(*op);
        have = true;
        break;
    }
    case 117: { // BroadcastNestedLoopJoin operator.proto:773-777 (planner.rs:1386-1436: NestedLoopJoinExec, BuildRight swaps the inputs)
        // Run by the hash join's node without keys: every pair is a candidate, the streamed side is probed.  Comet's serde sends the
        // shapes whose output follows the streamed side (operators.scala:2258-2266); the others would need the build side's rows merged
        // across partitions.
        op->kind = OpKind::HashJoin;
        int64_t join_type = 0, build_side = 0;
        while (b.next()) {
            if (b.field == 1) join_type = b.i64();
            else if (b.field == 2) build_side = b.i64();
            else if (b.field == 3 && b.wire == 2) op->join_condition = decode_join_condition(b.sub());
            else b.skip();
        }
        if (op->children.size() != 2) throw PlanError("nested-loop join expects two children");
        if (join_type < 0 || join_type > 5) throw PlanError("unknown join type " + std::to_string(join_type));
        if (build_side != 0 && build_side != 1) throw PlanError("unknown build side " + std::to_string(build_side));
        op->join_type = (JoinType)join_type;
        op->build_left = build_side == 0;
        const JoinType jt = op->join_type;
        const bool accepted = jt == JoinType::Inner || (jt == JoinType::LeftOuter && !op->build_left) || (jt == JoinType::RightOuter && op->build_left) ||
                              ((jt == JoinType::LeftSemi || jt == JoinType::LeftAnti) && !op->build_left);
        if (!accepted) {
            static const char* names[] = {"inner", "left outer", "right outer", "full outer", "left semi", "left anti"};
            throw Unsupported(std::string(names[join_type]) + " nested-loop join with " + (op->build_left ? "BuildLeft" : "BuildRight") +
                              " (only inner, left outer / semi / anti with BuildRight and right outer with BuildLeft: the output follows the streamed side)");
        }
        const auto &ls = op->children[0]->schema, &rs = op->children[1]->schema;
        if (ls.empty() || rs.empty()) throw Unsupported("a nested-loop join side without columns");
        op->schema = ls;
        if (jt != JoinType::LeftSemi && jt != JoinType::LeftAnti) op->schema.insert(op->schema.end(), rs.begin(), rs.end());
        resolve_join_condition(*op);
        have = true;
        break;
    }
    default:
        throw Unsupported("operator field " + std::to_string(f) + " is outside the GPU hot path");
    }
    if (!have) throw PlanError("operator not decoded");
    return op;
}

int sort_key_bits(const DType& t) {
    switch (t.id) {
    case TypeId::Bool: return 1;
    case TypeId::Int8: return 8;
    case TypeId::Int16: return 16;
    case TypeId::Int32: case TypeId::Date: case TypeId::Float32: return 32;
    case TypeId::Int64: case TypeId::Timestamp: case TypeId::TimestampNtz: case TypeId::Float64: return 64;
    case TypeId::Decimal: return t.precision <= 18 ? 64 : 128;
    case TypeId::String: return 32; // the rank of a dictionary code
    default: throw Unsupported("sort key of type " + t.str());
    }
}

OperatorP decode_plan(const uint8_t* data, size_t len) {
    try {
        return decode_operator(PbReader(data, len));
    } catch (const PbError& e) {
        throw PlanError(e.what());
    }
}

std::string expr_str(const Expr& e) {
    std::ostringstream o;
    static const char* names[] = {"lit", "col", "unbound", "+", "-", "*", "/", "=", "!=", ">", ">=", "<", "<=", "isnull",
                                  "isnotnull", "and", "or", "not", "cast", "checkoverflow", "neg", "if", "in", "strpred"};
    o << names[(int)e.kind];
    if (e.kind == ExprKind::Bound) o << e.index;
    o << ":" << e.type.str();
    if (!e.children.empty()) {
        o << "(";
        for (size_t i = 0; i < e.children.size(); i++) o << (i ? "," : "") << expr_str(*e.children[i]);
        o << ")";
    }
    return o.str();
}

} // namespace cb200
