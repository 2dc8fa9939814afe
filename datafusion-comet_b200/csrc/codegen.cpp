// codegen.cpp -- expression tree -> straight-line CUDA, spliced into device/cb_kernels.cuh.
//
// Every emitted operation names the reference rule it implements; the arithmetic itself is the
// hand-written device library device/cb_math.h (host-tested against the oracle).
#include "codegen.h"
#include <mutex>
#include "device/cb_params.h"
#include "ranges.h"

#include <algorithm>
#include <climits>
#include <cstring>
#include <functional>
#include <memory>
#include <set>
#include <sstream>

namespace cb200 {

int phys_bytes(Phys p) {
    switch (p) {
    case Phys::Bitmap: return 0;
    case Phys::I8: return 1;
    case Phys::I16: return 2;
    case Phys::I32: case Phys::F32: case Phys::Dict32: return 4;
    case Phys::I64: case Phys::F64: return 8;
    case Phys::I128: return 16;
    }
    return 0;
}

size_t GeneratedKernel::dyn_smem(int n_groups) const {
    size_t s = (entry == "cb_pipeline_agg" ? 128 : 256) + (size_t)stages * stage_bytes; // barrier area: CB_BAR_BYTES of the select kernels
    if (hash) return s;
    // grouped dense pipelines keep thread-private accumulators in shared memory even when the key has ONE value (a dictionary of
    // cardinality 1); only ungrouped pipelines (CB_G1) hold them in registers
    if (!word_kinds.empty() && !ungrouped) s += (size_t)std::max(n_groups, 1) * n_words * threads * 8;
    return s;
}

namespace {

struct Val {
    std::string v;   // C expression / variable holding the value
    std::string n;   // C expression for "is null" ("" = never null)
    DType type;
    bool narrow = false; // decimal held in a cb::i64 (its proven bound is < 2^63)
    bool nullable() const { return !n.empty(); }
};
const u128r R63 = (u128r)1 << 63;

std::string ctype(const DType& t) {
    switch (t.id) {
    case TypeId::Bool: return "bool";
    case TypeId::Int8: case TypeId::Int16: case TypeId::Int32: case TypeId::Date: return "cb::i32";
    case TypeId::Int64: case TypeId::Timestamp: case TypeId::TimestampNtz: return "cb::i64";
    case TypeId::Float32: return "float";
    case TypeId::Float64: return "double";
    case TypeId::Decimal: return "cb::i128";
    default: throw Unsupported("no device representation for " + t.str());
    }
}

std::string u64lit(uint64_t v) {
    std::ostringstream o;
    o << v << "ull";
    return o.str();
}
std::string i128lit(unsigned __int128 v) {
    std::ostringstream o;
    o << "cb::mk128(" << u64lit((uint64_t)v) << ", (cb::i64)" << u64lit((uint64_t)(v >> 64)) << ")";
    return o.str();
}
unsigned __int128 pow10_128(int e) {
    unsigned __int128 r = 1;
    for (int i = 0; i < e; i++) r *= 10;
    return r;
}
std::string bound_args(int precision) { // (lo, hi) of 10^p
    unsigned __int128 b = pow10_128(precision);
    return u64lit((uint64_t)b) + ", " + u64lit((uint64_t)(b >> 64));
}
std::string f64lit(double d) {
    uint64_t bits;
    memcpy(&bits, &d, 8);
    return "__longlong_as_double((cb::i64)" + u64lit(bits) + ")";
}
std::string f32lit(float f) {
    uint32_t bits;
    memcpy(&bits, &f, 4);
    std::ostringstream o;
    o << "__uint_as_float(" << bits << "u)";
    return o.str();
}

struct Emitter {
    const PipelineSpec& spec;
    std::ostringstream body;
    std::map<std::string, Val> cse;
    int next_id = 0;
    bool uses_err = false;
    std::vector<u128r> col_bounds; // assumed (kernel-validated) magnitude bound per staged column
    std::vector<bool> col_masked;  // columns whose value mask is accumulated (decimal inputs of aggregate pipelines)

    std::map<std::string, int> str_slot; // StrPred key -> PipeParams::smask index

    explicit Emitter(const PipelineSpec& s) : spec(s) {
        const std::vector<ExprP> sp = str_preds_of(s);
        for (size_t i = 0; i < sp.size(); i++) str_slot[std::to_string(sp[i]->children[0]->index) + "@" + str_pred_key(*sp[i])] = (int)i;
        for (auto& c : s.cols) {
            u128r b = RSAT;
            if (c.type.is_decimal()) {
                if (c.assume_bits > 0 && c.assume_bits < 127) b = (u128r)1 << c.assume_bits; // (v ^ sign) < 2^k  =>  |v| <= 2^k
                if (c.phys == Phys::I64 || c.phys == Phys::I32) b = std::min(b, R63); // narrow storage: |v| <= 2^63 (INT64_MIN)
            }
            col_bounds.push_back(b);
            col_masked.push_back(s.sink == SinkKind::Agg && c.type.is_decimal());
        }
    }
    u128r bound_of(const Expr& e) const { return expr_maxabs(e, col_bounds); }
    static std::string W(const Val& v) { return v.narrow ? "cb::i128_from_i64(" + v.v + ")" : v.v; } // as cb::i128
    std::string declw(const std::string& init) { std::string n = fresh(); body << "    cb::i128 " << n << " = " << init << ";\n"; return n; }
    std::string decln(const std::string& init) { std::string n = fresh(); body << "    cb::i64 " << n << " = " << init << ";\n"; return n; }

    std::string fresh(const char* prefix = "v") { return std::string(prefix) + std::to_string(next_id++); }

    static std::string or_null(const std::string& a, const std::string& b) {
        if (a.empty()) return b;
        if (b.empty()) return a;
        return "(" + a + " || " + b + ")";
    }
    std::string key_of(const Expr& e) {
        std::ostringstream o;
        o << (int)e.kind << "|" << e.type.str() << "|" << e.index << "|" << e.lit_null << "|" << e.lit_i64 << "|";
        uint64_t fb;
        memcpy(&fb, &e.lit_f64, 8);
        o << fb << "|" << (uint64_t)e.lit_dec << "," << (uint64_t)(e.lit_dec >> 64) << "|" << (int)e.eval_mode << "|"
          << e.fail_on_error << "|" << e.negated << "|" << e.wide_decimal << "|" << e.integral_div << e.check_divide_overflow << "|" << e.return_type.str() << "(";
        if (e.kind == ExprKind::StrPred) o << str_pred_key(e) << "|" << e.in_has_null << "|";
        for (auto& c : e.children) o << key_of(*c) << ",";
        o << ")";
        return o.str();
    }

    // declare `type name = init;` and return name
    std::string decl(const DType& t, const std::string& init) {
        std::string name = fresh();
        body << "    " << ctype(t) << " " << name << " = " << init << ";\n";
        return name;
    }
    std::string declb(const std::string& init) {
        std::string name = fresh("b");
        body << "    bool " << name << " = " << init << ";\n";
        return name;
    }

    // Branch guard: inside IF / CASE branches the reference evaluates the branch only on the rows that take it
    // (CaseExpr evaluates `then` under the selection), so ANSI / arrow overflow errors of rows that do not take
    // the branch must not fire.  Values are still computed (and ignored) for every row.
    std::string guard;
    std::string base_guard; // hash pipelines evaluate every row slot (no early return for filtered rows): errors only from kept rows
    Val emit(const Expr& e) {
        std::string k = guard.empty() ? key_of(e) : guard + "|" + key_of(e);
        auto it = cse.find(k);
        if (it != cse.end()) return it->second;
        Val r = emit_uncached(e);
        cse[k] = r;
        return r;
    }

    Val load_col(int slot) {
        const SourceCol& c = spec.cols.at(slot);
        Val r;
        r.type = c.type;
        std::string s = std::to_string(slot);
        if (c.has_validity) r.n = declb("!cb::ldv(t.val[" + s + "], r)");
        std::string notnull = r.n.empty() ? "" : "if (!" + r.n + ") ";
        if (!base_guard.empty()) notnull = r.n.empty() ? "if (in_range) " : "if (in_range && !" + r.n + ") ";
        if (c.type.is_decimal()) {
            bool narrow = col_bounds[slot] < R63;
            if (c.phys == Phys::I128) {
                std::string raw = declw("cb::ld<cb::i128>(t.col[" + s + "], r)");
                if (col_masked[slot]) body << "    " << notnull << "acc.vm_or(" << s << ", " << raw << ");\n";
                if (narrow) { r.v = decln("(cb::i64)" + raw + ".lo"); r.narrow = true; }
                else r.v = raw;
            } else { // decimal stored as int64 / int32 (Parquet physical types)
                std::string raw = decln(c.phys == Phys::I64 ? "cb::ld<cb::i64>(t.col[" + s + "], r)" : "(cb::i64)cb::ld<cb::i32>(t.col[" + s + "], r)");
                if (col_masked[slot]) body << "    " << notnull << "acc.vm_or64(" << s << ", " << raw << ");\n";
                r.v = raw;
                r.narrow = true;
            }
            return r;
        }
        std::string init;
        switch (c.phys) {
        case Phys::Bitmap: init = "cb::ldv(t.col[" + s + "], r)"; break;
        case Phys::I8: init = "(cb::i32)cb::ld<signed char>(t.col[" + s + "], r)"; break;
        case Phys::I16: init = "(cb::i32)cb::ld<short>(t.col[" + s + "], r)"; break;
        case Phys::I32: case Phys::Dict32: init = "cb::ld<cb::i32>(t.col[" + s + "], r)"; break;
        case Phys::I64: init = "cb::ld<cb::i64>(t.col[" + s + "], r)"; break;
        case Phys::F32: init = "cb::ld<float>(t.col[" + s + "], r)"; break;
        case Phys::F64: init = "cb::ld<double>(t.col[" + s + "], r)"; break;
        case Phys::I128: init = "cb::ld<cb::i128>(t.col[" + s + "], r)"; break;
        }
        if (c.phys == Phys::Dict32 || c.type.is_string()) { // dictionary codes of a string column
            r.v = fresh("k");
            body << "    cb::i32 " << r.v << " = " << init << ";\n";
        } else {
            r.v = decl(c.type, init);
        }
        return r;
    }

    Val emit_uncached(const Expr& e) {
        switch (e.kind) {
        case ExprKind::Bound: return load_col(e.index);
        case ExprKind::Unbound: throw PlanError("unbound reference reached code generation");
        case ExprKind::Literal: return emit_literal(e);
        case ExprKind::Add: case ExprKind::Sub: case ExprKind::Mul: case ExprKind::Div: return emit_arith(e);
        case ExprKind::Eq: case ExprKind::Neq: case ExprKind::Gt: case ExprKind::GtEq: case ExprKind::Lt: case ExprKind::LtEq:
            return emit_cmp(e);
        case ExprKind::And: case ExprKind::Or: return emit_logic(e);
        case ExprKind::Not: {
            Val c = emit(*e.children[0]);
            Val r;
            r.type = e.type;
            r.v = declb("!" + c.v);
            r.n = c.n;
            return r;
        }
        case ExprKind::IsNull: case ExprKind::IsNotNull: {
            Val c = emit(*e.children[0]);
            Val r;
            r.type = e.type;
            std::string isnull = c.n.empty() ? "false" : c.n;
            r.v = declb(e.kind == ExprKind::IsNull ? isnull : "!(" + isnull + ")");
            return r;
        }
        case ExprKind::Cast: return emit_cast(e);
        case ExprKind::CheckOverflow: return emit_check_overflow(e);
        case ExprKind::UnaryMinus: return emit_neg(e);
        case ExprKind::If: {
            Val c = emit(*e.children[0]);
            std::string ct = c.n.empty() ? c.v : declb("!" + c.n + " && " + c.v); // NULL condition -> else branch
            const std::string outer = guard;
            guard = outer.empty() ? ct : declb(outer + " && " + ct);
            Val a = emit(*e.children[1]);
            guard = outer.empty() ? "!(" + ct + ")" : declb(outer + " && !(" + ct + ")");
            Val b = emit(*e.children[2]);
            guard = outer;
            Val r;
            r.type = e.type;
            if (e.type.is_decimal()) {
                if (a.narrow && b.narrow) { r.v = decln(ct + " ? " + a.v + " : " + b.v); r.narrow = true; }
                else r.v = declw(ct + " ? " + W(a) + " : " + W(b));
            } else
            r.v = decl(e.type, ct + " ? " + a.v + " : " + b.v);
            if (a.nullable() || b.nullable())
                r.n = declb(ct + " ? " + (a.n.empty() ? "false" : a.n) + " : " + (b.n.empty() ? "false" : b.n));
            return r;
        }
        case ExprKind::In: return emit_in(e);
        case ExprKind::StrPred: return emit_str_pred(e);
        }
        throw PlanError("unhandled expression kind");
    }

    Val emit_literal(const Expr& e) {
        Val r;
        r.type = e.type;
        if (e.lit_null) {
            if (e.type.id == TypeId::Null) throw Unsupported("untyped NULL literal");
            if (e.type.is_decimal()) { r.v = "((cb::i64)0)"; r.narrow = true; }
            else r.v = decl(e.type, "0");
            r.n = "true";
            return r;
        }
        switch (e.type.id) {
        case TypeId::Bool: r.v = e.lit_i64 ? "true" : "false"; break;
        case TypeId::Int8: case TypeId::Int16: case TypeId::Int32: case TypeId::Date:
            r.v = "((cb::i32)" + std::to_string((int32_t)e.lit_i64) + ")";
            if ((int32_t)e.lit_i64 == INT32_MIN) r.v = "((cb::i32)0x80000000u)";
            break;
        case TypeId::Int64: case TypeId::Timestamp: case TypeId::TimestampNtz:
            r.v = "((cb::i64)" + u64lit((uint64_t)e.lit_i64) + ")";
            break;
        case TypeId::Float32: r.v = f32lit((float)e.lit_f64); break;
        case TypeId::Float64: r.v = f64lit(e.lit_f64); break;
        case TypeId::Decimal:
            if (bound_of(e) < R63) { r.v = "((cb::i64)" + u64lit((uint64_t)e.lit_dec) + ")"; r.narrow = true; }
            else r.v = declw(i128lit(e.lit_dec));
            break;
        default: throw Unsupported("literal of type " + e.type.str());
        }
        return r;
    }

    void raise(const std::string& cond, int bit) {
        uses_err = true;
        body << "    if (" << (base_guard.empty() ? "" : base_guard + " && ") << (guard.empty() ? "" : guard + " && ") << cond << ") cb::set_err(p, " << bit << ");\n";
    }

    // ---- arithmetic --------------------------------------------------------------------------------
    Val emit_arith(const Expr& e) {
        Val l = emit(*e.children[0]), rr = emit(*e.children[1]);
        Val r;
        r.type = e.type;
        std::string nn = or_null(l.n, rr.n);
        std::string valid = nn.empty() ? "true" : "!" + nn;
        const DType &lt = l.type, &rt = rr.type;
        if (lt.is_decimal() && e.kind == ExprKind::Div) {
            // decimal_div / decimal_integral_div (spark-expr/src/math_funcs/div.rs:75-190): only rows where both sides are valid are
            // evaluated (try_binary); a zero divisor is an error in ANSI mode and yields 0 otherwise (unreachable: the JVM serde wraps
            // the divisor in nullIf(= 0) outside ANSI mode)
            const int s1 = lt.scale, s2 = rt.scale, s3 = e.type.scale;
            const int l_exp = std::max(0, s2 + s3 + 1 - s1), r_exp = std::max(0, s1 - (s2 + s3 + 1));
            std::string ok = fresh("b"), fits = fresh("b");
            r.v = fresh();
            body << "    cb::i128 " << r.v << " = cb::mk128(0, 0); bool " << ok << " = true, " << fits << " = true;\n";
            body << "    if (" << valid << ") " << ok << " = cb::dec_div(" << W(l) << ", " << W(rr) << ", " << l_exp << ", " << r_exp << ", "
                 << (e.integral_div ? "true" : "false") << ", " << r.v << ", " << fits << ");\n";
            if (e.eval_mode == EvalMode::Ansi) {
                raise(valid + " && !" + ok, 3);
                if (e.integral_div && e.check_divide_overflow) raise(valid + " && " + ok + " && !" + fits, 1);
            }
            r.n = nn;
            return r;
        }
        if (lt.is_decimal()) {
            int op = e.kind == ExprKind::Add ? 0 : e.kind == ExprKind::Sub ? 1 : 2;
            const u128r raw = r_binary_raw(e, bound_of(*e.children[0]), bound_of(*e.children[1]));
            const int natural = op == 2 ? lt.scale + rt.scale : std::max(lt.scale, rt.scale);
            // Range proof: when the exact result provably stays inside i128 (plain) / the output precision
            // (wide, no rescale) the checks of the reference can never fire and are not emitted.
            bool unchecked = e.wide_decimal ? (natural == e.type.scale && raw <= r_prec_max(e.type.precision)) : raw < RSAT;
            if (unchecked) {
                Val u = emit_unchecked(op, l, rr, lt, rt, raw);
                if (!u.v.empty()) { u.type = e.type; u.n = nn; return u; }
            }
            if (e.wide_decimal) {
                // wide_decimal_binary_expr.rs:179-291
                std::string ok = fresh("b");
                r.v = fresh();
                body << "    cb::i128 " << r.v << " = cb::mk128(0, 0); bool " << ok << " = false;\n";
                body << "    if (" << valid << ") " << ok << " = ";
                if (op == 2)
                    body << "cb::wide_mul_fast(" << W(l) << ", " << W(rr) << ", " << (natural - e.type.scale) << ", " << e.type.precision << ", " << r.v
                         << ");\n";
                else
                    body << "cb::wide_addsub(" << W(l) << ", " << (natural - lt.scale) << ", " << W(rr) << ", " << (natural - rt.scale) << ", "
                         << (op == 1 ? "true" : "false") << ", " << (natural - e.type.scale) << ", " << e.type.precision << ", " << r.v << ");\n";
                if (e.eval_mode == EvalMode::Ansi) raise(valid + " && !" + ok, 1);
                r.n = declb("!" + ok); // overflow -> NULL (Legacy/Try); null inputs -> NULL
                return r;
            }
            // arrow-arith decimal_op (planner.rs:1126 fallthrough): checked i128, evaluated only on valid rows
            std::string err = fresh("e");
            r.v = fresh();
            body << "    cb::i128 " << r.v << " = cb::mk128(0, 0); bool " << err << " = false;\n";
            body << "    if (" << valid << ") " << r.v << " = ";
            if (op == 2) body << "cb::dec_mul_plain(" << W(l) << ", " << W(rr) << ", " << err << ");\n";
            else
                body << (op == 0 ? "cb::dec_add_plain(" : "cb::dec_sub_plain(") << W(l) << ", " << (natural - lt.scale) << ", " << W(rr) << ", "
                     << (natural - rt.scale) << ", " << err << ");\n";
            raise(err, 0); // arrow: "Overflow happened on ..." fails the query
            r.n = nn;
            return r;
        }
        if (lt.is_float()) {
            const char* opc = e.kind == ExprKind::Add ? "+" : e.kind == ExprKind::Sub ? "-" : e.kind == ExprKind::Mul ? "*" : "/";
            // IEEE arithmetic, no contraction: each node rounds once like the reference's per-node arrays
            std::string fn = lt.id == TypeId::Float64
                                 ? (e.kind == ExprKind::Add ? "__dadd_rn" : e.kind == ExprKind::Sub ? "__dsub_rn" : e.kind == ExprKind::Mul ? "__dmul_rn" : "__ddiv_rn")
                                 : (e.kind == ExprKind::Add ? "__fadd_rn" : e.kind == ExprKind::Sub ? "__fsub_rn" : e.kind == ExprKind::Mul ? "__fmul_rn" : "__fdiv_rn");
            (void)opc;
            // Float32: the hardware returns the canonical NaN 0x7FFFFFFF; f32_x86_nan restores the reference's (x86) NaN bits
            if (lt.id == TypeId::Float64) r.v = decl(e.type, fn + "(" + l.v + ", " + rr.v + ")");
            else r.v = decl(e.type, "cb::f32_x86_nan(" + l.v + ", " + rr.v + ", " + fn + "(" + l.v + ", " + rr.v + "))");
            r.n = nn;
            if (e.kind == ExprKind::Div && e.eval_mode != EvalMode::Legacy) {
                // checked_div (checked_arithmetic.rs:53-128; planner.rs:1094-1125 routes float Divide there under TRY / ANSI):
                // a zero divisor is NULL in TRY mode and DIVIDE_BY_ZERO in ANSI mode; everything else is IEEE
                std::string z = declb(rr.v + (lt.id == TypeId::Float64 ? " == 0.0" : " == 0.0f"));
                if (e.eval_mode == EvalMode::Ansi) raise(valid + " && " + z, 3);
                else r.n = or_null(nn, z);
            }
            return r;
        }
        // integers: Legacy wraps (arrow-arith *_wrapping); Try -> NULL, Ansi -> error (checked_arithmetic.rs:53-128)
        int bits = lt.id == TypeId::Int8 ? 8 : lt.id == TypeId::Int16 ? 16 : lt.id == TypeId::Int32 ? 32 : 64;
        if (e.kind == ExprKind::Div) {
            // Legacy: arrow-arith `div` (checked: zero divisor / MIN / -1 fail the query); TRY -> NULL, ANSI -> Spark errors
            // (checked_div, checked_arithmetic.rs:45,90-100)
            std::string err = fresh("e"), q = fresh();
            body << "    int " << err << " = 0; cb::i64 " << q << " = 0;\n";
            body << "    if (" << valid << ") " << q << " = cb::i64_div_checked((cb::i64)" << l.v << ", (cb::i64)" << rr.v << ", " << bits << ", " << err << ");\n";
            r.v = decl(e.type, "(" + ctype(e.type) + ")" + q);
            if (e.eval_mode == EvalMode::Try) r.n = or_null(nn, err + " != 0");
            else {
                raise(err + " == 1", e.eval_mode == EvalMode::Ansi ? 3 : 4);
                raise(err + " == 2", e.eval_mode == EvalMode::Ansi ? 1 : 0);
                r.n = nn;
            }
            return r;
        }
        std::string wide = fresh("w");
        const char* opc = e.kind == ExprKind::Add ? "+" : e.kind == ExprKind::Sub ? "-" : "*";
        if (bits < 64) {
            body << "    cb::i64 " << wide << " = (cb::i64)" << l.v << " " << opc << " (cb::i64)" << rr.v << ";\n";
            std::string wrapped = "(cb::i32)cb::wrap_int(" + wide + ", " + std::to_string(bits) + ")";
            r.v = decl(e.type, wrapped);
            if (e.eval_mode != EvalMode::Legacy) {
                const std::string lim = std::to_string((1LL << (bits - 1)) - 1);
                std::string ovf = declb("(" + wide + " < -" + lim + "ll - 1 || " + wide + " > " + lim + "ll)");
                if (e.eval_mode == EvalMode::Ansi) { raise(valid + " && " + ovf, 1); r.n = nn; }
                else r.n = or_null(nn, ovf);
            } else r.n = nn;
        } else {
            if (e.eval_mode == EvalMode::Legacy) {
                r.v = decl(e.type, "(cb::i64)((cb::u64)" + l.v + " " + opc + " (cb::u64)" + rr.v + ")");
                r.n = nn;
            } else {
                std::string ovf = fresh("b");
                r.v = fresh();
                body << "    cb::i64 " << r.v << "; bool " << ovf << " = cb::i64_" << (e.kind == ExprKind::Add ? "add" : e.kind == ExprKind::Sub ? "sub" : "mul")
                     << "_overflow(" << l.v << ", " << rr.v << ", " << r.v << ");\n";
                if (e.eval_mode == EvalMode::Ansi) { raise(valid + " && " + ovf, 1); r.n = nn; }
                else r.n = or_null(nn, ovf);
            }
        }
        return r;
    }

    // exact decimal op whose result magnitude is proven < 2^127 (`raw`): no overflow handling needed.
    // Returns an empty Val when no cheap form exists (caller falls back to the checked path).
    Val emit_unchecked(int op, const Val& l, const Val& rr, const DType& lt, const DType& rt, u128r raw) {
        Val r;
        if (op == 2) {
            if (l.narrow && rr.narrow) {
                if (raw < R63) { r.v = decln(l.v + " * " + rr.v); r.narrow = true; }
                else r.v = declw("cb::mul_i64_i64(" + l.v + ", " + rr.v + ")");
            } else if (l.narrow || rr.narrow) {
                const Val &w = l.narrow ? rr : l, &nv = l.narrow ? l : rr;
                r.v = declw("cb::mul_i128_i64(" + w.v + ", " + nv.v + ")");
            } else r.v = declw("cb::mul_i128_wrap(" + l.v + ", " + rr.v + ")");
            return r;
        }
        int ms = std::max(lt.scale, rt.scale), lup = ms - lt.scale, rup = ms - rt.scale;
        if (lup > 18 || rup > 18) return r; // scale factors beyond i64: keep the generic path
        std::string F1 = "((cb::i64)" + u64lit((uint64_t)pow10_128(lup)) + ")", F2 = "((cb::i64)" + u64lit((uint64_t)pow10_128(rup)) + ")";
        const char* o = op == 0 ? " + " : " - ";
        if (raw < R63 && l.narrow && rr.narrow) {
            std::string a = lup ? l.v + " * " + F1 : l.v, b = rup ? rr.v + " * " + F2 : rr.v;
            r.v = decln(a + o + b);
            r.narrow = true;
            return r;
        }
        std::string a = lup ? "cb::mul_i128_i64(" + W(l) + ", " + F1 + ")" : W(l), b = rup ? "cb::mul_i128_i64(" + W(rr) + ", " + F2 + ")" : W(rr);
        r.v = declw(std::string(op == 0 ? "cb::i128_add(" : "cb::i128_sub(") + a + ", " + b + ")");
        return r;
    }

    // ---- comparisons (arrow-ord cmp; floats by IEEE totalOrder) -------------------------------------
    Val emit_cmp(const Expr& e) {
        Val l = emit(*e.children[0]), rr = emit(*e.children[1]);
        Val r;
        r.type = e.type;
        r.n = or_null(l.n, rr.n);
        std::string a = l.v, b = rr.v;
        const DType& t = l.type;
        std::string expr;
        if (t.is_decimal() && l.narrow && rr.narrow) {
            const char* opc = e.kind == ExprKind::Eq ? "==" : e.kind == ExprKind::Neq ? "!=" : e.kind == ExprKind::Lt ? "<" : e.kind == ExprKind::LtEq ? "<=" : e.kind == ExprKind::Gt ? ">" : ">=";
            expr = "(" + a + " " + opc + " " + b + ")";
        } else if (t.is_decimal()) {
            a = W(l); b = W(rr);
            switch (e.kind) {
            case ExprKind::Eq: expr = "cb::i128_eq(" + a + ", " + b + ")"; break;
            case ExprKind::Neq: expr = "!cb::i128_eq(" + a + ", " + b + ")"; break;
            case ExprKind::Lt: expr = "cb::i128_lt(" + a + ", " + b + ")"; break;
            case ExprKind::LtEq: expr = "cb::i128_le(" + a + ", " + b + ")"; break;
            case ExprKind::Gt: expr = "cb::i128_lt(" + b + ", " + a + ")"; break;
            default: expr = "cb::i128_le(" + b + ", " + a + ")"; break;
            }
        } else {
            if (t.id == TypeId::Float64) {
                a = "cb::f64_total_key((cb::u64)__double_as_longlong(" + a + "))";
                b = "cb::f64_total_key((cb::u64)__double_as_longlong(" + b + "))";
            } else if (t.id == TypeId::Float32) {
                a = "cb::f32_total_key(__float_as_uint(" + a + "))";
                b = "cb::f32_total_key(__float_as_uint(" + b + "))";
            }
            const char* opc = e.kind == ExprKind::Eq ? "==" : e.kind == ExprKind::Neq ? "!=" : e.kind == ExprKind::Lt ? "<" : e.kind == ExprKind::LtEq ? "<=" : e.kind == ExprKind::Gt ? ">" : ">=";
            expr = "(" + a + " " + opc + " " + b + ")";
        }
        r.v = declb(expr);
        return r;
    }

    // ---- Kleene AND / OR (arrow and_kleene / or_kleene) ---------------------------------------------
    Val emit_logic(const Expr& e) {
        Val l = emit(*e.children[0]), rr = emit(*e.children[1]);
        Val r;
        r.type = e.type;
        bool is_and = e.kind == ExprKind::And;
        if (!l.nullable() && !rr.nullable()) {
            r.v = declb(l.v + (is_and ? " && " : " || ") + rr.v);
            return r;
        }
        std::string ln = l.n.empty() ? "false" : l.n, rn = rr.n.empty() ? "false" : rr.n;
        std::string lt = declb("!" + ln + " && " + l.v), lf = declb("!" + ln + " && !" + l.v);
        std::string rt = declb("!" + rn + " && " + rr.v), rf = declb("!" + rn + " && !" + rr.v);
        std::string T = declb(is_and ? lt + " && " + rt : lt + " || " + rt);
        std::string F = declb(is_and ? lf + " || " + rf : lf + " && " + rf);
        r.v = T;
        r.n = declb("!" + T + " && !" + F);
        return r;
    }

    Val emit_cast(const Expr& e) {
        Val c = emit(*e.children[0]);
        const DType &from = c.type, &to = e.type;
        Val r;
        r.type = to;
        r.n = c.n;
        if (from == to) { r.v = c.v; r.narrow = c.narrow; return r; }
        if ((from.is_integer() || from.is_float()) && (to.is_integer() || to.is_float())) {
            r.v = decl(to, "(" + ctype(to) + ")" + c.v);
            return r;
        }
        std::string valid = c.n.empty() ? "true" : "!" + c.n;
        if (from.is_integer() && to.is_decimal()) {
            // Spark Cast(int -> decimal(p,s)): value * 10^s, out of precision -> NULL (Legacy/Try) / error (ANSI)
            std::string ok = fresh("b");
            r.v = fresh();
            body << "    cb::i128 " << r.v << " = cb::mk128(0, 0); bool " << ok << " = cb::dec_rescale_check(cb::i128_from_i64((cb::i64)" << c.v
                 << "), " << to.scale << ", " << to.precision << ", " << r.v << ");\n";
            if (e.eval_mode == EvalMode::Ansi) raise(valid + " && !" + ok, 1);
            r.n = or_null(c.n, "!" + ok);
            return r;
        }
        if (from.is_decimal() && to.is_decimal()) {
            std::string ok = fresh("b");
            r.v = fresh();
            body << "    cb::i128 " << r.v << " = cb::mk128(0, 0); bool " << ok << " = cb::dec_rescale_check(" << W(c) << ", "
                 << (to.scale - from.scale) << ", " << to.precision << ", " << r.v << ");\n";
            if (e.eval_mode == EvalMode::Ansi) raise(valid + " && !" + ok, 1);
            r.n = or_null(c.n, "!" + ok);
            return r;
        }
        throw Unsupported("cast " + from.str() + " -> " + to.str());
    }

    Val emit_check_overflow(const Expr& e) {
        const Expr& ch = *e.children[0];
        // planner.rs:606-613: WideDecimalBinaryExpr already checked -> skip when the types agree
        if ((ch.kind == ExprKind::Add || ch.kind == ExprKind::Sub || ch.kind == ExprKind::Mul) && ch.wide_decimal && ch.type == e.type)
            return emit(ch);
        // planner.rs:617-637: Cast(decimal->decimal) + CheckOverflow fuse into DecimalRescaleCheckOverflow
        if (ch.kind == ExprKind::Cast && ch.children[0]->type.is_decimal() && ch.type == e.type) {
            Val c = emit(*ch.children[0]);
            std::string valid = c.n.empty() ? "true" : "!" + c.n;
            Val r;
            r.type = e.type;
            std::string ok = fresh("b");
            r.v = fresh();
            body << "    cb::i128 " << r.v << " = cb::mk128(0, 0); bool " << ok << " = cb::dec_rescale_check(" << W(c) << ", "
                 << (e.type.scale - ch.children[0]->type.scale) << ", " << e.type.precision << ", " << r.v << ");\n";
            if (e.fail_on_error) raise(valid + " && !" + ok, 1);
            r.n = or_null(c.n, "!" + ok);
            return r;
        }
        // checkoverflow.rs:105-200: bound check only
        Val c = emit(ch);
        Val r = c;
        r.type = e.type;
        if (bound_of(ch) <= r_prec_max(e.type.precision)) return r; // range proof: the check can never fire
        std::string valid = c.n.empty() ? "true" : "!" + c.n;
        std::string ok = declb("cb::dec_fits(" + W(c) + ", " + bound_args(e.type.precision) + ")");
        if (e.fail_on_error) { raise(valid + " && !" + ok, 1); r.n = c.n; }
        else r.n = or_null(c.n, "!" + ok);
        return r;
    }

    Val emit_neg(const Expr& e) {
        Val c = emit(*e.children[0]);
        Val r;
        r.type = e.type;
        r.n = c.n;
        const DType& t = c.type;
        if (t.is_decimal()) {
            if (c.narrow && bound_of(*e.children[0]) < R63) { r.v = decln("-" + c.v); r.narrow = true; } // |v| < 2^63: cannot overflow
            else r.v = declw("cb::i128_neg(" + W(c) + ")"); // an i64 holding INT64_MIN negates to 2^63
        }
        else if (t.is_float()) r.v = decl(t, (t.id == TypeId::Float64 ? "cb::f64_neg(" : "cb::f32_neg(") + c.v + ")"); // exact sign flip, see cb_math.h
        else if (t.id == TypeId::Int64) r.v = decl(t, "(cb::i64)(0ull - (cb::u64)" + c.v + ")");
        else {
            int bits = t.id == TypeId::Int8 ? 8 : t.id == TypeId::Int16 ? 16 : 32;
            r.v = decl(t, "(cb::i32)cb::wrap_int(-(cb::i64)" + c.v + ", " + std::to_string(bits) + ")");
        }
        if (e.fail_on_error && t.is_integer()) { // negative.rs: ANSI overflow on MIN
            std::string valid = c.n.empty() ? "true" : "!" + c.n;
            raise(valid + " && " + c.v + " != 0 && " + r.v + " == " + c.v, 1);
        }
        return r;
    }

    // String predicate: one bit per dictionary code, computed on the host side of the launch (k_str_pred); here only the lookup by the
    // code the kernel already staged.  The literal never enters the source, so plans that differ only in literals share one kernel.
    // A NULL row is NULL and its code (which Arrow leaves unspecified) is never used; a valid code outside the mask raises error bit 5.
    Val emit_str_pred(const Expr& e) {
        Val c = emit(*e.children[0]);
        auto it = str_slot.find(std::to_string(e.children[0]->index) + "@" + str_pred_key(e));
        if (it == str_slot.end()) throw PlanError("internal: string predicate without a mask slot");
        const std::string m = "p.smask[" + std::to_string(it->second) + "]";
        const std::string valid = c.n.empty() ? "true" : "!" + c.n;
        std::string ok = declb(valid + " && (cb::u32)" + c.v + " < (cb::u32)" + m + ".n_entries");
        uses_err = true;
        body << "    if (" << (base_guard.empty() ? "" : base_guard + " && ") << valid << " && !" << ok << ") cb::set_err(p, 5);\n";
        std::string hit = declb(ok + " && ((" + m + ".bits[(cb::u32)" + c.v + " >> 5] >> ((cb::u32)" + c.v + " & 31u)) & 1u) != 0u");
        Val r;
        r.type = e.type;
        if (e.str_op == StrOp::In) { // Spark In: NULL value -> NULL; match -> TRUE; else NULL if the list has a NULL, else FALSE
            r.v = e.negated ? declb("!" + hit) : hit;
            r.n = e.in_has_null ? or_null(c.n, "!" + hit) : c.n;
        } else {
            r.v = hit;
            r.n = c.n;
        }
        return r;
    }

    Val emit_in(const Expr& e) { // Spark In: NULL value -> NULL; match -> TRUE; else NULL if list has NULL, else FALSE
        Val v = emit(*e.children[0]);
        bool list_has_null = false;
        std::string any = "false";
        for (size_t i = 1; i < e.children.size(); i++) {
            const Expr& m = *e.children[i];
            if (m.lit_null) { list_has_null = true; continue; }
            Val mv = emit(m);
            if (v.type.is_decimal()) any += (v.narrow && mv.narrow) ? " || (" + v.v + " == " + mv.v + ")" : " || cb::i128_eq(" + W(v) + ", " + W(mv) + ")";
            else if (v.type.id == TypeId::Float64) any += " || (__double_as_longlong(" + v.v + ") == __double_as_longlong(" + mv.v + "))";
            else if (v.type.id == TypeId::Float32) any += " || (__float_as_uint(" + v.v + ") == __float_as_uint(" + mv.v + "))";
            else any += " || (" + v.v + " == " + mv.v + ")";
        }
        Val r;
        r.type = e.type;
        std::string hit = declb(any);
        r.v = e.negated ? declb("!" + hit) : hit;
        if (list_has_null) r.n = or_null(v.n, "!" + hit);
        else r.n = v.n;
        return r;
    }
};

// ---- aggregate slot planning ----------------------------------------------------------------------
struct SlotPlan {
    std::vector<int> kinds;                 // per word
    std::map<std::string, int> dedup;       // (kind|expr|cond) -> first word
    int add(int kind, const std::string& key, int n_words = 1) {
        std::string k = std::to_string(kind) + "|" + key;
        auto it = dedup.find(k);
        if (it != dedup.end()) return it->second;
        int w = (int)kinds.size();
        kinds.push_back(kind);
        if (n_words == 2) kinds.push_back(W_DD_LO);
        dedup[k] = w;
        return w;
    }
};

struct AggLayout { // where each aggregate finds its totals at finalize time
    int w_sum = -1, w_cnt = -1, w_bits = -1, w_bad = -1, w_minmax = -1, w_abs = -1;
    bool is_f64_sum = false;
};

std::string header(const PipelineSpec& s, const std::string& defs) {
    std::ostringstream o;
    o << "// generated by comet_b200 codegen -- do not edit\n";
    o << defs;
    if (const char* x = getenv("CB200_JIT_DEFS")) { // tuning experiments: "CB_X_FOO=1;CB_X_BAR=2" -> #define lines (part of the source, hence of the cache key)
        std::string d = x;
        size_t i = 0;
        while (i < d.size()) {
            size_t j = d.find(';', i);
            if (j == std::string::npos) j = d.size();
            std::string one = d.substr(i, j - i);
            size_t eq = one.find('=');
            if (!one.empty()) o << "#define " << (eq == std::string::npos ? one : one.substr(0, eq) + " " + one.substr(eq + 1)) << "\n";
            i = j + 1;
        }
    }
    o << "#define CB_NCOLS " << s.cols.size() << "\n#define CB_TILE " << s.tile << "\n#define CB_STAGES " << s.stages
      << "\n#define CB_THREADS " << s.threads << "\n";
    o << "#include \"cb_math.h\"\n";
    o << "constexpr __host__ __device__ int cb_col_bytes(int c) { return ";
    for (size_t i = 0; i < s.cols.size(); i++) o << "c == " << i << " ? " << phys_bytes(s.cols[i].phys) << " : ";
    o << "0; }\n";
    o << "constexpr __host__ __device__ bool cb_col_masked(int c) { return ";
    for (size_t i = 0; i < s.cols.size(); i++) o << "c == " << i << " ? " << (s.sink == SinkKind::Agg && s.cols[i].type.is_decimal() ? "true" : "false") << " : ";
    o << "false; }\n";
    o << "constexpr __host__ __device__ bool cb_col_has_val(int c) { return ";
    for (size_t i = 0; i < s.cols.size(); i++) o << "c == " << i << " ? " << (s.cols[i].has_validity ? "true" : "false") << " : ";
    o << "false; }\n";
    return o.str();
}

uint64_t fnv1a(const std::string& s) {
    uint64_t h = 1469598103934665603ull;
    for (unsigned char c : s) { h ^= c; h *= 1099511628211ull; }
    return h;
}

int stage_bytes_of(const PipelineSpec& s) {
    int b = 0;
    for (auto& c : s.cols) {
        int w = phys_bytes(c.phys);
        int colb = w == 0 ? s.tile / 8 : s.tile * w;
        b += (colb + 127) / 128 * 128;
        if (c.has_validity) b += (s.tile / 8 + 127) / 128 * 128;
    }
    return b;
}

int out_width(const DType& t) { return t.id == TypeId::Bool ? 1 : t.arrow_width(); }

// bits a group key occupies in the packed 64-bit hash-table key (0 = cannot be packed)
int key_bits(const DType& t) {
    switch (t.id) {
    case TypeId::Bool: return 1;
    case TypeId::Int8: return 8;
    case TypeId::Int16: return 16;
    case TypeId::Int32: case TypeId::Date: return 32;
    case TypeId::String: return 32; // dictionary code
    case TypeId::Int64: case TypeId::Timestamp: case TypeId::TimestampNtz: return 64;
    case TypeId::Decimal: return t.precision <= 18 ? 64 : 0;
    default: return 0;
    }
}

// store a value into a raw 16-byte output slot
std::string to_slot(const Val& v, const std::string& dst) {
    const DType& t = v.type;
    std::ostringstream o;
    if (t.is_decimal() && v.narrow) o << dst << "[0] = (cb::u64)" << v.v << "; " << dst << "[1] = (cb::u64)(" << v.v << " >> 63);";
    else if (t.is_decimal()) o << dst << "[0] = " << v.v << ".lo; " << dst << "[1] = (cb::u64)" << v.v << ".hi;";
    else if (t.id == TypeId::Float64) o << dst << "[0] = (cb::u64)__double_as_longlong(" << v.v << ");";
    else if (t.id == TypeId::Float32) o << dst << "[0] = (cb::u64)__float_as_uint(" << v.v << ");";
    else if (t.id == TypeId::Bool) o << dst << "[0] = " << v.v << " ? 1ull : 0ull;";
    else o << dst << "[0] = (cb::u64)(cb::i64)" << v.v << ";";
    return o.str();
}

} // namespace

// ---- memo: the same plan shape is generated again for every batch / every short-lived plan handle ------------------
namespace {
void sig_expr(std::ostringstream& o, const Expr& e) {
    uint64_t fb;
    memcpy(&fb, &e.lit_f64, 8);
    o << (int)e.kind << '|' << e.type.str() << '|' << e.index << '|' << e.lit_null << '|' << e.lit_i64 << '|' << fb << '|' << (uint64_t)e.lit_dec << ','
      << (uint64_t)(e.lit_dec >> 64) << '|' << e.lit_str << '|' << (int)e.eval_mode << '|' << e.fail_on_error << '|' << e.negated << '|' << e.wide_decimal << '|' << e.integral_div << e.check_divide_overflow << '|'
      << e.return_type.str() << '(';
    if (e.kind == ExprKind::StrPred) o << str_pred_key(e) << '|' << e.in_has_null << '|';
    for (auto& c : e.children) { sig_expr(o, *c); o << ','; }
    o << ')';
}
std::string spec_signature(const PipelineSpec& s) {
    std::ostringstream o;
    o << (int)s.sink << ';' << (int)s.mode << ';' << s.ungrouped << ';' << s.hash << (s.stream ? "s" : "") << (s.masked ? "m" : "") << ';' << s.tile << ';' << s.stages << ';' << s.threads << ';' << s.ltile << ";C";
    for (auto& c : s.cols) o << c.src_index << ':' << c.type.str() << ':' << (int)c.phys << ':' << c.has_validity << ':' << c.assume_bits << (c.layout_nullable && !c.has_validity ? "L" : "") << ',';
    o << ";P";
    for (auto& e : s.predicates) { sig_expr(o, *e); o << ';'; }
    o << ";O";
    for (auto& e : s.outputs) { sig_expr(o, *e); o << ';'; }
    o << ";K";
    for (size_t i = 0; i < s.keys.size(); i++) { sig_expr(o, *s.keys[i]); o << (i < s.key_nullable.size() && s.key_nullable[i]) << ';'; }
    o << ";A";
    for (auto& a : s.aggs) {
        o << (int)a.kind << ':' << (int)a.mode << ':' << a.datatype.str() << ':' << a.sum_datatype.str() << ':' << (int)a.eval_mode << '[';
        for (auto& c : a.children) { sig_expr(o, *c); o << ','; }
        o << "]F";
        if (a.filter) sig_expr(o, *a.filter);
        o << ';';
    }
    o << ";S";
    for (auto& v : s.state_slots) { for (int x : v) o << x << ','; o << ';'; }
    return o.str();
}
std::mutex g_memo_mu;
std::map<std::string, GeneratedKernel> g_memo;
GeneratedKernel generate_pipeline_uncached(const PipelineSpec& spec);
} // namespace

std::string pipeline_signature(const PipelineSpec& spec) { return spec_signature(spec); }

std::vector<int> widen_word_map(const GeneratedKernel& from, const GeneratedKernel& to) {
    if (from.role_words.size() != to.role_words.size()) return {};
    std::vector<int> map((size_t)to.n_words, -1);
    auto set = [&](int w, int o) {
        if (map[(size_t)w] >= 0 && map[(size_t)w] != o) return false; // two words of `from` would merge into one
        map[(size_t)w] = o;
        return true;
    };
    for (size_t r = 0; r < to.role_words.size(); r++) {
        const int w = to.role_words[r], o = from.role_words[r];
        if ((w < 0) != (o < 0)) return {};
        if (w < 0) continue;
        if (!set(w, o)) return {};
        if (to.word_kinds[(size_t)w] == W_DD_HI && !set(w + 1, o + 1)) return {};
    }
    for (int w = 0; w < to.n_words; w++)
        if (map[(size_t)w] < 0 || from.word_kinds.at((size_t)map[(size_t)w]) != to.word_kinds[(size_t)w]) return {};
    return map;
}

std::string str_pred_key(const Expr& e) {
    std::ostringstream o;
    o << (int)e.str_op << ':' << e.str_lits.size();
    for (auto& l : e.str_lits) o << ':' << l.size() << '=' << l; // length-prefixed: any bytes
    return o.str();
}

std::vector<ExprP> str_preds_of(const PipelineSpec& spec) {
    std::vector<ExprP> out;
    std::set<std::string> seen;
    std::function<void(const ExprP&)> walk = [&](const ExprP& e) {
        if (!e) return;
        if (e->kind == ExprKind::StrPred) {
            if (seen.insert(std::to_string(e->children[0]->index) + "@" + str_pred_key(*e)).second) out.push_back(e);
            return;
        }
        for (auto& c : e->children) walk(c);
    };
    for (auto& e : spec.predicates) walk(e);
    for (auto& e : spec.outputs) walk(e);
    for (auto& e : spec.keys) walk(e);
    for (auto& a : spec.aggs)
        if (a.mode == AggMode::Partial) {
            for (auto& c : a.children) walk(c);
            walk(a.filter);
        }
    if (out.size() > CB_MAX_STR_PREDS)
        throw Unsupported("more than " + std::to_string(CB_MAX_STR_PREDS) + " distinct string predicates in one fused pipeline");
    return out;
}

GeneratedKernel generate_pipeline(const PipelineSpec& spec) {
    const std::string sig = spec_signature(spec);
    {
        std::lock_guard<std::mutex> lk(g_memo_mu);
        auto it = g_memo.find(sig);
        if (it != g_memo.end()) return it->second;
    }
    GeneratedKernel g = generate_pipeline_uncached(spec);
    std::lock_guard<std::mutex> lk(g_memo_mu);
    if (g_memo.size() > 4096) g_memo.clear(); // plan shapes are few; this only bounds a pathological caller
    g_memo[sig] = g;
    return g;
}

// =================================================================================================
namespace {
GeneratedKernel generate_pipeline_uncached(const PipelineSpec& spec) {
    GeneratedKernel g;
    g.threads = spec.threads;
    g.tile = spec.tile;
    g.stages = spec.stages;
    g.stage_bytes = stage_bytes_of(spec);
    if (spec.cols.empty()) throw Unsupported("pipeline without input columns");
    if (spec.cols.size() > 24) throw Unsupported("more than 24 staged input columns");

    Emitter em(spec);
    if (spec.sink == SinkKind::Agg && spec.hash) em.base_guard = "in_range"; // hash pipelines also visit the row slots past the end of the tile
    // predicates first: `keep` = every predicate TRUE (FilterExec drops NULL and FALSE)
    std::string keep = "true";
    for (auto& p : spec.predicates) {
        Val v = em.emit(*p);
        keep += " && " + (v.n.empty() ? v.v : "(!" + v.n + " && " + v.v + ")");
    }
    std::ostringstream tu;

    if (spec.sink == SinkKind::Count) {
        em.body << "    return " << keep << ";\n";
        if (spec.ltile <= 0 || spec.tile % spec.ltile) throw PlanError("count pass: stage tile must be a multiple of the logical tile");
        tu << header(spec, "#define CB_KERNEL_SELECT 1\n#define CB_SELECT_COUNT 1\n#define CB_NOUT 0\n#define CB_LTILE " + std::to_string(spec.ltile) + "\n");
        tu << "#include \"cb_kernels.cuh\"\nnamespace cb {\n";
        tu << "CB_D bool cb_row_keep(const Tile& t, int r, i64 grow, const PipeParams& p) {\n    (void)grow; (void)p;\n" << em.body.str() << "}\n} // namespace cb\n";
        g.entry = "cb_select_count";
    } else if (spec.sink == SinkKind::Select) {
        if (spec.outputs.size() > 16) throw Unsupported("more than 16 output columns");
        em.body << "    if (!(" << keep << ")) return false;\n";
        std::ostringstream defs;
        defs << "#define CB_KERNEL_SELECT 1\n#define CB_NOUT " << spec.outputs.size() << "\n#define CB_SEL_MASKED " << (spec.masked ? 1 : 0) << "\n";
        std::vector<Val> outs;
        for (size_t i = 0; i < spec.outputs.size(); i++) {
            Val v = em.emit(*spec.outputs[i]);
            // strings travel as dictionary codes: only a plain column reference can be projected (the node re-attaches the dictionary)
            if (v.type.is_string() && spec.outputs[i]->kind != ExprKind::Bound) throw Unsupported("string expressions in a fused projection");
            outs.push_back(v);
            em.body << "    " << to_slot(v, "o.v[" + std::to_string(i) + "]") << " o.valid[" << i << "] = "
                    << (v.n.empty() ? "true" : "!" + v.n) << ";\n";
            OutCol oc;
            oc.type = v.type;
            oc.nullable = v.nullable();
            g.out_cols.push_back(oc);
            g.out_bytes.push_back(v.type.is_string() ? 4 : out_width(v.type));
        }
        em.body << "    return true;\n";
        tu << header(spec, defs.str());
        tu << "constexpr __host__ __device__ int cb_out_bytes(int c) { return ";
        for (size_t i = 0; i < outs.size(); i++) tu << "c == " << i << " ? " << g.out_bytes[i] << " : ";
        tu << "0; }\n";
        tu << "constexpr __host__ __device__ bool cb_out_nullable(int c) { return ";
        for (size_t i = 0; i < outs.size(); i++) tu << "c == " << i << " ? " << (g.out_cols[i].nullable ? "true" : "false") << " : ";
        tu << "false; }\n";
        tu << "#include \"cb_kernels.cuh\"\nnamespace cb {\n";
        tu << "CB_D bool cb_row_select(const Tile& t, int r, i64 grow, const PipeParams& p, SelOut& o) {\n    (void)grow; (void)p;\n"
           << em.body.str() << "}\n} // namespace cb\n";
        g.entry = "cb_pipeline_select";
    } else {
        // ---------------- aggregate ----------------
        if (spec.hash) {
            // no early return: the table update is warp-cooperative, absent / filtered rows take part with keep_ = false.  Errors
            // of expressions evaluated below must still come from kept rows only.
            em.body << "    const bool keep_ = in_range && (" << keep << ");\n";
            em.base_guard = "keep_";
        } else em.body << "    (void)in_range;\n    if (!(" << keep << ")) return;\n";
        SlotPlan slots;
        std::vector<AggLayout> layout(spec.aggs.size());
        // one accumulator update: `if (cond) acc.add_*(g, w, v)` on the dense paths, the warp-cooperative `acc.h_*(cond, w, v)`
        // (every lane takes part, see cb_kernels.cuh) on the hash path
        const bool H = spec.hash;
        auto upd = [&](const std::string& op, const std::string& cond, int w, const std::string& val = "") {
            std::ostringstream o;
            const std::string ws = std::to_string(w);
            if (H) {
                if (op == "count") o << "acc.h_count(" << cond << ", " << ws << ");";
                else if (op == "wrap") o << "acc.h_add_wrap(" << cond << ", " << ws << ", " << val << ");";
                else if (op == "wide") o << "acc.h_add_i64_wide(" << cond << ", " << ws << ", " << val << ");";
                else if (op == "i128") o << "acc.h_add_i128(" << cond << ", " << ws << ", " << val << ");";
                else if (op == "f64") o << "acc.h_add_f64(" << cond << ", " << ws << ", " << val << ");";
                else if (op == "min") o << "acc.h_min(" << cond << ", " << ws << ", " << val << ");";
                else o << "acc.h_max(" << cond << ", " << ws << ", " << val << ");";
            } else {
                o << "if (" << cond << ") ";
                if (op == "count") o << "acc.add_i64_wrap(g, " << ws << ", 1);";
                else if (op == "wrap") o << "acc.add_i64_wrap(g, " << ws << ", " << val << ");";
                else if (op == "wide") o << "acc.add_i64_wide(g, " << ws << ", " << val << ");";
                else if (op == "i128") o << "acc.add_i128(g, " << ws << ", " << val << ");";
                else if (op == "f64") o << "acc.add_f64(g, " << ws << ", " << val << ");";
                else if (op == "min") o << "acc.min_i64(g, " << ws << ", " << val << ");";
                else o << "acc.max_i64(g, " << ws << ", " << val << ");";
            }
            em.body << "    " << o.str() << "\n";
        };
        auto absval = [&](const std::string& iv) { return "cb::i128_abs_of_i64(" + iv + ")"; };
        // group id.  dense: mixed radix over key codes, NULL key -> last slot of that key.
        //           hash : key columns packed into one 64-bit word -> slot of the global table.
        std::string gid = "0";
        std::string null_group_cond;
        std::ostringstream unpack; // hash: cb_unpack_key body (reverse of the packing)
        if (spec.hash) {
            // Key columns are packed, in order, into 64-bit words: [value bits][null bit if nullable]; a key never straddles
            // words.  One word: the packed word IS the table key (single 128-bit probe).  More: see find_slot_multi.
            struct KeyPlan { Val v; int bits; bool nullable; int word; };
            std::vector<KeyPlan> kp;
            int n_words_k = 1, used = 0;
            for (size_t k = 0; k < spec.keys.size(); k++) {
                KeyPlan q;
                q.v = em.emit(*spec.keys[k]);
                const DType& kt = spec.keys[k]->type;
                q.bits = key_bits(kt);
                // The packing must not depend on whether THIS batch carries a validity buffer (a later batch may): every key
                // reserves its null flag.  Exception: a single 64-bit key sends NULL rows to the reserved NULL-key group, which
                // leaves the packing of non-NULL keys untouched.
                q.nullable = true;
                if (q.bits == 0) throw Unsupported("group key of type " + kt.str() + " cannot be packed into 64-bit hash key words");
                if (q.bits == 64 && spec.keys.size() == 1) {
                    null_group_cond = q.v.n;
                    q.nullable = false;
                }
                int need = q.bits + (q.nullable ? 1 : 0);
                if (need > 64) { // a nullable 64-bit key among several: its null flag opens the next word
                    if (used > 0) { n_words_k++; used = 0; }
                    q.word = n_words_k - 1;
                    used = 64;
                    kp.push_back(q);
                    continue;
                }
                if (used + need > 64) { n_words_k++; used = 0; }
                q.word = n_words_k - 1;
                used += need;
                kp.push_back(q);
            }
            // nullable 64-bit keys in multi-key groups: value fills a word, the null flag travels in an extra flags word
            std::vector<size_t> wide_nullable;
            for (size_t k = 0; k < kp.size(); k++) if (kp[k].nullable && kp[k].bits == 64) wide_nullable.push_back(k);
            int flags_word = -1;
            if (!wide_nullable.empty()) flags_word = n_words_k++;
            if (n_words_k > 4) throw Unsupported("group keys need more than 256 packed bits");
            g.key_words = n_words_k;
            std::vector<std::string> pk(n_words_k);
            for (int w = 0; w < n_words_k; w++) { pk[w] = em.fresh("pk"); em.body << "    cb::u64 " << pk[w] << " = 0;\n"; }
            std::vector<std::string> unpack_steps;
            for (size_t k = 0; k < kp.size(); k++) {
                const KeyPlan& q = kp[k];
                const Val& kv = q.v;
                const DType& kt = spec.keys[k]->type;
                const int bits = q.bits;
                const bool wide_null = q.nullable && bits == 64;
                const bool inline_null = q.nullable && !wide_null;
                const std::string& packed = pk[q.word];
                const std::string isn = kv.n.empty() ? "false" : kv.n;
                std::string raw;
                if (kt.is_decimal()) {
                    if (kv.narrow) raw = "(cb::u64)" + kv.v;
                    else {
                        // a NULL key packs as 0 whatever bytes its slot holds (Arrow leaves them unspecified): only valid keys count
                        const std::string valid = kv.n.empty() ? "" : " && !" + kv.n;
                        em.body << "    if (keep_" << valid << " && !cb::i128_fits_i64(" << kv.v << ")) atomicOr(p.hflags, 4);\n";
                        raw = kv.v + ".lo";
                    }
                } else if (kt.id == TypeId::Bool) raw = "(" + kv.v + " ? 1ull : 0ull)";
                else raw = "(cb::u64)(cb::i64)" + kv.v;
                std::string mask = bits == 64 ? "0xffffffffffffffffull" : u64lit((1ull << bits) - 1);
                if (q.nullable && !kv.n.empty()) raw = "(" + kv.n + " ? 0ull : " + raw + ")";
                if (bits == 64) em.body << "    " << packed << " = " << raw << ";\n";
                else em.body << "    " << packed << " = (" << packed << " << " << bits << ") | (" << raw << " & " << mask << ");\n";
                if (inline_null) em.body << "    " << packed << " = (" << packed << " << 1) | (" << isn << " ? 1ull : 0ull);\n";
                if (wide_null) em.body << "    " << pk[flags_word] << " = (" << pk[flags_word] << " << 1) | (" << isn << " ? 1ull : 0ull);\n";
                // unpack (emitted in reverse order below): consumes the same bits from k<word>
                std::ostringstream u;
                std::string kc = std::to_string(k), kwv = "k" + std::to_string(q.word);
                u << "    {\n";
                if (inline_null) u << "      bool isnull = (" << kwv << " & 1ull) != 0; " << kwv << " >>= 1;\n";
                else if (wide_null) u << "      bool isnull = (k" << flags_word << " & 1ull) != 0; k" << flags_word << " >>= 1;\n";
                else u << "      bool isnull = null_group;\n";
                if (bits == 64) u << "      cb::u64 raw = " << kwv << "; " << kwv << " = 0;\n";
                else u << "      cb::u64 raw = " << kwv << " & " << mask << "; " << kwv << " >>= " << bits << ";\n";
                if (kt.is_decimal()) u << "      cb::fin_store_i128(fp, " << kc << ", g, cb::i128_from_i64((cb::i64)raw), !isnull);\n";
                else if (kt.id == TypeId::Bool) u << "      cb::fin_store_u8(fp, " << kc << ", g, (int)raw, !isnull);\n";
                else if (bits == 64) u << "      cb::fin_store_i64(fp, " << kc << ", g, (cb::i64)raw, !isnull);\n";
                else {
                    int w = kt.is_string() ? 4 : kt.arrow_width();
                    std::string sx = bits == 8 ? "(cb::i32)(signed char)raw" : bits == 16 ? "(cb::i32)(short)raw" : "(cb::i32)raw";
                    u << "      cb::fin_store_i32(fp, " << kc << ", g, " << sx << ", !isnull, " << w << ");\n";
                }
                u << "    }\n";
                unpack_steps.push_back(u.str());
            }
            for (int w = 0; w < n_words_k; w++) unpack << "    cb::u64 k" << w << " = kw[" << w << "]; (void)k" << w << ";\n";
            for (auto it = unpack_steps.rbegin(); it != unpack_steps.rend(); ++it) unpack << *it;
            {
                std::string arr = em.fresh("kw");
                em.body << "    cb::u64 " << arr << "[" << n_words_k << "] = {";
                for (int w = 0; w < n_words_k; w++) em.body << (w ? ", " : "") << pk[w];
                em.body << "};\n";
                if (!null_group_cond.empty()) em.body << "    if (keep_ && " << null_group_cond << ") atomicOr(p.hflags, 8);\n";
                em.body << "    acc.begin(keep_, " << arr << ", " << (null_group_cond.empty() ? "false" : null_group_cond) << ");\n";
            }
        } else if (!spec.ungrouped) {
            for (size_t k = 0; k < spec.keys.size(); k++) {
                Val kv = em.emit(*spec.keys[k]);
                std::string code = kv.type.id == TypeId::Bool && spec.cols[spec.keys[k]->index].phys == Phys::Bitmap ? "(" + kv.v + " ? 1 : 0)" : kv.v;
                if (kv.nullable()) code = "(" + kv.n + " ? p.key_card[" + std::to_string(k) + "] - 1 : " + code + ")";
                gid = "(" + gid + ") * p.key_card[" + std::to_string(k) + "] + " + code;
            }
        }
        if (!spec.hash) em.body << "    const int g = " << gid << ";\n";
        int w_rows = slots.add(W_WRAP64, "cnt|true"); // rows passing the filter == COUNT(*) == non-null count of never-null inputs
        upd("count", "true", w_rows);
        // Which inputs share a word is decided by the null tests of every column that ever carried validity (layout_nullable), not
        // by this batch's alone, so a later batch without validity keeps the layout.  `km` emits the aggregate inputs as if those
        // columns had validity; only the strings it returns -- the slot dedup keys -- are used.  A spec where the two agree keys
        // the slots by `em`'s own strings.
        PipelineSpec lspec;
        std::unique_ptr<Emitter> km;
        if (std::any_of(spec.cols.begin(), spec.cols.end(), [](const SourceCol& c) { return c.layout_nullable && !c.has_validity; })) {
            lspec = spec;
            for (auto& c : lspec.cols) c.has_validity = c.has_validity || c.layout_nullable;
            km.reset(new Emitter(lspec));
            km->base_guard = em.base_guard;
        }
        // the FILTER clause, then the children: `cond` = the row passes the filter and every child is non-NULL
        auto input_cond = [](Emitter& e, const AggExpr& a, std::vector<Val>& cv) {
            std::string cond = "true";
            if (a.filter) {
                Val f = e.emit(*a.filter);
                cond = f.n.empty() ? f.v : "(!" + f.n + " && " + f.v + ")";
            }
            for (auto& c : a.children) cv.push_back(e.emit(*c));
            for (auto& v : cv) if (v.nullable()) cond += " && !" + v.n;
            return cond;
        };

        for (size_t ai = 0; ai < spec.aggs.size(); ai++) {
            const AggExpr& a = spec.aggs[ai];
            AggLayout& L = layout[ai];
            if (a.mode == AggMode::Partial) {
                // per-aggregate FILTER clause: NULL/FALSE excludes the row (sum_decimal.rs:452-458)
                std::vector<Val> cv, kcv;
                const std::string cond = input_cond(em, a, cv);
                const std::string condkey = km ? input_cond(*km, a, kcv) : cond;
                const Val& v = cv[0];
                const std::string vkey = km ? kcv[0].v : v.v; // the value's name in the slot keys
                std::string use = cond == "true" ? "true" : em.declb(cond);
                // non-null (and filter-passing) row count of this input: COUNT, AVG count, !is_empty
                auto cnt_slot = [&]() {
                    std::string k = "cnt|" + condkey;
                    bool first = slots.dedup.count(std::to_string((int)W_WRAP64) + "|" + k) == 0;
                    int w = slots.add(W_WRAP64, k);
                    if (first) upd("count", use, w);
                    return w;
                };
                switch (a.kind) {
                case AggKind::Count:
                    L.w_cnt = cnt_slot();
                    break;
                case AggKind::Sum: case AggKind::Avg: {
                    bool dec = a.datatype.is_decimal();
                    bool f64 = !dec && (a.kind == AggKind::Avg || a.datatype.is_float());
                    L.w_cnt = cnt_slot();
                    if (dec) {
                        bool first = slots.dedup.count(std::to_string((int)W_SUM128) + "|sum|" + vkey + "|" + condkey) == 0;
                        L.w_sum = slots.add(W_SUM128, "sum|" + vkey + "|" + condkey);
                        if (first) {
                            // per-thread 64-bit partials are exact while rows/thread * |v| < 2^63 (host caps rows/thread at 2^CB_RPT_LOG2)
                            u128r vb = em.bound_of(*a.children[0]);
                            if (spec.hash) upd(v.narrow ? "wide" : "i128", use, L.w_sum, v.v); // table words are full 128-bit totals: always sign-extend + carry
                            else if (v.narrow && vb < (R63 >> CB_RPT_LOG2)) upd("wrap", use, L.w_sum, v.v);
                            else if (v.narrow) upd("wide", use, L.w_sum, v.v);
                            else upd("i128", use, L.w_sum, v.v);
                        }
                    } else if (f64) {
                        L.is_f64_sum = true;
                        std::string dv = v.type.id == TypeId::Float64 ? v.v : "(double)" + v.v;
                        bool first = slots.dedup.count(std::to_string((int)W_DD_HI) + "|dd|" + vkey + "|" + condkey) == 0;
                        L.w_sum = slots.add(W_DD_HI, "dd|" + vkey + "|" + condkey, 2);
                        if (first) upd("f64", use, L.w_sum, dv);
                    } else if (a.eval_mode != EvalMode::Legacy) {
                        // SumInt ANSI / TRY (sum_int.rs:176-390): the reference adds row by row with add_checked, so whether it
                        // overflows depends on the row order.  The exact 128-bit sum and the exact sum of magnitudes decide it for
                        // EVERY order: sum|v| <= i64::MAX => no prefix of any order can overflow; total out of range => every
                        // order overflows (the last prefix is the total); anything else is order-dependent (finalize raises it).
                        std::string iv = "(cb::i64)" + v.v;
                        bool first = slots.dedup.count(std::to_string((int)W_SUM128) + "|csum|" + vkey + "|" + condkey) == 0;
                        L.w_sum = slots.add(W_SUM128, "csum|" + vkey + "|" + condkey);
                        L.w_abs = slots.add(W_SUM128, "cabs|" + vkey + "|" + condkey);
                        if (first) { upd("wide", use, L.w_sum, iv); upd("i128", use, L.w_abs, absval(iv)); }
                    } else { // SumInt Legacy: wrapping i64 (sum_int.rs:432)
                        bool first = slots.dedup.count(std::to_string((int)W_WRAP64) + "|isum|" + vkey + "|" + condkey) == 0;
                        L.w_sum = slots.add(W_WRAP64, "isum|" + vkey + "|" + condkey);
                        if (first) upd("wrap", use, L.w_sum, "(cb::i64)" + v.v);
                    }
                    break;
                }
                case AggKind::Min: case AggKind::Max: {
                    L.w_cnt = cnt_slot();
                    std::string key = v.type.is_decimal() ? (v.narrow ? v.v : "(cb::i64)" + v.v + ".lo")
                                      : v.type.id == TypeId::Float64 ? "cb::f64_total_key((cb::u64)__double_as_longlong(" + v.v + "))"
                                                                     : "(cb::i64)" + v.v;
                    // the words hold 64-bit keys: a decimal(p <= 18) value outside them (invalid input) is refused, never compared by its low word
                    if (v.type.is_decimal() && !v.narrow) em.raise(use + " && !cb::i128_fits_i64(" + v.v + ")", 6);
                    bool mn = a.kind == AggKind::Min;
                    std::string sk = std::string(mn ? "min|" : "max|") + vkey + "|" + condkey;
                    bool first = slots.dedup.count(std::to_string((int)(mn ? W_MIN : W_MAX)) + "|" + sk) == 0;
                    L.w_minmax = slots.add(mn ? W_MIN : W_MAX, sk);
                    if (first) upd(mn ? "min" : "max", use, L.w_minmax, key);
                    break;
                }
                }
            } else {
                // ---- Final / PartialMerge: merge state columns (merge_batch semantics) ----
                const std::vector<int>& sc = spec.state_slots.at(ai);
                auto col = [&](int i) { Expr b; b.kind = ExprKind::Bound; b.index = sc[i]; b.type = spec.cols[sc[i]].type; return em.emit(b); };
                std::string tag = "agg" + std::to_string(ai);
                switch (a.kind) {
                case AggKind::Count: { // count merge = sum of partial counts
                    Val c = col(0);
                    L.w_cnt = slots.add(W_WRAP64, tag + "cnt");
                    upd("wrap", c.n.empty() ? "true" : "!" + c.n, L.w_cnt, c.v);
                    break;
                }
                case AggKind::Sum:
                    if (a.datatype.is_decimal()) { // sum_decimal.rs:540-607
                        Val s = col(0), e = col(1);
                        std::string snull = s.n.empty() ? "false" : s.n;
                        L.w_sum = slots.add(W_SUM128, tag + "sum");
                        L.w_cnt = slots.add(W_WRAP64, tag + "cnt");
                        L.w_bad = slots.add(W_WRAP64, tag + "bad");
                        std::string bad = em.declb("!" + e.v + " && " + snull), ok = em.declb("!" + e.v + " && !(" + snull + ")");
                        upd("count", bad, L.w_bad);
                        upd("i128", ok, L.w_sum, Emitter::W(s));
                        upd("count", ok, L.w_cnt);
                    } else if (a.datatype.is_integer() && a.eval_mode != EvalMode::Legacy) { // sum_int.rs:236-243 (ANSI), :331-389 (TRY)
                        Val s = col(0);
                        std::string snull = s.n.empty() ? "false" : s.n;
                        L.w_sum = slots.add(W_SUM128, tag + "sum");
                        L.w_abs = slots.add(W_SUM128, tag + "abs");
                        L.w_cnt = slots.add(W_WRAP64, tag + "cnt");
                        std::string ok;
                        if (a.eval_mode == EvalMode::Try) { // state (sum, has_all_nulls): overflowed = !has_all_nulls && sum IS NULL
                            Val e = col(1);
                            L.w_bad = slots.add(W_WRAP64, tag + "bad");
                            upd("count", em.declb("!" + e.v + " && " + snull), L.w_bad);
                            ok = em.declb("!" + e.v + " && !(" + snull + ")");
                        } else ok = em.declb("!(" + snull + ")");
                        upd("wide", ok, L.w_sum, s.v);
                        upd("i128", ok, L.w_abs, absval(s.v));
                        upd("count", ok, L.w_cnt);
                    } else if (a.datatype.is_integer()) { // sum_int.rs:497-528
                        Val s = col(0);
                        L.w_sum = slots.add(W_WRAP64, tag + "sum");
                        L.w_cnt = slots.add(W_WRAP64, tag + "cnt");
                        const std::string ok = s.n.empty() ? "true" : "!" + s.n;
                        upd("wrap", ok, L.w_sum, s.v);
                        upd("count", ok, L.w_cnt);
                    } else {
                        Val s = col(0);
                        L.is_f64_sum = true;
                        L.w_sum = slots.add(W_DD_HI, tag + "sum", 2);
                        L.w_cnt = slots.add(W_WRAP64, tag + "cnt");
                        const std::string ok = s.n.empty() ? "true" : "!" + s.n;
                        upd("f64", ok, L.w_sum, "(double)" + s.v);
                        upd("count", ok, L.w_cnt);
                    }
                    break;
                case AggKind::Avg:
                    if (a.datatype.is_decimal()) { // avg_decimal.rs:542-595
                        Val s = col(0), c = col(1);
                        L.w_sum = slots.add(W_SUM128, tag + "sum");
                        L.w_cnt = slots.add(W_WRAP64, tag + "cnt");
                        L.w_bad = slots.add(W_WRAP64, tag + "bad");
                        std::string cnull = c.n.empty() ? "false" : c.n, snull = s.n.empty() ? "false" : s.n;
                        upd("wrap", "!" + cnull, L.w_cnt, c.v);
                        upd("count", "(" + snull + " || " + cnull + ")", L.w_bad);
                        upd("i128", "!" + snull, L.w_sum, Emitter::W(s));
                    } else { // avg.rs:165-175 (ungrouped), :279-309 (grouped)
                        // A NULL partial sum or count adds nothing: the ungrouped accumulator merges with arrow's null-skipping
                        // `sum`, and its Partial emits a NULL sum for a partition that saw no batch (avg.rs:148-153).  The bytes
                        // under a NULL slot are unspecified in Arrow, so they are never read.
                        Val s = col(0), c = col(1);
                        L.is_f64_sum = true;
                        L.w_sum = slots.add(W_DD_HI, tag + "sum", 2);
                        L.w_cnt = slots.add(W_WRAP64, tag + "cnt");
                        upd("f64", s.n.empty() ? "true" : "!" + s.n, L.w_sum, s.v);
                        upd("wrap", c.n.empty() ? "true" : "!" + c.n, L.w_cnt, c.v);
                    }
                    break;
                case AggKind::Min: case AggKind::Max: {
                    Val s = col(0);
                    bool mn = a.kind == AggKind::Min;
                    L.w_cnt = slots.add(W_WRAP64, tag + "cnt");
                    L.w_minmax = slots.add(mn ? W_MIN : W_MAX, tag + "mm");
                    std::string key = s.type.is_decimal() ? (s.narrow ? s.v : "(cb::i64)" + s.v + ".lo")
                                      : s.type.id == TypeId::Float64 ? "cb::f64_total_key((cb::u64)__double_as_longlong(" + s.v + "))"
                                                                     : "(cb::i64)" + s.v;
                    const std::string ok = s.n.empty() ? "true" : "!" + s.n;
                    if (s.type.is_decimal() && !s.narrow) em.raise(ok + " && !cb::i128_fits_i64(" + s.v + ")", 6);
                    upd(mn ? "min" : "max", ok, L.w_minmax, key);
                    upd("count", ok, L.w_cnt);
                    break;
                }
                }
            }
        }
        g.n_words = (int)slots.kinds.size();
        g.word_kinds = slots.kinds;
        g.role_words.push_back(w_rows);
        for (const AggLayout& L : layout)
            for (int w : {L.w_sum, L.w_cnt, L.w_bits, L.w_bad, L.w_minmax, L.w_abs}) g.role_words.push_back(w);

        // ---------------- finalize program: totals -> state columns (Partial) / results (Final) -------
        std::ostringstream fin;
        int oc = 0;
        if (spec.hash) {
            for (size_t k = 0; k < spec.keys.size(); k++) {
                OutCol o;
                o.type = spec.keys[k]->type;
                o.nullable = true;
                g.out_cols.push_back(o);
                g.out_bytes.push_back(o.type.is_string() ? 4 : out_width(o.type));
                oc++;
            }
            g.n_key_cols = (int)spec.keys.size();
            g.hash = true;
        }
        auto add_out = [&](const DType& t, bool nullable) {
            OutCol o;
            o.type = t;
            o.nullable = nullable;
            g.out_cols.push_back(o);
            g.out_bytes.push_back(out_width(t));
            return oc++;
        };
        auto T128 = [](int w) { return "cb::fin_i128(T, " + std::to_string(w) + ")"; };
        auto T64 = [](int w) { return "(cb::i64)T[" + std::to_string(w) + " * 2]"; };
        auto TDD = [](int w) { return "cb::fin_dd(T, " + std::to_string(w) + ")"; };
        for (size_t ai = 0; ai < spec.aggs.size(); ai++) {
            const AggExpr& a = spec.aggs[ai];
            const AggLayout& L = layout[ai];
            bool partial = a.mode != AggMode::Final; // Partial and PartialMerge emit state columns
            std::string A = "a" + std::to_string(ai);
            fin << "    { // aggregate " << ai << "\n";
            switch (a.kind) {
            case AggKind::Count: {
                int c = add_out(mk_type(TypeId::Int64), false);
                fin << "      cb::fin_store_i64(fp, " << c << ", g, " << T64(L.w_cnt) << ", true);\n";
                break;
            }
            case AggKind::Sum:
                if (a.datatype.is_decimal()) {
                    // exact total; overflow decided by the certificate (see DESIGN.md "decimal sums")
                    fin << "      cb::i128 s = " << T128(L.w_sum) << "; cb::i64 n = " << T64(L.w_cnt) << ";\n";
                    fin << "      bool bad = " << (L.w_bad >= 0 ? T64(L.w_bad) + " > 0" : "false") << ";\n";
                    fin << "      int cert = cb::sum_cert(cb::cert_level(n, fp.cert_b[" << ai << "][0], fp.cert_b[" << ai << "][1], " << a.datatype.precision
                        << "), cb::dec_fits_p(s, " << a.datatype.precision << ")); // 0 fits, 1 overflow, 2 order-dependent\n";
                    fin << "      if (n > 0 && !bad && cert == 2) cb::set_err_raw(fp.err, 2);\n";
                    fin << "      bool ovf = bad || (n > 0 && cert != 0);\n";
                    if (a.eval_mode == EvalMode::Ansi) fin << "      if (n > 0 && !bad && cert == 1) cb::set_err_raw(fp.err, 1); // certain overflow only: an order-dependent sum is reported as such\n";
                    if (partial) {
                        int c0 = add_out(a.datatype, true), c1 = add_out(mk_type(TypeId::Bool), false);
                        // state(): sum = Some(0) while empty, None after overflow (sum_decimal.rs:526-538)
                        fin << "      cb::fin_store_i128(fp, " << c0 << ", g, ovf ? cb::mk128(0, 0) : s, !ovf);\n";
                        fin << "      cb::fin_store_u8(fp, " << c1 << ", g, (n == 0 && !bad) ? 1 : 0, true);\n";
                    } else {
                        int c0 = add_out(a.datatype, true);
                        fin << "      bool ok = !ovf && n > 0;\n";
                        fin << "      cb::fin_store_i128(fp, " << c0 << ", g, ok ? s : cb::mk128(0, 0), ok);\n";
                    }
                } else if (a.datatype.is_integer() && a.eval_mode != EvalMode::Legacy) {
                    fin << "      cb::i128 s = " << T128(L.w_sum) << ", ab = " << T128(L.w_abs) << "; cb::i64 n = " << T64(L.w_cnt) << ";\n";
                    fin << "      bool bad = " << (L.w_bad >= 0 ? T64(L.w_bad) + " > 0" : "false") << ";\n";
                    fin << "      bool fits = s.hi == ((cb::i64)s.lo >> 63), absfits = ab.hi == 0 && (cb::i64)ab.lo >= 0;\n";
                    fin << "      int cert = absfits ? 0 : !fits ? 1 : 2; // 0 no order overflows, 1 every order overflows, 2 order-dependent\n";
                    fin << "      if (n > 0 && !bad && cert == 2) cb::set_err_raw(fp.err, 2);\n";
                    fin << "      bool ovf = bad || (n > 0 && cert != 0);\n";
                    if (a.eval_mode == EvalMode::Ansi) {
                        fin << "      if (bad || (n > 0 && cert == 1)) cb::set_err_raw(fp.err, 1);\n";
                        int c0 = add_out(mk_type(TypeId::Int64), true);
                        fin << "      cb::fin_store_i64(fp, " << c0 << ", g, (n > 0 && !ovf) ? (cb::i64)s.lo : 0, n > 0 && !ovf);\n";
                    } else if (partial) { // TRY state(): sum = Some(0) while all-null, None after overflow; has_all_nulls (sum_int.rs:322-329)
                        int c0 = add_out(mk_type(TypeId::Int64), true), c1 = add_out(mk_type(TypeId::Bool), false);
                        fin << "      cb::fin_store_i64(fp, " << c0 << ", g, (n > 0 && !ovf) ? (cb::i64)s.lo : 0, !ovf);\n";
                        fin << "      cb::fin_store_u8(fp, " << c1 << ", g, (n == 0 && !bad) ? 1 : 0, true);\n";
                    } else { // TRY evaluate(): NULL when all inputs were NULL or the sum overflowed (sum_int.rs:310-316)
                        int c0 = add_out(mk_type(TypeId::Int64), true);
                        fin << "      bool ok = n > 0 && !ovf;\n";
                        fin << "      cb::fin_store_i64(fp, " << c0 << ", g, ok ? (cb::i64)s.lo : 0, ok);\n";
                    }
                } else if (a.datatype.is_integer()) {
                    int c0 = add_out(mk_type(TypeId::Int64), true);
                    fin << "      cb::i64 n = " << T64(L.w_cnt) << ";\n";
                    fin << "      cb::fin_store_i64(fp, " << c0 << ", g, n > 0 ? " << T64(L.w_sum) << " : 0, n > 0);\n";
                } else {
                    int c0 = add_out(a.datatype, true);
                    fin << "      cb::i64 n = " << T64(L.w_cnt) << "; double s = " << TDD(L.w_sum) << ";\n";
                    if (a.datatype.id == TypeId::Float32) fin << "      cb::fin_store_f32(fp, " << c0 << ", g, n > 0 ? (float)s : 0.0f, n > 0);\n";
                    else fin << "      cb::fin_store_f64(fp, " << c0 << ", g, n > 0 ? s : 0.0, n > 0);\n";
                }
                break;
            case AggKind::Avg:
                if (a.datatype.is_decimal()) {
                    int sp = a.sum_datatype.precision;
                    fin << "      cb::i128 s = " << T128(L.w_sum) << "; cb::i64 n = " << T64(L.w_cnt) << ";\n";
                    fin << "      bool bad = " << (L.w_bad >= 0 ? T64(L.w_bad) + " > 0" : "false") << ";\n";
                    // addends: input rows (Partial) / merged state rows (Final, PartialMerge: `n` is the merged COUNT there)
                    fin << "      int cert = cb::sum_cert(cb::cert_level(" << (a.mode == AggMode::Partial ? "n" : "(cb::i64)T[CB_W_ROWS * 2]") << ", fp.cert_b[" << ai
                        << "][0], fp.cert_b[" << ai << "][1], " << sp << "), cb::dec_fits_p(s, " << sp << "));\n";
                    fin << "      if (n > 0 && !bad && cert == 2) cb::set_err_raw(fp.err, 2);\n";
                    fin << "      bool notnull = !bad && !(n > 0 && cert != 0);\n";
                    if (partial) { // state(): sums and counts share is_not_null as validity (avg_decimal.rs:640-656)
                        int c0 = add_out(a.sum_datatype, true), c1 = add_out(mk_type(TypeId::Int64), true);
                        fin << "      cb::fin_store_i128(fp, " << c0 << ", g, s, notnull);\n";
                        fin << "      cb::fin_store_i64(fp, " << c1 << ", g, n, notnull);\n";
                    } else {
                        int c0 = add_out(a.datatype, true);
                        if (a.eval_mode == EvalMode::Ansi) fin << "      if (n > 0 && (bad || cert == 1)) cb::set_err_raw(fp.err, 1);\n";
                        int d = a.datatype.scale - a.sum_datatype.scale;
                        if (d < 0) d = 0;
                        fin << "      cb::i128 r = cb::mk128(0, 0); bool ok = notnull && n > 0 && cb::avg_decimal_eval(s, n, " << d << ", "
                            << a.datatype.precision << ", r);\n";
                        fin << "      cb::fin_store_i128(fp, " << c0 << ", g, ok ? r : cb::mk128(0, 0), ok);\n";
                    }
                } else {
                    fin << "      cb::i64 n = " << T64(L.w_cnt) << "; double s = " << TDD(L.w_sum) << ";\n";
                    if (partial) {
                        int c0 = add_out(mk_type(TypeId::Float64), false), c1 = add_out(mk_type(TypeId::Int64), false);
                        fin << "      cb::fin_store_f64(fp, " << c0 << ", g, s, true);\n      cb::fin_store_i64(fp, " << c1 << ", g, n, true);\n";
                    } else {
                        int c0 = add_out(mk_type(TypeId::Float64), true);
                        fin << "      cb::fin_store_f64(fp, " << c0 << ", g, n != 0 ? __ddiv_rn(s, (double)n) : 0.0, n != 0);\n";
                    }
                }
                break;
            case AggKind::Min: case AggKind::Max: {
                int c0 = add_out(a.datatype, true);
                fin << "      cb::i64 n = " << T64(L.w_cnt) << "; cb::i64 k = " << T64(L.w_minmax) << ";\n";
                if (a.datatype.is_decimal()) fin << "      cb::fin_store_i128(fp, " << c0 << ", g, cb::i128_from_i64(k), n > 0);\n";
                else if (a.datatype.id == TypeId::Float64)
                    fin << "      cb::fin_store_f64(fp, " << c0 << ", g, __longlong_as_double(cb::f64_total_key((cb::u64)k)), n > 0);\n";
                else if (a.datatype.arrow_width() == 8) fin << "      cb::fin_store_i64(fp, " << c0 << ", g, k, n > 0);\n";
                else fin << "      cb::fin_store_i32(fp, " << c0 << ", g, (cb::i32)k, n > 0, " << a.datatype.arrow_width() << ");\n";
                break;
            }
            }
            fin << "    }\n";
        }

        // claim-first probing when the input rows are state rows: a Final / PartialMerge operator, or one with a merging aggregate
        bool merges_state = spec.mode != AggMode::Partial;
        for (auto& a : spec.aggs) if (a.mode != AggMode::Partial) merges_state = true;
        std::ostringstream defs;
        g.ungrouped = spec.ungrouped;
        defs << "#define CB_KERNEL_AGG 1\n#define CB_WORDS " << g.n_words << "\n#define CB_G1 " << (spec.ungrouped ? 1 : 0) << "\n#define CB_W_ROWS " << w_rows
             << "\n#define CB_HASH " << (spec.hash ? 1 : 0) << "\n#define CB_KEY_WORDS " << (spec.hash ? g.key_words : 1) << "\n#define CB_STREAM " << (spec.hash && spec.stream ? 1 : 0)
             << "\n#define CB_CAS_FIRST " << (spec.hash && merges_state ? 1 : 0) << "\n";
        tu << header(spec, defs.str());
        tu << "constexpr __host__ __device__ int cb_word_kind(int w) { return ";
        for (size_t i = 0; i < slots.kinds.size(); i++) tu << "w == " << i << " ? " << slots.kinds[i] << " : ";
        tu << "0; }\n";
        tu << "#include \"cb_kernels.cuh\"\nnamespace cb {\n";
        tu << "CB_D void cb_row_agg(const Tile& t, int r, i64 grow, const PipeParams& p, Acc& acc, bool in_range) {\n    (void)grow;\n" << em.body.str() << "}\n";
        tu << "CB_D void cb_finalize_group(const FinParams& fp, int g, const u64* T) {\n" << fin.str() << "}\n";
        if (spec.hash) tu << "CB_D void cb_unpack_key(const FinParams& fp, int g, const u64* kw, bool null_group) {\n" << unpack.str() << "}\n";
        tu << "} // namespace cb\n";
        g.entry = "cb_pipeline_agg";
        g.finalize_entry = "cb_finalize";
    }
    g.source = tu.str();
    std::ostringstream k;
    k << std::hex << fnv1a(g.source) << "_" << g.source.size();
    g.key = k.str();
    return g;
}
} // namespace

} // namespace cb200
