// layout_test.cpp -- test-only driver of the aggregate accumulator layout (codegen.cpp), linked with the plan decoder (plan.cpp) and
// without the CUDA runtime by tests/test_batch_layouts_cpu.py.  Not part of libcomet_b200.so.
#include "codegen.h"

#include <cstdio>

using namespace cb200;

namespace {

Phys phys_of_type(const DType& t) { // exec_internal.h phys_of, strings as dictionary codes (the staged form of a key)
    switch (t.id) {
    case TypeId::Bool: return Phys::Bitmap;
    case TypeId::Int8: return Phys::I8;
    case TypeId::Int16: return Phys::I16;
    case TypeId::Int32: case TypeId::Date: return Phys::I32;
    case TypeId::Int64: case TypeId::Timestamp: case TypeId::TimestampNtz: return Phys::I64;
    case TypeId::Float32: return Phys::F32;
    case TypeId::Float64: return Phys::F64;
    case TypeId::Decimal: return Phys::I128;
    default: return Phys::Dict32;
    }
}

// The pipeline of a Partial HashAggregate over a Scan, every scan column staged in its own slot: column c carries validity in this
// batch when bit c of `validity` is set, and an earlier batch gave it validity when bit c of `layout` is set.
GeneratedKernel agg_layout(const uint8_t* plan, size_t len, uint32_t validity, uint32_t layout, int hash) {
    OperatorP op = decode_plan(plan, len);
    if (op->kind != OpKind::HashAgg || op->children.empty()) throw PlanError("expected a HashAggregate over a scan");
    const std::vector<DType>& in = op->children[0]->schema;
    if (in.size() > 24) throw PlanError("more than 24 columns");
    PipelineSpec s;
    for (size_t c = 0; c < in.size(); c++) {
        SourceCol sc;
        sc.src_index = (int)c;
        sc.type = in[c];
        sc.phys = phys_of_type(in[c]);
        sc.has_validity = (validity >> c) & 1;
        sc.layout_nullable = (layout >> c) & 1;
        s.cols.push_back(sc);
    }
    s.sink = SinkKind::Agg;
    s.mode = op->mode;
    s.ungrouped = op->grouping.empty();
    s.hash = hash != 0;
    s.keys = op->grouping;
    s.key_nullable.assign(s.keys.size(), false);
    for (auto& a : op->aggs) {
        if (a.mode != AggMode::Partial) throw PlanError("expected Partial-mode aggregates");
        s.aggs.push_back(a);
        s.state_slots.push_back({});
    }
    return generate_pipeline(s);
}

int fail(const std::exception& e, char* err, size_t cap) {
    snprintf(err, cap, "%s", e.what());
    return -1;
}

} // namespace

extern "C" {
// The accumulator layout: out = [n_words, n_roles, word kinds..., role words...].  Returns 0, or -1 with the error in `err`.
int lt_layout(const uint8_t* plan, size_t len, uint32_t validity, uint32_t layout, int hash, int* out, int cap, char* err, size_t err_cap) {
    try {
        const GeneratedKernel g = agg_layout(plan, len, validity, layout, hash);
        const int need = 2 + g.n_words + (int)g.role_words.size();
        if (need > cap) throw PlanError("output too small");
        int at = 0;
        out[at++] = g.n_words;
        out[at++] = (int)g.role_words.size();
        for (int k : g.word_kinds) out[at++] = k;
        for (int w : g.role_words) out[at++] = w;
        return 0;
    } catch (const std::exception& e) {
        return fail(e, err, err_cap);
    }
}

// widen_word_map from the layout of the batches so far (columns in `from` nullable) to the one of a batch whose validity adds the
// columns of `to`: out[w] = the word new word w starts from.  Returns the new word count, -2 when the layouts do not correspond, or
// -1 with the error in `err`.
int lt_widen(const uint8_t* plan, size_t len, uint32_t from, uint32_t to, int hash, int* out, int cap, char* err, size_t err_cap) {
    try {
        const GeneratedKernel a = agg_layout(plan, len, from, 0, hash), b = agg_layout(plan, len, to, from | to, hash);
        const std::vector<int> map = widen_word_map(a, b);
        if (map.empty()) return -2;
        if ((int)map.size() > cap) throw PlanError("output too small");
        for (size_t w = 0; w < map.size(); w++) out[w] = map[w];
        return (int)map.size();
    } catch (const std::exception& e) {
        return fail(e, err, err_cap);
    }
}
}
