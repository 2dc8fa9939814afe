// ranges_test.cpp -- test-only driver of the magnitude bounds (ranges.h), linked with the plan decoder (plan.cpp) and without the CUDA
// runtime by tests/test_ranges_cpu.py.  Not part of libcomet_b200.so.
#include "plan.h"
#include "ranges.h"

#include <cstdio>

using namespace cb200;

extern "C" {
// expr_maxabs of the first expression of a Projection plan, given |column c| <= bounds[c] (bounds: n_cols (lo, hi) pairs, 2^127 =
// unbounded).  Writes the bound as (lo, hi); returns 0, or -1 with the decode error in `err`.
int rt_maxabs(const uint8_t* plan, size_t len, int n_cols, const uint64_t* bounds, uint64_t* out, char* err, size_t cap) {
    try {
        OperatorP op = decode_plan(plan, len);
        if (op->kind != OpKind::Projection || op->project_list.empty()) throw PlanError("expected a Projection");
        std::vector<u128r> b((size_t)n_cols);
        for (int c = 0; c < n_cols; c++) b[(size_t)c] = (u128r)bounds[2 * c] | (u128r)bounds[2 * c + 1] << 64;
        const u128r r = expr_maxabs(*op->project_list[0], b);
        out[0] = (uint64_t)r;
        out[1] = (uint64_t)(r >> 64);
        return 0;
    } catch (const std::exception& e) {
        snprintf(err, cap, "%s", e.what());
        return -1;
    }
}
}
