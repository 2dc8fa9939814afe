// strpred_test.cpp -- test-only driver of device/cb_strpred.h on the host (the matcher the mask kernel k_str_pred runs), built with
// g++ by tests/test_string_predicates_cpu.py like host_math_test.cpp.
#include "device/cb_strpred.h"

#include <vector>

// op: cb::StrOp.  Literal i is lits[lit_off[i], lit_off[i + 1]); for SP_LIKE, lits[lit_off[0], lit_off[1]) is the pattern text.
// Returns the predicate's value (0 / 1) on s[0, n), or -1 when the LIKE pattern does not compile.
extern "C" int cb_sp_eval(int op, const unsigned char* s, int n, const unsigned char* lits, const int* lit_off, int n_lits) {
    cb::StrPredDev d{};
    d.op = op;
    d.n_lits = n_lits;
    d.lit_off = lit_off;
    d.lit = lits;
    std::vector<unsigned short> items;
    if (op == cb::SP_LIKE) {
        const int len = lit_off[1] - lit_off[0];
        items.resize((size_t)len + 1);
        const int k = cb::sp_like_compile(lits + lit_off[0], len, items.data());
        if (k < 0) return -1;
        d.pat = items.data();
        d.pat_len = k;
    }
    return cb::sp_eval(d, s, n) ? 1 : 0;
}
