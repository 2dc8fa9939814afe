// cb_kernels.cuh -- hand-written sm_90a kernel skeletons for the fused scan -> filter -> project
// -> {compact | aggregate} pipelines.  A pipeline kernel = this file + one generated `cb_prog`
// block (the plan's expression tree spliced into straight-line code by codegen.cpp) compiled by
// NVRTC for sm_90a at createPlan time.  Everything that decides performance lives here:
//
//   * persistent CTAs (grid = #SMs x CTAs/SM), each looping over row tiles;
//   * TMA bulk staging: one elected thread issues `cp.async.bulk.shared::cluster.global` per input
//     column per tile into a CB_STAGES-deep shared-memory ring, completion via mbarrier tx-count;
//     rows are then read from shared memory, so HBM traffic is exactly one read of every input
//     column and bytes-in-flight do not cost registers;
//   * aggregation: thread-private partial aggregates (registers for the ungrouped case, a
//     bank-conflict-free shared-memory slice per thread for <= a few dozen groups), 64-bit fast
//     path with an exact 128-bit escape, then a fixed-order intra-CTA tree and per-CTA partials in
//     global memory merged by a finalize kernel => exact integer results, deterministic floats;
//   * selection: warp-ballot + popc prefix for in-tile compaction and a decoupled look-back scan
//     over tile descriptors for the global output offsets (single pass, stable row order).
//
// Replaces (reference, all CPU): DataFusion FilterExec / ProjectionExec / AggregateExec as wired by
// native/core/src/execution/planner.rs:1230-1385 and the accumulators in
// native/spark-expr/src/agg_funcs/{sum_decimal,avg_decimal,avg,sum_int}.rs.
#ifndef CB_KERNELS_CUH
#define CB_KERNELS_CUH

namespace cb {

} // namespace cb
#include "cb_params.h"
namespace cb {

// ------------------------------------------------------------------------------------------------
// PTX wrappers: mbarrier + TMA 1-D bulk copy (SASS: UBLKCP / SYNCS)
// ------------------------------------------------------------------------------------------------
CB_D u32 smem_u32(const void* p) { return (u32)__cvta_generic_to_shared(p); }
CB_D void mbar_init(u64* bar, u32 count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
CB_D void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
CB_D void mbar_expect_tx(u64* bar, u32 bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
CB_D void mbar_wait(u64* bar, u32 parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "CB_WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra CB_DONE_%=;\n"
        "bra CB_WAIT_%=;\n"
        "CB_DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
CB_D void mbar_arrive(u64* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
CB_D u64 l2_evict_first_policy() {
    u64 pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
CB_D void tma_bulk_g2s(void* dst_smem, const void* src_gmem, u32 bytes, u64* bar, u64 policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}

// ------------------------------------------------------------------------------------------------
// staged tile view handed to the generated row program
// ------------------------------------------------------------------------------------------------
struct Tile {
    const u8* col[CB_MAX_COLS]; // shared-memory slabs of the current stage
    const u8* val[CB_MAX_COLS]; // shared-memory validity slabs (or nullptr)
};
template <typename T> CB_D T ld(const u8* slab, int r) { return reinterpret_cast<const T*>(slab)[r]; }
CB_D bool ldv(const u8* vslab, int r) { return (vslab[r >> 3] >> (r & 7)) & 1; }

CB_D void set_err(const PipeParams& p, int bit) { atomicOr(p.err, 1 << bit); }

} // namespace cb

// =================================================================================================
// The generated program supplies (see codegen.cpp):
//   CB_NCOLS, CB_COL_BYTES(c) (constexpr array cb_col_bytes[]), cb_col_has_val[],
//   CB_TILE, CB_STAGES, CB_THREADS,
//   and for the aggregate kernel: CB_WORDS (8-byte accumulator words per group), CB_G1 (ungrouped),
//   cb_word_kind(w) (0 = i64 sum w/ 128-bit escape, 1 = f64 double-double hi, 2 = dd lo,
//                   3 = i64 wrapping sum / count, 4 = min i64 key, 5 = max i64 key),
//   `cb_row_agg(const cb::Tile&, int r, i64 grow, Acc&)`  or
//   `cb_row_select(const cb::Tile&, int r, i64 grow, SelOut&) -> bool`.
// =================================================================================================

#if defined(CB_KERNEL_AGG) || defined(CB_KERNEL_SELECT)
namespace cb {

// bytes of one column slab in a stage (cb_col_bytes == 0: bit-packed booleans)
constexpr __host__ __device__ int slab_bytes(int c) {
    return ((cb_col_bytes(c) == 0 ? CB_TILE / 8 : CB_TILE * cb_col_bytes(c)) + 127) / 128 * 128;
}
constexpr __host__ __device__ int stage_bytes() {
    int b = 0;
    for (int c = 0; c < CB_NCOLS; c++) {
        b += slab_bytes(c);
        if (cb_col_has_val(c)) b += (CB_TILE / 8 + 127) / 128 * 128;
    }
    return b;
}

// Issue the bulk copies of one tile into one stage.  Called by a single thread.
CB_D void issue_tile(const PipeParams& p, int tile, u8* stage_base, u64* bar, u64 policy) {
    i64 row0 = (i64)tile * CB_TILE;
    i64 rem = p.n_rows - row0;
    int rows = rem < CB_TILE ? (int)rem : CB_TILE;
    u32 total = 0;
    u32 bytes_c[CB_NCOLS], bytes_v[CB_NCOLS];
#pragma unroll
    for (int c = 0; c < CB_NCOLS; c++) {
        bytes_c[c] = cb_col_bytes(c) == 0 ? (u32)((((rows + 7) >> 3) + 15) & ~15) : (u32)((rows * cb_col_bytes(c) + 15) & ~15);
        bytes_v[c] = cb_col_has_val(c) ? (u32)((((rows + 7) >> 3) + 15) & ~15) : 0u;
        total += bytes_c[c] + bytes_v[c];
    }
    mbar_expect_tx(bar, total);
    u8* dst = stage_base;
#pragma unroll
    for (int c = 0; c < CB_NCOLS; c++) {
        tma_bulk_g2s(dst, p.col[c] + (cb_col_bytes(c) == 0 ? (row0 >> 3) : row0 * cb_col_bytes(c)), bytes_c[c], bar, policy);
        dst += slab_bytes(c);
        if (cb_col_has_val(c)) {
            tma_bulk_g2s(dst, p.val[c] + (row0 >> 3), bytes_v[c], bar, policy);
            dst += (CB_TILE / 8 + 127) / 128 * 128;
        }
    }
}
CB_D void tile_view(u8* stage_base, Tile& t) {
    u8* ptr = stage_base;
#pragma unroll
    for (int c = 0; c < CB_NCOLS; c++) {
        t.col[c] = ptr;
        ptr += slab_bytes(c);
        if (cb_col_has_val(c)) { t.val[c] = ptr; ptr += (CB_TILE / 8 + 127) / 128 * 128; }
        else t.val[c] = nullptr;
    }
}

} // namespace cb
#endif

// =================================================================================================
// AGGREGATE kernel
// =================================================================================================
#ifdef CB_KERNEL_AGG
namespace cb {
struct Acc;
// dense / ungrouped: called for rows of the tile only.  hash: called by whole warps for every slot of the tile, `in_range` false
// for the slots past the last row (the warp-cooperative table update needs convergent lanes).
CB_D void cb_row_agg(const Tile& t, int r, i64 grow, const PipeParams& p, Acc& acc, bool in_range);

// Thread-private accumulator file.  Word (g, w) of thread t lives at acc[(g*CB_WORDS + w)*CB_THREADS + t]
// (8-byte words interleaved across threads => every warp access is bank-conflict-free no matter
// which group each lane updates).  For the ungrouped case the words are registers.
#ifndef CB_KEY_WORDS
#define CB_KEY_WORDS 1
#endif
#ifndef CB_HASH
#define CB_HASH 0
#endif
#define CB_EMPTY_KEY 0xffffffffffffffffull
#ifndef CB_STREAM
#define CB_STREAM 0
#endif
#ifndef CB_CAS_FIRST
#define CB_CAS_FIRST 0
#endif

#if CB_HASH
// ---- hash aggregation: accumulators live in a global open-addressing table, updated with atomics -------------
// The table is fed WARP-COOPERATIVELY.  Lanes of a warp hold 32 consecutive rows; rows with equal keys that sit next to each
// other (clustered inputs: ~4 lines per order in Config 4) form a RUN.  Per run, one lane -- its head -- probes the key table
// once and issues one atomic per accumulator word with the run's combined value (segmented shuffle reduction); the other lanes
// never touch the table.  Round 1 probed and issued 2-3 returning atomics per ROW and ran at < 5 % of the HBM roofline: the kernel
// was bound by L2 atomic throughput, not by the 24 bytes per row it streams.
//
// CB_STREAM (Partial aggregates over inputs whose equal keys sit next to each other -- the host samples that): no key table at
// all.  Every run becomes a NEW state row: its head draws a fresh id and STORES the run's combined words (the arrays need no
// zero-fill).  A key whose rows are split over several runs appears in several state rows; that is a valid Partial result (the
// Final stage merges state rows by key, as it does for the reference's own early-emitting partial aggregates), and it turns the
// partial stage from ~8 dependent random HBM round trips per group into a stream.
struct Acc {
    const PipeParams* p;
    u64 vm[2 * CB_NCOLS];
    // state of the current row iteration (begin() sets it)
    bool shared_g;  // CB_STREAM: g is the reserved NULL-key group, which other runs update too (atomics instead of stores)
    int g;          // group id (valid on head lanes)
    int run_end;    // last lane of this lane's run
    bool head, keep;
    CB_D void vm_or(int c, i128 raw) { u64 s = (u64)(raw.hi >> 63); vm[2 * c] |= raw.lo ^ s; vm[2 * c + 1] |= (u64)raw.hi ^ s; }
    CB_D void vm_or64(int c, i64 raw) { vm[2 * c] |= (u64)raw ^ (u64)(raw >> 63); }

    // slot s = 16 bytes {key or tag, gid}: one 128-bit L2 load answers "is it my key, and which group"
    CB_D int wait_gid(u32 s) const {
        int g_;
        while ((g_ = *((volatile i32*)&p->hkeys[2 * (size_t)s + 1])) < 0) {}
        return g_;
    }
    CB_D static u64 mix64(u64 h) { h ^= h >> 33; h *= 0xff51afd7ed558ccdull; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 33; return h; }
    CB_D static u64 key_tag(const u64* kw) { // CB_KEY_WORDS > 1: 64-bit tag of all key words, never the empty pattern
        u64 h = 0x9e3779b97f4a7c15ull;
#pragma unroll
        for (int i = 0; i < CB_KEY_WORDS; i++) {
            u64 x = mix64(kw[i] + h);
            h = (h << 5 | h >> 59) ^ x;
        }
        return h == CB_EMPTY_KEY ? 0ull : h;
    }
    CB_D bool same_key(int g_, const u64* kw) const {
        const u64* k = p->hkey_of_gid + (size_t)g_ * CB_KEY_WORDS;
        bool eq = true;
#pragma unroll
        for (int i = 0; i < CB_KEY_WORDS; i++) eq = eq && __ldcg(k + i) == kw[i];
        return eq;
    }

    // Fresh group ids for the lanes with `need` (warp-collective: every lane calls it).  One atomic per warp on the counter of the
    // warp's home id range; a full range sends the lanes that did not fit to the next one.  -1: every range is full.
    CB_D int alloc_gids(bool need) {
        const u32 lane = threadIdx.x & 31u;
        const int R = p->max_groups / CB_GID_RANGES;
        u32 r = (blockIdx.x * (CB_THREADS / 32) + (threadIdx.x >> 5)) % CB_GID_RANGES;
        int gn = -1;
        for (int tries = 0; tries < CB_GID_RANGES; tries++) {
            const u32 cm = __ballot_sync(0xffffffffu, need);
            if (!cm) break;
            const int leader = __ffs(cm) - 1;
            int base = 0;
            if ((int)lane == leader) base = atomicAdd(&p->hflags[CB_HFLAG_CTR + r], __popc(cm));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (need) {
                const int local = base + __popc(cm & ((1u << lane) - 1u));
                if (base >= 0 && local < R) { gn = (int)r * R + local; need = false; } // (a counter that ran past R stays there: the host clamps)
            }
            r = (r + 1u) % CB_GID_RANGES;
        }
        return gn;
    }

    // Group ids of the head lanes' keys, inserting new keys.  Called by the whole warp (convergent).
    //   probe   : linear probing from the key's home slot; a hit on a published slot resolves the lane, an empty slot is claimed
    //             with a CAS, a slot whose id is not published yet leaves the lane PENDING (no spinning here: the publisher may be
    //             a lane of this very warp that is waiting at the next step)
    //   claim   : the lanes that claimed a slot draw consecutive DENSE group ids with ONE atomic per warp, store the key words of
    //             their group and publish the id into the slot
    //   pending : now it is safe to wait for the other claimer's publication; wide keys compare the stored words and go on probing
    //             after a tag collision
    CB_D void resolve(const u64* kw, bool want, bool null_group) {
        const u32 lane = threadIdx.x & 31u, mask = p->hmask;
        g = 0;
        shared_g = false;
#if CB_STREAM
        {
            (void)mask;
            bool fresh = want;
            if (want && null_group) { g = p->max_groups + 1; shared_g = true; fresh = false; }
            (void)lane;
            if (__any_sync(0xffffffffu, fresh)) {
                int gn = alloc_gids(fresh);
                if (fresh) {
                    if (gn < 0) { atomicOr(p->hflags, CB_HF_FULL); gn = p->max_groups; shared_g = true; } // out of state rows: the host grows the arrays and repeats the launch
                    else {
#pragma unroll
                        for (int i = 0; i < CB_KEY_WORDS; i++) p->hkey_of_gid[(size_t)gn * CB_KEY_WORDS + i] = kw[i];
                    }
                    g = gn;
                }
            }
            return;
        }
#endif
        bool unresolved = want;
        if (want && null_group) { g = p->max_groups + 1; unresolved = false; }           // reserved group of the NULL key
        if (CB_KEY_WORDS == 1 && unresolved && kw[0] == CB_EMPTY_KEY) { atomicOr(p->hflags, CB_HF_SENTINEL); g = p->max_groups; unresolved = false; } // the key equal to the empty pattern
        const u64 tag = CB_KEY_WORDS == 1 ? kw[0] : key_tag(kw);
        u32 s = (CB_KEY_WORDS == 1 ? (u32)mix64(tag) : (u32)(tag ^ (tag >> 32))) & mask;
        u32 probes = 0;
        while (__any_sync(0xffffffffu, unresolved)) {
            bool claimed = false, pending = false;
            if (unresolved) {
                while (true) {
                    if (probes++ > mask) { atomicOr(p->hflags, CB_HF_FULL); g = p->max_groups; unresolved = false; break; } // table full: cannot happen (host sizes it)
#if CB_CAS_FIRST
                    // merging state rows: most keys are new, so claim first and look second -- one L2 / HBM round trip instead of two
                    ulonglong2 slot;
                    slot.x = atomicCAS((unsigned long long*)&p->hkeys[2 * (size_t)s], (unsigned long long)CB_EMPTY_KEY, (unsigned long long)tag);
                    if (slot.x == CB_EMPTY_KEY) { claimed = true; break; }
                    slot.y = slot.x == tag ? __ldcg(&p->hkeys[2 * (size_t)s + 1]) : 0ull;
#else
                    ulonglong2 slot = __ldcg(reinterpret_cast<const ulonglong2*>(p->hkeys) + s);
                    if (slot.x == CB_EMPTY_KEY) {
                        const u64 prev = atomicCAS((unsigned long long*)&p->hkeys[2 * (size_t)s], (unsigned long long)CB_EMPTY_KEY, (unsigned long long)tag);
                        if (prev == CB_EMPTY_KEY) { claimed = true; break; }
                        slot.x = prev;
                        slot.y = ~0ull; // somebody else just took it: its id may not be out yet
                    }
#endif
                    if (slot.x == tag) {
                        const int gs = (i32)(u32)slot.y;
                        if (gs < 0) { pending = true; break; }
                        if (CB_KEY_WORDS == 1 || gs >= p->max_groups || same_key(gs, kw)) { g = gs; unresolved = false; break; }
                    }
                    s = (s + 1u) & mask;
                }
            }
            (void)lane;
            if (__any_sync(0xffffffffu, claimed)) {
                int gn = alloc_gids(claimed);
                if (claimed) {
                    if (gn < 0) { atomicOr(p->hflags, CB_HF_FULL); gn = p->max_groups; } // cannot happen: host sizes max_groups >= rows
                    else {
#pragma unroll
                        for (int i = 0; i < CB_KEY_WORDS; i++) p->hkey_of_gid[(size_t)gn * CB_KEY_WORDS + i] = kw[i];
                    }
                    if (CB_KEY_WORDS > 1) __threadfence(); // readers of a wide key compare the stored words once they see the id; a one-word key IS the slot key
                    *((volatile i32*)&p->hkeys[2 * (size_t)s + 1]) = gn;
                    g = gn;
                    unresolved = false;
                }
            }
            if (pending) {
                const int gs = wait_gid(s);
                if (CB_KEY_WORDS > 1) __threadfence(); // the claimer's key words are visible once its id is
                if (CB_KEY_WORDS == 1 || gs >= p->max_groups || same_key(gs, kw)) { g = gs; unresolved = false; }
                else s = (s + 1u) & mask; // tag collision: keep probing
            }
        }
    }

    // start of a row iteration: run structure of the warp's 32 rows + group ids of the run heads
    CB_D void begin(bool keep_, const u64* kw, bool null_group) {
        const u32 lane = threadIdx.x & 31u;
        keep = keep_;
        bool same_prev = lane != 0;
#pragma unroll
        for (int i = 0; i < CB_KEY_WORDS; i++) {
            const u64 up = __shfl_up_sync(0xffffffffu, kw[i], 1); // every lane shuffles: `a && shfl()` would let lane 0 skip the collective
            same_prev = same_prev & (up == kw[i]);
        }
        const bool prev_keep = __shfl_up_sync(0xffffffffu, (int)keep_, 1) != 0;
        const bool prev_null = __shfl_up_sync(0xffffffffu, (int)null_group, 1) != 0;
        head = keep_ && !(same_prev && prev_keep && prev_null == null_group);
        const u32 stops = __ballot_sync(0xffffffffu, head) | ~__ballot_sync(0xffffffffu, keep_); // a run ends before the next head / absent row
        const u32 above = lane == 31u ? 0u : (stops & ~((2u << lane) - 1u));
        run_end = above ? __ffs(above) - 2 : 31;
        resolve(kw, head, null_group);
    }

    CB_D u64* W(int w) const { return p->htotals + ((size_t)g * CB_WORDS + w) * 2; }
    CB_D void store2(int w, u64 a, u64 b) const { *reinterpret_cast<ulonglong2*>(W(w)) = make_ulonglong2(a, b); } // CB_STREAM: the run's word, written once
    CB_D bool in_run(int off) const { return (int)(threadIdx.x & 31u) + off <= run_end; }
    // count of rows of the run with `c`: no shuffles needed, the ballot has it
    CB_D void h_count(bool c, int w) {
        const u32 lane = threadIdx.x & 31u;
        const u32 m = __ballot_sync(0xffffffffu, keep && c);
        if (head) {
            const u32 run = (run_end == 31 ? 0xffffffffu : ((2u << run_end) - 1u)) & ~((1u << lane) - 1u);
            const int n = __popc(m & run);
            if (CB_STREAM && !shared_g) { store2(w, (u64)n, 0ull); return; }
            if (n) atomicAdd((unsigned long long*)W(w), (unsigned long long)n);
        }
    }
    CB_D void h_add_wrap(bool c, int w, i64 v) { // wrapping 64-bit sum (SumInt Legacy, merged counts)
        u64 x = (keep && c) ? (u64)v : 0ull;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) { const u64 o = __shfl_down_sync(0xffffffffu, x, off); if (in_run(off)) x += o; }
        if (CB_STREAM && head && !shared_g) { store2(w, x, 0ull); return; }
        if (head && x) atomicAdd((unsigned long long*)W(w), (unsigned long long)x);
    }
    CB_D void h_add_i128(bool c, int w, i128 v) { // exact 128-bit sum: (lo, hi) words with carry
        u64 lo = (keep && c) ? v.lo : 0ull;
        i64 hi = (keep && c) ? v.hi : 0;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const u64 olo = __shfl_down_sync(0xffffffffu, lo, off);
            const i64 ohi = __shfl_down_sync(0xffffffffu, hi, off);
            if (in_run(off)) { const u64 n = lo + olo; hi += ohi + (n < lo ? 1 : 0); lo = n; }
        }
        if (CB_STREAM && head && !shared_g) { store2(w, lo, (u64)hi); return; }
#ifdef CB_X_NOCARRY
        if (head && (lo | (u64)hi)) { u64* s = W(w); if (lo) atomicAdd((unsigned long long*)&s[0], (unsigned long long)lo); if (hi) atomicAdd((unsigned long long*)&s[1], (unsigned long long)hi); return; } // timing experiment
#endif
        if (head && (lo | (u64)hi)) {
            u64* s = W(w);
            u64 carry = 0;
            if (lo) { const u64 old = atomicAdd((unsigned long long*)&s[0], (unsigned long long)lo); carry = (old + lo) < old ? 1ull : 0ull; }
            const u64 h2 = (u64)hi + carry;
            if (h2) atomicAdd((unsigned long long*)&s[1], (unsigned long long)h2);
        }
    }
    CB_D void h_add_i64_wide(bool c, int w, i64 v) { h_add_i128(c, w, i128_from_i64(v)); }
    CB_D void h_add_f64(bool c, int w, double x) { // double-double: run partial in lane order, then one 128-bit CAS loop per run
        dd a;
        a.hi = (keep && c) ? x : 0.0;
        a.lo = 0.0;
        bool any = keep && c;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            dd o;
            o.hi = __shfl_down_sync(0xffffffffu, a.hi, off);
            o.lo = __shfl_down_sync(0xffffffffu, a.lo, off);
            const bool oany = __shfl_down_sync(0xffffffffu, (int)any, off) != 0;
            if (in_run(off) && oany) { if (any) dd_add_dd(a, o); else a = o; any = true; }
        }
        if (CB_STREAM && head && !shared_g) { store2(w, (u64)__double_as_longlong(any ? a.hi : 0.0), (u64)__double_as_longlong(any ? a.lo : 0.0)); return; }
        if (!(head && any)) return;
        u64* s = W(w);
        u64 o0 = __ldcg(&s[0]), o1 = __ldcg(&s[1]);
        while (true) {
            dd t;
            t.hi = __longlong_as_double((i64)o0);
            t.lo = __longlong_as_double((i64)o1);
            dd_add_dd(t, a);
            u64 n0 = (u64)__double_as_longlong(t.hi), n1 = (u64)__double_as_longlong(t.lo), r0, r1;
            asm volatile(
                "{\n"
                ".reg .b128 cmp, nv, res;\n"
                "mov.b128 cmp, {%3, %4};\n"
                "mov.b128 nv, {%5, %6};\n"
                "atom.relaxed.gpu.global.cas.b128 res, [%2], cmp, nv;\n"
                "mov.b128 {%0, %1}, res;\n"
                "}\n"
                : "=l"(r0), "=l"(r1)
                : "l"(s), "l"(o0), "l"(o1), "l"(n0), "l"(n1)
                : "memory");
            if (r0 == o0 && r1 == o1) return;
            o0 = r0; o1 = r1;
        }
    }
    CB_D void h_min(bool c, int w, i64 key) {
        i64 x = (keep && c) ? key : (i64)0x7fffffffffffffffll;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) { const i64 o = __shfl_down_sync(0xffffffffu, x, off); if (in_run(off) && o < x) x = o; }
        if (CB_STREAM && head && !shared_g) { store2(w, (u64)x, 0ull); return; }
        if (head && x != (i64)0x7fffffffffffffffll) atomicMin((long long*)W(w), (long long)x);
    }
    CB_D void h_max(bool c, int w, i64 key) {
        i64 x = (keep && c) ? key : (i64)0x8000000000000000ll;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) { const i64 o = __shfl_down_sync(0xffffffffu, x, off); if (in_run(off) && o > x) x = o; }
        if (CB_STREAM && head && !shared_g) { store2(w, (u64)x, 0ull); return; }
        if (head && x != (i64)0x8000000000000000ll) atomicMax((long long*)W(w), (long long)x);
    }
};
#else
struct Acc {
#if CB_G1
    u64 r[CB_WORDS];
#else
    u64* base; // shared memory, already offset by threadIdx.x
#endif
    const PipeParams* p;
    u64 vm[2 * CB_NCOLS]; // OR of (value ^ sign) per staged column: validates range assumptions, feeds the host certificate

    CB_D void vm_or(int c, i128 raw) { u64 s = (u64)(raw.hi >> 63); vm[2 * c] |= raw.lo ^ s; vm[2 * c + 1] |= (u64)raw.hi ^ s; }
    CB_D void vm_or64(int c, i64 raw) { vm[2 * c] |= (u64)raw ^ (u64)(raw >> 63); }

    CB_D u64& word(int g, int w) {
#if CB_G1
        (void)g;
        return r[w];
#else
        return base[(g * CB_WORDS + w) * CB_THREADS];
#endif
    }
    // exact escape: add a full 128-bit value to the global spill accumulator (rare path)
    CB_D void spill128(int g, int w, i128 v) {
        u64* s = p->spill + ((size_t)g * CB_WORDS + w) * 2;
        u64 old = atomicAdd((unsigned long long*)&s[0], (unsigned long long)v.lo);
        u64 carry = (old + v.lo) < old ? 1ull : 0ull;
        atomicAdd((unsigned long long*)&s[1], (unsigned long long)((u64)v.hi + carry));
    }
    // decimal / wide integer sum: 64-bit thread-private partial when |v| < 2^46, else exact escape
    CB_D void add_i128(int g, int w, i128 v) {
        i64 lo = (i64)v.lo;
        bool small = (v.hi == (lo >> 63)) && (lo < (1ll << 46)) && (lo > -(1ll << 46));
        if (small) word(g, w) += (u64)lo;
        else spill128(g, w, v);
    }
    CB_D void add_i64_wide(int g, int w, i64 v) { add_i128(g, w, i128_from_i64(v)); }
    CB_D void add_i64_wrap(int g, int w, i64 v) { word(g, w) += (u64)v; }          // SumInt Legacy, counts
    CB_D void add_f64(int g, int w, double x) {                                     // double-double in words w, w+1
        dd a;
        a.hi = __longlong_as_double((i64)word(g, w));
        a.lo = __longlong_as_double((i64)word(g, w + 1));
        dd_add_double(a, x);
        word(g, w) = (u64)__double_as_longlong(a.hi);
        word(g, w + 1) = (u64)__double_as_longlong(a.lo);
    }
    CB_D void min_i64(int g, int w, i64 key) { i64 c = (i64)word(g, w); if (key < c) word(g, w) = (u64)key; }
    CB_D void max_i64(int g, int w, i64 key) { i64 c = (i64)word(g, w); if (key > c) word(g, w) = (u64)key; }
};

#endif // CB_HASH

CB_D u64 acc_identity(int kind) {
    switch (kind) {
    case 4: return 0x7fffffffffffffffull; // min
    case 5: return 0x8000000000000000ull; // max
    default: return 0ull;
    }
}

// combine two partial words of the same kind (used in the intra-CTA tree)
struct Pair128 { u64 a, b; };
CB_D Pair128 shfl_xor_pair(Pair128 v, int m) {
    Pair128 r;
    r.a = __shfl_xor_sync(0xffffffffu, v.a, m);
    r.b = __shfl_xor_sync(0xffffffffu, v.b, m);
    return r;
}

CB_D void consumer_bar() { asm volatile("bar.sync 1, %0;" ::"n"(CB_THREADS) : "memory"); }

// CB_THREADS consumer threads + one producer warp.  The producer's elected lane keeps the CB_STAGES-deep
// ring full with TMA bulk copies (full[s]: tx-count mbarrier); each consumer warp releases a stage through
// empty[s] as soon as IT is done with it, so no CTA-wide barrier sits on the streaming path.
extern "C" __global__ void __launch_bounds__(CB_THREADS + 32, 1) cb_pipeline_agg(const __grid_constant__ PipeParams p) {
    extern __shared__ __align__(128) u8 smem[];
    constexpr int SB = stage_bytes();
    constexpr int NW = CB_THREADS / 32;
    u64* full = reinterpret_cast<u64*>(smem);                  // CB_STAGES mbarriers
    u64* empty = full + CB_STAGES;                             // CB_STAGES mbarriers
    u8* stages = smem + 128;
    u64* accmem = reinterpret_cast<u64*>(stages + (size_t)CB_STAGES * SB);
    const int tid = threadIdx.x;
    static_assert(2 * CB_STAGES * 8 <= 128, "barrier area");

    if (tid == 0) {
        for (int s = 0; s < CB_STAGES; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], NW); }
        mbar_fence_init();
    }
    __syncthreads();

    const int first = blockIdx.x, step = gridDim.x;
    const int my_tiles = first < p.n_tiles ? (p.n_tiles - first + step - 1) / step : 0;

    if (tid >= CB_THREADS) { // ---------------- producer warp ----------------
        if (tid == CB_THREADS) {
            const u64 policy = l2_evict_first_policy();
            for (int k = 0; k < my_tiles; k++) {
                const int s = k % CB_STAGES, u = k / CB_STAGES;
                if (u > 0) mbar_wait(&empty[s], (u32)((u - 1) & 1));
                issue_tile(p, first + k * step, stages + (size_t)s * SB, &full[s], policy);
            }
        }
        return;
    }

    Acc acc;
    acc.p = &p;
#pragma unroll
    for (int c = 0; c < 2 * CB_NCOLS; c++) acc.vm[c] = 0;
#if CB_HASH
    (void)accmem;
#elif CB_G1
#pragma unroll
    for (int w = 0; w < CB_WORDS; w++) acc.r[w] = acc_identity(cb_word_kind(w));
#else
    acc.base = accmem + tid;
    for (int g = 0; g < p.n_groups; g++)
        for (int w = 0; w < CB_WORDS; w++) acc.word(g, w) = acc_identity(cb_word_kind(w));
#endif

    for (int k = 0; k < my_tiles; k++) {
        const int s = k % CB_STAGES;
        mbar_wait(&full[s], (u32)((k / CB_STAGES) & 1));
        Tile t;
        tile_view(stages + (size_t)s * SB, t);
        const int tile = first + k * step;
        const i64 row0 = (i64)tile * CB_TILE;
        const i64 rem = p.n_rows - row0;
        const int rows = rem < CB_TILE ? (int)rem : CB_TILE;
#if CB_HASH
        static_assert(CB_TILE % CB_THREADS == 0, "hash tiles are whole warps");
#pragma unroll 2
        for (int r = tid; r < CB_TILE; r += CB_THREADS) cb_row_agg(t, r, row0 + r, p, acc, r < rows);
#else
#pragma unroll 2
        for (int r = tid; r < rows; r += CB_THREADS) cb_row_agg(t, r, row0 + r, p, acc, true);
#endif
        __syncwarp();
        if ((tid & 31) == 0) mbar_arrive(&empty[s]); // this warp is done with stage s
    }

    // ---- publish the value masks (warp OR-reduce, one atomic per warp and word) ----------------------
#pragma unroll
    for (int c = 0; c < 2 * CB_NCOLS; c++) {
        if (!cb_col_masked(c >> 1)) continue;
        u32 lo = __reduce_or_sync(0xffffffffu, (u32)acc.vm[c]), hi = __reduce_or_sync(0xffffffffu, (u32)(acc.vm[c] >> 32));
        u64 m = ((u64)hi << 32) | lo;
        if ((tid & 31) == 0 && m) atomicOr((unsigned long long*)&p.vmask[c], (unsigned long long)m);
    }

#if CB_HASH
    return; // the table is the running total: nothing to fold
#else
    // ---- fold thread-private partials into one per-CTA partial per (group, word) -------------------
    // fixed butterfly order inside a warp, fixed warp order across the CTA => deterministic.
    __shared__ Pair128 wred[NW];
    const int lane = tid & 31, wid = tid >> 5;
    const int ng = p.n_groups;
    u64* out = reinterpret_cast<u64*>(p.partials) + (size_t)blockIdx.x * ng * CB_WORDS * 2;
    for (int g = 0; g < ng; g++) {
#pragma unroll
        for (int w = 0; w < CB_WORDS; w++) {
            const int kind = cb_word_kind(w);
            if (kind == 2) continue; // dd lo handled with its hi word
            Pair128 v;
            u64 x = acc.word(g, w);
            if (kind == 0) { v.a = x; v.b = (u64)((i64)x >> 63); }              // sign-extend to 128
            else if (kind == 1) { v.a = x; v.b = acc.word(g, w + 1); }           // (hi, lo) doubles
            else { v.a = x; v.b = 0; }
#pragma unroll
            for (int m = 16; m >= 1; m >>= 1) {
                Pair128 o = shfl_xor_pair(v, m);
                if (kind == 0) { i128 s = i128_add(mk128(v.a, (i64)v.b), mk128(o.a, (i64)o.b)); v.a = s.lo; v.b = (u64)s.hi; }
                else if (kind == 1) {
                    // butterfly: both partners must compute the same value => order operands by lane
                    dd A, B;
                    bool lowfirst = (lane & m) == 0;
                    A.hi = __longlong_as_double((i64)(lowfirst ? v.a : o.a)); A.lo = __longlong_as_double((i64)(lowfirst ? v.b : o.b));
                    B.hi = __longlong_as_double((i64)(lowfirst ? o.a : v.a)); B.lo = __longlong_as_double((i64)(lowfirst ? o.b : v.b));
                    dd_add_dd(A, B);
                    v.a = (u64)__double_as_longlong(A.hi); v.b = (u64)__double_as_longlong(A.lo);
                }
                else if (kind == 3) v.a += o.a;
                else if (kind == 4) v.a = (u64)(((i64)o.a < (i64)v.a) ? (i64)o.a : (i64)v.a);
                else v.a = (u64)(((i64)o.a > (i64)v.a) ? (i64)o.a : (i64)v.a);
            }
            if (lane == 0) wred[wid] = v;
            consumer_bar();
            if (tid == 0) {
                Pair128 t = wred[0];
                for (int i = 1; i < NW; i++) {
                    Pair128 o = wred[i];
                    if (kind == 0) { i128 s = i128_add(mk128(t.a, (i64)t.b), mk128(o.a, (i64)o.b)); t.a = s.lo; t.b = (u64)s.hi; }
                    else if (kind == 1) {
                        dd A, B;
                        A.hi = __longlong_as_double((i64)t.a); A.lo = __longlong_as_double((i64)t.b);
                        B.hi = __longlong_as_double((i64)o.a); B.lo = __longlong_as_double((i64)o.b);
                        dd_add_dd(A, B);
                        t.a = (u64)__double_as_longlong(A.hi); t.b = (u64)__double_as_longlong(A.lo);
                    }
                    else if (kind == 3) t.a += o.a;
                    else if (kind == 4) t.a = (u64)(((i64)o.a < (i64)t.a) ? (i64)o.a : (i64)t.a);
                    else t.a = (u64)(((i64)o.a > (i64)t.a) ? (i64)o.a : (i64)t.a);
                }
                out[((size_t)g * CB_WORDS + w) * 2 + 0] = t.a;
                out[((size_t)g * CB_WORDS + w) * 2 + 1] = t.b;
            }
            consumer_bar();
        }
    }
#endif // !CB_HASH
}

} // namespace cb
#endif // CB_KERNEL_AGG


// =================================================================================================
// fold + finalize (aggregate pipelines): per-CTA partials -> running totals -> output columns
// =================================================================================================
#ifdef CB_KERNEL_AGG
namespace cb {


CB_D void set_err_raw(i32* err, int bit) { atomicOr(err, 1 << bit); }
CB_D i128 fin_i128(const u64* T, int w) { return mk128(T[w * 2], (i64)T[w * 2 + 1]); }
CB_D double fin_dd(const u64* T, int w) { return __longlong_as_double((i64)T[w * 2]); } // normalised: hi = round(hi + lo)
CB_D void fin_store_i128(const FinParams& fp, int c, int g, i128 v, bool valid) {
    reinterpret_cast<i128*>(fp.out[c])[g] = v; fp.outv[c][g] = valid ? 1 : 0;
}
CB_D void fin_store_i64(const FinParams& fp, int c, int g, i64 v, bool valid) {
    reinterpret_cast<i64*>(fp.out[c])[g] = v; fp.outv[c][g] = valid ? 1 : 0;
}
CB_D void fin_store_f64(const FinParams& fp, int c, int g, double v, bool valid) {
    reinterpret_cast<double*>(fp.out[c])[g] = v; fp.outv[c][g] = valid ? 1 : 0;
}
CB_D void fin_store_f32(const FinParams& fp, int c, int g, float v, bool valid) {
    reinterpret_cast<float*>(fp.out[c])[g] = v; fp.outv[c][g] = valid ? 1 : 0;
}
CB_D void fin_store_u8(const FinParams& fp, int c, int g, int v, bool valid) {
    fp.out[c][g] = (u8)v; fp.outv[c][g] = valid ? 1 : 0;
}
CB_D void fin_store_i32(const FinParams& fp, int c, int g, i32 v, bool valid, int width) {
    if (width == 4) reinterpret_cast<i32*>(fp.out[c])[g] = v;
    else if (width == 2) reinterpret_cast<short*>(fp.out[c])[g] = (short)v;
    else reinterpret_cast<signed char*>(fp.out[c])[g] = (signed char)v;
    fp.outv[c][g] = valid ? 1 : 0;
}

CB_D void cb_finalize_group(const FinParams& fp, int g, const u64* T);
#if CB_HASH
CB_D void cb_unpack_key(const FinParams& fp, int g, const u64* kw, bool null_group); // kw: CB_KEY_WORDS packed words

// non-zero identities (MIN / MAX words) for a fresh range of group ids; all-zero layouts use a memset instead
extern "C" __global__ void cb_hash_init(u64* totals, long long first, long long n) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    i += first;
#pragma unroll
    for (int w = 0; w < CB_WORDS; w++) { totals[(i * CB_WORDS + w) * 2] = acc_identity(cb_word_kind(w)); totals[(i * CB_WORDS + w) * 2 + 1] = 0; }
}
// re-insert every group's key into a fresh key table under its (possibly relocated) id; ids: see CB_GID_RANGES
extern "C" __global__ void cb_hash_rehash(const u64* key_of_gid, int range_rows, const i32* counters, u64* hkeys, u32 mask) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)range_rows * CB_GID_RANGES) return;
    const int r = (int)(idx / range_rows), l = (int)(idx % range_rows);
    if (l >= counters[r]) return;
    const int g = (int)idx;
#if CB_KEY_WORDS > 1
    u64 kw[CB_KEY_WORDS];
#pragma unroll
    for (int i = 0; i < CB_KEY_WORDS; i++) kw[i] = key_of_gid[(size_t)g * CB_KEY_WORDS + i];
    const u64 key = Acc::key_tag(kw); // distinct keys may share a tag: each takes its own slot
    u32 s = (u32)(key ^ (key >> 32)) & mask;
#else
    u64 key = key_of_gid[g];
    u32 s = (u32)Acc::mix64(key) & mask;
#endif
    while (true) {
        u64 prev = atomicCAS((unsigned long long*)&hkeys[2 * (size_t)s], (unsigned long long)CB_EMPTY_KEY, (unsigned long long)key);
        if (prev == CB_EMPTY_KEY) { *((i32*)&hkeys[2 * (size_t)s + 1]) = g; return; }
        s = (s + 1u) & mask;
    }
}
#endif

// one thread per (group, word): fixed CTA order => deterministic
extern "C" __global__ void cb_fold(const __grid_constant__ FinParams fp) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    int total = fp.n_groups * CB_WORDS;
    if (idx >= total) return;
    int w = idx % CB_WORDS;
    int kind = cb_word_kind(w);
    if (kind == 2) return;
    u64 a, b;
    if (fp.first) { a = acc_identity(kind); b = 0; if (kind == 0) b = 0; }
    else { a = fp.totals[idx * 2]; b = fp.totals[idx * 2 + 1]; }
    for (int c = 0; c < fp.n_ctas; c++) {
        const u64* P = fp.partials + ((size_t)c * total + idx) * 2;
        u64 pa = P[0], pb = P[1];
        if (kind == 0) { i128 s = i128_add(mk128(a, (i64)b), mk128(pa, (i64)pb)); a = s.lo; b = (u64)s.hi; }
        else if (kind == 1) {
            dd A, B;
            A.hi = __longlong_as_double((i64)a); A.lo = __longlong_as_double((i64)b);
            B.hi = __longlong_as_double((i64)pa); B.lo = __longlong_as_double((i64)pb);
            dd_add_dd(A, B);
            a = (u64)__double_as_longlong(A.hi); b = (u64)__double_as_longlong(A.lo);
        }
        else if (kind == 3) a += pa;
        else if (kind == 4) a = (u64)(((i64)pa < (i64)a) ? (i64)pa : (i64)a);
        else a = (u64)(((i64)pa > (i64)a) ? (i64)pa : (i64)a);
    }
    if (kind == 0) {
        i128 s = i128_add(mk128(a, (i64)b), mk128(fp.spill[idx * 2], (i64)fp.spill[idx * 2 + 1]));
        a = s.lo; b = (u64)s.hi;
        fp.spill[idx * 2] = 0; fp.spill[idx * 2 + 1] = 0;
    }
    fp.totals[idx * 2] = a;
    fp.totals[idx * 2 + 1] = b;
}

extern "C" __global__ void cb_finalize(const __grid_constant__ FinParams fp) {
    int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= fp.n_groups) return;
    const u64* T = fp.totals + (size_t)g * CB_WORDS * 2;
#if CB_HASH
    // output row g: groups 0..n_hash_groups-1 in id order, then the reserved groups that were used
    int gid = g;
    bool is_sentinel = false, is_null_group = false;
    if (g < fp.n_hash_groups) { // the g-th id in (range, local) order
        int lo = 0, hi = CB_GID_RANGES - 1;
        while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (fp.gid_prefix[mid] <= g) lo = mid; else hi = mid - 1; }
        gid = lo * fp.gid_range + (g - fp.gid_prefix[lo]);
    }
    if (g >= fp.n_hash_groups) {
        int extra = g - fp.n_hash_groups;
        if (fp.sentinel_used && extra == 0) is_sentinel = true;
        else is_null_group = true;
        gid = is_sentinel ? fp.max_groups : fp.max_groups + 1;
    }
    const u64* TH = fp.totals + (size_t)gid * CB_WORDS * 2;
    fp.present[g] = 1;
    u64 kw[CB_KEY_WORDS];
#pragma unroll
    for (int i = 0; i < CB_KEY_WORDS; i++) kw[i] = (is_sentinel || is_null_group) ? (is_sentinel ? CB_EMPTY_KEY : 0ull) : fp.hkeys[(size_t)gid * CB_KEY_WORDS + i];
    cb_unpack_key(fp, g, kw, is_null_group);
    cb_finalize_group(fp, g, TH);
    return;
#else
    fp.present[g] = (i64)T[CB_W_ROWS * 2] > 0 ? 1 : 0;
#endif
    cb_finalize_group(fp, g, T);
}

} // namespace cb
#endif // CB_KERNEL_AGG (fold/finalize)

// =================================================================================================
// SELECT kernels: filter + project + stable compaction in two streaming passes
//
//   pass 1  cb_select_count   stages only the columns the predicates read; every warp owns a contiguous span of each
//                             tile and writes how many of its rows pass to sel_off[tile * NW + warp]
//   (scan)  k_scan_chunks / k_scan_totals (aot_kernels.cu): exclusive prefix sum of those counts
//   pass 2  cb_pipeline_select re-evaluates the predicate, evaluates the projections and writes every kept row at
//                             its final position (stable row order, like FilterExec)
//
// A single-pass compaction needs a tile's predecessors' totals before it can write (decoupled look-back); with one
// resident CTA per SM that wait sits on every tile's critical path and the first version ran at 10% of HBM peak.  Two
// passes cost a second read of the predicate columns (4 of 20..36 bytes per row in Config 1) and in exchange both are
// barrier-free streams with the same TMA ring / producer warp as the aggregate kernel.
// =================================================================================================
#ifdef CB_KERNEL_SELECT
namespace cb {

#ifndef CB_SEL_MASKED
#define CB_SEL_MASKED 0
#endif
#define CB_BAR_BYTES 256                     // up to 16 stages: narrow pipelines (pass 1 reads 4 bytes per row) need depth to keep enough bytes in flight
// Pass 1 stages CB_TILE rows at a time but counts per LOGICAL tile of CB_LTILE rows (= pass 2's CB_TILE): its rows are
// 4 bytes wide, and a 1024-row stage would leave each warp ~170 cycles per tile at HBM speed -- less than one
// barrier wait + release costs.
#ifndef CB_LTILE
#define CB_LTILE CB_TILE
#endif
constexpr int SEL_NW = CB_THREADS / 32;      // consumer warps
constexpr int SEL_RPW = CB_LTILE / SEL_NW;   // contiguous rows of a logical tile owned by one warp
constexpr int SEL_ROUNDS = SEL_RPW / 32;
constexpr int SEL_SUB = CB_TILE / CB_LTILE;  // logical tiles per stage
static_assert(CB_LTILE % (SEL_NW * 32) == 0 && CB_TILE % CB_LTILE == 0, "tile must be a multiple of 32 rows per warp");

// barriers + producer warp shared by both passes; returns false for the producer warp (which is done)
#define CB_SELECT_PROLOGUE()                                                                                          \
    extern __shared__ __align__(128) u8 smem[];                                                                       \
    constexpr int SB = stage_bytes();                                                                                 \
    u64* full = reinterpret_cast<u64*>(smem);                                                                         \
    u64* empty = full + CB_STAGES;                                                                                    \
    u8* stages = smem + CB_BAR_BYTES;                                                                                 \
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;                                                     \
    static_assert(2 * CB_STAGES * 8 <= CB_BAR_BYTES, "barrier area");                                                 \
    if (tid == 0) {                                                                                                   \
        for (int s = 0; s < CB_STAGES; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], SEL_NW); }                 \
        mbar_fence_init();                                                                                            \
    }                                                                                                                 \
    __syncthreads();                                                                                                  \
    const int first = blockIdx.x, step = gridDim.x;                                                                   \
    const int my_tiles = first < p.n_tiles ? (p.n_tiles - first + step - 1) / step : 0;                               \
    if (tid >= CB_THREADS) {                                                                                          \
        if (tid == CB_THREADS) {                                                                                      \
            const u64 policy = l2_evict_first_policy();                                                               \
            for (int k = 0; k < my_tiles; k++) {                                                                      \
                const int s = k % CB_STAGES, u = k / CB_STAGES;                                                       \
                if (u > 0) mbar_wait(&empty[s], (u32)((u - 1) & 1));                                                  \
                issue_tile(p, first + k * step, stages + (size_t)s * SB, &full[s], policy);                           \
            }                                                                                                         \
        }                                                                                                             \
        return;                                                                                                       \
    }

#ifdef CB_SELECT_COUNT
CB_D bool cb_row_keep(const Tile& t, int r, i64 grow, const PipeParams& p);

extern "C" __global__ void __launch_bounds__(CB_THREADS + 32, 1) cb_select_count(const __grid_constant__ PipeParams p) {
    CB_SELECT_PROLOGUE()
    for (int k = 0; k < my_tiles; k++) {
        const int s = k % CB_STAGES;
        mbar_wait(&full[s], (u32)((k / CB_STAGES) & 1));
        Tile t;
        tile_view(stages + (size_t)s * SB, t);
        const int tile = first + k * step;
        const i64 row0 = (i64)tile * CB_TILE;
        const i64 rem = p.n_rows - row0;
        const int rows = rem < CB_TILE ? (int)rem : CB_TILE;
        int cnt[SEL_SUB];
#pragma unroll
        for (int sub = 0; sub < SEL_SUB; sub++) {
            cnt[sub] = 0;
            u32 mine = 0; // lane q keeps the keep-mask of round q: the SEL_ROUNDS words of (logical tile, warp) leave as one coalesced store
#pragma unroll
            for (int q = 0; q < SEL_ROUNDS; q++) {
                const int r = sub * CB_LTILE + wid * SEL_RPW + q * 32 + lane;
                const bool keep = r < rows ? cb_row_keep(t, r, row0 + r, p) : false;
                const u32 bal = __ballot_sync(0xffffffffu, keep);
                cnt[sub] += __popc(bal);
                if (lane == q) mine = bal;
            }
            if (p.sel_mask && lane < SEL_ROUNDS && sub * CB_LTILE + wid * SEL_RPW + lane * 32 < rows)
                p.sel_mask[((row0 + sub * CB_LTILE + wid * SEL_RPW) >> 5) + lane] = mine;
        }
        __syncwarp();
        if (lane == 0) {
            mbar_arrive(&empty[s]); // this warp is done with stage s
            const i64 n_ltiles = (p.n_rows + CB_LTILE - 1) / CB_LTILE;
#pragma unroll
            for (int sub = 0; sub < SEL_SUB; sub++) {
                const i64 lt = (i64)tile * SEL_SUB + sub;
                if (lt < n_ltiles) p.sel_off[(size_t)lt * SEL_NW + wid] = (u32)cnt[sub];
            }
        }
    }
}

#else // ---- pass 2 --------------------------------------------------------------------------------------------

struct SelOut {
    // filled by the generated program for one row: CB_NOUT values (raw 16-byte slots) + validity
    u64 v[CB_NOUT][2];
    bool valid[CB_NOUT];
};

CB_D bool cb_row_select(const Tile& t, int r, i64 grow, const PipeParams& p, SelOut& o);

CB_D void store_out(u8* base, int bytes, i64 idx, const u64* v) {
    if (bytes == 16) { reinterpret_cast<ulonglong2*>(base)[idx] = make_ulonglong2(v[0], v[1]); }
    else if (bytes == 8) reinterpret_cast<u64*>(base)[idx] = v[0];
    else if (bytes == 4) reinterpret_cast<u32*>(base)[idx] = (u32)v[0];
    else if (bytes == 2) reinterpret_cast<u16*>(base)[idx] = (u16)v[0];
    else base[idx] = (u8)v[0];
}

extern "C" __global__ void __launch_bounds__(CB_THREADS + 32, 1) cb_pipeline_select(const __grid_constant__ PipeParams p) {
    CB_SELECT_PROLOGUE()
    // where a warp's kept rows go: scanned pass-1 counts, or the row itself when nothing is filtered.  The two loads are
    // issued one tile ahead so their latency (longer than a tile's share of HBM time) overlaps the previous tile.
    // (the two halves stay separate registers until the tile is processed: adding them at load time would wait for them)
    // (prefetch distance TWO tiles: with one, 34 % of this kernel's stall samples sat on the register move that consumes the loads)
    struct Pre {
        u32 chunk, off;
#if CB_SEL_MASKED
        u32 mask[SEL_ROUNDS];
#endif
    };
    Pre pre1, pre2; // for the next tile / the one after it
    auto load_base = [&](int tile, Pre& o) {
        const size_t e = (size_t)tile * SEL_NW + wid;
        o.chunk = p.sel_chunk[e / CB_SCAN_CHUNK];
        o.off = p.sel_off[e];
#if CB_SEL_MASKED
        const u32* mw = p.sel_mask + ((((i64)tile * CB_TILE) + wid * SEL_RPW) >> 5); // the warp's rows of this tile: SEL_ROUNDS consecutive words
#pragma unroll
        for (int q = 0; q < SEL_ROUNDS; q++) o.mask[q] = __ldg(mw + q);
#endif
    };
    const bool filtered = p.sel_off != nullptr;
    pre1.chunk = pre1.off = pre2.chunk = pre2.off = 0;
#if CB_SEL_MASKED
#pragma unroll
    for (int q = 0; q < SEL_ROUNDS; q++) pre1.mask[q] = pre2.mask[q] = 0;
#endif
    if (filtered && my_tiles > 0) load_base(first, pre1);
    if (filtered && my_tiles > 1) load_base(first + step, pre2);
    // tile k reads its slot (loaded two tiles ago) and refills it for tile k + 2; even tiles use pre1, odd ones pre2 -- no register
    // ever waits for a load younger than two tiles
    auto process = [&](const int k, Pre& slot) {
        const int s = k % CB_STAGES;
        const Pre cur = slot;
        if (filtered && k + 2 < my_tiles) load_base(first + (k + 2) * step, slot);
        const u32 cur_chunk = cur.chunk, cur_off = cur.off;
        mbar_wait(&full[s], (u32)((k / CB_STAGES) & 1));
        Tile t;
        tile_view(stages + (size_t)s * SB, t);
        const int tile = first + k * step;
        const i64 row0 = (i64)tile * CB_TILE;
        const i64 rem = p.n_rows - row0;
        const int rows = rem < CB_TILE ? (int)rem : CB_TILE;
        i64 wbase = filtered ? (i64)cur_chunk + (i64)cur_off : row0 + (i64)wid * SEL_RPW;
#if CB_NOUT <= 4
#pragma unroll
#else
#pragma unroll 1
#endif
        for (int q = 0; q < SEL_ROUNDS; q++) {
            const int r = wid * SEL_RPW + q * 32 + lane;
            SelOut o;
#if CB_SEL_MASKED
            // pass 1 already decided: its keep bits are this round's ballot, and only kept rows run the projections
            const u32 bal = (wid * SEL_RPW + q * 32 < rows) ? cur.mask[q] : 0u; // words past the last row were never written
            const bool keep = r < rows && ((bal >> lane) & 1u) != 0;
            if (keep) (void)cb_row_select(t, r, row0 + r, p, o);
#else
            const bool keep = r < rows ? cb_row_select(t, r, row0 + r, p, o) : false;
            const u32 bal = __ballot_sync(0xffffffffu, keep);
#endif
            const int rank = __popc(bal & ((1u << lane) - 1u));
            if (keep) {
#pragma unroll
                for (int c = 0; c < CB_NOUT; c++) store_out(p.out[c], cb_out_bytes(c), wbase + rank, o.v[c]);
            }
#pragma unroll
            for (int c = 0; c < CB_NOUT; c++) {
                if (!cb_out_nullable(c)) continue;
                // the warp's kept rows occupy output bits [wbase, wbase + popc(bal)): compress the validity bits in
                // keep order (lane j's bit lands at its rank) and OR them into the zeroed bitmap
                u32 packed = __reduce_or_sync(0xffffffffu, (keep && o.valid[c]) ? (1u << rank) : 0u);
                if (lane == 0 && bal != 0) {
                    const u64 bits = (u64)packed << (wbase & 31);
                    if ((u32)bits) atomicOr(&p.out_valid[c][wbase >> 5], (u32)bits);
                    if ((bits >> 32) != 0) atomicOr(&p.out_valid[c][(wbase >> 5) + 1], (u32)(bits >> 32));
                }
            }
            wbase += __popc(bal);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]); // this warp is done with stage s
    };
    for (int k = 0; k < my_tiles; k += 2) {
        process(k, pre1);
        if (k + 1 < my_tiles) process(k + 1, pre2);
    }
}
#endif // CB_SELECT_COUNT

} // namespace cb
#endif // CB_KERNEL_SELECT

#endif // CB_KERNELS_CUH
