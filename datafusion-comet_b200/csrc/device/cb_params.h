// cb_params.h -- kernel parameter blocks shared by the device skeletons (cb_kernels.cuh) and the host
// executor (exec.cpp, agg.cpp).  Plain structs over the cb_math.h typedefs so both sides agree on layout.
#ifndef CB_PARAMS_H
#define CB_PARAMS_H
#include "cb_math.h"
namespace cb {

// pipeline kernels (filled by exec.cpp / agg.cpp; passed __grid_constant__)
#define CB_MAX_COLS 24
#define CB_MAX_OUT 24
#define CB_MAX_KEYS 4

#define CB_SCAN_CHUNK 4096
#define CB_MAX_STR_PREDS 8  // distinct string predicates one pipeline evaluates

// a string predicate's value per dictionary code: bit c & 31 of word c >> 5, for codes [0, n_entries) (see exec_internal.h StrMasks)
struct StrMask {
    const u32* bits;
    i32 n_entries;
};

struct PipeParams {
    const u8* col[CB_MAX_COLS];      // input column value buffers (16-byte aligned, padded)
    const u8* val[CB_MAX_COLS];      // validity bitmaps (LSB order) or nullptr
    i64 n_rows;
    i32 n_tiles;
    i32 n_groups;                    // dense aggregate: number of group slots (>=1)
    i32 key_card[CB_MAX_KEYS];       // dense aggregate: cardinality of each key (incl. null slot)
    u8* out[CB_MAX_OUT];             // select: output value buffers
    u32* out_valid[CB_MAX_OUT];      // select: output validity bitmap words (zeroed) or nullptr
    // select (two passes): pass 1 writes the rows each (tile, warp) keeps into sel_off[tile * NW + warp]; an exclusive
    // scan over chunks of CB_SCAN_CHUNK entries turns it into output offsets (sel_off: within the chunk, sel_chunk:
    // of the chunk); pass 2 writes the kept rows at sel_chunk[e / CB_SCAN_CHUNK] + sel_off[e].  nullptr = keep all.
    u32* sel_off;
    u32* sel_chunk;
    u32* sel_mask;                   // select: keep bit of every row (bit r & 31 of word r >> 5), written by pass 1, read by pass 2 when it is
                                     //         compiled CB_SEL_MASKED (then pass 2 neither stages nor re-evaluates the predicate columns)
    i64* out_count;                  // select: total rows kept
    u8* partials;                    // agg: per-CTA partial slots [grid][n_groups][CB_WORDS] x 16 B
    u64* spill;                      // agg: exact 128-bit escape accumulators [n_groups][CB_WORDS][2]
    i32* err;                        // error flags (bit 0: arithmetic overflow, bit1: ansi error...)
    u64* vmask;                      // agg: per staged column OR of (value ^ sign) over valid rows [CB_MAX_COLS][2] (lo, hi)
    // hash aggregation.  Key table in HBM: 16-byte slots {packed 64-bit key (all-ones = empty), dense group id handed out
    // at claim time (-1 until published)}.  Accumulators are DENSE by group id: htotals[gid][CB_WORDS][2],
    // hkey_of_gid[gid]; ids max_groups / max_groups+1 are reserved for the key equal to the empty pattern and for the
    // NULL key of a single nullable 64-bit key column.
    u64* hkeys;                      // [cap][2]: {packed key, group id in the low 32 bits (all-ones = not published)}
    u64* hkey_of_gid;
    u64* htotals;
    u32 hmask;                       // cap - 1 (cap is a power of two)
    i32 max_groups;
    i32* hflags;                     // [0] bit 0: sentinel key seen, bit 1: out of group ids / table full, bit 2: key does not fit
                                     //     the 64-bit packing, bit 3: NULL-key group used;
                                     // [CB_HFLAG_CTR + r], r < CB_GID_RANGES: group ids handed out in id range r (see below)
    StrMask smask[CB_MAX_STR_PREDS]; // string predicates, in the order codegen.h str_preds_of lists them
};
// Group ids come from CB_GID_RANGES independent counters, not one: range r owns the ids [r * R, (r + 1) * R), R = max_groups /
// CB_GID_RANGES, and every warp draws from its home range (spilling to the next one when it is full).  One counter for the whole
// grid serialised in the L2 atomic unit: 29 % of the hash kernel's stall samples sat on its result.  Output row o of finalize is
// the o-th id in (range, local) order -- FinParams::gid_prefix maps it back.
#define CB_GID_RANGES 64
#define CB_HFLAG_CTR 16
#define CB_HFLAG_WORDS (CB_HFLAG_CTR + CB_GID_RANGES)
// hflags[0] bits
#define CB_HF_SENTINEL 1    // a key equal to the empty-slot pattern was seen (reserved group max_groups)
#define CB_HF_FULL 2        // out of group ids / key table full
#define CB_HF_WIDE_KEY 4    // a decimal(p > 18) key does not fit the 64-bit packing
#define CB_HF_NULL_GROUP 8  // the NULL-key group (reserved group max_groups + 1) was used


// fold / finalize kernels of aggregate pipelines
struct FinParams {
    const u64* partials; // [n_ctas][n_groups][CB_WORDS][2]
    u64* spill;          // [n_groups][CB_WORDS][2]  (zeroed again after folding)
    u64* totals;         // [n_groups][CB_WORDS][2]
    i32 n_ctas, n_groups, first;
    u8* out[CB_MAX_OUT];   // finalize: value buffers, one element per group
    u8* outv[CB_MAX_OUT];  // finalize: validity, one byte per group
    u8* present;           // finalize: 1 if the group saw at least one row
    i32* err;
    const u64* hkeys;      // hash aggregation: hkey_of_gid (nullptr for dense aggregation); output row r < n_hash_groups is group r
    i32 n_hash_groups;     // hash aggregation: groups handed out; reserved groups follow as output rows when used
    i32 max_groups;
    i32 sentinel_used;     // hash aggregation: slot `cap` holds the key equal to the EMPTY sentinel
    i32 null_group_used;   // hash aggregation: slot `cap+1` holds the all-NULL key (single nullable 64-bit key)
    i32 gid_range;         // hash aggregation: ids per range (max_groups / CB_GID_RANGES)
    i32 gid_prefix[CB_GID_RANGES + 1]; // hash aggregation: output row of the first id of each range (exclusive prefix of the per-range counts)
    u64 cert_b[CB_MAX_OUT][2]; // per aggregate: bound (lo, hi) on the magnitude of any single addend of a decimal SUM / AVG, from the observed value
                               // masks through the range propagation (hi = ~0: unbounded); finalize turns it into a per-group certificate (cb::cert_level)
};

} // namespace cb
#endif
