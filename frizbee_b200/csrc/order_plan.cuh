// order_plan.cuh — the row rule of the ordered call (frz_match_list_ordered, DESIGN.md §4.15) and the pick step of its
// top-K select.  Shared by the device kernels (order.cu, and the LSD sort's OrderKey in sort.cu), the host call (host.cu)
// and a CPU build (tests/harness/order_harness.cpp).
//
// L0 is the list the call orders: the index-ordered list, reversed for the *_DESC strategies.  Each row carries a 112-bit
// order key whose descending unsigned order is the call's order, so every key is unique and no step resolves ties:
//   ATTR_DESC / ATTR_ASC                      [a : 64][r : 16][x : 32]
//   SCORE_THEN_ATTR_DESC / SCORE_THEN_ATTR_ASC [r : 16][a : 64][x : 32]
// where a is the attribute value mapped to an unsigned key (frz_order_attr_key: null is 0, below every value in both
// directions), r = clamp(score + boost[index], 0, 65535) (the raw score without a boost), and x = index under the *_DESC
// strategies, ~index otherwise (frz_collapse_key's rule), so equal a and r keep L0's order.  The key is stored as hi (the
// top 64 bits) and lo (the low 48 bits).
//
// The select narrows the list most-significant digit first, 8 bits per pass (digit shift s: bits [s, s + 8) of the key).
// A digit that is the same in every key of the list is skipped (frz_order_digits), so a tie-heavy attribute costs no pass
// over its constant bits.  Each pass histograms the digit over the remaining candidates and picks (frz_order_pick) the
// bucket that holds the need-th key: the buckets above it are selected, and the bucket becomes the next candidate set,
// unless it is taken whole.
#pragma once
#include <stdint.h>

#include "batch_plan.cuh"

#include "frz_hd.cuh"

// Orders (FRZ_ORDER_*): bit 0 set is ascending attribute order, orders from kFrzOrderScoreFirst on rank by r first.
constexpr uint32_t kFrzOrderScoreFirst = 2;   // FRZ_ORDER_SCORE_THEN_ATTR_DESC
constexpr uint32_t kFrzOrderCount = 4;
constexpr uint32_t kFrzOrderDigitBits = 8;
constexpr uint32_t kFrzOrderBins = 1u << kFrzOrderDigitBits;
constexpr uint32_t kFrzOrderKeyBits = 112;
constexpr uint32_t kFrzOrderMaxDigits = kFrzOrderKeyBits / kFrzOrderDigitBits;   // 14
// The one-block sort's capacity (order.cu): a selection of at most this many rows is sorted in shared memory.
constexpr uint32_t kFrzOrderBlockRows = 4096;

struct FrzOrderKey {
    uint64_t hi;   // key bits [48, 112)
    uint64_t lo;   // key bits [0, 48)
};

// The call's attribute, boost and order on the device.
struct FrzOrderDev {
    const int64_t* values;   // the attribute: values[i] for i < n_values; null past it
    const int16_t* boost;    // boost[i] for i < n_boost, 0 past it (n_boost == 0: no boost)
    uint64_t n_values;
    uint32_t n_boost;
    uint32_t order;          // FRZ_ORDER_*
    uint32_t reversed;       // 1: the *_DESC strategies (L0 is in descending index order)
    uint32_t pad_;
};

// Device state of one select (order.cu), zeroed before the key kernel.
struct FrzOrderState {
    unsigned long long n;            // the list's length
    unsigned long long vary_hi;      // bits that differ between keys: OR of the keys ... (these four words in this order)
    unsigned long long vary_lo;
    unsigned long long flip_hi;      // ... and OR of their complements (a bit varies where both are set)
    unsigned long long flip_lo;
    unsigned long long n_sel;        // rows selected so far (positions in the selection list)
    unsigned long long n_cand[2];    // candidates written by the passes of each parity
    unsigned long long need;         // rows still to select from the candidates
    unsigned int bucket;             // the last pick (frz_order_pick)
    unsigned int take;
    unsigned int finished;           // the selection is complete: later passes do nothing
    unsigned int done_blocks;        // last-block counter of a pass (self-resetting)
};

// The unsigned key of attribute value v: v ascending (asc) or descending maps to descending keys, and null (INT64_MIN)
// maps to 0 in both directions.  Every other value maps to 1 .. 2^64 - 1: INT64_MIN + 1 is 1 under DESC, INT64_MAX is 1
// under ASC.
FRZ_HD uint64_t frz_order_attr_key(int64_t v, bool asc) {
    const uint64_t u = (uint64_t)v;
    return asc ? (1ull << 63) - u : u ^ (1ull << 63);
}

// i's value in the attribute
FRZ_HD int64_t frz_order_value(const int64_t* values, uint64_t n_values, uint32_t index) {
    return index < n_values ? values[index] : (int64_t)(1ull << 63);
}

// The order key of a row from its parts (boost: boost[index], 0 without one; value: the attribute's value)
FRZ_HD FrzOrderKey frz_order_key(uint32_t order, bool reversed, uint32_t score, int32_t boost, uint32_t index, int64_t value) {
    const uint64_t r = frz_batch_ranked_value(score, boost);
    const uint64_t a = frz_order_attr_key(value, (order & 1u) != 0);
    const uint64_t x = reversed ? index : (uint32_t)~index;
    FrzOrderKey k;
    if (order < kFrzOrderScoreFirst) {
        k.hi = a;
        k.lo = r << 32 | x;
    } else {
        k.hi = r << 48 | a >> 16;
        k.lo = (a & 0xFFFFu) << 32 | x;
    }
    return k;
}

// The order key of the list row (index, score) under o
FRZ_HD FrzOrderKey frz_order_row_key(const FrzOrderDev& o, uint32_t index, uint32_t score) {
    const int32_t b = index < o.n_boost ? (int32_t)o.boost[index] : 0;
    return frz_order_key(o.order, o.reversed != 0, score, b, index, frz_order_value(o.values, o.n_values, index));
}

// a is ahead of b in the call's order
FRZ_HD bool frz_order_ahead(const FrzOrderKey& a, const FrzOrderKey& b) { return a.hi > b.hi || (a.hi == b.hi && a.lo > b.lo); }

// The digit of key bits [shift, shift + 8), shift a multiple of 8 below 112.
FRZ_HD uint32_t frz_order_digit(const FrzOrderKey& k, uint32_t shift) {
    return (uint32_t)((shift >= 48 ? k.hi >> (shift - 48) : k.lo >> shift) & (kFrzOrderBins - 1));
}

// The digit shifts the select visits, most significant first: those where some key bit varies (vary_*: the bits set in
// some key and clear in another).  Returns their number (<= kFrzOrderMaxDigits).  The LSD sort visits them in reverse.
FRZ_HD uint32_t frz_order_digits(uint64_t vary_hi, uint64_t vary_lo, uint32_t* shifts) {
    uint32_t n = 0;
    const FrzOrderKey v = {vary_hi, vary_lo};
    for (int32_t s = (int32_t)(kFrzOrderKeyBits - kFrzOrderDigitBits); s >= 0; s -= (int32_t)kFrzOrderDigitBits)
        if (frz_order_digit(v, (uint32_t)s)) shifts[n++] = (uint32_t)s;
    return n;
}

// The pick of one pass.  Candidates whose digit is above `bucket` are selected; those equal to it are selected too when
// `take`, else they are the next pass's candidates, of which need - above are still to select.
struct FrzOrderPick {
    uint32_t bucket;   // kFrzOrderBins: none (need == 0)
    uint32_t take;
    uint64_t above;    // candidates whose digit is above bucket
};

// hist: the pass's digit counts over the candidates (need <= their sum).  n_sel: rows selected before this pass.  fit: 0,
// or the capacity of a later sort that cuts the selection to its first `need` rows itself: the bucket is then taken whole
// as soon as the whole selection fits in it, so the select may stop above the need-th key.  Without fit the bucket is
// taken only when it completes the need exactly, and the select ends with exactly the need rows of largest key.
FRZ_HD FrzOrderPick frz_order_pick(const uint32_t* hist, uint64_t need, uint64_t n_sel, uint64_t fit) {
    FrzOrderPick p = {kFrzOrderBins, 1u, 0};
    if (need == 0) return p;
    uint32_t b = kFrzOrderBins - 1;
    while (b > 0 && p.above + hist[b] < need) p.above += hist[b--];
    p.bucket = b;
    const uint64_t through = p.above + hist[b];
    p.take = through == need || (fit && n_sel + through <= fit);
    return p;
}
