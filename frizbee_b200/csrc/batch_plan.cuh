// batch_plan.cuh — per-query position arithmetic of the batched top-K call (frz_match_list_batch_top, DESIGN.md §4.11).
// Shared by the device kernel (batch.cu: k_batch_top) and a CPU build (tests/harness/batch_plan_harness.cpp).
//
// Query j of a sub-batch owns rows [j * k, j * k + rows) of the sub-batch's output, rows = min(k, total_j).  Its index-ordered
// list (already reversed for the *_DESC strategies, as the scoring kernels write it) becomes its first `rows` rows:
//   index-ordered strategies  the list's first `rows` entries;
//   score strategies          the list's stable sort by descending score, cut at `rows`.  The cut is found from two 256-bin
//                             histograms (high, then low score byte): the threshold score T, the rows above it, and how many
//                             rows scoring exactly T are kept (the first ones in list order).  The kept rows are then ordered
//                             by (descending score, list position), which is the stable sort's order.
//
// A scoped or ranked query (frz_match_list_batch) first drops the rows of its list that are not members of its subset
// (frz_batch_member); its total is the members' count.  It is then ordered as above on the value
//   v = ranked ? clamp(score + boost[index], 0, 65535) : score                       (frz_batch_ranked_value)
// and a ranked query is ordered by v under every strategy (the strategy's direction only orders ties, through the list).
// An index-ordered query that is not ranked keeps its first `rows` members in list order.
#pragma once
#include <stdint.h>

#include "frz_hd.cuh"

constexpr int kFrzBatchBins = 256;
// Largest k the batched device path serves: the kept rows of a query are sorted in one block's shared memory.
constexpr uint32_t kFrzBatchMaxK = 1024;

// a query's total when its survivor lists overflowed (a real total is at most 2^32 - 1)
constexpr uint64_t kFrzBatchOverflow = ~0ull;

FRZ_HD uint64_t frz_batch_rows(uint64_t k, uint64_t total) { return k < total ? k : total; }
FRZ_HD uint64_t frz_batch_row0(uint64_t j, uint64_t k) { return j * k; }

// The bin of a descending walk over hist[bins - 1 .. 0] that holds the want-th entry (1 <= want <= sum of hist), and in
// *above the entries of the bins above it.
FRZ_HD int frz_batch_select(const uint32_t* hist, int bins, uint64_t want, uint64_t* above) {
    uint64_t acc = 0;
    int b = bins - 1;
    for (; b > 0; b--) {
        if (acc + hist[b] >= want) break;
        acc += hist[b];
    }
    *above = acc;
    return b;
}

// The cut of a score-ordered query: rows with score > threshold are kept, and the first `eq_keep` rows (in list order)
// scoring exactly `threshold`.
struct FrzBatchCut {
    uint32_t threshold;
    uint64_t eq_keep;
};
// hi: histogram of score >> 8 over the list; lo: histogram of score & 255 over the rows whose high byte is the selected bin
// (the caller builds lo after frz_batch_cut_hi).  rows >= 1.
FRZ_HD int frz_batch_cut_hi(const uint32_t* hi, uint64_t rows, uint64_t* above_hi) {
    return frz_batch_select(hi, kFrzBatchBins, rows, above_hi);
}
FRZ_HD FrzBatchCut frz_batch_cut_lo(const uint32_t* lo, int hi_bin, uint64_t above_hi, uint64_t rows) {
    uint64_t above_lo = 0;
    const int lo_bin = frz_batch_select(lo, kFrzBatchBins, rows - above_hi, &above_lo);
    FrzBatchCut c;
    c.threshold = (uint32_t)hi_bin << 8 | (uint32_t)lo_bin;
    c.eq_keep = rows - above_hi - above_lo;
    return c;
}
// eq_before: rows scoring exactly the threshold that come before this one in the list
FRZ_HD bool frz_batch_keep(uint32_t score, const FrzBatchCut& c, uint64_t eq_before) {
    return score > c.threshold || (score == c.threshold && eq_before < c.eq_keep);
}
// Sort key of a kept row: ascending keys are the stable descending-score order.
FRZ_HD uint64_t frz_batch_key(uint32_t score, uint32_t list_pos) { return (uint64_t)(0xFFFFu - score) << 32 | list_pos; }
FRZ_HD uint32_t frz_batch_key_pos(uint64_t key) { return (uint32_t)key; }

// Membership of a row in a subset bitmap over the indices [0, n_bits) (frz_subset: rows appended after the subset was made
// lie past n_bits and are not members).
FRZ_HD bool frz_batch_member(const uint32_t* bits, uint64_t n_bits, uint32_t index) {
    return index < n_bits && (bits[index >> 5] >> (index & 31) & 1u);
}
// The ranked value of a row, in 32-bit arithmetic: boost is boost[index], or 0 for an index past the boost array.
FRZ_HD uint32_t frz_batch_ranked_value(uint32_t score, int32_t boost) {
    const int32_t v = (int32_t)score + boost;
    return v < 0 ? 0u : v > 0xFFFF ? 0xFFFFu : (uint32_t)v;
}
