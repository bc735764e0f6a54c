// batch_order_plan.cuh — per-query arithmetic of the batched ordered call's sub-batches (frz_match_list_batch_ordered,
// DESIGN.md §4.11 "Ordered queries").  Shared by the device kernels (order.cu: k_batch_order_*, collapse.cu:
// k_batch_collapse_*_key), host.cu and a CPU build (tests/harness/batch_order_harness.cpp).
//
// An ordered sub-batch holds only ordered queries.  Its stages up to the index-ordered lists are those of every sub-batch;
// then, per query slot j:
//   keys      the order key (order_plan.cuh) of each of its list rows, in list order: 16 bytes per list row;
//   cand      two candidate lists of list_stride positions.  The first starts as the query's rows (frz_batch_order_member:
//             the list rows in its subset and, with groups, kept by its collapse), and the select's passes ping-pong
//             between the two after that;
//   sel       the selection, kFrzOrderBlockRows positions (k <= kFrzBatchMaxK, so a selection always fits the block sort);
//   state     a FrzOrderState: n is the query's row count (its total), the masks are the OR of its rows' keys and of their
//             complements;
//   hist      the select's 256-bin histogram, zero between passes;
//   best_lo   with grouped queries, the second round table (collapse_plan.cuh's two-step max) of n_groups_max entries,
//             beside the existing best table; zero on allocation, and the rounds leave it zero.
// Pass p of the select handles the query's p-th varying digit (frz_batch_order_shift), so every query visits exactly its
// own varying digits, most significant first, and a query with fewer of them has finished before the later passes.
#pragma once
#include <stdint.h>

#include "batch_collapse_plan.cuh"
#include "order_plan.cuh"

#include "frz_hd.cuh"

// Launches of the select: one per digit a key can have, and the last one that ends every query's selection.
constexpr uint32_t kFrzBatchOrderPasses = kFrzOrderMaxDigits + 1;

// Slot offsets, in elements of each array
FRZ_HD uint64_t frz_batch_order_keys_at(uint32_t j, uint64_t list_stride) { return (uint64_t)j * list_stride; }
FRZ_HD uint64_t frz_batch_order_cand_at(uint32_t j, uint64_t list_stride) { return (uint64_t)j * 2 * list_stride; }
FRZ_HD uint64_t frz_batch_order_sel_at(uint32_t j) { return (uint64_t)j * kFrzOrderBlockRows; }
FRZ_HD uint64_t frz_batch_order_hist_at(uint32_t j) { return (uint64_t)j * kFrzOrderBins; }

// Device bytes an ordered query slot adds to a sub-batch over lists of list_rows rows: its FrzOrderDev record, its keys,
// its two candidate lists, the selection, the state, the histogram, and with grouped queries (n_groups_max > 0) a best_lo
// table.
FRZ_HD uint64_t frz_batch_order_bytes(uint64_t n_groups_max, uint64_t list_rows) {
    return sizeof(FrzOrderDev) + list_rows * (sizeof(FrzOrderKey) + 2 * sizeof(uint32_t)) + kFrzOrderBlockRows * sizeof(uint32_t) +
           sizeof(FrzOrderState) + kFrzOrderBins * sizeof(uint32_t) + n_groups_max * sizeof(unsigned long long);
}
// Queries per ordered sub-batch within `budget` bytes, when a query needs base bytes without its groups and ordering (0:
// fewer than two fit, and the ordered queries run the single-query call).
FRZ_HD uint64_t frz_batch_order_fit(uint64_t budget, uint64_t base, uint64_t n_groups_max, uint64_t list_rows) {
    const uint64_t q = budget / (base + frz_batch_collapse_bytes(n_groups_max, list_rows) + frz_batch_order_bytes(n_groups_max, list_rows));
    return q >= 2 ? q : 0;
}

// The varying bits of a query's rows: set in some key and clear in another (the state's OR masks).
FRZ_HD FrzOrderKey frz_batch_order_vary(const FrzOrderState& s) { return FrzOrderKey{s.vary_hi & s.flip_hi, s.vary_lo & s.flip_lo}; }

// The p-th varying digit of `vary`, most significant first: true and its shift in *shift when the query has more than p
// varying digits (frz_order_digits' p-th entry), false otherwise.
FRZ_HD bool frz_batch_order_shift(const FrzOrderKey& vary, uint32_t p, uint32_t* shift) {
    uint32_t n = 0;
    for (int32_t s = (int32_t)(kFrzOrderKeyBits - kFrzOrderDigitBits); s >= 0; s -= (int32_t)kFrzOrderDigitBits) {
        if (!frz_order_digit(vary, (uint32_t)s)) continue;
        if (n++ == p) {
            *shift = (uint32_t)s;
            return true;
        }
    }
    return false;
}

// The member rule: list row `index` is one of the query's rows when it is a member of its subset (bits == nullptr: no
// subset) and, for a grouped query (ids != nullptr), kept by its collapse (counts: its count table, taken: the row's flag).
// Non-members never enter the select: no key value can stand for "not a row", since an all-zero key is a legitimate row.
FRZ_HD bool frz_batch_order_member(const uint32_t* bits, uint64_t n_bits, const uint32_t* ids, uint64_t n_ids, const uint32_t* counts,
                                   uint32_t per_group, bool taken, uint32_t index) {
    if (bits && !frz_batch_member(bits, n_bits, index)) return false;
    if (!ids) return true;
    const uint32_t g = frz_collapse_group(ids, n_ids, index);
    return frz_collapse_keep(g, g == kFrzGroupNone ? 0u : counts[g], per_group, taken);
}

// The rows the block sort reads: every row of the query when they fit it (the select is skipped), else the selection.
FRZ_HD bool frz_batch_order_whole(uint64_t n_rows) { return n_rows <= kFrzOrderBlockRows; }
