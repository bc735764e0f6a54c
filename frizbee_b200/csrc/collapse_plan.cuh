// collapse_plan.cuh — the row rule of the collapsed call (frz_match_list_collapsed, DESIGN.md §4.12).  Shared by the
// device kernels (collapse.cu) and a CPU build (tests/harness/collapse_harness.cpp).
//
// L is the list the uncollapsed call returns (frz_match_list_ranked with the whole list, frz_match_list_subset or
// frz_match_list).  A row of L is kept when it is in no group, or when fewer than per_group earlier rows of L share its
// group.  The kernels see L before it is ordered (the index-ordered list, reversed for the *_DESC strategies), so each row
// carries an order key whose descending order is L's order:
//   high 32 bits  clamp(score + boost[index], 0, 65535) for a ranked call (frz_batch_ranked_value), else the score under
//                 a by-score strategy with a non-empty matcher, else 0;
//   low 32 bits   index under the *_DESC strategies, ~index otherwise.
// Keys are unique, so the first row of a group in L is the one with the largest key.  A group with at most per_group rows
// keeps them all.  An over-full group is resolved in per_group rounds: a round finds the largest key among the group's rows
// not yet taken (a max over the group's table entry) and takes that row.
#pragma once
#include <stdint.h>

#include "batch_plan.cuh"
#include "order_plan.cuh"

#if defined(__CUDACC__)
#define FRZ_CP_HD __host__ __device__ __forceinline__
#else
#define FRZ_CP_HD inline
#endif

constexpr uint32_t kFrzGroupNone = 0xFFFFFFFFu;            // FRZ_GROUP_NONE
constexpr uint64_t kFrzCollapseMaxPerGroup = 32;           // per_group above this (other than "no cap") is unsupported

// What the high half of the order key holds.
enum FrzCollapseOrder : uint8_t {
    FRZ_COLLAPSE_BY_INDEX = 0,   // index strategies, and the empty matcher unranked: 0
    FRZ_COLLAPSE_BY_SCORE = 1,   // by-score strategies with a non-empty matcher: the score
    FRZ_COLLAPSE_BY_KEY = 2,     // ranked calls: clamp(score + boost, 0, 65535)
};

// The group of a corpus index: ids[index] for index < n_ids, none past the array (rows appended after the handle).
FRZ_CP_HD uint32_t frz_collapse_group(const uint32_t* ids, uint64_t n_ids, uint32_t index) {
    return index < n_ids ? ids[index] : kFrzGroupNone;
}

// The order key of a row; boost is boost[index] (0 past the boost array), read only by FRZ_COLLAPSE_BY_KEY.
FRZ_CP_HD uint64_t frz_collapse_key(uint8_t order, bool reversed, uint32_t score, int32_t boost, uint32_t index) {
    const uint32_t primary = order == FRZ_COLLAPSE_BY_KEY ? frz_batch_ranked_value(score, boost)
                           : order == FRZ_COLLAPSE_BY_SCORE ? score : 0u;
    return (uint64_t)primary << 32 | (reversed ? index : ~index);
}

// A row of an over-full group not yet taken: it takes part in the next round.
FRZ_CP_HD bool frz_collapse_contends(uint32_t group, uint32_t count, uint32_t per_group, bool taken) {
    return group != kFrzGroupNone && count > per_group && !taken;
}

// The table entry a round's max is taken over: 0 is an empty entry, so a row's entry is its key + 1 (keys are below 2^48).
// The round's winner is the contender whose entry equals the max; it resets the entry to 0 for the next round, and a
// contender that reads the reset value cannot mistake itself for the winner.
FRZ_CP_HD uint64_t frz_collapse_entry(uint64_t key) { return key + 1; }

// The row is in C: no group, a group of at most per_group rows, or taken in a round.
FRZ_CP_HD bool frz_collapse_keep(uint32_t group, uint32_t count, uint32_t per_group, bool taken) {
    return group == kFrzGroupNone || count <= per_group || taken;
}

// Rounds on the order key (frz_match_list_ordered_collapsed and the ordered column call, DESIGN.md §4.15.1).  There L is the
// ordered call's list, so a row's key is its 112-bit FrzOrderKey (order_plan.cuh): unique, and the first row of a group in L
// is the one with the largest key.  The count pass and the keep rule above are unchanged; only a round differs.  The key
// does not fit one 64-bit atomic, and every value of hi is legitimate (INT64_MAX under ATTR_DESC is hi = 2^64 - 1), so
// hi + 1 could overflow.  A round takes the max in two steps over two tables, best_hi and best_lo, zero between rounds:
//   1. best_hi[group] = the largest hi among the group's contenders (frz_collapse_hi_entry);
//   2. best_lo[group] = the largest lo + 1 among the contenders whose hi equals best_hi (frz_collapse_lo_entry; the
//      others offer 0, which never raises the entry);
//   3. the contender whose lo + 1 equals best_lo is taken (frz_collapse_key_takes) and resets both entries to 0.
// Why this is safe:
//   - lo holds the index part x, so lo is unique within the list: the take test needs only best_lo.
//   - A contender that reads a reset best_lo cannot mistake itself for the winner: lo + 1 >= 1.
//   - A reset best_hi of 0 is right for the next round.  In round r < per_group an over-full group still has count - r >
//     per_group - r >= 1 contenders, so each max is over a non-empty set; a group whose contenders all have hi = 0 (null
//     attribute values under ATTR_*) keeps best_hi = 0, which step 2 matches.
//   - Every over-full group has one winner per round, which resets its entries, so both tables are zero after the rounds.
FRZ_CP_HD uint64_t frz_collapse_hi_entry(const FrzOrderKey& k) { return k.hi; }
FRZ_CP_HD uint64_t frz_collapse_lo_entry(const FrzOrderKey& k, uint64_t best_hi) { return k.hi == best_hi ? k.lo + 1 : 0; }
FRZ_CP_HD bool frz_collapse_key_takes(const FrzOrderKey& k, uint64_t best_lo) { return k.lo + 1 == best_lo; }
