// batch_columns_plan.cuh — per-row arithmetic of the batched column call (frz_match_list_batch_columns, DESIGN.md §4.13
// "Batched column calls").  Shared by the device kernels (batch_columns.cu), host.cu and a CPU build
// (tests/harness/batch_columns_harness.cpp).
//
// Each column of a sub-batch is scanned by the batched stages for the queries that have a pattern in it; every query's
// list for that column is then folded into the query's accumulator, one u32 per row:
//   bits  0..15  the saturating sum of the folded columns' scores
//   bit  16      the OR of their exact flags
//   bits 24..31  how many columns the row has matched so far
// The columns are folded in order and a list holds a row at most once, so fold p of a query (its p-th folded column)
// only extends rows that matched all p earlier ones.  A row is a match of the query when it matched every folded column
// (frz_columns_matched).  A column whose matcher has no pattern folds the rows that are live in it, with score 0, and is
// not folded at all when none of its rows was removed.  A row removed in a column never enters that column's list, so
// "matched every folded column" also means "live in every column": the rule k_keep<LiveInColumns> applies to the
// single-query call.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define FRZ_BK_HD __host__ __device__ __forceinline__
#else
#define FRZ_BK_HD inline
#endif

// Most columns a batched query folds (the matched count is 8 bits); a call with more columns runs the single-query call.
constexpr uint32_t kFrzBatchMaxColumns = 255;

// How query j of a sub-batch folds column c (uploaded with the patterns, [c][j]).
constexpr uint8_t kFrzColumnLive = 0xFE;   // no pattern: the rows live in the column
constexpr uint8_t kFrzColumnSkip = 0xFF;   // no pattern and no removed row: not folded
struct FrzColumnFold {
    uint8_t slot;   // the query's slot in the column's batched stages (< kFrzBatchMaxSub), or kFrzColumnLive / kFrzColumnSkip
    uint8_t pass;   // columns the query folds before this one
};

// The accumulator of a row after fold `pass` with a record of the column (score, exact).
FRZ_BK_HD uint32_t frz_columns_fold(uint32_t acc, uint32_t pass, uint32_t score, uint32_t exact) {
    if ((acc >> 24) != pass) return acc;   // it missed an earlier column
    const uint32_t s = (acc & 0xFFFFu) + score;
    return (pass + 1) << 24 | (acc & 0x10000u) | (exact ? 0x10000u : 0u) | (s > 0xFFFFu ? 0xFFFFu : s);
}
// A match of a query that folds `need` columns.
FRZ_BK_HD bool frz_columns_matched(uint32_t acc, uint32_t need) { return (acc >> 24) == need; }
FRZ_BK_HD uint32_t frz_columns_score(uint32_t acc) { return acc & 0xFFFFu; }
FRZ_BK_HD uint32_t frz_columns_exact(uint32_t acc) { return (acc >> 16) & 1u; }

// Position of the p-th match (index order) of a list of `total` matches, reversed under the *_DESC strategies.
FRZ_BK_HD uint64_t frz_columns_pos(uint64_t p, uint64_t total, bool reversed) { return reversed ? total - 1 - p : p; }

// Device bytes a query adds to a sub-batch for n_cols columns over lists of list_rows rows: its accumulator, its error
// word, the patterns of its further columns (pattern_bytes each), its fold records and its column count.
FRZ_BK_HD uint64_t frz_batch_columns_bytes(uint64_t n_cols, uint64_t list_rows, uint64_t pattern_bytes) {
    return list_rows * sizeof(uint32_t) + sizeof(uint32_t) + (n_cols - 1) * pattern_bytes + n_cols * sizeof(FrzColumnFold) + 1;
}
