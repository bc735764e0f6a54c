// subset_match_plan.cuh — the bitmap fold of frz_subset_match (DESIGN.md §4.19).  Shared by the device kernel
// (subset_match.cu), the host call (host.cu) and the CPU build (tests/harness/subset_match_harness.cpp).
//
// Row i of the text corpus T is in frz_match_list_into(m, T, 0) exactly when it is live, every non-negated compiled
// pattern's length gate and prefilter accept it, and no negated pattern's do (src/matcher/algo.rs:85-100 pushes every
// prefiltered haystack; src/matcher/multi.rs:84-152 ANDs the patterns).  So the fill needs each pattern's prefilter
// survivor bitmap only, one bit per index (word w holds indices 32w .. 32w + 31, the layout of a subset's bits), and folds
// them word by word into the subset's bitmap:
//   the first step     bits = start & base & (indices below n), start being the first non-negated pattern's survivors,
//                      or T's live rows when every pattern is negated or there is none;
//   a non-negated one  bits &= survivors;
//   a negated one      bits &= ~survivors.
// The last step also writes each chunk's member count (kFrzWhereChunk indices), which the subset fills' common tail scans.
#pragma once
#include <stdint.h>

#include "frz_hd.cuh"
#include "where_plan.cuh"

#include <vector>

enum : uint32_t { kFrzFoldFirst = 0, kFrzFoldAnd = 1, kFrzFoldAndNot = 2 };

// One fold step on the device.
struct FrzSubsetFoldDev {
    const uint32_t* surv;        // the step's survivor bitmap; nullptr: T's live rows, read from slot_meta / slot_of
    const uint32_t* slot_meta;   // T's slot metadata and inverse permutation (surv == nullptr)
    const uint16_t* slot_of;
    const uint32_t* base;        // has_base (first step only): the base's bitmap over [0, n_base)
    uint32_t* bits;              // in/out: ceil(n / 32) words (may be `base`: each word is read, then written)
    uint32_t* chunk_count;       // out, the last step only (else nullptr): members per chunk of kFrzWhereChunk indices
    uint64_t n;                  // the subset's corpus's length
    uint64_t n_base;
    uint32_t has_base;
    uint32_t op;                 // kFrzFoldFirst, kFrzFoldAnd or kFrzFoldAndNot
};

// the bits of `word` whose indices are below n
FRZ_HD uint32_t frz_fold_below(uint64_t word, uint64_t n) {
    const uint64_t lo = word * 32;
    return lo >= n ? 0u : n - lo >= 32 ? 0xFFFFFFFFu : (1u << (uint32_t)(n - lo)) - 1u;
}

// the members of the base in `word` (all bits without a base; base_word is read only below n_base)
FRZ_HD uint32_t frz_fold_base(uint32_t has_base, uint32_t base_word, uint64_t word, uint64_t n_base) {
    return has_base ? base_word & frz_fold_below(word, n_base) : 0xFFFFFFFFu;
}

// one step of the fold on one word: cur is the word so far (not read by the first step), surv the step's survivors,
// base the base's members (frz_fold_base) and below the indices below n (frz_fold_below); both matter to the first
// step only, because every later step keeps a subset of its bits
FRZ_HD uint32_t frz_fold_word(uint32_t op, uint32_t cur, uint32_t surv, uint32_t base, uint32_t below) {
    if (op == kFrzFoldFirst) return surv & base & below;
    return op == kFrzFoldAnd ? cur & surv : cur & ~surv;
}

// One step of a fill: the compiled pattern whose survivors it folds (-1: T's live rows) and how.
struct FrzSubsetMatchStep {
    int32_t pattern;
    uint32_t op;
};

// (host) The steps for compiled patterns with these negation flags, in the multi-pattern loop's order: the first
// non-negated pattern (else T's live rows) starts, then every other pattern in its order.  No pattern: the live rows.
inline std::vector<FrzSubsetMatchStep> frz_subset_match_steps(const std::vector<bool>& negated) {
    std::vector<FrzSubsetMatchStep> steps;
    int32_t first = -1;
    for (size_t i = 0; i < negated.size() && first < 0; i++)
        if (!negated[i]) first = (int32_t)i;
    steps.push_back(FrzSubsetMatchStep{first, kFrzFoldFirst});
    for (size_t i = 0; i < negated.size(); i++)
        if ((int32_t)i != first) steps.push_back(FrzSubsetMatchStep{(int32_t)i, negated[i] ? kFrzFoldAndNot : kFrzFoldAnd});
    return steps;
}

// (host) Whether step k's prefilter reads T's slot metadata masked to the rows that can still be members
// (k_subset_meta) rather than T's own.  Every step after the first is masked by the members so far: their number is on
// the device only, and the masked form measured faster at every density tried, while a mask pass that removes nothing
// costs about 5 % of a prefilter step.  The first step is masked by the base when there is one and it leaves
// rows out (base_members < n).  DESIGN.md §4.19 has the measurements.
FRZ_HD bool frz_subset_match_masked(uint32_t step, bool has_base, uint64_t base_members, uint64_t n) {
    return step > 0 || (has_base && base_members < n);
}
