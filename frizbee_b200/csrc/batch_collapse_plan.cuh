// batch_collapse_plan.cuh — per-query arithmetic of the batched collapsed call (frz_match_list_batch_collapsed, DESIGN.md
// §4.11 "Collapsed queries").  Shared by the device kernels (collapse.cu, batch.cu: k_batch_top<CollapsedKey>), host.cu and
// a CPU build (tests/harness/batch_collapse_harness.cpp).
//
// A sub-batch with grouped queries holds, per query slot, a count table and a round table of G entries (G: the largest
// n_groups among the call's batched grouped queries) and one taken flag per list row.  A grouped query owns the tables of
// its slot: the queries that want their counts back take the first slots, so the counts they read back are one prefix of
// the count tables.  Query j takes part in the first rounds(per_group_j) of the sub-batch's max over its queries' rounds;
// the row rule itself (order key, contend and keep) is collapse_plan.cuh's, applied to the query's subset members only.
#pragma once
#include <stdint.h>

#include "collapse_plan.cuh"

#include "frz_hd.cuh"

// The groups of one query of a sub-batch, uploaded with its pattern (ids == nullptr: the query has no groups).
struct FrzBatchCollapse {
    const uint32_t* ids;   // group of index i < n_ids (frz_groups); indices past it are in no group
    uint64_t n_ids;
    uint64_t table;        // first entry of the query's count and round tables (frz_batch_collapse_table)
    uint32_t per_group;    // 1..32, or 0xFFFFFFFF: no cap
    uint8_t order;         // FrzCollapseOrder
    uint8_t pad[3];
};

// The rounds a query takes part in: per_group when capped, none without a cap (every count fits).
FRZ_HD uint32_t frz_batch_collapse_rounds(uint64_t per_group) {
    return per_group <= kFrzCollapseMaxPerGroup ? (uint32_t)per_group : 0u;
}
FRZ_HD bool frz_batch_collapse_in_round(uint32_t per_group, uint32_t round) { return round < frz_batch_collapse_rounds(per_group); }

// The first table entry of slot `slot` when every slot holds n_groups_max entries.
FRZ_HD uint64_t frz_batch_collapse_table(uint32_t slot, uint64_t n_groups_max) { return (uint64_t)slot * n_groups_max; }

// Device bytes a query slot adds to a sub-batch for tables of n_groups_max entries over lists of list_rows rows: a u32 count
// and a u64 round entry per group, a taken flag per row, and its record.  0 when no query of the call has groups.
FRZ_HD uint64_t frz_batch_collapse_bytes(uint64_t n_groups_max, uint64_t list_rows) {
    return n_groups_max ? n_groups_max * (sizeof(uint32_t) + sizeof(unsigned long long)) + list_rows + sizeof(FrzBatchCollapse) : 0;
}
// Queries per sub-batch within `budget` bytes, when a query needs base bytes without its groups (0: fewer than two fit, and
// the grouped queries run the single-query call).
FRZ_HD uint64_t frz_batch_collapse_fit(uint64_t budget, uint64_t base, uint64_t n_groups_max, uint64_t list_rows) {
    const uint64_t q = budget / (base + frz_batch_collapse_bytes(n_groups_max, list_rows));
    return q >= 2 ? q : 0;
}

// Slots of a sub-batch's ns queries: slot[j] for a grouped query, those with wants[j] first, both in query order; the
// slot of a query without groups is unused.  Returns the number of slots whose counts are read back.
FRZ_HD uint32_t frz_batch_collapse_slots(const uint8_t* grouped, const uint8_t* wants, uint32_t ns, uint32_t* slot) {
    uint32_t next = 0;
    for (uint32_t j = 0; j < ns; j++)
        if (grouped[j] && wants[j]) slot[j] = next++;
    const uint32_t n_back = next;
    for (uint32_t j = 0; j < ns; j++) {
        if (grouped[j] && !wants[j]) slot[j] = next++;
        else if (!grouped[j]) slot[j] = 0;
    }
    return n_back;
}
