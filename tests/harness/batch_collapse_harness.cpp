// CPU build of frizbee_b200/csrc/batch_collapse_plan.cuh: one sub-batch of the batched collapsed call as collapse.cu's
// k_batch_collapse_* kernels and batch.cu's k_batch_top<CollapsedKey> run it, sequentially, through the headers' own
// functions: slots and shared tables, the count pass over subset members, the rounds each query takes part in, and the
// keep rule (tests/test_batch_collapsed_host.py).
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../frizbee_b200/csrc/batch_collapse_plan.cuh"

struct M {
    uint32_t index;
    uint16_t score;
    uint8_t exact, pad;
};

extern "C" uint64_t h_record_bytes() { return sizeof(FrzBatchCollapse); }
extern "C" uint64_t h_collapse_bytes(uint64_t n_groups_max, uint64_t list_rows) { return frz_batch_collapse_bytes(n_groups_max, list_rows); }
extern "C" uint64_t h_collapse_fit(uint64_t budget, uint64_t base, uint64_t n_groups_max, uint64_t list_rows) {
    return frz_batch_collapse_fit(budget, base, n_groups_max, list_rows);
}
extern "C" uint32_t h_rounds(uint64_t per_group) { return frz_batch_collapse_rounds(per_group); }

// Query j: list[j] (n[j] rows, index-ordered, reversed for the *_DESC strategies), groups ids[j] (nullptr: none) over
// n_ids[j] indices, per_group[j] as the call takes it (1..32 or UINT64_MAX), order[j] (FrzCollapseOrder), boost[j] over
// n_boost[j] indices, subset bits[j] over n_bits[j] indices (nullptr: every row).  Writes keep[j][i] (the row is one of
// the query's rows) and, for the queries with wants[j], their counts as one prefix of the count tables into counts_back.
// Returns the slots read back, or UINT32_MAX when a round table is not zero after the rounds.
extern "C" uint32_t h_batch_collapse(uint32_t ns, const M* const* list, const uint64_t* n, const uint32_t* const* ids, const uint64_t* n_ids,
                                     const uint64_t* per_group, const uint8_t* order, const uint8_t* reversed, const int16_t* const* boost,
                                     const uint64_t* n_boost, const uint32_t* const* bits, const uint64_t* n_bits, const uint8_t* wants,
                                     uint64_t n_groups_max, uint8_t* const* keep, uint32_t* counts_back) {
    std::vector<uint8_t> grouped(ns), want(ns);
    std::vector<uint32_t> slot(ns);
    for (uint32_t j = 0; j < ns; j++) {
        grouped[j] = ids[j] != nullptr;
        want[j] = grouped[j] && wants[j];
    }
    const uint32_t n_back = frz_batch_collapse_slots(grouped.data(), want.data(), ns, slot.data());
    std::vector<FrzBatchCollapse> c(ns);
    uint32_t rounds = 0;
    for (uint32_t j = 0; j < ns; j++) {
        c[j] = FrzBatchCollapse();
        if (!grouped[j]) continue;
        c[j].ids = ids[j];
        c[j].n_ids = n_ids[j];
        c[j].per_group = per_group[j] == UINT64_MAX ? 0xFFFFFFFFu : (uint32_t)per_group[j];
        c[j].order = order[j];
        c[j].table = frz_batch_collapse_table(slot[j], n_groups_max);
        rounds = std::max(rounds, frz_batch_collapse_rounds(per_group[j]));
    }
    std::vector<uint32_t> counts(ns * n_groups_max, 0);
    std::vector<uint64_t> best(ns * n_groups_max, 0);
    std::vector<std::vector<uint8_t>> taken(ns);
    auto group = [&](uint32_t j, uint64_t i) {
        const uint32_t x = list[j][i].index;
        if (bits[j] && !frz_batch_member(bits[j], n_bits[j], x)) return kFrzGroupNone;
        return frz_collapse_group(c[j].ids, c[j].n_ids, x);
    };
    auto entry = [&](uint32_t j, uint64_t i) {
        const M& r = list[j][i];
        const int32_t b = c[j].order == FRZ_COLLAPSE_BY_KEY && r.index < n_boost[j] ? boost[j][r.index] : 0;
        return frz_collapse_entry(frz_collapse_key(c[j].order, reversed[j] != 0, r.score, b, r.index));
    };
    for (uint32_t j = 0; j < ns; j++) {   // the count pass
        if (!grouped[j]) continue;
        taken[j].assign(n[j], 0);
        for (uint64_t i = 0; i < n[j]; i++)
            if (group(j, i) != kFrzGroupNone) counts[c[j].table + group(j, i)]++;
    }
    for (uint32_t r = 0; r < rounds; r++) {
        for (uint32_t j = 0; j < ns; j++) {
            if (!grouped[j] || !frz_batch_collapse_in_round(c[j].per_group, r)) continue;
            uint32_t* cnt = counts.data() + c[j].table;
            uint64_t* bst = best.data() + c[j].table;
            auto contends = [&](uint64_t i) {
                const uint32_t g = group(j, i);
                return g != kFrzGroupNone && frz_collapse_contends(g, cnt[g], c[j].per_group, taken[j][i] != 0);
            };
            for (uint64_t i = 0; i < n[j]; i++)   // the max pass
                if (contends(i)) bst[group(j, i)] = std::max(bst[group(j, i)], entry(j, i));
            for (uint64_t i = 0; i < n[j]; i++) {   // the take pass
                if (contends(i) && entry(j, i) == bst[group(j, i)]) {
                    taken[j][i] = 1;
                    bst[group(j, i)] = 0;
                }
            }
        }
    }
    for (uint64_t e : best)
        if (e) return UINT32_MAX;
    for (uint32_t j = 0; j < ns; j++) {   // k_batch_top<CollapsedKey>'s member()
        for (uint64_t i = 0; i < n[j]; i++) {
            const uint32_t x = list[j][i].index;
            bool in = !bits[j] || frz_batch_member(bits[j], n_bits[j], x);
            if (in && grouped[j]) {
                const uint32_t g = frz_collapse_group(c[j].ids, c[j].n_ids, x);
                in = frz_collapse_keep(g, g == kFrzGroupNone ? 0u : counts[c[j].table + g], c[j].per_group, taken[j][i] != 0);
            }
            keep[j][i] = in;
        }
    }
    memcpy(counts_back, counts.data(), n_back * n_groups_max * sizeof(uint32_t));
    return n_back;
}
