// CPU build of frizbee_b200/csrc/collapse_plan.cuh: the order keys, and the count pass, rounds and keep rule of the
// collapsed call as collapse.cu and host.cu's CollapseKeep run them, sequentially, through the header's own functions
// (tests/test_collapsed_host.py).
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../frizbee_b200/csrc/collapse_plan.cuh"

struct M {
    uint32_t index;
    uint16_t score;
    uint8_t exact, pad;
};

static uint64_t row_key(const M& r, uint8_t order, uint8_t reversed, const int16_t* boost, uint64_t n_boost) {
    const int32_t b = order == FRZ_COLLAPSE_BY_KEY && r.index < n_boost ? boost[r.index] : 0;
    return frz_collapse_key(order, reversed != 0, r.score, b, r.index);
}

// keys[i] = the order key of list[i]
extern "C" void h_collapse_keys(const M* list, uint64_t n, uint8_t order, uint8_t reversed, const int16_t* boost, uint64_t n_boost,
                                uint64_t* keys) {
    for (uint64_t i = 0; i < n; i++) keys[i] = row_key(list[i], order, reversed, boost, n_boost);
}

// The collapse of the unordered list (index-ordered, reversed for the *_DESC strategies): counts[n_groups] and keep[n].
// per_group == 0 stands for no cap (no rounds, every row kept).
extern "C" void h_collapse(const M* list, uint64_t n, const uint32_t* ids, uint64_t n_ids, uint64_t n_groups, uint32_t per_group,
                           uint8_t order, uint8_t reversed, const int16_t* boost, uint64_t n_boost, uint8_t* keep, uint32_t* counts) {
    const uint32_t cap = per_group ? per_group : 0xFFFFFFFFu;
    std::vector<uint8_t> taken(n, 0);
    std::vector<uint64_t> best(n_groups, 0);
    memset(counts, 0, n_groups * sizeof(uint32_t));
    auto group = [&](uint64_t i) { return frz_collapse_group(ids, n_ids, list[i].index); };
    for (uint64_t i = 0; i < n; i++)
        if (group(i) != kFrzGroupNone) counts[group(i)]++;
    auto contends = [&](uint64_t i) {
        const uint32_t g = group(i);
        return g != kFrzGroupNone && frz_collapse_contends(g, counts[g], cap, taken[i] != 0);
    };
    for (uint32_t r = 0; per_group && r < per_group; r++) {
        for (uint64_t i = 0; i < n; i++) {   // the max pass
            if (!contends(i)) continue;
            const uint64_t e = frz_collapse_entry(row_key(list[i], order, reversed, boost, n_boost));
            if (e > best[group(i)]) best[group(i)] = e;
        }
        for (uint64_t i = 0; i < n; i++) {   // the take pass
            if (!contends(i)) continue;
            if (frz_collapse_entry(row_key(list[i], order, reversed, boost, n_boost)) == best[group(i)]) {
                taken[i] = 1;
                best[group(i)] = 0;
            }
        }
    }
    for (uint64_t j = 0; j < n_groups; j++)
        if (best[j]) counts[j] = 0xFFFFFFFFu;   // the table must be zero again after the rounds
    for (uint64_t i = 0; i < n; i++) {
        const uint32_t g = group(i);
        keep[i] = frz_collapse_keep(g, g == kFrzGroupNone ? 0u : counts[g], cap, taken[i] != 0);
    }
}
