// CPU build of the rounds on the order key (frizbee_b200/csrc/collapse_plan.cuh's two-step max, with order_plan.cuh's keys)
// as collapse.cu's k_collapse_count / k_collapse_max_hi / k_collapse_max_lo / k_collapse_take_key and host.cu's
// CollapseKeep run them, through the headers' own functions (tests/test_ordered_collapsed_host.py).  Each pass visits the
// rows in a fresh random order, standing for any interleaving of the kernels' atomics.
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <numeric>
#include <random>
#include <vector>

#include "../../frizbee_b200/csrc/collapse_plan.cuh"

struct M {
    uint32_t index;
    uint16_t score;
    uint8_t exact, pad;
};

// The collapse of the list L0 (index-ordered, reversed for the *_DESC strategies) by the order key of
// (values, boost, order, reversed): counts[n_groups] and keep[n].  per_group == 0 stands for no cap.  Returns 1 when both
// round tables are zero after the rounds, 0 otherwise.
extern "C" int h_ordered_collapse(const M* list, uint64_t n, const int64_t* values, uint64_t n_values, const int16_t* boost,
                                  uint32_t n_boost, uint32_t order, int reversed, const uint32_t* ids, uint64_t n_ids,
                                  uint64_t n_groups, uint32_t per_group, uint64_t seed, uint8_t* keep, uint32_t* counts) {
    FrzOrderDev o{};
    o.values = values;
    o.n_values = n_values;
    o.boost = boost;
    o.n_boost = n_boost;
    o.order = order;
    o.reversed = reversed != 0;
    std::vector<FrzOrderKey> keys(n);   // k_order_keys
    for (uint64_t i = 0; i < n; i++) keys[i] = frz_order_row_key(o, list[i].index, list[i].score);
    const uint32_t cap = per_group ? per_group : 0xFFFFFFFFu;
    std::vector<uint8_t> taken(n, 0);
    std::vector<uint64_t> best_hi(n_groups, 0), best_lo(n_groups, 0);
    memset(counts, 0, n_groups * sizeof(uint32_t));
    auto group = [&](uint64_t i) { return frz_collapse_group(ids, n_ids, list[i].index); };
    for (uint64_t i = 0; i < n; i++)
        if (group(i) != kFrzGroupNone) counts[group(i)]++;
    auto contends = [&](uint64_t i) {
        const uint32_t g = group(i);
        return g != kFrzGroupNone && frz_collapse_contends(g, counts[g], cap, taken[i] != 0);
    };
    std::mt19937_64 rng(seed);
    std::vector<uint64_t> visit(n);
    std::iota(visit.begin(), visit.end(), 0);
    auto shuffled = [&]() -> const std::vector<uint64_t>& {
        std::shuffle(visit.begin(), visit.end(), rng);
        return visit;
    };
    for (uint32_t r = 0; per_group && r < per_group; r++) {
        for (uint64_t i : shuffled()) {   // k_collapse_max_hi
            if (!contends(i)) continue;
            const uint64_t e = frz_collapse_hi_entry(keys[i]);
            if (e > best_hi[group(i)]) best_hi[group(i)] = e;
        }
        for (uint64_t i : shuffled()) {   // k_collapse_max_lo
            if (!contends(i)) continue;
            const uint64_t e = frz_collapse_lo_entry(keys[i], best_hi[group(i)]);
            if (e > best_lo[group(i)]) best_lo[group(i)] = e;
        }
        for (uint64_t i : shuffled()) {   // k_collapse_take_key: a winner's reset is seen by the rows visited after it
            if (!contends(i)) continue;
            if (frz_collapse_key_takes(keys[i], best_lo[group(i)])) {
                taken[i] = 1;
                best_hi[group(i)] = 0;
                best_lo[group(i)] = 0;
            }
        }
    }
    for (uint64_t i = 0; i < n; i++) {   // CollapseKeep
        const uint32_t g = group(i);
        keep[i] = frz_collapse_keep(g, g == kFrzGroupNone ? 0u : counts[g], cap, taken[i] != 0);
    }
    for (uint64_t j = 0; j < n_groups; j++)
        if (best_hi[j] || best_lo[j]) return 0;
    return 1;
}
