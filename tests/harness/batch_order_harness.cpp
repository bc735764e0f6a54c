// CPU build of frizbee_b200/csrc/batch_order_plan.cuh: one ordered sub-batch of the batched ordered call as order.cu's
// k_batch_order_* kernels and collapse.cu's k_batch_collapse_*_key kernels run it, sequentially, through the headers' own
// functions: keys, slots and shared tables, the count pass over subset members, the rounds on the order key each query
// takes part in, the member rule, the select's passes (each query's p-th varying digit in pass p) and the block sort
// (tests/test_batch_ordered_host.py).
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../frizbee_b200/csrc/batch_order_plan.cuh"

struct M {
    uint32_t index;
    uint16_t score;
    uint8_t exact, pad;
};

extern "C" uint64_t h_sizes(uint32_t which) {
    return which == 0 ? sizeof(FrzOrderDev) : which == 1 ? sizeof(FrzOrderKey) : which == 2 ? sizeof(FrzOrderState) : kFrzBatchOrderPasses;
}
extern "C" uint64_t h_order_bytes(uint64_t n_groups_max, uint64_t list_rows) { return frz_batch_order_bytes(n_groups_max, list_rows); }
extern "C" uint64_t h_order_fit(uint64_t budget, uint64_t base, uint64_t n_groups_max, uint64_t list_rows) {
    return frz_batch_order_fit(budget, base, n_groups_max, list_rows);
}
// frz_batch_order_shift for p = 0, 1, ... while it finds a digit: the shifts → shifts, their number returned
extern "C" uint32_t h_shifts(uint64_t vary_hi, uint64_t vary_lo, uint32_t* shifts) {
    uint32_t p = 0;
    while (p < kFrzBatchOrderPasses && frz_batch_order_shift(FrzOrderKey{vary_hi, vary_lo}, p, &shifts[p])) p++;
    return p;
}
// frz_order_row_key's parts, for the test's own restatement of the varying digits
extern "C" void h_key(const M* row, const int64_t* values, uint64_t n_values, const int16_t* boost, uint32_t n_boost, uint32_t order,
                      int reversed, uint64_t* hi_lo) {
    FrzOrderDev o{};
    o.values = values;
    o.n_values = n_values;
    o.boost = boost;
    o.n_boost = n_boost;
    o.order = order;
    o.reversed = reversed != 0;
    const FrzOrderKey k = frz_order_row_key(o, row->index, row->score);
    hi_lo[0] = k.hi;
    hi_lo[1] = k.lo;
}

// Query j: list[j] (n[j] rows, index-ordered, reversed when reversed[j]), attribute values[j] over n_values[j] indices,
// boost[j] over n_boost[j] indices (nullptr: none), order[j], subset bits[j] over n_bits[j] indices (nullptr: every row),
// groups ids[j] (nullptr: none) over n_ids[j] indices with per_group[j] (1..32 or UINT64_MAX), counts wanted when
// wants[j].  Writes each query's first min(k, total) list positions in order to pos[j * k ..], its total to totals[j], the
// digit shifts its passes visited to visited[j * kFrzBatchOrderPasses ..] and their number to n_visited[j], and the counts
// of the queries that want them, as one prefix of the count tables, to counts_back.  Returns the slots read back, or
// UINT32_MAX when a round table is not zero after the rounds or a selection outgrows kFrzOrderBlockRows.
extern "C" uint32_t h_batch_order(uint32_t ns, uint64_t k, const M* const* list, const uint64_t* n, const uint8_t* reversed,
                                  const int64_t* const* values, const uint64_t* n_values, const int16_t* const* boost,
                                  const uint64_t* n_boost, const uint32_t* order, const uint32_t* const* bits, const uint64_t* n_bits,
                                  const uint32_t* const* ids, const uint64_t* n_ids, const uint64_t* per_group, const uint8_t* wants,
                                  uint64_t n_groups_max, uint32_t* pos, uint64_t* totals, uint32_t* visited, uint32_t* n_visited,
                                  uint32_t* counts_back) {
    std::vector<uint8_t> grouped(ns), want(ns);
    std::vector<uint32_t> slot(ns);
    for (uint32_t j = 0; j < ns; j++) {
        grouped[j] = ids[j] != nullptr;
        want[j] = grouped[j] && wants[j];
    }
    const uint32_t n_back = frz_batch_collapse_slots(grouped.data(), want.data(), ns, slot.data());
    std::vector<FrzBatchCollapse> c(ns);
    std::vector<FrzOrderDev> od(ns);
    std::vector<std::vector<FrzOrderKey>> keys(ns);
    uint32_t rounds = 0;
    for (uint32_t j = 0; j < ns; j++) {
        od[j] = FrzOrderDev();
        od[j].values = values[j];
        od[j].n_values = n_values[j];
        od[j].boost = boost[j];
        od[j].n_boost = boost[j] ? (uint32_t)n_boost[j] : 0;
        od[j].order = order[j];
        od[j].reversed = reversed[j];
        keys[j].resize(n[j]);
        for (uint64_t i = 0; i < n[j]; i++) keys[j][i] = frz_order_row_key(od[j], list[j][i].index, list[j][i].score);   // k_batch_order_keys
        c[j] = FrzBatchCollapse();
        if (!grouped[j]) continue;
        c[j].ids = ids[j];
        c[j].n_ids = n_ids[j];
        c[j].per_group = per_group[j] == UINT64_MAX ? 0xFFFFFFFFu : (uint32_t)per_group[j];
        c[j].table = frz_batch_collapse_table(slot[j], n_groups_max);
        rounds = std::max(rounds, frz_batch_collapse_rounds(per_group[j]));
    }
    std::vector<uint32_t> counts(ns * n_groups_max, 0);
    std::vector<uint64_t> best_hi(ns * n_groups_max, 0), best_lo(ns * n_groups_max, 0);
    std::vector<std::vector<uint8_t>> taken(ns);
    auto group = [&](uint32_t j, uint64_t i) {
        const uint32_t x = list[j][i].index;
        if (bits[j] && !frz_batch_member(bits[j], n_bits[j], x)) return kFrzGroupNone;
        return frz_collapse_group(c[j].ids, c[j].n_ids, x);
    };
    for (uint32_t j = 0; j < ns; j++) {   // k_batch_collapse_count
        taken[j].assign(n[j], 0);
        if (!grouped[j]) continue;
        for (uint64_t i = 0; i < n[j]; i++)
            if (group(j, i) != kFrzGroupNone) counts[c[j].table + group(j, i)]++;
    }
    for (uint32_t r = 0; r < rounds; r++) {
        for (uint32_t j = 0; j < ns; j++) {
            if (!grouped[j] || !frz_batch_collapse_in_round(c[j].per_group, r)) continue;
            uint32_t* cnt = counts.data() + c[j].table;
            uint64_t* bh = best_hi.data() + c[j].table;
            uint64_t* bl = best_lo.data() + c[j].table;
            auto contends = [&](uint64_t i) {
                const uint32_t g = group(j, i);
                return g != kFrzGroupNone && frz_collapse_contends(g, cnt[g], c[j].per_group, taken[j][i] != 0);
            };
            for (uint64_t i = 0; i < n[j]; i++)   // k_batch_collapse_max_hi
                if (contends(i)) bh[group(j, i)] = std::max(bh[group(j, i)], frz_collapse_hi_entry(keys[j][i]));
            for (uint64_t i = 0; i < n[j]; i++)   // k_batch_collapse_max_lo
                if (contends(i)) bl[group(j, i)] = std::max(bl[group(j, i)], frz_collapse_lo_entry(keys[j][i], bh[group(j, i)]));
            for (uint64_t i = 0; i < n[j]; i++) {   // k_batch_collapse_take_key
                if (contends(i) && frz_collapse_key_takes(keys[j][i], bl[group(j, i)])) {
                    taken[j][i] = 1;
                    bh[group(j, i)] = 0;
                    bl[group(j, i)] = 0;
                }
            }
        }
    }
    for (uint64_t e : best_hi)
        if (e) return UINT32_MAX;
    for (uint64_t e : best_lo)
        if (e) return UINT32_MAX;
    for (uint32_t j = 0; j < ns; j++) {
        // k_batch_order_members
        std::vector<uint32_t> rows;
        FrzOrderState st = FrzOrderState();
        const uint32_t* cnt = grouped[j] ? counts.data() + c[j].table : nullptr;
        for (uint64_t i = 0; i < n[j]; i++) {
            if (!frz_batch_order_member(bits[j], n_bits[j], c[j].ids, c[j].n_ids, cnt, c[j].per_group, grouped[j] && taken[j][i],
                                        list[j][i].index))
                continue;
            rows.push_back((uint32_t)i);
            const FrzOrderKey& kk = keys[j][i];
            st.vary_hi |= kk.hi;
            st.vary_lo |= kk.lo;
            st.flip_hi |= ~kk.hi;
            st.flip_lo |= ~kk.lo & ((1ull << 48) - 1);
        }
        st.n = rows.size();
        totals[j] = st.n;
        n_visited[j] = 0;
        // k_batch_order_pass, launches 0 .. kFrzBatchOrderPasses - 1
        std::vector<uint32_t> sel, cand = rows;
        const FrzOrderKey vary = frz_batch_order_vary(st);
        for (uint32_t p = 0; p < kFrzBatchOrderPasses && !st.finished && k && !frz_batch_order_whole(st.n); p++) {
            uint32_t prev = 0, cur = 0;
            if (p > 0 && !frz_batch_order_shift(vary, p - 1, &prev)) break;
            const bool has_digit = frz_batch_order_shift(vary, p, &cur);
            const bool first = p == 0;
            const uint32_t bucket = first ? 0u : st.bucket;
            const bool take = !first && st.take != 0;
            const bool count = has_digit && !take;
            const std::vector<uint32_t>& in = p <= 1 ? rows : cand;
            std::vector<uint32_t> next;
            uint32_t hist[kFrzOrderBins] = {};
            for (uint32_t x : in) {
                bool keep = true, selected = false;
                if (!first) {
                    const uint32_t d = frz_order_digit(keys[j][x], prev);
                    keep = d == bucket && !take;
                    selected = d > bucket || (d == bucket && take);
                }
                if (selected) sel.push_back(x);
                if (keep && count) {
                    next.push_back(x);
                    hist[frz_order_digit(keys[j][x], cur)]++;
                }
            }
            if (!count) {
                st.finished = 1;
                continue;
            }
            visited[j * kFrzBatchOrderPasses + n_visited[j]++] = cur;
            const uint64_t need = first ? std::min<uint64_t>(k, st.n) : st.need;
            const FrzOrderPick pk = frz_order_pick(hist, need, sel.size(), kFrzOrderBlockRows);
            st.bucket = pk.bucket;
            st.take = pk.take;
            st.need = need - pk.above;
            cand.swap(next);
        }
        // k_batch_order_sort
        if (!k) continue;
        std::vector<uint32_t> picked = frz_batch_order_whole(st.n) ? rows : sel;
        if (picked.size() > kFrzOrderBlockRows) return UINT32_MAX;
        std::sort(picked.begin(), picked.end(), [&](uint32_t a, uint32_t b) { return frz_order_ahead(keys[j][a], keys[j][b]); });
        const uint64_t m = frz_batch_rows(k, st.n);
        for (uint64_t r = 0; r < m; r++) pos[frz_batch_row0(j, k) + r] = picked[r];
    }
    memcpy(counts_back, counts.data(), n_back * n_groups_max * sizeof(uint32_t));
    return n_back;
}
