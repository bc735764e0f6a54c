// CPU build of frizbee_b200/csrc/batch_plan.cuh for scoped and ranked queries: the per-query top-K of a batch sub-batch as
// k_batch_top<ScopedKey> (batch.cu) runs it, sequentially, through the header's own functions
// (tests/test_batch_scoped_host.py).
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../frizbee_b200/csrc/batch_plan.cuh"

struct M {
    uint32_t index;
    uint16_t score;
    uint8_t exact, pad;
};

// lists: the q index-ordered lists back to back (counts[j] each); by_score[j]: the query's strategy orders by score.
// scoped[j]: only members of the bitmap bits[j] over [0, n_bits[j]) are rows; ranked[j]: the rows are ordered by
// clamp(score + boost[j][index], 0, 65535) (boost 0 at and past n_boost[j]) under every strategy.
// Query j's first min(k, members) rows → out[j * k ...], their number → n_out[j], the members' count → n_total[j].
extern "C" void h_batch_scoped_top(const M* lists, const uint64_t* counts, const uint8_t* by_score, const uint8_t* scoped,
                                   const uint32_t* const* bits, const uint64_t* n_bits, const uint8_t* ranked,
                                   const int16_t* const* boost, const uint32_t* n_boost, uint64_t q, uint64_t k, M* out,
                                   uint64_t* n_out, uint64_t* n_total) {
    const M* list = lists;
    for (uint64_t j = 0; j < q; list += counts[j], j++) {
        const uint64_t n_list = counts[j];
        auto member = [&](const M& m) { return !scoped[j] || frz_batch_member(bits[j], n_bits[j], m.index); };
        auto value = [&](const M& m) -> uint32_t {
            if (!ranked[j]) return m.score;
            return frz_batch_ranked_value(m.score, m.index < n_boost[j] ? (int32_t)boost[j][m.index] : 0);
        };
        uint64_t total = 0;
        for (uint64_t i = 0; i < n_list; i++) total += member(list[i]);
        n_total[j] = total;
        const uint64_t rows = frz_batch_rows(k, total);
        n_out[j] = rows;
        M* o = out + frz_batch_row0(j, k);
        if (rows == 0) continue;
        if (!ranked[j] && !by_score[j]) {   // the members' head
            uint64_t kept = 0;
            for (uint64_t i = 0; i < n_list && kept < rows; i++)
                if (member(list[i])) o[kept++] = list[i];
            continue;
        }
        uint32_t hist[kFrzBatchBins] = {};
        for (uint64_t i = 0; i < n_list; i++)
            if (member(list[i])) hist[value(list[i]) >> 8]++;
        uint64_t above_hi = 0;
        const int hb = frz_batch_cut_hi(hist, rows, &above_hi);
        memset(hist, 0, sizeof hist);
        for (uint64_t i = 0; i < n_list; i++)
            if (member(list[i]) && (value(list[i]) >> 8) == (uint32_t)hb) hist[value(list[i]) & 255]++;
        const FrzBatchCut cut = frz_batch_cut_lo(hist, hb, above_hi, rows);
        std::vector<uint64_t> keys;
        uint64_t eq = 0;
        for (uint64_t i = 0; i < n_list; i++) {
            if (!member(list[i])) continue;
            const uint32_t v = value(list[i]);
            if (frz_batch_keep(v, cut, eq)) keys.push_back(frz_batch_key(v, (uint32_t)i));
            eq += v == cut.threshold;
        }
        std::sort(keys.begin(), keys.end());
        for (uint64_t i = 0; i < rows && i < keys.size(); i++) o[i] = list[frz_batch_key_pos(keys[i])];
        if (keys.size() != rows) n_out[j] = ~0ull;   // the cut must keep exactly `rows` rows
    }
}
