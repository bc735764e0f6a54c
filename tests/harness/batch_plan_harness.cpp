// CPU build of frizbee_b200/csrc/batch_plan.cuh: the per-query top-K of a batch sub-batch as k_batch_top (batch.cu) runs
// it, sequentially, through the header's own functions (tests/test_batch_host.py).
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
// Query j's first min(k, counts[j]) rows → out[j * k ...], their number → n_out[j].
extern "C" void h_batch_top(const M* lists, const uint64_t* counts, const uint8_t* by_score, uint64_t q, uint64_t k, M* out,
                            uint64_t* n_out) {
    const M* list = lists;
    for (uint64_t j = 0; j < q; list += counts[j], j++) {
        const uint64_t total = counts[j];
        const uint64_t rows = frz_batch_rows(k, total);
        n_out[j] = rows;
        M* o = out + frz_batch_row0(j, k);
        if (rows == 0) continue;
        if (!by_score[j]) {
            memcpy(o, list, rows * sizeof(M));
            continue;
        }
        uint32_t hist[kFrzBatchBins] = {};
        for (uint64_t i = 0; i < total; i++) hist[list[i].score >> 8]++;
        uint64_t above_hi = 0;
        const int hb = frz_batch_cut_hi(hist, rows, &above_hi);
        memset(hist, 0, sizeof hist);
        for (uint64_t i = 0; i < total; i++)
            if ((list[i].score >> 8) == (uint32_t)hb) hist[list[i].score & 255]++;
        const FrzBatchCut cut = frz_batch_cut_lo(hist, hb, above_hi, rows);
        std::vector<uint64_t> keys;
        uint64_t eq = 0;
        for (uint64_t i = 0; i < total; i++) {
            const uint32_t s = list[i].score;
            if (frz_batch_keep(s, cut, eq)) keys.push_back(frz_batch_key(s, (uint32_t)i));
            eq += s == cut.threshold;
        }
        std::sort(keys.begin(), keys.end());
        for (uint64_t i = 0; i < rows && i < keys.size(); i++) o[i] = list[frz_batch_key_pos(keys[i])];
        if (keys.size() != rows) n_out[j] = ~0ull;   // the cut must keep exactly `rows` rows
    }
}
