// CPU build of frizbee_b200/csrc/batch_columns_plan.cuh for tests/test_batch_columns_host.py: one query's join of a batched
// column call, run as the device runs it (batch_columns.cu) — the fold of every column in order, then the compaction.
#include <stdint.h>

#include <vector>

#include "../../frizbee_b200/csrc/batch_columns_plan.cuh"

// frz_match / FrzMatchDev
struct FrzMatchDev {
    uint32_t index;
    uint16_t score;
    uint8_t exact;
    uint8_t pad;
};

extern "C" {

uint64_t h_columns_bytes(uint64_t n_cols, uint64_t rows, uint64_t pattern_bytes) {
    return frz_batch_columns_bytes(n_cols, rows, pattern_bytes);
}

uint32_t h_fold(uint32_t acc, uint32_t pass, uint32_t score, uint32_t exact) { return frz_columns_fold(acc, pass, score, exact); }

// Column c: lists[c] (n_list[c] index-ordered records, those of the rows live in it) when has_pattern[c], else the rows
// with live[c][i] != 0 (live[c] == nullptr: no row removed, the column is not folded).  The query's matches → out, in
// index order or reversed; returns their number.
uint64_t h_join(uint64_t n, uint32_t n_cols, const FrzMatchDev* const* lists, const uint64_t* n_list, const uint8_t* const* live,
                const uint8_t* has_pattern, int reversed, FrzMatchDev* out) {
    std::vector<uint32_t> acc(n, 0);
    uint32_t need = 0;
    for (uint32_t c = 0; c < n_cols; c++) {
        FrzColumnFold f;
        f.pass = (uint8_t)need;
        f.slot = has_pattern[c] ? 0 : live[c] ? kFrzColumnLive : kFrzColumnSkip;
        if (f.slot == kFrzColumnSkip) continue;
        need++;
        if (f.slot == kFrzColumnLive) {
            for (uint64_t i = 0; i < n; i++)
                if (live[c][i]) acc[i] = frz_columns_fold(acc[i], f.pass, 0, 0);
        } else {
            for (uint64_t i = 0; i < n_list[c]; i++) {
                const FrzMatchDev& r = lists[c][i];
                acc[r.index] = frz_columns_fold(acc[r.index], f.pass, r.score, r.exact);
            }
        }
    }
    uint64_t total = 0;
    for (uint64_t i = 0; i < n; i++) total += frz_columns_matched(acc[i], need);
    uint64_t p = 0;
    for (uint64_t i = 0; i < n; i++) {
        if (!frz_columns_matched(acc[i], need)) continue;
        FrzMatchDev r;
        r.index = (uint32_t)i;
        r.score = (uint16_t)frz_columns_score(acc[i]);
        r.exact = (uint8_t)frz_columns_exact(acc[i]);
        r.pad = 0;
        out[frz_columns_pos(p++, total, reversed != 0)] = r;
    }
    return total;
}

}  // extern "C"
