// CPU build of frizbee_b200/csrc/rank_plan.cuh for tests/test_rank_host.py: the chunk rules one by one, and the whole
// refinement of frz_attr_rank with the kernels' per-row steps (rank.cu) run in loops, std::sort in place of the LSD sort.
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../frizbee_b200/csrc/rank_plan.cuh"

namespace {
struct Bytes {
    const uint8_t* p;
    uint8_t operator()(int i) const { return p[i]; }
};
}  // namespace

extern "C" uint64_t h_rank_text_chunk(const uint8_t* text, uint32_t len, uint32_t off, uint32_t fold, uint32_t desc) {
    return frz_rank_text_chunk(Bytes{text}, len, off, fold != 0, desc != 0);
}
extern "C" uint64_t h_rank_attr_chunk(int64_t v, uint32_t desc) { return frz_rank_attr_chunk(v, desc != 0); }
extern "C" uint32_t h_rank_chunk_ends(uint64_t chunk, uint32_t text, uint32_t desc) { return frz_rank_chunk_ends(chunk, text != 0, desc != 0); }
extern "C" uint32_t h_rank_fold4(uint32_t x) { return frz_rank_fold4(x); }

// the sort key of a round as (hi, lo), and the digit shifts the LSD sort visits for the masks of a round's keys
extern "C" void h_rank_sort_key(uint32_t seg, uint64_t chunk, uint64_t* hi_lo) {
    const FrzOrderKey k = frz_rank_sort_key(seg, chunk);
    hi_lo[0] = k.hi;
    hi_lo[1] = k.lo;
}
extern "C" uint32_t h_rank_key_seg(uint64_t hi, uint64_t lo) { return frz_rank_key_seg(FrzOrderKey{hi, lo}); }
extern "C" uint32_t h_order_digits(uint64_t vary_hi, uint64_t vary_lo, uint32_t* shifts) { return frz_order_digits(vary_hi, vary_lo, shifts); }

// a and b: the texts padded with zeros to whole 16-byte units
extern "C" uint32_t h_rank_common(const uint8_t* a, uint32_t len_a, const uint8_t* b, uint32_t len_b, uint32_t off, uint32_t fold) {
    const auto unit = [&](int t, uint32_t u, uint32_t* w) { memcpy(w, (t ? b : a) + 16 * u, 16); };
    return frz_rank_common(unit, len_a, len_b, off, fold != 0);
}

// The ranks of n rows under n_keys keys.  Key k: is_text[k]; values[k] (n values) or texts[k] with offs[k] (n + 1
// offsets); desc[k], fold[k].  ranked[i]: row i is ranked.  out[i]: its rank or INT64_MIN.  Returns the rounds run.
extern "C" uint32_t h_rank(uint32_t n, uint32_t n_keys, const uint32_t* is_text, const uint32_t* desc, const uint32_t* fold,
                           const int64_t* const* values, const uint8_t* const* texts, const uint64_t* const* offs,
                           const uint8_t* ranked, int64_t* out) {
    // padded copies: the kernels read whole units
    std::vector<std::vector<std::vector<uint8_t>>> pad(n_keys);
    for (uint32_t k = 0; k < n_keys; k++) {
        if (!is_text[k]) continue;
        pad[k].resize(n);
        for (uint32_t i = 0; i < n; i++) {
            const uint64_t len = offs[k][i + 1] - offs[k][i];
            pad[k][i].assign((len + 15) / 16 * 16 + 16, 0);
            memcpy(pad[k][i].data(), texts[k] + offs[k][i], len);
        }
    }
    const auto len_of = [&](uint32_t k, uint32_t i) { return (uint32_t)(offs[k][i + 1] - offs[k][i]); };
    std::vector<uint32_t> seg_of(n, kFrzRankNone), at_row(n), skip(n), list;
    std::vector<uint32_t> seg_rep(n), seg_at(n);   // FrzRankDev::segs
    std::vector<FrzOrderKey> keys(n);
    std::vector<uint8_t> heads(n, 0);
    for (uint32_t i = 0; i < n; i++)   // k_rank_init
        if (ranked[i]) {
            if (list.empty()) { seg_rep[0] = i; seg_at[0] = frz_rank_at(0, 0); skip[0] = kFrzRankNone; }
            list.push_back(i);
            seg_of[i] = 0;
        }
    const uint32_t m = (uint32_t)list.size();
    uint32_t rounds = 0;
    while (!list.empty()) {
        rounds++;
        for (uint32_t row : list) {   // k_rank_skip
            const uint32_t s = seg_of[row], at = seg_at[s], k = frz_rank_at_key(at);
            if (!is_text[k] || row == seg_rep[s]) continue;
            const uint8_t* a = pad[k][row].data();
            const uint8_t* b = pad[k][seg_rep[s]].data();
            const auto unit = [&](int t, uint32_t u, uint32_t* w) { memcpy(w, (t ? b : a) + 16 * u, 16); };
            const uint32_t c = frz_rank_common(unit, len_of(k, row), len_of(k, seg_rep[s]), frz_rank_at_off(at), fold[k] != 0);
            skip[s] = std::min(skip[s], c);
        }
        for (uint32_t row : list) {   // k_rank_chunk
            const uint32_t s = seg_of[row];
            uint32_t at = seg_at[s];
            const uint32_t k = frz_rank_at_key(at);
            uint64_t chunk;
            if (is_text[k]) {
                if (skip[s] != kFrzRankNone) at += skip[s];
                chunk = frz_rank_text_chunk(Bytes{pad[k][row].data()}, len_of(k, row), frz_rank_at_off(at), fold[k] != 0, desc[k] != 0);
            } else {
                chunk = frz_rank_attr_chunk(values[k][row], desc[k] != 0);
            }
            keys[row] = frz_rank_sort_key(s, chunk);
            at_row[row] = at;
        }
        std::vector<uint32_t> sorted = list;   // the LSD sort: descending sort key
        std::stable_sort(sorted.begin(), sorted.end(), [&](uint32_t x, uint32_t y) { return frz_order_ahead(keys[x], keys[y]); });
        std::vector<uint32_t> next;
        const uint64_t c = sorted.size();
        for (uint64_t j = 0; j < c; j++) {   // k_rank_split
            const uint32_t row = sorted[j];
            const FrzOrderKey kk = keys[row];
            const uint32_t s = frz_rank_key_seg(kk);
            uint64_t parent = j, first = j;
            while (parent > 0 && frz_rank_key_seg(keys[sorted[parent - 1]]) == s) parent--;
            while (first > 0 && frz_rank_key_eq(keys[sorted[first - 1]], kk)) first--;
            const uint32_t seg = s + (uint32_t)(first - parent);
            const bool alone = first == j && (j + 1 == c || !frz_rank_key_eq(keys[sorted[j + 1]], kk));
            const uint32_t at = at_row[row], k = frz_rank_at_key(at);
            const uint64_t chunk = ~((kk.hi & 0xFFFFu) << 48 | kk.lo);
            uint32_t place = 0;
            const bool more = !alone && frz_rank_next(at, frz_rank_chunk_ends(chunk, is_text[k] != 0, desc[k] != 0), n_keys, &place);
            seg_of[row] = seg;
            if (first == j) {
                if (more) { seg_rep[seg] = row; seg_at[seg] = place; skip[seg] = kFrzRankNone; }
                else heads[seg] = 1;
            }
            if (more) next.push_back(row);
        }
        list.swap(next);
    }
    std::vector<int64_t> before(m + 1, 0);   // k_rank_heads + the scan
    for (uint32_t p = 0; p < m; p++) before[p + 1] = before[p] + heads[p];
    for (uint32_t i = 0; i < n; i++) out[i] = seg_of[i] == kFrzRankNone ? INT64_MIN : before[seg_of[i]];
    return rounds;
}
