// Host build of frizbee_b200/csrc/unicode_path.cuh (the code the GPU unicode kernel runs) + the host-side needle
// compilation of frizbee_b200/csrc/unicode_needle.h, exported for tests/test_unicode_device_code.py.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../frizbee_b200/csrc/unicode_needle.h"
#include "../../frizbee_b200/csrc/unicode_path.cuh"
#include "../../frizbee_b200/csrc/indices_path.cuh"

namespace {
struct Flat {
    const uint8_t* p;
    uint8_t operator()(int i) const { return p[i]; }
};
FrzUScoring scoring_of(const uint16_t* s9, bool u8) {
    // order of frz_scoring: match, mismatch, gap_open, gap_extend, prefix, cap, case, exact, delim
    auto sat_sub = [](uint32_t a, uint32_t b) { return a > b ? a - b : 0u; };
    auto sat_add = [](uint32_t a, uint32_t b) { return a + b > 0xffffu ? 0xffffu : a + b; };
    const uint32_t m = u8 ? 0xff : 0xffff;
    FrzUScoring sc;
    sc.gex = s9[3] & m; sc.gopx = sat_sub(s9[2], s9[3]) & m; sc.match_x = sat_add(s9[0], s9[1]) & m; sc.mismatch = s9[1] & m;
    sc.case_bonus = s9[6] & m; sc.cap_bonus = s9[5] & m; sc.delim_bonus = s9[8] & m; sc.prefix_bonus = s9[4] & m;
    sc.raw_match = s9[0]; sc.raw_gap_open = s9[2]; sc.raw_gap_extend = s9[3]; sc.raw_prefix = s9[4]; sc.raw_cap = s9[5];
    sc.raw_case = s9[6]; sc.raw_delim = s9[8]; sc.exact_bonus = s9[7];
    return sc;
}
}  // namespace

extern "C" {
int h_build_needle(const uint8_t* needle, size_t n, int case_sensitive, FrzUNeedle* out) { return frz_build_uneedle(needle, n, case_sensitive != 0, out) ? 1 : 0; }
int h_needle_has_uppercase(const uint8_t* needle, size_t n) { return frz_needle_has_uppercase(needle, n) ? 1 : 0; }
// the product's case tables, scalar by scalar (tests/test_unicode_device_code.py checks them against an independent derivation)
uint32_t h_scalar_flip(uint32_t cp) { return frz_unicode_detail::scalar_flip(cp); }
int h_scalar_is_uppercase(uint32_t cp) { return frz_unicode_detail::scalar_is_uppercase(cp) ? 1 : 0; }
int h_prefilter(const uint8_t* needle, size_t n, int case_sensitive, const uint8_t* hay, int len, int lanes, int max_typos,
                int* start, int* end) {
    FrzUNeedle nd;
    if (!frz_build_uneedle(needle, n, case_sensitive != 0, &nd)) return -1;
    Flat h{hay};
    return frzu::prefilter(nd, h, len, lanes, max_typos, start, end) ? 1 : 0;
}
int h_sw_score(const uint8_t* needle, size_t n, int case_sensitive, const uint16_t* scoring9, const uint8_t* hay, int len,
               int include_prefix, int lanes, int score_bits) {
    FrzUNeedle nd;
    if (!frz_build_uneedle(needle, n, case_sensitive != 0, &nd)) return -1;
    const FrzUScoring sc = scoring_of(scoring9, score_bits == 8);
    std::vector<uint16_t> scratch((size_t)2 * (nd.n + 1) * lanes);
    Flat h{hay};
    return (int)frzu::sw_score(nd, sc, h, len, include_prefix != 0, lanes, score_bits == 8, scratch.data());
}
int h_sw_indices(const uint8_t* needle, size_t n, int case_sensitive, int unicode, const uint16_t* scoring9, const uint8_t* hay, int len,
                 int start_pos, int max_typos, int lanes, int score_bits, uint32_t* out, int cap, int* n_out) {
    FrzUNeedle nd;
    if (!frz_build_uneedle(needle, n, case_sensitive != 0, &nd)) return -1;
    const FrzUScoring sc = scoring_of(scoring9, score_bits == 8);
    std::vector<uint16_t> scratch(frzi::indices_scratch_elems(unicode ? nd.n : nd.nbytes, lanes));
    Flat h{hay};
    return (int)frzi::sw_indices(nd, unicode != 0, sc, h, len, start_pos, max_typos, lanes, score_bits == 8, scratch.data(), out, cap, n_out);
}
int h_lit_find(const uint8_t* needle, size_t n, int case_sensitive, const uint16_t* scoring9, const uint8_t* hay, int len, int mode,
               int* pos, uint32_t* score) {
    FrzUNeedle nd;
    if (!frz_build_uneedle(needle, n, case_sensitive != 0, &nd)) return -1;
    const FrzUScoring sc = scoring_of(scoring9, false);
    Flat h{hay};
    return frzu::lit_find(nd, sc, h, len, mode, pos, score) ? 1 : 0;
}

// The same kernels on a ready needle and scoring: the library's own (frz_matcher_debug_unicode), so that the tests run
// with exactly the constants the GPU kernels receive.
size_t h_uneedle_size() { return sizeof(FrzUNeedle); }
size_t h_uscoring_size() { return sizeof(FrzUScoring); }
void h_scoring_of(const uint16_t* scoring9, int score_bits, FrzUScoring* out) { *out = scoring_of(scoring9, score_bits == 8); }
int h_sw_score_c(const FrzUNeedle* nd, const FrzUScoring* sc, const uint8_t* hay, int len, int include_prefix, int lanes, int score_bits) {
    std::vector<uint16_t> scratch((size_t)2 * (nd->n + 1) * lanes);
    Flat h{hay};
    return (int)frzu::sw_score(*nd, *sc, h, len, include_prefix != 0, lanes, score_bits == 8, scratch.data());
}
int h_sw_indices_c(const FrzUNeedle* nd, int unicode, const FrzUScoring* sc, const uint8_t* hay, int len, int start_pos, int max_typos,
                   int lanes, int score_bits, uint32_t* out, int cap, int* n_out) {
    std::vector<uint16_t> scratch(frzi::indices_scratch_elems(unicode ? nd->n : nd->nbytes, lanes));
    Flat h{hay};
    return (int)frzi::sw_indices(*nd, unicode != 0, *sc, h, len, start_pos, max_typos, lanes, score_bits == 8, scratch.data(), out, cap, n_out);
}
int h_lit_find_c(const FrzUNeedle* nd, const FrzUScoring* sc, const uint8_t* hay, int len, int mode, int* pos, uint32_t* score) {
    Flat h{hay};
    return frzu::lit_find(*nd, *sc, h, len, mode, pos, score) ? 1 : 0;
}
}
