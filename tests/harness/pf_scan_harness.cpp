// Host build of frizbee_b200/csrc/prefilter_scan.cuh — the scanning prefilter forms (window_k0 / _k1 / _k2 / _many) and
// the literal matcher that the kernels run per thread — for tests/test_kernel_logic_cpu.py.  The haystack is read as the
// kernels read the packed corpus: little-endian words of its contiguous bytes, zero padded past the end.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../frizbee_b200/csrc/prefilter_scan.cuh"

using namespace frzpf;

namespace {

struct HostAcc {
    const uint32_t* w;
    uint32_t word(uint32_t i) const { return w[i]; }
};

std::vector<uint32_t> words_of(const uint8_t* hay, int len) {
    std::vector<uint32_t> v((size_t)(len + 3) / 4 + 4, 0u);
    if (len) memcpy(v.data(), hay, (size_t)len);
    return v;
}

// the needle of a long pattern as k_scan_window_long stages it (prefilter.cu: stage_long_pat), its per-position data
// from the case_needle pairs c / flip with the probes host.cu: compile_pattern derives from them
struct LongTab {
    std::vector<uint8_t> c, flip, om, tg;
    LongPat view(const FrzPatternDev& p) const {
        LongPat l;
        l.c = c.data(); l.flip = flip.data(); l.om = om.data(); l.tg = tg.data();
        l.n = p.n; l.pf_lanes = p.pf_lanes; l.sw_lanes = p.sw_lanes; l.max_typos = p.max_typos; l.matching = p.matching;
        l.col_classes = p.col_classes; l.n_distinct = 0;
        l.raw_match = p.raw_match; l.raw_case = p.raw_case; l.raw_prefix = p.raw_prefix; l.raw_cap = p.raw_cap;
        l.raw_delim = p.raw_delim; l.exact_bonus = p.exact_bonus;
        return l;
    }
};
LongTab long_tab(const uint8_t* c, const uint8_t* flip, int n) {
    LongTab t;
    t.c.assign(c, c + n);
    t.flip.assign(flip, flip + n);
    for (int i = 0; i < n; i++) {
        t.om.push_back(flip[i] != c[i] ? 0x20 : 0);
        t.tg.push_back(flip[i] != c[i] ? (uint8_t)(c[i] | 0x20) : c[i]);
    }
    return t;
}

// the form k_match_indices runs for the pattern's typo mode; -1 = no prefilter form (NONE / LITERAL)
template <class P>
int window(const FrzPatternDev& pat, const P& p, const uint8_t* hay, int len, int* start, int* end) {
    const std::vector<uint32_t> w = words_of(hay, len);
    const HostAcc a{w.data()};
    switch (pat.typo_mode) {
        case FRZ_T_0: return window_k0(a, p, len, start, end) ? 1 : 0;
        case FRZ_T_1: return window_k1(a, p, len, start, end) ? 1 : 0;
        case FRZ_T_2: return window_k2(a, p, len, start, end) ? 1 : 0;
        case FRZ_T_MANY: return window_many(a, p, len, start, end) ? 1 : 0;
        default: return -1;
    }
}

template <class P>
int literal(const P& p, const uint8_t* hay, int len, int* pos, uint32_t* score) {
    const std::vector<uint32_t> w = words_of(hay, len);
    return lit_find(HostAcc{w.data()}, p, len, pos, score) ? 1 : 0;
}

}  // namespace

extern "C" {
size_t h_pattern_size() { return sizeof(FrzPatternDev); }

// The scanning form of the pattern's typo mode on a FrzPatternDev (needles of up to FRZ_MAX_NEEDLE bytes).
// Returns 1/0 = matched, -1 = the typo mode has no prefilter form.
int h_scan_window(const void* pat_bytes, const uint8_t* hay, int len, int* start, int* end) {
    FrzPatternDev pat;
    memcpy(&pat, pat_bytes, sizeof pat);
    return window(pat, pat, hay, len, start, end);
}

// The same on a LongPat (needles of more than FRZ_MAX_NEEDLE bytes): c / flip are the needle's n case_needle pairs.
int h_scan_window_long(const void* pat_bytes, const uint8_t* c, const uint8_t* flip, const uint8_t* hay, int len, int* start,
                       int* end) {
    FrzPatternDev pat;
    memcpy(&pat, pat_bytes, sizeof pat);
    const LongTab t = long_tab(c, flip, pat.n);
    return window(pat, t.view(pat), hay, len, start, end);
}

// lit_find on the pattern (c == nullptr) or on its LongPat.  Returns 1/0 = matched; *pos, *score.
int h_lit_find(const void* pat_bytes, const uint8_t* c, const uint8_t* flip, const uint8_t* hay, int len, int* pos,
               uint32_t* score) {
    FrzPatternDev pat;
    memcpy(&pat, pat_bytes, sizeof pat);
    if (!c) return literal(pat, hay, len, pos, score);
    const LongTab t = long_tab(c, flip, pat.n);
    return literal(t.view(pat), hay, len, pos, score);
}

// the probes host.cu: compile_pattern stored for the first min(n, FRZ_MAX_NEEDLE) positions
void h_pattern_probes(const void* pat_bytes, uint8_t* om, uint8_t* tg) {
    FrzPatternDev pat;
    memcpy(&pat, pat_bytes, sizeof pat);
    memcpy(om, pat.om, FRZ_MAX_NEEDLE);
    memcpy(tg, pat.tg, FRZ_MAX_NEEDLE);
}
}
