// Host build of the long-needle scorers for tests/test_long_needle_cpu.py: the wavefront arithmetic of k_sw_long
// (sw_wave.cuh) and generic_score (sw_generic.cuh) over a needle view as k_sw_long_thread reads it.  The scoring constants
// come from the real library (frz_matcher_debug_pattern); the needle bytes and case flips from the test.
#include <stdint.h>
#include <string.h>

#include "../../frizbee_b200/csrc/sw_generic.cuh"
#include "../../frizbee_b200/csrc/sw_wave.cuh"

namespace {
struct HostHay {
    const uint8_t* p;
    uint32_t operator()(int i) const { return p[i]; }
};
// the members generic_score reads (sw.cu: LongNeedle)
struct HostLongNeedle {
    const uint8_t *c, *flip;
    int n, sw_lanes, score_bits;
    int32_t gap_extend, gap_open_x, match_x, mismatch, case_bonus, cap_bonus, delim_bonus, prefix_bonus;
};
}  // namespace

extern "C" {
size_t h_pattern_size() { return sizeof(FrzPatternDev); }
// wave_score of window[0..W) at the pattern's sw_lanes; -2 for an unsupported argument
int h_sw_wave(const void* pat_bytes, const uint8_t* nc, const uint8_t* nf, int n, const uint8_t* window, int W, int include_prefix) {
    FrzPatternDev pat;
    memcpy(&pat, pat_bytes, sizeof pat);
    if (W > FRZ_SW_MAX_WINDOW || n > FRZ_LONG_NEEDLE) return -2;
    const frzwave::WaveConst k = frzwave::wave_const(pat);
    switch (pat.sw_lanes) {
        case 8: return (int)frzwave::wave_score<8>(HostHay{window}, W, nc, nf, n, include_prefix != 0, k);
        case 16: return (int)frzwave::wave_score<16>(HostHay{window}, W, nc, nf, n, include_prefix != 0, k);
        case 32: return (int)frzwave::wave_score<32>(HostHay{window}, W, nc, nf, n, include_prefix != 0, k);
        default: return -2;
    }
}
// generic_score (k_sw_long_thread) of window[0..W) for the needle nc / nf of n bytes
int h_sw_generic_long(const void* pat_bytes, const uint8_t* nc, const uint8_t* nf, int n, const uint8_t* window, int W,
                      int include_prefix) {
    FrzPatternDev p;
    memcpy(&p, pat_bytes, sizeof p);
    if (W > FRZ_SW_MAX_WINDOW || n > FRZ_LONG_NEEDLE) return -2;
    const HostLongNeedle nv{nc, nf, n, p.sw_lanes, p.score_bits, p.gap_extend, p.gap_open_x, p.match_x, p.mismatch, p.case_bonus,
                            p.cap_bonus, p.delim_bonus, p.prefix_bonus};
    return (int)frzsw::generic_score(HostHay{window}, W, nv, include_prefix != 0);
}
}
