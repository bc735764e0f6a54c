// Host build of frizbee_b200/csrc/sw_generic.cuh — the scorers of k_sw_generic (windows of 129..1024 bytes, greedy
// above) — for tests/test_kernel_logic_cpu.py.  The pattern constants come from the real library
// (frz_matcher_debug_pattern).
#include <stdint.h>
#include <string.h>

#include "../../frizbee_b200/csrc/sw_generic.cuh"

using namespace frzsw;

namespace {
struct HostHay {
    const uint8_t* p;
    uint32_t operator()(int i) const { return p[i]; }
};
}  // namespace

extern "C" {
size_t h_pattern_size() { return sizeof(FrzPatternDev); }
// generic_score of window[0..W), W <= FRZ_SW_MAX_WINDOW
int h_sw_generic(const void* pat_bytes, const uint8_t* window, int W, int include_prefix) {
    FrzPatternDev pat;
    memcpy(&pat, pat_bytes, sizeof pat);
    if (W > FRZ_SW_MAX_WINDOW) return -2;
    return (int)generic_score(HostHay{window}, W, pat, include_prefix != 0);
}
// greedy_score of window[0..W): -1 when the needle does not match
int h_greedy(const void* pat_bytes, const uint8_t* window, int W, int include_prefix) {
    FrzPatternDev pat;
    memcpy(&pat, pat_bytes, sizeof pat);
    return greedy_score(HostHay{window}, W, pat, include_prefix != 0);
}
}
