// Host build of frizbee_b200/csrc/sw_core.cuh — the register Smith-Waterman core the GPU kernels run — for
// tests/test_kernel_logic_cpu.py.  The pattern constants come from the real library (frz_matcher_debug_pattern).
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../frizbee_b200/csrc/sw_core.cuh"

using namespace frzsw;

namespace {
template <int LANES, int COLS, bool WRAP8, int VAR, int CC>
uint32_t run_one(const FrzPatternDev& pat, const uint8_t* window, int W, int startlo, bool include_prefix, int* exact_eq) {
    // stage the window the way the kernel receives it: 16-byte units with `startlo` bytes of junk in front
    constexpr int NU = (CC + 15) / 16 + 1;
    uint8_t raw[NU * 16];
    for (int i = 0; i < NU * 16; i++) raw[i] = (uint8_t)(0xA5 ^ i);        // junk before the window and after it
    for (int i = 0; i < W && startlo + i < NU * 16; i++) raw[startlo + i] = window[i];
    uint4 u[NU];
    memcpy(u, raw, sizeof u);
    // (the kernel zero-fills units past the window's last unit)
    const int last_u = W > 0 ? (startlo + W - 1) >> 4 : -1;
    for (int k = 0; k < NU; k++) if (k > last_u) u[k] = make_uint4(0, 0, 0, 0);
    uint32_t hw[CC / 4];
    window_from_units<CC>(u, (uint32_t)startlo, W, hw);
    std::vector<uint32_t> smem(2 * 64 * kSwThreads);
    const uint32_t score = SwCore<LANES, COLS, WRAP8, VAR, CC>::run(hw, W, pat, include_prefix, smem.data());
    *exact_eq = window_equals_needle(hw, W, pat) ? 1 : 0;
    return score;
}

// VAR bit of SwCore's per-lane gap penalties (sw_core.cuh: kSwVarLanePen)
constexpr int kLanePen = 16;

template <int LANES, bool WRAP8, int VAR>
int dispatch_cc(const FrzPatternDev& pat, const uint8_t* w, int W, int startlo, bool pre, int cols, int cc, int* eq) {
    if (cols == 128) {
        constexpr int V = VAR & kLanePen;   // the 128-column kernel classifies the bonus per lane
        switch (cc) {   // column-limited forms of the 128-column variant (groundwork, DESIGN.md §8 item 6)
            case 80: return (int)run_one<LANES, 128, WRAP8, V, 80>(pat, w, W, startlo, pre, eq);
            case 96: return (int)run_one<LANES, 128, WRAP8, V, 96>(pat, w, W, startlo, pre, eq);
            case 112: return (int)run_one<LANES, 128, WRAP8, V, 112>(pat, w, W, startlo, pre, eq);
            default: return (int)run_one<LANES, 128, WRAP8, V, 128>(pat, w, W, startlo, pre, eq);
        }
    }
    switch (cc) {
        case 40: return (int)run_one<LANES, 64, WRAP8, VAR, 40>(pat, w, W, startlo, pre, eq);
        case 48: return (int)run_one<LANES, 64, WRAP8, VAR, 48>(pat, w, W, startlo, pre, eq);
        case 56: return (int)run_one<LANES, 64, WRAP8, VAR, 56>(pat, w, W, startlo, pre, eq);
        case 64: return (int)run_one<LANES, 64, WRAP8, VAR, 64>(pat, w, W, startlo, pre, eq);
    }
    return -1;
}
template <int LANES>
int dispatch(const FrzPatternDev& pat, const uint8_t* w, int W, int startlo, bool pre, int cols, int cc, int wrap8, int var, int* eq) {
    if (wrap8) return dispatch_cc<LANES, true, 0>(pat, w, W, startlo, pre, cols, cc, eq);
    {
        switch (var) {
            case 8: return dispatch_cc<LANES, false, 8>(pat, w, W, startlo, pre, cols, cc, eq);
            case kLanePen: return dispatch_cc<LANES, false, kLanePen>(pat, w, W, startlo, pre, cols, cc, eq);
            case 8 | kLanePen: return dispatch_cc<LANES, false, 8 | kLanePen>(pat, w, W, startlo, pre, cols, cc, eq);
        }
    }
    return dispatch_cc<LANES, false, 0>(pat, w, W, startlo, pre, cols, cc, eq);
}
}  // namespace

extern "C" {
size_t h_pattern_size() { return sizeof(FrzPatternDev); }
// the pattern fields that pick the SwCore instantiation: wrap8, col_classes, and whether frz_launch_sw (sw.cu) takes the
// per-lane gap penalty variant (gap_extend == 0 < gap_open_x, no WRAP8)
void h_pattern_flags(const void* pat_bytes, int* wrap8, int* col_classes, int* lane_pen) {
    FrzPatternDev pat;
    memcpy(&pat, pat_bytes, sizeof pat);
    *wrap8 = pat.wrap8;
    *col_classes = pat.col_classes;
    *lane_pen = !pat.wrap8 && pat.gap_extend == 0 && pat.gap_open_x > 0;
}
// score of SwCore<lanes, cols, wrap8, var, cc> on window[0..W) staged at byte offset `startlo` of its first unit
int h_swcore(const void* pat_bytes, const uint8_t* window, int W, int startlo, int include_prefix, int lanes, int cols, int cc,
             int wrap8, int var, int* exact_eq) {
    FrzPatternDev pat;
    memcpy(&pat, pat_bytes, sizeof pat);
    switch (lanes) {
        case 8: return dispatch<8>(pat, window, W, startlo, include_prefix != 0, cols, cc, wrap8, var, exact_eq);
        case 16: return dispatch<16>(pat, window, W, startlo, include_prefix != 0, cols, cc, wrap8, var, exact_eq);
        case 32: return dispatch<32>(pat, window, W, startlo, include_prefix != 0, cols, cc, wrap8, var, exact_eq);
        case 64: return dispatch<64>(pat, window, W, startlo, include_prefix != 0, cols, cc, wrap8, var, exact_eq);
    }
    return -1;
}
}
