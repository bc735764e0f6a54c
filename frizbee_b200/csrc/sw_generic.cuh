// sw_generic.cuh — the per-thread scorers of k_sw_generic (sw.cu): the row-major Smith-Waterman of windows of
// 129..1024 bytes and the greedy scorer of longer windows (src/smith_waterman/greedy.rs:7-91).  Like sw_core.cuh this
// is FRZ_SW_FN code over a byte accessor (`hay(i)` = byte i of the window), so the same source is compiled by nvcc for
// the kernel and by g++ for tests/test_kernel_logic_cpu.py, which runs it on the CPU against the oracle.
#pragma once
#include <stdint.h>

#include "sw_core.cuh"

namespace frzsw {

constexpr int kGenCols = FRZ_SW_MAX_WINDOW + 64;

// Not force-inlined on the device: k_sw_generic calls it for rare > 1024-byte windows and nvcc decides.
#if defined(__CUDACC__)
#define FRZ_SW_GREEDY_FN __device__
#else
#define FRZ_SW_GREEDY_FN inline
#endif

template <class Hay>
FRZ_SW_GREEDY_FN int greedy_score(const Hay& hay, int W, const FrzPatternDev& p, bool include_prefix) {
    const int n = p.n;
    if (n > W) return -1;
    auto sat_add = [](uint32_t a, uint32_t b) { uint32_t r = a + b; return r > 0xffffu ? 0xffffu : r; };
    auto sat_sub = [](uint32_t a, uint32_t b) { return a > b ? a - b : 0u; };
    uint32_t score = 0;
    int hi = 0;
    bool delim_enabled = false, prev_lower = false, prev_delim = false;
    for (int ni = 0; ni < n; ni++) {
        const int hstart = hi;
        bool matched = false;
        while (hi <= W - n + ni) {
            const uint32_t hc = hay(hi);
            const bool is_digit = hc - '0' <= 9u, is_upper = hc - 'A' <= 25u, is_lower = hc - 'a' <= 25u;
            const bool is_delim = hc < 128 && !(is_lower || is_upper || is_digit);
            if (!is_delim) delim_enabled = true;
            if (p.c[ni] != hc && p.flip[ni] != hc) {
                prev_delim = delim_enabled && is_delim;
                prev_lower = is_lower;
                hi++;
                continue;
            }
            score = sat_add(score, p.raw_match);
            if (hi != hstart && ni != 0) {
                uint32_t gl = (uint32_t)(hi - hstart);
                gl = gl > 0 ? gl - 1 : 0;
                if (gl > 0xffffu) gl = 0xffffu;
                uint32_t mul = (uint32_t)p.raw_gap_extend * gl;
                if (mul > 0xffffu) mul = 0xffffu;
                score = sat_sub(score, sat_add(p.raw_gap_open, mul));
            }
            if (p.c[ni] == hc) score = sat_add(score, p.raw_case);
            if (is_upper && prev_lower) score = sat_add(score, p.raw_cap);
            if (include_prefix && hi == 0) score = sat_add(score, p.raw_prefix);
            if (prev_delim && !is_delim) score = sat_add(score, p.raw_delim);
            prev_delim = delim_enabled && is_delim;
            prev_lower = is_lower;
            hi++;
            matched = true;
            break;
        }
        if (!matched) return -1;
    }
    return (int)score;
}

// Score of a window of W <= FRZ_SW_MAX_WINDOW bytes: a literal row-major restatement of the reference with true
// element-width arithmetic (u8 or u16 lanes, pat.sw_lanes wide chunks).
template <class Hay>
FRZ_SW_FN uint32_t generic_score(const Hay& hay, int W, const FrzPatternDev& pat, bool include_prefix) {
    const int L = pat.sw_lanes;
    const uint32_t lane_mask = pat.score_bits == 8 ? 0xffu : 0xffffu;  // real element width
    uint16_t Hp[kGenCols], Hc[kGenCols], bon[kGenCols];
    uint8_t Mp[kGenCols], Mc[kGenCols], hb[kGenCols];
    const int nch = (W + L - 1) / L, cols = nch * L;
    bool pl = false, pd = false;
    for (int c = 0; c < cols; c++) {
        uint32_t b = c < W ? hay(c) : 0;
        hb[c] = (uint8_t)b;
        bool up = b - 'A' <= 25u, lo = b - 'a' <= 25u, dg = b - '0' <= 9u;
        bool dl = !(up || lo || dg || b > 127);
        // wrapping adds in the element width (ascii.rs:98-101)
        uint32_t bo = 0;
        if (pd && !dl) bo = (bo + pat.delim_bonus) & lane_mask;
        if (up && pl) bo = (bo + pat.cap_bonus) & lane_mask;
        if (c == 0 && include_prefix) bo = (bo + pat.prefix_bonus) & lane_mask;
        bo = (bo + pat.match_x) & lane_mask;
        bon[c] = (uint16_t)bo;
        Hp[c] = 0; Mp[c] = 0;
        pl = lo; pd = dl;
    }
    auto bonus_at = [&](int c) -> uint32_t { return bon[c]; };
    for (int i = 0; i < pat.n; i++) {
        for (int c = 0; c < cols; c++) {
            uint32_t b = hb[c];
            bool e = b == pat.c[i], f = b == pat.flip[i];
            bool m = e || f;
            uint32_t dg = c > 0 ? Hp[c - 1] : 0;
            if (m) dg = (dg + bonus_at(c)) & lane_mask;
            dg = dg > (uint32_t)pat.mismatch ? dg - pat.mismatch : 0;
            if (e) dg = (dg + pat.case_bonus) & lane_mask;
            uint32_t upv = Hp[c];
            upv = upv > (uint32_t)pat.gap_extend ? upv - pat.gap_extend : 0;
            if (Mp[c]) upv = upv > (uint32_t)pat.gap_open_x ? upv - pat.gap_open_x : 0;
            Hc[c] = (uint16_t)max(dg, upv);
            Mc[c] = m;
        }
        for (int ch = 0; ch < nch; ch++) {
            const int lo = ch * L;
            uint32_t gex = pat.gap_extend;
            for (int s = 1; s < L; s <<= 1) {
                for (int c = lo + L - 1; c >= lo; c--) {
                    int src = c - s;
                    if (src < 0) continue;
                    if (src < lo && src < lo - L) continue;  // only the adjacent chunk feeds in
                    uint32_t pen = (gex + (Mc[src] ? (uint32_t)pat.gap_open_x : 0u)) & lane_mask;
                    uint32_t v = Hc[src];
                    v = v > pen ? v - pen : 0;
                    if (v > Hc[c]) Hc[c] = (uint16_t)v;
                }
                gex = (gex + gex) & lane_mask;
            }
        }
        for (int c = 0; c < cols; c++) { Hp[c] = Hc[c]; Mp[c] = Mc[c]; }
    }
    uint32_t mx = 0;
    for (int c = 0; c < cols; c++) mx = max(mx, (uint32_t)Hp[c]);
    return mx;
}

}  // namespace frzsw
