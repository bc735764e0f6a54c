// sw_wave.cuh — the arithmetic of k_sw_long (sw.cu): the Smith-Waterman score of one window of up to FRZ_SW_MAX_WINDOW
// bytes against a needle of FRZ_MAX_NEEDLE + 1 .. FRZ_LONG_NEEDLE bytes, scored by one warp as a systolic wavefront.
//
// The reference evaluates the matrix in LANES-column chunks (u16 family: LANES 8, 16 or 32).  Cell (row i, chunk j)
// depends on (i - 1, j), on the last cell of (i - 1, j - 1) (diagonal) and on the final cells of (i, j - 1): the in-row
// gap scan is a log-step doubling over the chunk whose steps reach LANES / 2 cells into the left chunk (generic_score in
// sw_generic.cuh is the row-major restatement that the CPU suite pins against the oracle).  So lane j of the warp owns
// chunk j and computes row t - j at step t: the row the left lane finished one step earlier.  What the right neighbour
// needs travels as a WaveLeft (the last LANES / 2 cells and match flags of the row, the last cell of the row before):
// by shuffle inside a pass of 32 chunks, through a per-row store between passes (windows of more than 32 chunks).
//
// The same source is compiled by g++ for tests/test_long_needle_cpu.py: wave_score runs the lanes of each step from the last
// to the first, so "the left lane's state" is still the previous step's, as a shuffle of the device loop reads it.
#pragma once
#include <stdint.h>

#include "frz_device.cuh"

#include "frz_hd.cuh"

namespace frzwave {

// scoring constants of the u16 family (FrzPatternDev's, as the reference splats them)
struct WaveConst {
    uint32_t gex, gopx, mismatch, case_bonus, delim_bonus, cap_bonus, prefix_bonus, match_x;
};
FRZ_HD WaveConst wave_const(const FrzPatternDev& p) {
    return WaveConst{(uint32_t)p.gap_extend, (uint32_t)p.gap_open_x, (uint32_t)p.mismatch, (uint32_t)p.case_bonus,
                     (uint32_t)p.delim_bonus, (uint32_t)p.cap_bonus, (uint32_t)p.prefix_bonus, (uint32_t)p.match_x};
}

// What chunk j - 1 hands chunk j for row i.  All zero for chunk 0: a zero cell minus a penalty never raises a cell, which
// is what the reference's "no cell to the left" amounts to.
template <int L>
struct WaveLeft {
    uint32_t hp[L / 4];   // final cells L/2 .. L-1 of row i, two 16-bit cells per word (cell L/2 + q: word q / 2, half q % 2)
    uint32_t m;           // their match flags, bit q = cell L/2 + q
    uint32_t diag;        // last cell of row i - 1
};

// One lane's chunk: the window bytes and per-column bonuses (packed) and the last row it computed.
template <int L>
struct WaveLane {
    uint32_t hb[L / 4];   // window bytes, four per word (zero past the window)
    uint32_t bon[L / 2];  // per-column bonus + match_x, two 16-bit values per word
    uint32_t h[L];        // cells of the last row computed (row -1: zeros)
    uint32_t m;           // match flags of that row
    uint32_t hlast_prev;  // last cell of the row before it
};

FRZ_HD uint32_t sat_sub(uint32_t a, uint32_t b) { return a > b ? a - b : 0u; }

// columns chunk * L .. chunk * L + L - 1 of a window of W bytes (hay(c) = byte c, read for c < W only); per-column bonus as
// generic_score computes it
template <int L, class Hay>
FRZ_HD void lane_load(WaveLane<L>& s, const Hay& hay, int chunk, int W, bool include_prefix, const WaveConst& k) {
#pragma unroll
    for (int q = 0; q < L / 4; q++) s.hb[q] = 0;
#pragma unroll
    for (int q = 0; q < L / 2; q++) s.bon[q] = 0;
    const int c0 = chunk * L;
    uint32_t pb = (c0 > 0 && c0 - 1 < W) ? hay(c0 - 1) : 0;
    bool pl = pb - 'a' <= 25u, pd = c0 > 0 && !(pb - 'A' <= 25u || pl || pb - '0' <= 9u || pb > 127);
#pragma unroll
    for (int r = 0; r < L; r++) {
        const int c = c0 + r;
        const uint32_t b = c < W ? hay(c) : 0u;
        const bool up = b - 'A' <= 25u, lo = b - 'a' <= 25u, dg = b - '0' <= 9u;
        const bool dl = !(up || lo || dg || b > 127);
        uint32_t bo = 0;
        if (pd && !dl) bo = (bo + k.delim_bonus) & 0xffffu;
        if (up && pl) bo = (bo + k.cap_bonus) & 0xffffu;
        if (c == 0 && include_prefix) bo = (bo + k.prefix_bonus) & 0xffffu;
        bo = (bo + k.match_x) & 0xffffu;
        s.hb[r / 4] |= b << (8 * (r % 4));
        s.bon[r / 2] |= bo << (16 * (r % 2));
        pl = lo; pd = dl;
    }
#pragma unroll
    for (int r = 0; r < L; r++) s.h[r] = 0;
    s.m = 0;
    s.hlast_prev = 0;
}

// what this lane hands its right neighbour after its last row
template <int L>
FRZ_HD WaveLeft<L> lane_out(const WaveLane<L>& s) {
    WaveLeft<L> o;
#pragma unroll
    for (int q = 0; q < L / 4; q++) o.hp[q] = s.h[L / 2 + 2 * q] | s.h[L / 2 + 2 * q + 1] << 16;
    o.m = s.m >> (L / 2);
    o.diag = s.hlast_prev;
    return o;
}
template <int L>
FRZ_HD WaveLeft<L> wave_left_zero() {
    WaveLeft<L> o;
#pragma unroll
    for (int q = 0; q < L / 4; q++) o.hp[q] = 0;
    o.m = 0;
    o.diag = 0;
    return o;
}

// row i of this lane's chunk, needle byte c / its case flip f
template <int L>
FRZ_HD void lane_row(WaveLane<L>& s, const WaveLeft<L>& left, uint32_t nc, uint32_t nf, const WaveConst& k) {
    uint32_t h[L];
    uint32_t m = 0;
#pragma unroll
    for (int r = 0; r < L; r++) {
        const uint32_t b = (s.hb[r / 4] >> (8 * (r % 4))) & 0xffu;
        const bool e = b == nc, mm = e || b == nf;
        uint32_t dg = r > 0 ? s.h[r - 1] : left.diag;
        if (mm) dg = (dg + ((s.bon[r / 2] >> (16 * (r % 2))) & 0xffffu)) & 0xffffu;
        dg = sat_sub(dg, k.mismatch);
        if (e) dg = (dg + k.case_bonus) & 0xffffu;
        uint32_t up = sat_sub(s.h[r], k.gex);
        if ((s.m >> r) & 1u) up = sat_sub(up, k.gopx);
        h[r] = dg > up ? dg : up;
        m |= (uint32_t)mm << r;
    }
    // log-step gap scan; descending in place, so cell r - s still holds the previous step's value
    uint32_t gexs = k.gex;
#pragma unroll
    for (int sh = 1; sh < L; sh <<= 1) {
#pragma unroll
        for (int r = L - 1; r >= 0; r--) {
            uint32_t v, mb;
            if (r >= sh) {
                v = h[r - sh];
                mb = (m >> (r - sh)) & 1u;
            } else {
                const int q = L / 2 + r - sh;   // cell of the left chunk's handed-over half
                v = (left.hp[q / 2] >> (16 * (q % 2))) & 0xffffu;
                mb = (left.m >> q) & 1u;
            }
            const uint32_t pen = (gexs + (mb ? k.gopx : 0u)) & 0xffffu;
            v = sat_sub(v, pen);
            if (v > h[r]) h[r] = v;
        }
        gexs = (gexs + gexs) & 0xffffu;
    }
    s.hlast_prev = s.h[L - 1];
#pragma unroll
    for (int r = 0; r < L; r++) s.h[r] = h[r];
    s.m = m;
}

template <int L>
FRZ_HD uint32_t lane_max(const WaveLane<L>& s) {
    uint32_t mx = 0;
#pragma unroll
    for (int r = 0; r < L; r++) mx = s.h[r] > mx ? s.h[r] : mx;
    return mx;
}

#if !defined(__CUDA_ARCH__)
// The device loop of k_sw_long run on one thread (the CPU suite's view of it): the maximum over the last row of the
// window's ceil(W / L) chunks, as generic_score.  nc / nf: needle bytes and their case flips, n of them.
template <int L, class Hay>
inline uint32_t wave_score(const Hay& hay, int W, const uint8_t* nc, const uint8_t* nf, int n, bool include_prefix,
                           const WaveConst& k) {
    const int nch = (W + L - 1) / L;
    static thread_local WaveLeft<L> store[FRZ_LONG_NEEDLE];
    WaveLane<L> st[32];
    uint32_t best = 0;
    for (int p0 = 0; p0 < nch; p0 += 32) {
        const int lanes = nch - p0 < 32 ? nch - p0 : 32;
        const bool has_next = p0 + 32 < nch;
        for (int j = 0; j < lanes; j++) lane_load<L>(st[j], hay, p0 + j, W, include_prefix, k);
        for (int t = 0; t < n + lanes - 1; t++) {
            for (int j = lanes - 1; j >= 0; j--) {
                const int i = t - j;
                if (i < 0 || i >= n) continue;
                const WaveLeft<L> left = j > 0 ? lane_out<L>(st[j - 1]) : p0 > 0 ? store[i] : wave_left_zero<L>();
                lane_row<L>(st[j], left, nc[i], nf[i], k);
                if (j == 31 && has_next) store[i] = lane_out<L>(st[j]);
            }
        }
        for (int j = 0; j < lanes; j++) best = lane_max<L>(st[j]) > best ? lane_max<L>(st[j]) : best;
    }
    return best;
}
#endif

}  // namespace frzwave
