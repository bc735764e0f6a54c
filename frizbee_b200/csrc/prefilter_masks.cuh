// prefilter_masks.cuh — the occurrence-mask windows of prefilter.cu (0 and 1 typo), in a header so that the SAME source
// is compiled by nvcc for the kernels and by g++ for tests/test_kernel_logic_cpu.py (one emulated lane at a time, the
// warp intrinsics reduced to their single-lane meaning).  See prefilter.cu for the algorithm notes.
#pragma once
#include <stdint.h>

#include "frz_device.cuh"

#if defined(__CUDACC__)
#define FRZ_PF_FN __device__ __forceinline__
#define FRZ_PF_LANE frz_lane()
#else
#define FRZ_PF_FN inline
#define FRZ_PF_LANE 0u
// ---- single-lane host stand-ins ----
inline uint32_t __dp4a(uint32_t a, uint32_t b, uint32_t c) {   // unsigned 8-bit dot product + accumulate
    for (int i = 0; i < 4; i++) c += ((a >> (8 * i)) & 0xff) * ((b >> (8 * i)) & 0xff);
    return c;
}
inline uint4 __ldg(const uint4* p) { return *p; }
inline void __syncwarp() {}
inline bool __any_sync(unsigned, bool p) { return p; }
inline int __reduce_max_sync(unsigned, int v) { return v; }
inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
inline int __ffsll(long long x) { return __builtin_ffsll(x); }
inline int min(int a, int b) { return a < b ? a : b; }
#endif

namespace frzpf {

FRZ_PF_FN uint32_t splat4(uint32_t b) { return b * 0x01010101u; }

// ---------------------------------------------------------------------------------------------
// Occurrence-mask windows (0 and 1 typo) for candidates staged in shared memory.
//
// The reference works on per-chunk occurrence bitmasks (`B::occ`, one compare+movemask per needle
// byte).  A GPU lane has no movemask, and the first two versions of this stage (nested scans, then a
// per-lane scanning automaton) spent most of their instructions on divergent
// byte scans.  Here each lane first builds, with uniform straight-line code,
// the 64-bit occurrence mask of every DISTINCT needle byte class over a 64-byte block of its haystack:
// 4 bytes per step — xor/or with the probe, exact zero-byte flags, and one DP4A that packs the four
// flags into mask bits (weights 1,2,4,8 / 16,...,128).  After that the reference's mask state machine
// runs literally (`clear_through_lowest`, `first_path_chunk_mask > second_path_chunk_mask`, ...),
// every `occ` being one shared-memory load.
// ---------------------------------------------------------------------------------------------
constexpr int kMaxDistinct = 16;

// 0x80 in every byte of x that is zero
FRZ_PF_FN uint32_t zero_flags(uint32_t x) {
    const uint32_t t = (x & 0x7f7f7f7fu) + 0x7f7f7f7fu;
#if defined(__CUDA_ARCH__)
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0x10;" : "=r"(r) : "r"(0x80808080u), "r"(t), "r"(x));  // a & ~b & ~c
    return r;
#else
    return 0x80808080u & ~t & ~x;
#endif
}

// occ[d][lane] = occurrence mask of distinct class d over bytes [64*blk, 64*blk+64) of the lane's haystack.
// `base` points at unit 0 of the lane's haystack, unit k at base + k — in the packed corpus, or in the lane's row of
// the shared-memory stage k_scan_window fills with cp.async (same layout).  `units` = ceil(len / 16) bounds the reads.
FRZ_PF_FN void build_block_masks(const uint4* base, int units, int blk, const FrzPatternDev& pat,
                                                  uint2 (*occ)[32], uint32_t lane) {
    uint32_t w[16];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (4 * blk + k < units) v = base[4 * blk + k];   // generic load: packed corpus or a shared-memory stage
        w[4 * k] = v.x; w[4 * k + 1] = v.y; w[4 * k + 2] = v.z; w[4 * k + 3] = v.w;
    }
    for (int d = 0; d < pat.n_distinct; d++) {
        const uint32_t om4 = splat4(pat.dc_om[d]), tg4 = splat4(pat.dc_tg[d]);
        uint32_t m[2] = {0u, 0u};
#pragma unroll
        for (int j = 0; j < 8; j++) {  // 8 bytes per step → 8 mask bits (scaled by 128)
            const uint32_t f0 = zero_flags((w[2 * j] | om4) ^ tg4);
            const uint32_t f1 = zero_flags((w[2 * j + 1] | om4) ^ tg4);
            const uint32_t v = __dp4a(f0, 0x08040201u, __dp4a(f1, 0x80402010u, 0u));  // = 128 * bits
            const int sh = 8 * (j & 3) - 7;
            m[j >> 2] |= sh < 0 ? (v >> 7) : (v << sh);
        }
        occ[d][lane] = make_uint2(m[0], m[1]);
    }
}

FRZ_PF_FN uint64_t lowmask64(int n) { return n >= 64 ? ~0ull : ((1ull << n) - 1); }
FRZ_PF_FN uint64_t u2_to_u64(uint2 v) { return (uint64_t)v.x | ((uint64_t)v.y << 32); }

// Window of the 0-typo prefilter (closed form, SURVEY.md Appendix A.2) from block masks.  Warp-wide;
// `active` lanes own a candidate of `len` bytes starting at unit pointer `base` (any length: 64-byte blocks).
FRZ_PF_FN bool masks_k0(const uint4* base, const FrzPatternDev& pat, const uint8_t* __restrict__ cid_s,
                                         uint2 (*occ)[32], int len, bool active, int* ostart, int* oend) {
    const int units = active ? (len + 15) >> 4 : 0;
    const uint32_t lane = FRZ_PF_LANE;
    const int n = pat.n;
    int ni = 0, start = 0, end = 0;
    bool alive = active && len > 0, found = false;
    const int max_len = __reduce_max_sync(0xffffffffu, active ? len : 0);
    for (int blk = 0; blk * 64 < max_len; blk++) {
        build_block_masks(base, units, blk, pat, occ, lane);
        __syncwarp();
        const int rem = len - blk * 64;
        const uint64_t valid = rem > 0 ? lowmask64(rem) : 0ull;
        // 1 + last occurrence of the last needle byte (whole haystack)
        const uint64_t lastm = u2_to_u64(occ[pat.cid[n - 1]][lane]) & valid;
        if (lastm) end = blk * 64 + 64 - __clzll((long long)lastm);
        uint64_t fc = valid;
        bool in_blk = alive && !found && rem > 0;
        while (__any_sync(0xffffffffu, in_blk)) {
            if (in_blk) {
                const uint64_t x = u2_to_u64(occ[cid_s[ni]][lane]) & fc;
                if (x) {
                    if (ni == 0) start = blk * 64 + __ffsll((long long)x) - 1;
                    fc &= ~(x ^ (x - 1));  // clear_through_lowest
                    if (++ni == n) { found = true; in_blk = false; }
                } else in_blk = false;
            }
        }
        __syncwarp();
    }
    *ostart = start;
    *oend = end;
    return found;
}

// match_haystack_1_typo (src/prefilter/algo/ascii_typos.rs:15-110) on block masks, chunk width L.
FRZ_PF_FN bool masks_k1(const uint4* base, const FrzPatternDev& pat, const uint8_t* __restrict__ cid_s,
                                         uint2 (*occ)[32], int len, bool active, int* ostart, int* oend) {
    const int units = active ? (len + 15) >> 4 : 0;
    const uint32_t lane = FRZ_PF_LANE;
    const int n = pat.n, L = pat.pf_lanes;
    int f = 0, s = 1, ms = 0x7fffffff, end = -1;
    // 0 running, 1 found, 2 rejected / idle
    int state = 2;
    if (active) state = n <= 1 ? 1 : (len == 0 ? 2 : 0);
    if (active && n <= 1) ms = 0;
    const int max_len = __reduce_max_sync(0xffffffffu, active ? len : 0);
    const uint64_t lmask = lowmask64(L);
    for (int blk = 0; blk * 64 < max_len; blk++) {
        build_block_masks(base, units, blk, pat, occ, lane);
        __syncwarp();
        const int rem = len - blk * 64;
        const uint64_t valid = rem > 0 ? lowmask64(rem) : 0ull;
        // find_end_pos_with_typos: 1 + last occurrence of either of the last two needle bytes, else len
        if (n >= 2) {
            const uint64_t lastm = (u2_to_u64(occ[pat.cid[n - 1]][lane]) | u2_to_u64(occ[pat.cid[n - 2]][lane])) & valid;
            if (lastm) end = blk * 64 + 64 - __clzll((long long)lastm);
        }
        int cs = blk * 64;                       // chunk start (absolute)
        bool in_blk = state == 0 && rem > 0;
        bool init = true;
        uint64_t fm = 0, sm = 0, fc = 0, sc = 0;
        while (__any_sync(0xffffffffu, in_blk)) {
            if (in_blk) {
                const int sh = cs - blk * 64;
                if (init) {  // new chunk: both path masks restart from the whole chunk
                    const uint64_t cm = (valid >> sh) & lmask;
                    fm = (u2_to_u64(occ[cid_s[f]][lane]) >> sh) & lmask;
                    sm = (u2_to_u64(occ[cid_s[s]][lane]) >> sh) & lmask;
                    fc = sc = cm;
                    init = false;
                }
                bool adv = false;
                const int cand = f + 1;
                if (cand > s) {
                    if (cand == n) { state = 1; in_blk = false; }
                    else { s = cand; sc = fc; sm = (u2_to_u64(occ[cid_s[s]][lane]) >> sh) & lmask; }
                } else if (cand == s && fc > sc) sc = fc;
                if (in_blk) {
                    const uint64_t x = fm & fc;
                    if (x) {
                        ms = min(ms, cs + __ffsll((long long)x) - 1);
                        f++;
                        fc &= ~(x ^ (x - 1));
                        fm = (u2_to_u64(occ[cid_s[f]][lane]) >> sh) & lmask;
                        adv = true;
                    }
                    const uint64_t y = sm & sc;
                    if (y) {
                        ms = min(ms, cs + __ffsll((long long)y) - 1);
                        s++;
                        if (s >= n) { state = 1; in_blk = false; }
                        else {
                            sc &= ~(y ^ (y - 1));
                            sm = (u2_to_u64(occ[cid_s[s]][lane]) >> sh) & lmask;
                            adv = true;
                        }
                    }
                    if (in_blk && !adv) {  // next chunk
                        cs += L;
                        init = true;
                        if (cs >= len) { state = 2; in_blk = false; }
                        else if (cs >= blk * 64 + 64) in_blk = false;  // continues in the next block
                    }
                }
            }
        }
        __syncwarp();
    }
    *ostart = ms == 0x7fffffff ? 0 : ms;
    *oend = end < 0 ? len : end;
    return state == 1;
}

// ---- single-chunk forms -------------------------------------------------------------------------------------
// When no haystack of the corpus exceeds 64 bytes and the emulated prefilter width is 64 lanes, a candidate is ONE block
// and ONE chunk: the chunk loop, the `>> sh` alignment and the lane mask of the general forms disappear, and a step that
// finds nothing rejects at once.  The masks are also re-indexed per needle POSITION (pos[i] = occ[cid[i]], stored behind
// the distinct classes in the same shared-memory array when n_distinct + n <= kMaxDistinct), so every step of the state
// machine costs one LDS.64 instead of two dependent loads (class id, then mask): phase B is latency-bound, the chain
// length is what matters.  Bit-identical to masks_k0 / masks_k1 (tests/test_kernel_logic_cpu.py).
FRZ_PF_FN bool single_chunk_ok(const FrzPatternDev& pat, uint32_t max_gunits) {
    return max_gunits <= 4 && pat.pf_lanes == 64 && pat.n_distinct > 0 && pat.n_distinct + pat.n <= kMaxDistinct;
}
FRZ_PF_FN void build_position_masks(const FrzPatternDev& pat, uint2 (*occ)[32], uint32_t lane) {
    const int nd = pat.n_distinct;
    for (int i = 0; i < pat.n; i++) occ[nd + i][lane] = occ[pat.cid[i]][lane];   // a lane only ever touches its own column
}

FRZ_PF_FN bool masks_k0_single(const uint4* base, const FrzPatternDev& pat, uint2 (*occ)[32], int len, bool active,
                               int* ostart, int* oend) {
    const uint32_t lane = FRZ_PF_LANE;
    const int n = pat.n, nd = pat.n_distinct;
    build_block_masks(base, active ? (len + 15) >> 4 : 0, 0, pat, occ, lane);
    build_position_masks(pat, occ, lane);
    const uint64_t valid = len > 0 ? lowmask64(len) : 0ull;
    const uint64_t lastm = u2_to_u64(occ[nd + n - 1][lane]) & valid;
    int start = 0, ni = 0;
    uint64_t fc = valid;
    bool run = active && len > 0, found = false;
    while (__any_sync(0xffffffffu, run)) {
        if (run) {
            const uint64_t x = u2_to_u64(occ[nd + ni][lane]) & fc;
            if (x) {
                if (ni == 0) start = __ffsll((long long)x) - 1;
                fc &= ~(x ^ (x - 1));  // clear_through_lowest
                if (++ni == n) { found = true; run = false; }
            } else run = false;
        }
    }
    *ostart = start;
    *oend = lastm ? 64 - __clzll((long long)lastm) : 0;
    return found;
}

FRZ_PF_FN bool masks_k1_single(const uint4* base, const FrzPatternDev& pat, uint2 (*occ)[32], int len, bool active,
                               int* ostart, int* oend) {
    const uint32_t lane = FRZ_PF_LANE;
    const int n = pat.n, nd = pat.n_distinct;
    build_block_masks(base, active ? (len + 15) >> 4 : 0, 0, pat, occ, lane);
    build_position_masks(pat, occ, lane);
    const uint64_t valid = len > 0 ? lowmask64(len) : 0ull;
    int end = -1;
    if (n >= 2) {   // find_end_pos_with_typos: 1 + last occurrence of either of the last two needle bytes, else len
        const uint64_t lastm = (u2_to_u64(occ[nd + n - 1][lane]) | u2_to_u64(occ[nd + n - 2][lane])) & valid;
        if (lastm) end = 64 - __clzll((long long)lastm);
    }
    int f = 0, s = 1, ms = 0x7fffffff;
    int state = 2;   // 0 running, 1 found, 2 rejected / idle
    if (active) state = n <= 1 ? 1 : (len == 0 ? 2 : 0);
    if (active && n <= 1) ms = 0;
    uint64_t fc = valid, sc = valid, fm = 0, sm = 0;
    if (state == 0) { fm = u2_to_u64(occ[nd][lane]); sm = u2_to_u64(occ[nd + 1][lane]); }
    while (__any_sync(0xffffffffu, state == 0)) {
        if (state == 0) {
            bool adv = false;
            const int cand = f + 1;
            if (cand > s) {
                if (cand == n) state = 1;
                else { s = cand; sc = fc; sm = u2_to_u64(occ[nd + s][lane]); }
            } else if (cand == s && fc > sc) sc = fc;
            if (state == 0) {
                const uint64_t x = fm & fc;
                if (x) {
                    ms = min(ms, __ffsll((long long)x) - 1);
                    f++;
                    fc &= ~(x ^ (x - 1));
                    fm = u2_to_u64(occ[nd + f][lane]);
                    adv = true;
                }
                const uint64_t y = sm & sc;
                if (y) {
                    ms = min(ms, __ffsll((long long)y) - 1);
                    s++;
                    if (s >= n) state = 1;
                    else {
                        sc &= ~(y ^ (y - 1));
                        sm = u2_to_u64(occ[nd + s][lane]);
                        adv = true;
                    }
                }
                if (state == 0 && !adv) state = 2;   // the next chunk would start at 64 >= len
            }
        }
    }
    *ostart = ms == 0x7fffffff ? 0 : ms;
    *oend = end < 0 ? len : end;
    return state == 1;
}

// ---- 2-typo / N-typo trackers on occurrence masks.  Checked against the oracle on the CPU
// (tests/test_kernel_logic_cpu.py) and on the GPU (tests/test_gpu_parity.py, every typo budget); the kernels call them
// whenever the needle has <= 16 distinct byte classes (see prefilter.cu).

// match_haystack_2_typos (src/prefilter/algo/ascii_typos.rs:113-251) on block masks: NP = 3 paths with their own
// chunk masks; NP = 2 is match_haystack_1_typo again (== masks_k1, kept as a cross-check).
template <int NP>
FRZ_PF_FN bool masks_paths(const uint4* base, const FrzPatternDev& pat, const uint8_t* __restrict__ cid_s,
                           uint2 (*occ)[32], int len, bool active, int* ostart, int* oend) {
    const int units = active ? (len + 15) >> 4 : 0;
    const uint32_t lane = FRZ_PF_LANE;
    const int n = pat.n, L = pat.pf_lanes, K = NP - 1;
    int idx[NP];
#pragma unroll
    for (int k = 0; k < NP; k++) idx[k] = k;
    int ms = 0x7fffffff, end = -1;
    int state = 2;   // 0 running, 1 found, 2 rejected / idle
    if (active) state = n <= K ? 1 : (len == 0 ? 2 : 0);
    if (active && n <= K) ms = 0;
    const int max_len = __reduce_max_sync(0xffffffffu, active ? len : 0);
    const uint64_t lmask = lowmask64(L);
    for (int blk = 0; blk * 64 < max_len; blk++) {
        build_block_masks(base, units, blk, pat, occ, lane);
        __syncwarp();
        const int rem = len - blk * 64;
        const uint64_t valid = rem > 0 ? lowmask64(rem) : 0ull;
        // find_end_pos_with_typos: 1 + last occurrence of any of the last K + 1 needle bytes, else len
        if (n > K) {
            uint64_t lastm = 0;
            for (int i = n - 1 - K; i < n; i++) lastm |= u2_to_u64(occ[pat.cid[i]][lane]);
            lastm &= valid;
            if (lastm) end = blk * 64 + 64 - __clzll((long long)lastm);
        }
        int cs = blk * 64;
        bool in_blk = state == 0 && rem > 0;
        bool init = true;
        uint64_t m[NP], c[NP];
#pragma unroll
        for (int k = 0; k < NP; k++) { m[k] = 0; c[k] = 0; }
        while (__any_sync(0xffffffffu, in_blk)) {
            if (in_blk) {
                const int sh = cs - blk * 64;
                if (init) {
                    const uint64_t cm = (valid >> sh) & lmask;
#pragma unroll
                    for (int k = 0; k < NP; k++) { m[k] = (u2_to_u64(occ[cid_s[idx[k]]][lane]) >> sh) & lmask; c[k] = cm; }
                    init = false;
                }
                bool adv = false;
#pragma unroll
                for (int k = 1; k < NP; k++) {
                    if (!in_blk) break;
                    const int cand = idx[k - 1] + 1;
                    if (cand > idx[k]) {
                        if (cand == n) { state = 1; in_blk = false; }
                        else { idx[k] = cand; c[k] = c[k - 1]; m[k] = (u2_to_u64(occ[cid_s[cand]][lane]) >> sh) & lmask; }
                    } else if (cand == idx[k] && c[k - 1] > c[k]) c[k] = c[k - 1];
                }
#pragma unroll
                for (int k = 0; k < NP; k++) {
                    if (!in_blk) break;
                    const uint64_t x = m[k] & c[k];
                    if (!x) continue;
                    ms = min(ms, cs + __ffsll((long long)x) - 1);
                    idx[k]++;
                    if (k > 0 && idx[k] >= n) { state = 1; in_blk = false; break; }
                    c[k] &= ~(x ^ (x - 1));
                    m[k] = (u2_to_u64(occ[cid_s[idx[k]]][lane]) >> sh) & lmask;
                    adv = true;
                }
                if (in_blk && !adv) {   // next chunk
                    cs += L;
                    init = true;
                    if (cs >= len) { state = 2; in_blk = false; }
                    else if (cs >= blk * 64 + 64) in_blk = false;
                }
            }
        }
        __syncwarp();
    }
    *ostart = ms == 0x7fffffff ? 0 : ms;
    *oend = end < 0 ? len : end;
    return state == 1;
}

// match_haystack_many_typos_impl (ascii_typos.rs:254-360) on block masks: k + 1 paths sharing one chunk mask, every
// path that matches the first available hit advances.
FRZ_PF_FN bool masks_many(const uint4* base, const FrzPatternDev& pat, const uint8_t* __restrict__ cid_s,
                          uint2 (*occ)[32], int len, bool active, int* ostart, int* oend) {
    const int units = active ? (len + 15) >> 4 : 0;
    const uint32_t lane = FRZ_PF_LANE;
    const int n = pat.n, L = pat.pf_lanes, K = pat.max_typos;   // K <= 15 (host guard)
    const int paths = K + 1;
    int idx[16];
    uint64_t nm[16];
    for (int k = 0; k < 16; k++) { idx[k] = 0; nm[k] = 0; }
    int ms = 0x7fffffff, end = -1;
    int state = 2;
    if (active) state = n <= K ? 1 : (len == 0 ? 2 : 0);
    if (active && n <= K) ms = 0;
    const int max_len = __reduce_max_sync(0xffffffffu, active ? len : 0);
    const uint64_t lmask = lowmask64(L);
    for (int blk = 0; blk * 64 < max_len; blk++) {
        build_block_masks(base, units, blk, pat, occ, lane);
        __syncwarp();
        const int rem = len - blk * 64;
        const uint64_t valid = rem > 0 ? lowmask64(rem) : 0ull;
        if (n > K) {
            uint64_t lastm = 0;
            for (int i = n - 1 - K; i < n; i++) lastm |= u2_to_u64(occ[pat.cid[i]][lane]);
            lastm &= valid;
            if (lastm) end = blk * 64 + 64 - __clzll((long long)lastm);
        }
        int cs = blk * 64;
        bool in_blk = state == 0 && rem > 0;
        bool init = true;
        uint64_t chunk_mask = 0;
        while (__any_sync(0xffffffffu, in_blk)) {
            if (in_blk) {
                const int sh = cs - blk * 64;
                if (init) {
                    chunk_mask = (valid >> sh) & lmask;
                    for (int k = 0; k < paths; k++) nm[k] = (u2_to_u64(occ[cid_s[idx[k]]][lane]) >> sh) & lmask;
                    init = false;
                }
                for (int k = 1; k < paths && in_blk; k++) {
                    const int cand = idx[k - 1] + 1;
                    if (cand > idx[k]) {
                        if (cand == n) { state = 1; in_blk = false; }
                        else { idx[k] = cand; nm[k] = (u2_to_u64(occ[cid_s[cand]][lane]) >> sh) & lmask; }
                    }
                }
                if (in_blk) {
                    uint64_t mm = 0;
                    for (int k = 0; k < paths; k++) mm |= nm[k];
                    const uint64_t matches = mm & chunk_mask;
                    if (!matches) {   // next chunk
                        cs += L;
                        init = true;
                        if (cs >= len) { state = 2; in_blk = false; }
                        else if (cs >= blk * 64 + 64) in_blk = false;
                    } else {
                        const int hit_pos = __ffsll((long long)matches) - 1;
                        const uint64_t hit = matches & lowmask64(hit_pos + 1);
                        ms = min(ms, cs + hit_pos);
                        for (int k = 0; k < paths && in_blk; k++) {
                            if (!(nm[k] & hit)) continue;
                            idx[k]++;
                            if (idx[k] == n) { state = 1; in_blk = false; }
                            else nm[k] = (u2_to_u64(occ[cid_s[idx[k]]][lane]) >> sh) & lmask;
                        }
                        chunk_mask &= ~(hit ^ (hit - 1));
                    }
                }
            }
        }
        __syncwarp();
    }
    *ostart = ms == 0x7fffffff ? 0 : ms;
    *oend = end < 0 ? len : end;
    return state == 1;
}

}  // namespace frzpf
