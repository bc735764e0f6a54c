// sw_core.cuh — the register Smith-Waterman core of sw.cu (SwCore, RowStore, window assembly), in a header so that
// the SAME source is compiled by nvcc for the kernels and by g++ for tests/test_kernel_logic_cpu.py, which runs it on
// the CPU against the oracle (the CUDA SIMD-in-register intrinsics get scalar stand-ins below).  See sw.cu for the
// algorithm notes.
#pragma once
#include <stdint.h>

#include "frz_device.cuh"

#if defined(__CUDACC__)
#define FRZ_SW_FN __device__ __forceinline__
#define FRZ_SW_TID ((int)threadIdx.x)
#else
// ---- host stand-ins of the device intrinsics (exact per-lane semantics) ----
#define FRZ_SW_FN inline
#define FRZ_SW_TID 0
inline uint32_t __byte_perm(uint32_t x, uint32_t y, uint32_t s) {   // the CUDA intrinsic uses 3 bits per selector nibble
    const uint64_t v = ((uint64_t)y << 32) | x;
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) {
        const uint32_t sel = (s >> (4 * i)) & 0x7;   // (nvcc masks bit 3: `__byte_perm(x, 0, 0xBB99)` is PRMT 0x3311)
        r |= ((uint32_t)(v >> (8 * sel)) & 0xff) << (8 * i);
    }
    return r;
}
inline uint32_t __vadd2(uint32_t a, uint32_t b) { return ((a + b) & 0xffffu) | (((a >> 16) + (b >> 16)) << 16); }
inline uint32_t __vminu2(uint32_t a, uint32_t b) {
    const uint32_t lo = (a & 0xffff) < (b & 0xffff) ? (a & 0xffff) : (b & 0xffff), hi = (a >> 16) < (b >> 16) ? (a >> 16) : (b >> 16);
    return lo | (hi << 16);
}
inline uint32_t __vmaxu2(uint32_t a, uint32_t b) {
    const uint32_t lo = (a & 0xffff) > (b & 0xffff) ? (a & 0xffff) : (b & 0xffff), hi = (a >> 16) > (b >> 16) ? (a >> 16) : (b >> 16);
    return lo | (hi << 16);
}
inline uint32_t __viaddmax_s16x2_relu(uint32_t a, uint32_t b, uint32_t c) {   // per signed 16-bit lane: max(a + b, c, 0)
    uint32_t r = 0;
    for (int h = 0; h < 2; h++) {
        const int16_t x = (int16_t)(a >> (16 * h)), y = (int16_t)(b >> (16 * h)), z = (int16_t)(c >> (16 * h));
        int32_t v = (int16_t)(x + y);
        if (z > v) v = z;
        if (v < 0) v = 0;
        r |= ((uint32_t)v & 0xffffu) << (16 * h);
    }
    return r;
}
inline uint32_t max(uint32_t a, uint32_t b) { return a > b ? a : b; }   // CUDA's global max()
inline uint32_t __umulhi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t sh) { return (uint32_t)(((((uint64_t)hi) << 32) | lo) >> (sh & 31)); }
#endif

namespace frzsw {

constexpr int kSwThreads = 128;
// The non-wrapping 64-lane kernel for <= 64-byte windows keeps the haystack/bonus rows in shared memory: that brings it
// to <= 168 registers, i.e. 3 blocks (3 warps per scheduler) per SM.
template <int LANES, bool WRAP8>
constexpr bool kSw64RowsInSmem = LANES == 64 && !WRAP8;
// SwCore VAR bit: per-lane gap penalties, for scorings with gap_extend == 0 < gap_open_x (see SwCore)
constexpr int kSwVarLanePen = 16;

FRZ_SW_FN uint32_t splat16(int v) { return ((uint32_t)v & 0xffffu) * 0x00010001u; }

// PRMT with the full selector: a nibble with bit 3 set replicates the SIGN bit of the selected byte (prmt.b32 default mode).
// `__byte_perm` cannot express this (it masks the selector to 3 bits per nibble), hence the inline PTX.
FRZ_SW_FN uint32_t prmt_sign(uint32_t x, uint32_t selector) {
#if defined(__CUDA_ARCH__)
    uint32_t d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(x), "r"(0u), "r"(selector));
    return d;
#else
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) {
        const uint32_t sel = (selector >> (4 * i)) & 0xf;
        uint32_t b = (sel & 4) ? 0u : (x >> (8 * (sel & 3))) & 0xff;
        if (sel & 8) b = (b & 0x80) ? 0xff : 0x00;
        r |= b << (8 * i);
    }
    return r;
#endif
}

// per-16-bit-lane: 0xFFFF where x == 0 else 0   (x lanes are in 0..255)
FRZ_SW_FN uint32_t eqmask16(uint32_t x) {
    return __byte_perm(__vadd2(x, 0xFFFFFFFFu), 0, 0x3311);  // high byte of (x - 1): 0xFF only for x == 0 → both bytes
}
// bitwise select (mask ? a : b) as ONE LOP3 (nvcc otherwise emits and / and-not / or: three)
FRZ_SW_FN uint32_t sel(uint32_t mask, uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    uint32_t d;
    asm("lop3.b32 %0, %1, %2, %3, 0xCA;" : "=r"(d) : "r"(mask), "r"(a), "r"(b));
    return d;
#else
    return (mask & a) | (~mask & b);
#endif
}

// max(a + b, c, 0) per signed 16-bit lane
FRZ_SW_FN uint32_t addmax_relu(uint32_t a, uint32_t b, uint32_t c) { return __viaddmax_s16x2_relu(a, b, c); }

// Register array, or (for the 128-column variant, whose two score rows already fill the register
// file) a conflict-free shared-memory column [r][thread].
template <int R, bool SMEM>
struct RowStore;
template <int R>
struct RowStore<R, false> {
    uint32_t v[R];
    FRZ_SW_FN RowStore(uint32_t*) {}
    FRZ_SW_FN uint32_t get(int r) const { return v[r]; }
    FRZ_SW_FN void set(int r, uint32_t x) { v[r] = x; }
};
template <int R>
struct RowStore<R, true> {
    uint32_t* base;
    FRZ_SW_FN RowStore(uint32_t* b) : base(b + FRZ_SW_TID) {}
    FRZ_SW_FN uint32_t get(int r) const { return base[r * kSwThreads]; }
    FRZ_SW_FN void set(int r, uint32_t x) { base[r * kSwThreads] = x; }
};

// The haystack lanes and the bonus row of one window, read together by every row of the recurrence.  PAIR: both in
// shared memory, interleaved per register [r][thread]{h, b}, so that a row reads each register's pair with one LDS.64.
template <int R, bool SMEM, bool PAIR>
struct HayRows {
    RowStore<R, SMEM> h, b;
    FRZ_SW_FN HayRows(uint32_t* s) : h(s), b(s + R * kSwThreads) {}
    FRZ_SW_FN uint32_t get_h(int r) const { return h.get(r); }
    FRZ_SW_FN void set_h(int r, uint32_t x) { h.set(r, x); }
    FRZ_SW_FN void set_b(int r, uint32_t x) { b.set(r, x); }
    FRZ_SW_FN uint2 get(int r) const { return make_uint2(h.get(r), b.get(r)); }
};
template <int R, bool SMEM>
struct HayRows<R, SMEM, true> {
    uint2* base;
    FRZ_SW_FN HayRows(uint32_t* s) : base(reinterpret_cast<uint2*>(s) + FRZ_SW_TID) {}
    FRZ_SW_FN uint32_t get_h(int r) const { return base[r * kSwThreads].x; }
    FRZ_SW_FN void set_h(int r, uint32_t x) { base[r * kSwThreads].x = x; }
    FRZ_SW_FN void set_b(int r, uint32_t x) { base[r * kSwThreads].y = x; }
    FRZ_SW_FN uint2 get(int r) const { return base[r * kSwThreads]; }
};

// VAR bit 3 (8): the per-column bonus is classified on the packed bytes (4 at a time) instead of per 16-bit lane — the
// default of the non-wrapping 64-lane kernel.  Forms that were tried and removed because they were slower: one-lane
// shifts as IMAD.HI + IMAD pairs instead of PRMT, the shifted match mask folded into the gap penalty with IMAD.HI, two
// column classes instead of four.
//
// VAR bit 4 (kSwVarLanePen): the gap penalties are formed per 16-bit lane with a select on the full match mask, as
// WRAP8 does.  The default form `base + mask * gap_open_x` is one 32-bit IMAD over both lanes of a register, which is
// exact only while the low lane's sum stays below 0x10000.  It does for gap_extend >= 1, but with gap_extend == 0 and
// gap_open_x > 0 the low lane of a non-matching column sums to exactly 0x10000, and the carry takes one point off the
// high lane's penalty.  frz_launch_sw (sw.cu) selects this variant for exactly that scoring.
//
// CC (<= COLS, multiple of 8) is the number of columns actually evaluated.  Cells never depend on cells to
// their right, and a cell in column >= W + needle_len can only hold a value that decayed from a cell to its
// left in the same row (it is past the reach of the diagonal/up chains that start inside the window, and zero
// padding never matches), so it can never be the unique row maximum: evaluating the first
// min(W + n, ceil(W / LANES) * LANES) columns gives the reference's score.  Not used with WRAP8 (no monotone
// arithmetic) or a needle containing NUL; pinned by tests/test_oracle_kat.py::test_column_limit_property.
template <int LANES, int COLS, bool WRAP8, int VAR = 0, int CC = COLS>
struct SwCore {
    static constexpr int R = CC / 2;       // registers per row
    static constexpr int RL = LANES / 2;   // registers per chunk
    static constexpr int NCH = (CC + LANES - 1) / LANES;
    static constexpr bool SMEM = COLS > 64 || kSw64RowsInSmem<LANES, WRAP8>;
    static constexpr bool PAIR = COLS <= 64 && SMEM;
    static constexpr size_t smem_bytes = SMEM ? 2 * R * kSwThreads * sizeof(uint32_t) : 0;
    static constexpr bool kGaplessLastRow = !WRAP8 && COLS <= 64;   // see run()

    // ---- diagonal + up of needle row i at register r, in place (H[r-1] must still hold row i-1).  up: the needle byte
    // is an uppercase letter (rare), whose exact-case bonus moves from the non-upper to the upper haystack bytes.
    static FRZ_SW_FN void diag_up(uint32_t (&H)[R], uint32_t (&M)[R], int r, uint2 hb, const FrzPatternDev& p, int i, bool up_row) {
        const uint32_t om16 = p.om16[i], tg16 = p.tg16[i];
        const uint32_t hv = hb.x, Bv = hb.y;
        if (!WRAP8) {
            // nm: 0 where the haystack byte matches needle[i] (either case), else 1
            const uint32_t nm = __vminu2((hv | om16) ^ tg16, 0x00010001u);
            const uint32_t nmfull = nm * 0xFFFFu;
            const uint32_t prevs = r > 0 ? __byte_perm(H[r - 1], H[r], 0x5432) : __byte_perm(0u, H[0], 0x5432);
            uint32_t Dv = Bv;
            if (up_row) {
                const uint32_t t = __vadd2(hv, splat16(-'A')), d = __vadd2(hv, splat16(-('Z' + 1)));
                const uint32_t up = __byte_perm(d & ~t, 0, 0x3311);
                Dv = __vadd2(Dv, sel(up, p.k_case, splat16(-p.case_bonus)));
            }
            // no ReLU here: max(H + upd, diag, 0) below clamps anyway, and VIADDMNMX has no zero operand, so the ReLU
            // form costs a register holding zero (or a PRMT rematerialising one per use)
            const uint32_t diag = __vadd2(prevs, sel(nmfull, p.k_neg_mis, Dv));
            const uint32_t upd = (VAR & kSwVarLanePen) ? sel(M[r] * 0xFFFFu, p.k_up_plain, p.k_up_open)
                                                       : p.k_up_open + M[r] * (uint32_t)p.gap_open_x;   // M[r] still row i-1
            H[r] = addmax_relu(H[r], upd, diag);
            M[r] = nm;
        } else {
            const bool folded = p.om[i] != 0;  // case-insensitive letter: exact-case mask differs from match mask
            const uint32_t mmn = eqmask16((hv | om16) ^ tg16);
            const uint32_t prevs = r > 0 ? __byte_perm(H[r - 1], H[r], 0x5432) : __byte_perm(0u, H[0], 0x5432);
            const uint32_t ex = folded ? eqmask16(hv ^ p.c16[i]) : mmn;
            uint32_t d = __vadd2(prevs, mmn & Bv) & 0x00FF00FFu;        // wrapping u8 add
            d = addmax_relu(d, p.k_neg_mis, 0u);                         // saturating sub
            const uint32_t diag = __vadd2(d, ex & p.k_case) & 0x00FF00FFu;  // wrapping u8 add
            const uint32_t upd = sel(M[r], p.k_up_open, p.k_up_plain);       // M[r] still row i-1
            H[r] = addmax_relu(H[r], upd, diag);
            M[r] = mmn;
        }
    }

    // hw: CC/4 words of window bytes, zero beyond W
    static FRZ_SW_FN uint32_t run(const uint32_t (&hw)[CC / 4], int W, const FrzPatternDev& p, bool include_prefix,
                                   uint32_t* smem) {
        HayRows<R, SMEM, PAIR> rows(smem);
        // expand bytes to one per 16-bit lane
#pragma unroll
        for (int i = 0; i < CC / 4; i++) {
            rows.set_h(2 * i, __byte_perm(hw[i], 0, 0x4140));
            rows.set_h(2 * i + 1, __byte_perm(hw[i], 0, 0x4342));
        }
        // ---- per-column bonus (ascii.rs:64-101) ----
        if ((VAR & 8) && !WRAP8) {
            // VAR bit 3 (set by every k_sw64 launch without wrap8): classify the haystack bytes four at a time on the
            // PACKED words (the flag of a byte is bit 7 of its position) and expand only the three masks the bonus needs.
            // Same values as the per-lane form below, about 40% fewer instructions and a smaller body.
            const uint32_t capb = p.k_cap, delb = p.k_delim;
            const uint32_t base2 = __vadd2(p.k_base, p.k_neg_mis);
            uint32_t prev_lo = 0, prev_dl = 0;   // flags of the previous word (byte 3 feeds byte 0 of this one)
#pragma unroll
            for (int k = 0; k < CC / 4; k++) {
                const uint32_t w = hw[k];
                const uint32_t x7 = w & 0x7f7f7f7fu;
                // lo <= b <= hi for bytes < 128: bit 7 of (x7 + 0x80 - lo) is "b >= lo", bit 7 of (x7 + 0x7f - hi) is "b > hi"
                const uint32_t up_f = (x7 + 0x01010101u * (0x80 - 'A')) & ~(x7 + 0x01010101u * (0x7f - 'Z')) & ~w;
                const uint32_t lo_f = (x7 + 0x01010101u * (0x80 - 'a')) & ~(x7 + 0x01010101u * (0x7f - 'z')) & ~w;
                const uint32_t dg_f = (x7 + 0x01010101u * (0x80 - '0')) & ~(x7 + 0x01010101u * (0x7f - '9')) & ~w;
                const uint32_t dl_f = ~(up_f | lo_f | dg_f | w);            // not letter, digit or >= 128 (padding zeros ARE delimiters)
                const uint32_t lo_sh = (lo_f << 8) | (prev_lo >> 24);       // flag of the previous byte
                const uint32_t dl_sh = (dl_f << 8) | (prev_dl >> 24);
                const uint32_t cap_f = up_f & lo_sh;
                const uint32_t del_f = dl_sh & ~dl_f;
                prev_lo = lo_f;
                prev_dl = dl_f;
#pragma unroll
                for (int h = 0; h < 2; h++) {   // expand bit 7 of bytes (2h, 2h+1) to 16-bit lane masks
                    const uint32_t sgn = h ? 0xBBAAu : 0x9988u;   // sign bit of byte 2h → low lane, of byte 2h+1 → high lane
                    const uint32_t cap_m = prmt_sign(cap_f, sgn), del_m = prmt_sign(del_f, sgn), up_m = prmt_sign(up_f, sgn);
                    uint32_t bonus = __vadd2(__vadd2(del_m & delb, cap_m & capb), base2);
                    if (k == 0 && h == 0 && include_prefix) bonus = __vadd2(bonus, (uint32_t)p.prefix_bonus & 0xffffu);
                    bonus = __vadd2(bonus, ~up_m & p.k_case);
                    rows.set_b(2 * k + h, bonus);
                }
            }
        } else {
            const uint32_t capb = p.k_cap, delb = p.k_delim, base = p.k_base;
            uint32_t prev_lower = 0, prev_delim = 0;  // masks of the previous register
#pragma unroll
            for (int r = 0; r < R; r++) {
                const uint32_t b = rows.get_h(r);
                // range tests on lanes in 0..255:  lo <= b <= hi  ⇔  (b-lo) >= 0 && (b-hi-1) < 0
                auto in_range = [&](int lo, int hi) {
                    uint32_t t = __vadd2(b, splat16(-lo));
                    uint32_t d = __vadd2(b, splat16(-(hi + 1)));
                    return __byte_perm(d & ~t, 0, 0x3311);   // high byte of each lane (0xFF or 0x00 here) → both bytes
                };
                const uint32_t upper = in_range('A', 'Z');
                const uint32_t lower = in_range('a', 'z');
                const uint32_t digit = in_range('0', '9');
                const uint32_t high = __byte_perm(__vadd2(b, splat16(-128)), 0, 0x3311) ^ 0xFFFFFFFFu;  // b >= 128
                const uint32_t delim = ~(upper | lower | digit | high);
                const uint32_t lower_sh = __byte_perm(prev_lower, lower, 0x5432);
                const uint32_t delim_sh = __byte_perm(prev_delim, delim, 0x5432);
                const uint32_t cap_m = upper & lower_sh;
                const uint32_t del_m = delim_sh & ~delim;
                uint32_t bonus = __vadd2(__vadd2(del_m & delb, cap_m & capb), base);
                if (r == 0 && include_prefix) bonus = __vadd2(bonus, (uint32_t)p.prefix_bonus & 0xffffu);
                if (WRAP8) bonus &= 0x00FF00FFu;
                // Non-wrapping variant stores D = bonus - mismatch + (exact-case bonus where the haystack byte
                // is not an uppercase letter): for a needle byte that is not an uppercase letter, "exact case"
                // ⇔ match && !upper(hay) (a lowercase letter matches {c, C}; a non-letter matches only itself),
                // so a matched cell's whole diagonal increment is D and the row needs no exact-case mask.
                if (!WRAP8) bonus = __vadd2(__vadd2(bonus, p.k_neg_mis), ~upper & p.k_case);
                rows.set_b(r, bonus);
                prev_lower = lower;
                prev_delim = delim;
            }
        }
        uint32_t H[R], M[R];
#pragma unroll
        for (int r = 0; r < R; r++) { H[r] = 0; M[r] = WRAP8 ? 0u : 0x00010001u; }  // row 0: no matches

        // fma-pipe helpers.  The ALU pipe (LOP3 / PRMT / VIADD / VIADDMNMX) issues one warp instruction
        // every two cycles per scheduler and the first version of this loop saturated it with the FMA
        // pipe idle.  Match masks are therefore kept as 0/1 per lane so that every
        // "penalty = base - mask * gap_open" is one IMAD, and lane shifts use IMAD / IMAD.HI too.
        const uint32_t gopx = (uint32_t)p.gap_open_x;
        for (int i = 0; i < p.n; i++) {
            const bool upper_row = (uint32_t)(p.c[i] - 'A') <= 25u;  // exact case ⇔ match && upper(hay)
            // ---- diagonal + up, in place, high register first.  <= 64 columns: one branch per row picks one of two
            // bodies, so the common one has no per-register test (the 128-column variant keeps the test: two bodies
            // make it spill).  The unroll count is explicit because a plain `#pragma unroll` leaves the rare copy
            // rolled, which puts H[] in local memory.
            if (COLS <= 64 && !WRAP8 && upper_row) {
#pragma unroll R
                for (int r = R - 1; r >= 0; r--) diag_up(H, M, r, rows.get(r), p, i, true);
            } else {
#pragma unroll R
                for (int r = R - 1; r >= 0; r--) diag_up(H, M, r, rows.get(r), p, i, COLS > 64 && !WRAP8 && upper_row);
            }
            // The last row's gap propagation cannot change the score.  Every gap penalty is <= 0 per lane and every cell
            // >= 0, so a gap step H[j] = max(H[j - s] + pen, H[j], 0) never raises a cell above the largest cell to its
            // left, and the maximum over the leading chunks read below is the one the diagonal + up step leaves.  Not
            // with WRAP8 (the u8 wrap makes the arithmetic non-monotone), and not for 128 columns, whose rows already
            // spill and which ptxas then spills further.
            if (kGaplessLastRow && i == p.n - 1) break;
            // ---- horizontal gap propagation, chunk by chunk (ascii_gap.rs gap_step!) ----
#pragma unroll
            for (int c = 0; c < NCH; c++) {
                const int lo = c * RL, hi = (lo + RL < R) ? lo + RL : R;
#pragma unroll
                for (int s = 1, si = 0; s < LANES; s <<= 1, si++) {
                    const uint32_t penA = p.k_pen_a[si];
                    const uint32_t penB = p.k_pen_b[si];
#pragma unroll
                    for (int r = hi - 1; r >= lo; r--) {
                        uint32_t sh, smm;
                        if (s == 1 && !WRAP8) {
                            sh = r == 0 ? __byte_perm(0u, H[0], 0x5432) : __byte_perm(H[r - 1], H[r], 0x5432);
                            smm = r == 0 ? __byte_perm(0u, M[0], 0x5432) : __byte_perm(M[r - 1], M[r], 0x5432);
                        } else if (s == 1) {
                            if (r == 0) { sh = __byte_perm(0u, H[0], 0x5432); smm = __byte_perm(0u, M[0], 0x5432); }
                            else { sh = __byte_perm(H[r - 1], H[r], 0x5432); smm = __byte_perm(M[r - 1], M[r], 0x5432); }
                        } else {
                            const int src = r - s / 2;
                            if (src < 0) continue;  // shifted-in lanes of the first chunk are zero: no-op
                            sh = H[src];
                            smm = M[src];
                        }
                        const uint32_t pen = WRAP8                    ? sel(smm, penB, penA)
                                             : (VAR & kSwVarLanePen) ? sel(smm * 0xFFFFu, penA, penB)
                                                                     : penB + smm * gopx;
                        H[r] = addmax_relu(sh, pen, H[r]);
                    }
                }
            }
        }
        // ---- max over the chunks the reference actually has: ceil(W / LANES) ----
        const int nch = (W + LANES - 1) / LANES;
        uint32_t mx = 0;
#pragma unroll
        for (int r = 0; r < R; r++)
            if (r < nch * RL) mx = __vmaxu2(mx, H[r]);
        return max(mx & 0xffffu, mx >> 16);
    }
};

// Window bytes [startlo, startlo + W) of the NU staged 16-byte units → COLS/4 zero-padded words.
template <int COLS>
FRZ_SW_FN void window_from_units(const uint4 (&u)[(COLS + 15) / 16 + 1], uint32_t startlo, int W,
                                                  uint32_t (&hw)[COLS / 4]) {
    constexpr int NU = (COLS + 15) / 16 + 1;
    uint32_t w[NU * 4 + 4];
#pragma unroll
    for (int k = 0; k < NU; k++) { w[4 * k] = u[k].x; w[4 * k + 1] = u[k].y; w[4 * k + 2] = u[k].z; w[4 * k + 3] = u[k].w; }
#pragma unroll
    for (int k = NU * 4; k < NU * 4 + 4; k++) w[k] = 0;
    const uint32_t ws = startlo >> 2, bs = (startlo & 3) * 8;
    if (ws & 2) {
#pragma unroll
        for (int k = 0; k < NU * 4 + 2; k++) w[k] = w[k + 2];
    }
    if (ws & 1) {
#pragma unroll
        for (int k = 0; k < NU * 4 + 3; k++) w[k] = w[k + 1];
    }
#pragma unroll
    for (int k = 0; k < COLS / 4; k++) {
        uint32_t v = __funnelshift_r(w[k], w[k + 1], bs);
        int rem = W - 4 * k;
        if (rem <= 0) v = 0;
        else if (rem < 4) v &= (1u << (8 * rem)) - 1;
        hw[k] = v;
    }
}

// exact = include_exact && needle_bytes == window (src/matcher/algo.rs:245); byte-exact compare
template <int NW>
FRZ_SW_FN bool window_equals_needle(const uint32_t (&hw)[NW], int W, const FrzPatternDev& p) {
    if (W != p.n) return false;
    bool eq = true;
#pragma unroll
    for (int k = 0; k < NW; k++) {
        uint32_t nw = 0;
#pragma unroll
        for (int b = 0; b < 4; b++)
            if (4 * k + b < p.n && 4 * k + b < FRZ_MAX_NEEDLE) nw |= (uint32_t)p.c[4 * k + b] << (8 * b);
        if (4 * k < p.n) eq = eq && (hw[k] == nw);
    }
    return eq;
}

}  // namespace frzsw
