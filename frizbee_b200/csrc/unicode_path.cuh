// unicode_path.cuh — the UNICODE = true specialisations of the hot path (SURVEY.md §8(f) rank 4), per haystack:
//   src/prefilter/algo/unicode.rs         match_haystack_unicode (0 typos), unicode_char_mask, find_last_unicode_char_pos
//   src/prefilter/algo/unicode_typos.rs   1 / 2 / N-typo path trackers, find_end_pos_with_unicode_typos
//   src/smith_waterman/algo/unicode.rs    score_haystack_unicode: rows are needle SCALARS, columns haystack BYTES
//   src/smith_waterman/algo/unicode_gap.rs  propagate_unicode_{8,16,32,64}_lane (continuation bytes are transport lanes)
//   src/literal/algo.rs:159-230           matches_at / score_at with UNICODE = true
//   src/smith_waterman/greedy.rs:7-91     match_greedy for windows > 1024 bytes
//
// Correctness path, not tuned: one thread runs one haystack start to finish, lane vectors are plain arrays and the
// two per-row state vectors live in a caller-provided scratch.  Everything here is `__host__ __device__` and reads
// the haystack through a byte accessor, so the same code is compiled for the GPU (unicode.cu, packed-corpus
// accessor) and for the CPU by tests/test_unicode_device_code.py, which checks it against the oracle without a GPU.
#pragma once
#include <stdint.h>

#include "frz_hd.cuh"

#define FRZ_U_MAX_SCALARS 64   // needle scalars (needle bytes are capped at 64)
#define FRZ_U_MAX_LANES 64
#define FRZ_U_MAX_WINDOW 1024  // src/smith_waterman/algo/mod.rs:18 (MAX_HAYSTACK_LEN)

// The needle as the unicode kernels see it (case_needle_unicode, src/prefilter/mod.rs:71-96) plus the byte-level
// case_needle pairs the greedy scorer uses (src/prefilter/mod.rs:49-65).
struct FrzUNeedle {
    uint8_t c[64];        // needle bytes
    uint8_t f[64];        // bytes of the case-flipped scalars, scalar by scalar (same lengths)
    uint8_t bflip[64];    // per-byte ASCII flip (case_needle), for match_greedy
    uint8_t off[FRZ_U_MAX_SCALARS];   // first byte of scalar i
    uint8_t len[FRZ_U_MAX_SCALARS];   // UTF-8 length of scalar i
    int32_t n;            // scalars
    int32_t nbytes;       // bytes
};

// scoring constants; `*_x` as the reference splats them into lanes (u8-truncated in the u8 family), raw_* in u16
struct FrzUScoring {
    int32_t gex, gopx, match_x, mismatch, case_bonus, cap_bonus, delim_bonus, prefix_bonus;
    int32_t raw_match, raw_gap_open, raw_gap_extend, raw_prefix, raw_cap, raw_case, raw_delim, exact_bonus;
};

namespace frzu {

FRZ_HD int ctz64(uint64_t m) {
#if defined(__CUDA_ARCH__)
    return __ffsll((long long)m) - 1;
#else
    return __builtin_ctzll(m);
#endif
}
FRZ_HD int clz64(uint64_t m) {
#if defined(__CUDA_ARCH__)
    return __clzll((long long)m);
#else
    return __builtin_clzll(m);
#endif
}

// ------------------------------------------------------------------------------------------------ prefilter
// Masks hold LANES meaningful low bits (u16/u32/u64 in the reference, src/prefilter/backend/mod.rs:45-114).
template <class Hay>
struct Pf {
    const FrzUNeedle& nd;
    const Hay& hay;
    int len;     // bytes visible through `hay` (a sub-slice view shifts `base`)
    int base;    // offset of this view inside the accessor
    int lanes;

    FRZ_HD uint64_t all() const { return lanes == 64 ? ~0ull : ((1ull << lanes) - 1); }
    FRZ_HD uint64_t first_n(int n) const { return n >= lanes ? all() : ((1ull << n) - 1); }
    FRZ_HD int lz(uint64_t m) const { return clz64(m) - (64 - lanes); }
    FRZ_HD static uint64_t ctl(uint64_t mask, uint64_t hit) { return mask & ~(hit ^ (hit - 1)); }  // clear_through_lowest
    // equality mask of the chunk at `pos`; lanes past the end are over-read garbage in the reference and masked by
    // every caller (the last-byte window is the shortest): "no match" here
    FRZ_HD uint64_t eq(int pos, uint8_t b) const {
        uint64_t m = 0;
        for (int i = 0; i < lanes; i++) {
            const int q = pos + i;
            if (q >= len) break;
            if (hay(base + q) == b) m |= 1ull << i;
        }
        return m;
    }
    FRZ_HD uint64_t prefix(int start, int cl, const uint8_t* ch) const {   // match_unicode_char_prefix
        uint64_t m = all();
        for (int k = 0; k < cl - 1; k++) m &= eq(start + k, ch[k]);
        return m;
    }
    FRZ_HD uint64_t variant(int start, uint64_t chunk_mask, int cl, const uint8_t* ch) const {  // char_variant_mask
        uint64_t mask = eq(start + cl - 1, ch[cl - 1]) & chunk_mask;
        if (mask && cl > 1) mask &= prefix(start, cl, ch);
        return mask;
    }
    FRZ_HD uint64_t char_mask(int start, int i) const {   // unicode_char_mask of needle scalar i
        const int cl = nd.len[i];
        if (start + cl > len) return 0;
        const uint64_t chunk_mask = first_n(len - (start + cl - 1));
        return variant(start, chunk_mask, cl, nd.c + nd.off[i]) | variant(start, chunk_mask, cl, nd.f + nd.off[i]);
    }
};

template <class Hay>
FRZ_HD int find_last_unicode_char_pos(const Pf<Hay>& p, int ni, int off) {
    Pf<Hay> s{p.nd, p.hay, p.len - off, p.base + off, p.lanes};
    const int len = s.len, cl = p.nd.len[ni];
    const uint8_t* c = p.nd.c + p.nd.off[ni];
    const uint8_t* f = p.nd.f + p.nd.off[ni];
    int start = len > s.lanes + cl - 1 ? len - (s.lanes + cl - 1) : 0;
    for (;;) {
        const uint64_t chunk_mask = s.first_n(len - (start + cl - 1));
        uint64_t mask = (s.eq(start + cl - 1, c[cl - 1]) | s.eq(start + cl - 1, f[cl - 1])) & chunk_mask;
        if (mask && cl > 1) mask &= s.prefix(start, cl, c) | s.prefix(start, cl, f);
        if (mask) return start + s.lanes - s.lz(mask) + cl - 1;
        if (start == 0) break;
        start = start > s.lanes ? start - s.lanes : 0;
    }
    return len;
}

template <class Hay>
FRZ_HD bool prefilter_k0(const Pf<Hay>& p, int* ostart, int* oend) {   // unicode.rs:120-222
    const int len = p.len, n = p.nd.n;
    if (len == 0) { *ostart = 0; *oend = 0; return false; }
    bool can_skip = true;
    int ms = 0, ni = 0, start = 0;
    while (start + p.nd.len[ni] <= len) {
        int char_len = p.nd.len[ni];
        uint64_t valid = p.first_n(len - (start + char_len - 1));
        uint64_t available = p.all();
        for (;;) {
            const uint64_t chunk_mask = available & valid;
            const int cl = p.nd.len[ni];
            const uint64_t mask = p.variant(start, chunk_mask, cl, p.nd.c + p.nd.off[ni]) |
                                  p.variant(start, chunk_mask, cl, p.nd.f + p.nd.off[ni]);
            if (!mask) break;
            available = Pf<Hay>::ctl(available, mask);
            if (can_skip) { ms = start + ctz64(mask); can_skip = false; }
            if (ni + 1 < n) {
                ni++;
                if (p.nd.len[ni] != char_len) {
                    if (start + p.nd.len[ni] > len) break;
                    char_len = p.nd.len[ni];
                    valid = p.first_n(len - (start + char_len - 1));
                }
            } else if (start + cl - 1 + p.lanes >= len) {
                *ostart = ms;
                *oend = start + p.lanes - p.lz(mask) + cl - 1;
                return true;
            } else {
                *ostart = ms;
                *oend = start + find_last_unicode_char_pos(p, ni, start);
                return true;
            }
        }
        start += p.lanes;
    }
    *ostart = ms;
    *oend = len;
    return false;
}

template <class Hay>
FRZ_HD int find_end_pos_with_typos(const Pf<Hay>& p, int max_typos) {   // unicode_typos.rs:486-508
    const int len = p.len, n = p.nd.n;
    const int first = n - 1 - max_typos;
    int start = len > p.lanes ? len - p.lanes : 0;
    for (;;) {
        int end_pos = 0;
        for (int i = first; i < n; i++) {
            const uint64_t mask = p.char_mask(start, i);
            if (mask) {
                const int e = start + p.lanes - p.lz(mask) + p.nd.len[i] - 1;
                if (e > end_pos) end_pos = e;
            }
        }
        if (end_pos) return end_pos;
        if (start == 0) break;
        start = start > p.lanes ? start - p.lanes : 0;
    }
    return len;
}

// unicode_typos.rs:336-472.  The 1- and 2-typo specialisations (:15-333) are the same tracker with the chunk masks
// kept per path; they are restated separately below because their tie handling differs (per-path chunk masks).
template <class Hay>
FRZ_HD bool prefilter_many(const Pf<Hay>& p, int max_typos, int* ostart, int* oend) {
    const int len = p.len, n = p.nd.n;
    if (n <= max_typos) { *ostart = 0; *oend = len; return true; }
    if (len == 0) { *ostart = 0; *oend = 0; return false; }
    const int path_count = max_typos + 1;   // <= 16 (host guard)
    int idx[16];
    uint64_t nm[16];
    for (int k = 0; k < path_count; k++) { idx[k] = 0; nm[k] = 0; }
    int ms = 0x7fffffff;
    for (int start = 0; start < len; start += p.lanes) {
        uint64_t chunk_mask = p.all();
        for (int k = 0; k < path_count; k++) nm[k] = p.char_mask(start, idx[k]);
        for (;;) {
            for (int k = 1; k < path_count; k++) {
                const int cand = idx[k - 1] + 1;
                if (cand > idx[k]) {
                    if (cand == n) { *ostart = ms; *oend = find_end_pos_with_typos(p, max_typos); return true; }
                    idx[k] = cand;
                    nm[k] = p.char_mask(start, cand);
                }
            }
            uint64_t mm = 0;
            for (int k = 0; k < path_count; k++) mm |= nm[k];
            const uint64_t matches = mm & chunk_mask;
            if (!matches) break;
            const int hit_pos = ctz64(matches);
            const uint64_t hit = matches & p.first_n(hit_pos + 1);
            if (start + hit_pos < ms) ms = start + hit_pos;
            for (int k = 0; k < path_count; k++) {
                if (!(nm[k] & hit)) continue;
                idx[k]++;
                if (idx[k] == n) { *ostart = ms; *oend = find_end_pos_with_typos(p, max_typos); return true; }
                nm[k] = p.char_mask(start, idx[k]);
            }
            chunk_mask = Pf<Hay>::ctl(chunk_mask, hit);
        }
    }
    *ostart = ms == 0x7fffffff ? 0 : ms;
    *oend = len;
    return false;
}

// unicode_typos.rs:15-143 (1 typo) and :146-333 (2 typos): NP = 2 or 3 paths with their own chunk masks
template <int NP, class Hay>
FRZ_HD bool prefilter_paths(const Pf<Hay>& p, int* ostart, int* oend) {
    const int len = p.len, n = p.nd.n;
    if (n <= NP - 1) { *ostart = 0; *oend = len; return true; }
    if (len == 0) { *ostart = 0; *oend = 0; return false; }
    int idx[NP];
    for (int k = 0; k < NP; k++) idx[k] = k;
    int ms = 0x7fffffff;
    for (int start = 0; start < len; start += p.lanes) {
        uint64_t m[NP], c[NP];
        for (int k = 0; k < NP; k++) { m[k] = p.char_mask(start, idx[k]); c[k] = p.all(); }
        for (;;) {
            bool advanced = false;
            for (int k = 1; k < NP; k++) {
                const int cand = idx[k - 1] + 1;
                if (cand > idx[k]) {
                    if (cand == n) { *ostart = ms; *oend = find_end_pos_with_typos(p, NP - 1); return true; }
                    idx[k] = cand; c[k] = c[k - 1]; m[k] = p.char_mask(start, cand);
                } else if (cand == idx[k] && c[k - 1] > c[k]) {
                    c[k] = c[k - 1];
                }
            }
            for (int k = 0; k < NP; k++) {
                const uint64_t x = m[k] & c[k];
                if (!x) continue;
                if (start + ctz64(x) < ms) ms = start + ctz64(x);
                idx[k]++;
                if (k > 0 && idx[k] >= n) { *ostart = ms; *oend = find_end_pos_with_typos(p, NP - 1); return true; }
                c[k] = Pf<Hay>::ctl(c[k], x);
                m[k] = p.char_mask(start, idx[k]);
                advanced = true;
            }
            if (!advanced) break;
        }
    }
    *ostart = ms == 0x7fffffff ? 0 : ms;
    *oend = len;
    return false;
}

// Prefilter::match_haystack_unicode* dispatch (src/matcher/algo.rs:171-193); max_typos < 0 = NO_PREFILTER
template <class Hay>
FRZ_HD bool prefilter(const FrzUNeedle& nd, const Hay& hay, int len, int lanes, int max_typos, int* start, int* end) {
    if (max_typos < 0) { *start = 0; *end = len; return true; }
    Pf<Hay> p{nd, hay, len, 0, lanes};
    if (max_typos == 0) return prefilter_k0(p, start, end);
    if (max_typos == 1) return prefilter_paths<2>(p, start, end);
    if (max_typos == 2) return prefilter_paths<3>(p, start, end);
    return prefilter_many(p, max_typos, start, end);
}

// ------------------------------------------------------------------------------------------------ Smith-Waterman
// Lane vectors of LANES u16 cells holding u8 or u16 values (wrapping add / zero-saturating sub / max),
// src/smith_waterman/backend/scalar.rs:163-354.
struct Ar {
    int lanes;
    uint16_t full;   // 0xFF or 0xFFFF
    FRZ_HD uint16_t add(uint16_t a, uint16_t b) const { return (uint16_t)((a + b) & full); }
    FRZ_HD static uint16_t subs(uint16_t a, uint16_t b) { return a > b ? (uint16_t)(a - b) : (uint16_t)0; }
    FRZ_HD static uint16_t mx(uint16_t a, uint16_t b) { return a > b ? a : b; }
};
// shift_right_padded::<L>: lane i takes a[i - L], the low L lanes take the top L lanes of `adj`
FRZ_HD uint16_t srp(const uint16_t* a, const uint16_t* adj, int lanes, int L, int i) { return i >= L ? a[i - L] : adj[lanes - L + i]; }

// propagate_unicode_N_lane (unicode_gap.rs:196-262): `row`/`pend` updated in place; cgex/adj_cgex/send/adj_send are
// scratch copies the steps mutate.
FRZ_HD void propagate_unicode(const Ar& A, uint16_t* row, uint16_t* pend, const uint16_t* adj_row, const uint16_t* adj_pend,
                              uint16_t* cgex, uint16_t* adj_cgex, uint16_t* send, uint16_t* adj_send, uint16_t gop, uint16_t gex) {
    const int L = A.lanes;
    uint16_t total = gex;
    uint16_t t_row[FRZ_U_MAX_LANES], t_pend[FRZ_U_MAX_LANES], t_a[FRZ_U_MAX_LANES], t_b[FRZ_U_MAX_LANES];
    for (int s = 1;; s <<= 1) {
        // unicode_gap_step::<s>
        for (int i = 0; i < L; i++) {
            const uint16_t sh_row = srp(row, adj_row, L, s, i);
            const uint16_t sh_pend = srp(pend, adj_pend, L, s, i);
            const uint16_t scalar_gex = Ar::subs(total, cgex[i]);
            const uint16_t crossed = sh_pend & send[i];
            const uint16_t pen = A.add(scalar_gex, gop & crossed);
            t_row[i] = Ar::mx(row[i], Ar::subs(sh_row, pen));
            t_pend[i] = Ar::mx(pend[i], Ar::subs(sh_pend, send[i]));
        }
        for (int i = 0; i < L; i++) { row[i] = t_row[i]; pend[i] = t_pend[i]; }
        if (s >= L / 2) break;
        // prepare_next_unicode_gap_step::<s>
        for (int i = 0; i < L; i++) {
            t_a[i] = A.add(cgex[i], srp(cgex, adj_cgex, L, s, i));
            t_b[i] = Ar::mx(send[i], srp(send, adj_send, L, s, i));
        }
        for (int i = L - 1; i >= 0; i--) {   // adjacent vectors shift in zeros: in place, high lane first
            adj_cgex[i] = A.add(adj_cgex[i], i >= s ? adj_cgex[i - s] : (uint16_t)0);
            adj_send[i] = Ar::mx(adj_send[i], i >= s ? adj_send[i - s] : (uint16_t)0);
        }
        for (int i = 0; i < L; i++) { cgex[i] = t_a[i]; send[i] = t_b[i]; }
        total = A.add(total, total);
    }
}

// match_greedy (src/smith_waterman/greedy.rs:7-91) on needle BYTES with the ASCII case pairs; -1 = None
template <class Hay>
FRZ_HD int greedy_score(const FrzUNeedle& nd, const FrzUScoring& sc, const Hay& hay, int W, bool include_prefix,
                        uint32_t* idx_out = nullptr) {   // idx_out: haystack position of every needle byte (nbytes entries)
    const int n = nd.nbytes;
    if (n > W) return -1;
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
            if (nd.c[ni] != hc && nd.bflip[ni] != hc) {
                prev_delim = delim_enabled && is_delim;
                prev_lower = is_lower;
                hi++;
                continue;
            }
            score += (uint32_t)sc.raw_match; if (score > 0xffffu) score = 0xffffu;
            if (hi != hstart && ni != 0) {
                uint32_t gl = (uint32_t)(hi - hstart);
                gl = gl > 0 ? gl - 1 : 0;
                if (gl > 0xffffu) gl = 0xffffu;
                uint32_t mul = (uint32_t)sc.raw_gap_extend * gl;
                if (mul > 0xffffu) mul = 0xffffu;
                uint32_t pen = (uint32_t)sc.raw_gap_open + mul;
                if (pen > 0xffffu) pen = 0xffffu;
                score = score > pen ? score - pen : 0;
            }
            auto sat_add = [&](int32_t b) { score += (uint32_t)b; if (score > 0xffffu) score = 0xffffu; };
            if (nd.c[ni] == hc) sat_add(sc.raw_case);
            if (is_upper && prev_lower) sat_add(sc.raw_cap);
            if (include_prefix && hi == 0) sat_add(sc.raw_prefix);
            if (prev_delim && !is_delim) sat_add(sc.raw_delim);
            prev_delim = delim_enabled && is_delim;
            prev_lower = is_lower;
            if (idx_out) idx_out[ni] = (uint32_t)hi;
            hi++;
            matched = true;
            break;
        }
        if (!matched) return -1;
    }
    return (int)score;
}

// score_haystack_unicode (unicode.rs:9-224).  `hay(i)` is byte i of the WINDOW (0 <= i < W).
// scratch: 2 * (n + 1) * lanes uint16 (previous chunk's row vectors and the pending-gap-open vectors of every row).
// Hfull / Mfull (optional, for the traceback): the whole score matrix and match masks, [(n + 1)][cols] with
// cols = (chunks + 1) * lanes and chunk 0 the zero column — the layout of src/smith_waterman/matrix.rs.
template <class Hay>
FRZ_HD uint32_t sw_score(const FrzUNeedle& nd, const FrzUScoring& sc, const Hay& hay, int W, bool include_prefix, int lanes,
                         bool u8, uint16_t* scratch, uint16_t* Hfull = nullptr, uint16_t* Mfull = nullptr, int cols = 0) {
    if (W > FRZ_U_MAX_WINDOW) {
        const int g = greedy_score(nd, sc, hay, W, include_prefix);
        return g < 0 ? 0u : (uint32_t)g;
    }
    const int n = nd.n;
    if (n == 0) return 0;
    const Ar A{lanes, (uint16_t)(u8 ? 0xFF : 0xFFFF)};
    const uint16_t FULL = A.full;
    uint16_t* Hprev = scratch;                         // [(n + 1)][lanes]: row r of the previous chunk
    uint16_t* pending = scratch + (n + 1) * lanes;     // [(n + 1)][lanes]
    for (int i = 0; i < 2 * (n + 1) * lanes; i++) scratch[i] = 0;
    if (Hfull) {
        for (int i = 0; i < cols; i++) { Hfull[i] = 0; Mfull[i] = 0; }                       // row 0
        for (int r = 1; r <= n; r++)
            for (int i = 0; i < lanes; i++) { Hfull[r * cols + i] = 0; Mfull[r * cols + i] = 0; }   // chunk 0
    }
    const uint16_t gex = (uint16_t)sc.gex, gop = (uint16_t)sc.gopx, mismatch = (uint16_t)sc.mismatch;
    bool prev_last_delim = false, prev_last_lower = false;
    uint16_t prev_cgex[FRZ_U_MAX_LANES], prev_sstart[FRZ_U_MAX_LANES], maxv[FRZ_U_MAX_LANES];
    for (int i = 0; i < lanes; i++) { prev_cgex[i] = 0; prev_sstart[i] = 0; maxv[i] = 0; }
    const int chunks = (W + lanes - 1) / lanes;
    for (int col = 0; col < chunks; col++) {
        const int cs = col * lanes;
        const int valid_lanes = W - cs < lanes ? W - cs : lanes;
        uint16_t sstart[FRZ_U_MAX_LANES], cgex[FRZ_U_MAX_LANES], bonuses[FRZ_U_MAX_LANES];
        bool sst[FRZ_U_MAX_LANES];
        bool last_lower = false, last_delim = false;
        {
            bool pl = prev_last_lower, pd = prev_last_delim;
            for (int i = 0; i < lanes; i++) {
                const int pos = cs + i;
                const uint8_t b = pos < W ? hay(pos) : (uint8_t)0;
                const bool valid = i < valid_lanes;
                const bool cont = b > 0x7f && b < 0xc0 && valid;
                sst[i] = !cont && valid;
                sstart[i] = sst[i] ? FULL : (uint16_t)0;
                cgex[i] = cont ? gex : (uint16_t)0;
                const bool up = b < 'Z' + 1 && b > 'A' - 1, lo = b < 'z' + 1 && b > 'a' - 1;
                const bool digit = b > '0' - 1 && b < '9' + 1;
                const bool dl = !(up || lo || digit || b > 127);
                uint16_t bn = 0;
                if (pd && !dl) bn = A.add(bn, (uint16_t)sc.delim_bonus);
                if (up && pl) bn = A.add(bn, (uint16_t)sc.cap_bonus);
                if (col == 0 && i == 0 && include_prefix) bn = A.add(bn, (uint16_t)sc.prefix_bonus);
                bonuses[i] = A.add(bn, (uint16_t)sc.match_x);
                pl = lo; pd = dl;
                if (i == lanes - 1) { last_lower = lo; last_delim = dl; }
            }
        }
        prev_last_lower = last_lower;
        prev_last_delim = last_delim;
        uint16_t prev_row[FRZ_U_MAX_LANES], up_gap[FRZ_U_MAX_LANES], row[FRZ_U_MAX_LANES], pend[FRZ_U_MAX_LANES];
        for (int i = 0; i < lanes; i++) { prev_row[i] = 0; up_gap[i] = 0; row[i] = 0; }
        uint16_t diag_in = 0;   // last lane of row r-1 in the previous chunk, before this chunk overwrites Hprev[r-1]
        uint16_t saved_prev_chunk_last = Hprev[0 * lanes + lanes - 1];   // row 0 is all zero
        for (int r = 1; r <= n; r++) {
            const int cl = nd.len[r - 1];
            const uint8_t* c = nd.c + nd.off[r - 1];
            const uint8_t* f = nd.f + nd.off[r - 1];
            diag_in = saved_prev_chunk_last;                      // score_matrix.get(r - 1, col - 1), top lane
            saved_prev_chunk_last = Hprev[r * lanes + lanes - 1];  // needed by row r + 1
            uint16_t mm[FRZ_U_MAX_LANES];
            for (int i = 0; i < lanes; i++) {
                bool e = sst[i], fl = sst[i];
                for (int k = 0; k < cl; k++) {
                    const int pos = cs + i + k;
                    const uint8_t b = pos < W ? hay(pos) : (uint8_t)0;
                    e = e && b == c[k];
                    fl = fl && b == f[k];
                }
                mm[i] = (e || fl) ? FULL : (uint16_t)0;
                uint16_t d = i > 0 ? prev_row[i - 1] : diag_in;
                d = A.add(d, mm[i] & bonuses[i]);
                d = Ar::subs(d, mismatch);
                d = A.add(d, e ? (uint16_t)sc.case_bonus : (uint16_t)0);
                d &= sstart[i];
                uint16_t u = Ar::subs(Ar::subs(prev_row[i], gex), up_gap[i] & gop);
                u &= sstart[i];
                row[i] = Ar::mx(d, u);
                pend[i] = mm[i];
            }
            uint16_t w_cgex[FRZ_U_MAX_LANES], w_adj_cgex[FRZ_U_MAX_LANES], w_send[FRZ_U_MAX_LANES], w_adj_send[FRZ_U_MAX_LANES];
            for (int i = 0; i < lanes; i++) { w_cgex[i] = cgex[i]; w_adj_cgex[i] = prev_cgex[i]; w_send[i] = sstart[i]; w_adj_send[i] = prev_sstart[i]; }
            propagate_unicode(A, row, pend, Hprev + r * lanes, pending + r * lanes, w_cgex, w_adj_cgex, w_send, w_adj_send, gop, gex);
            for (int i = 0; i < lanes; i++) {
                Hprev[r * lanes + i] = row[i];       // becomes "previous chunk" for the next chunk
                pending[r * lanes + i] = pend[i];
                prev_row[i] = row[i];
                up_gap[i] = mm[i];
                if (Hfull) { Hfull[r * cols + (col + 1) * lanes + i] = row[i]; Mfull[r * cols + (col + 1) * lanes + i] = mm[i]; }
            }
        }
        for (int i = 0; i < lanes; i++) { maxv[i] = Ar::mx(maxv[i], row[i]); prev_cgex[i] = cgex[i]; prev_sstart[i] = sstart[i]; }
    }
    uint16_t m = 0;
    for (int i = 0; i < lanes; i++) m = Ar::mx(m, maxv[i]);
    return m;
}

// ------------------------------------------------------------------------------------------------ literal modes
FRZ_HD bool in_range(uint8_t b, uint8_t lo, uint8_t hi) { return b >= lo && b <= hi; }
FRZ_HD bool lit_is_delim(uint8_t b) { return b <= 127 && !(in_range(b, '0', '9') || in_range(b, 'a', 'z') || in_range(b, 'A', 'Z')); }

template <class Hay>
FRZ_HD bool lit_matches_at(const FrzUNeedle& nd, const Hay& hay, int pos) {   // literal/algo.rs:159-170
    for (int i = 0; i < nd.n; i++) {
        const int cl = nd.len[i], o = nd.off[i];
        bool a = true, b = true;
        for (int k = 0; k < cl; k++) {
            const uint8_t h = hay(pos + o + k);
            a = a && h == nd.c[o + k];
            b = b && h == nd.f[o + k];
        }
        if (!a && !b) return false;
    }
    return true;
}
template <class Hay>
FRZ_HD uint32_t lit_score_at(const FrzUNeedle& nd, const FrzUScoring& sc, const Hay& hay, int hl, int pos) {  // :183-225
    uint32_t score = 0;
    for (int i = 0; i < nd.n; i++) {
        const int cl = nd.len[i], o = nd.off[i], st = pos + o;
        bool exact_case = true;
        for (int k = 0; k < cl; k++) exact_case = exact_case && hay(st + k) == nd.c[o + k];
        uint32_t s = (uint32_t)sc.raw_match;
        if (exact_case) s += (uint32_t)sc.raw_case;
        if (st == 0) s += (uint32_t)sc.raw_prefix;
        else {
            const uint8_t byte = hay(st), prev = hay(st - 1);
            if (in_range(byte, 'A', 'Z') && in_range(prev, 'a', 'z')) s += (uint32_t)sc.raw_cap;
            if (lit_is_delim(prev) && !lit_is_delim(byte)) s += (uint32_t)sc.raw_delim;
        }
        score = (score + s) & 0xffffu;
    }
    if (pos == 0 && nd.nbytes == hl) score = (score + (uint32_t)sc.exact_bonus) & 0xffffu;
    return score;
}
// LiteralImpl::find with UNICODE = true (literal/algo.rs:234-313); mode = FRZ_MATCHING_* (1 exact, 2 prefix, 3 suffix, 4 substring)
template <class Hay>
FRZ_HD bool lit_find(const FrzUNeedle& nd, const FrzUScoring& sc, const Hay& hay, int hl, int mode, int* opos, uint32_t* oscore) {
    const int n = nd.nbytes;
    if (hl < n) return false;
    if (mode == 4) {
        bool have = false;
        for (int pos = 0; pos + n <= hl; pos++) {
            if (!lit_matches_at(nd, hay, pos)) continue;
            const uint32_t s = lit_score_at(nd, sc, hay, hl, pos);
            if (!have || s > *oscore) { have = true; *opos = pos; *oscore = s; }
        }
        return have;
    }
    const int pos = mode == 3 ? hl - n : 0;
    if (mode == 1 && hl != n) return false;
    if (!lit_matches_at(nd, hay, pos)) return false;
    *opos = pos;
    *oscore = lit_score_at(nd, sc, hay, hl, pos);
    return true;
}

}  // namespace frzu
