// prefilter_scan.cuh — the scanning prefilter forms of prefilter.cu (window_k0 / _k1 / _k2 / _many over word probes of the
// haystack: needles with more than 16 distinct byte classes, long needles, k_match_indices) and the ASCII literal matcher,
// in a header so that the SAME source is compiled by nvcc for the kernels and by g++ for tests/test_kernel_logic_cpu.py
// (one thread; the few intrinsics they use have host stand-ins here and in prefilter_masks.cuh).
//
// The haystack is read through an accessor A with `uint32_t word(uint32_t w)`: little-endian 32-bit word w of the
// haystack's contiguous bytes.  The forms read whole words, up to 3 bytes past the haystack's end (zero padding of the
// packed corpus).  The needle is read through P: FrzPatternDev (needles of up to FRZ_MAX_NEEDLE bytes) or LongPat.
#pragma once
#include <stdint.h>

#include "../../include/frz_cuda.h"
#include "frz_device.cuh"
#include "prefilter_masks.cuh"

#if defined(__CUDACC__)
#define FRZ_SCAN_INL __device__ __forceinline__
#define FRZ_SCAN_FN __device__
#else
#define FRZ_SCAN_INL inline
#define FRZ_SCAN_FN inline
// ---- host stand-ins ----
inline int __ffs(int x) { return __builtin_ffs(x); }
inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
#endif

namespace frzpf {

// first position in [from, to) whose byte b satisfies (b | om) == tg, else -1
template <class A>
FRZ_SCAN_INL int find_first(const A& a, uint32_t om4, uint32_t tg4, int from, int to) {
    if (from >= to) return -1;
    int w = from >> 2;
    const int wend = (to + 3) >> 2;
    uint32_t x = (a.word(w) | om4) ^ tg4;
    x |= (1u << ((from & 3) * 8)) - 1;  // bytes below `from` can never look like a hit
    for (;;) {
        // lowest flagged byte is always a true zero byte (borrows only travel upwards)
        uint32_t z = (x - 0x01010101u) & ~x & 0x80808080u;
        if (z) {
            int p = w * 4 + ((__ffs(z) - 1) >> 3);
            return p < to ? p : -1;
        }
        if (++w >= wend) return -1;
        x = (a.word(w) | om4) ^ tg4;
    }
}

FRZ_SCAN_INL uint32_t zero_bytes_exact(uint32_t x) {
    return ~(((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x | 0x7f7f7f7fu);  // 0x80 in every zero byte
}

// last position in [from, to) matching either probe (om1,tg1) or (om2,tg2), else -1
template <class A>
FRZ_SCAN_INL int find_last2(const A& a, uint32_t om1, uint32_t tg1, uint32_t om2, uint32_t tg2, int from, int to) {
    if (from >= to) return -1;
    int w = (to - 1) >> 2;
    const int w0 = from >> 2;
    for (;;) {
        uint32_t v = a.word(w);
        uint32_t z = zero_bytes_exact((v | om1) ^ tg1) | zero_bytes_exact((v | om2) ^ tg2);
        int lo = w * 4;
        if (to - lo < 4) z &= (1u << ((to - lo) * 8)) - 1;          // drop bytes >= to
        if (from > lo) z &= ~((1u << ((from - lo) * 8)) - 1);       // drop bytes < from
        if (z) return lo + ((31 - __clz(z)) >> 3);
        if (--w < w0) return -1;
    }
}

// The needle as the prefilter forms below read it (template parameter P): FrzPatternDev itself for needles of up to
// FRZ_MAX_NEEDLE bytes (per-position data in the constant bank), LongPat for longer ones (per-position data staged from
// FrzNeedleTab into shared memory, scalars from the pattern).  The forms use the same member names on both.
struct LongPat {
    const uint8_t *c, *flip, *om, *tg;   // shared memory
    int n, pf_lanes, sw_lanes, max_typos, matching, col_classes, n_distinct;
    uint32_t raw_match, raw_case, raw_prefix, raw_cap, raw_delim, exact_bonus;
};

struct Probe {
    uint32_t om, tg;
};
template <class P>
FRZ_SCAN_INL Probe probe_of(const P& p, int i) { return Probe{splat4(p.om[i]), splat4(p.tg[i])}; }

// ---- Prefilter::match_haystack (0 typos): closed form of src/prefilter/algo/ascii.rs:6-54 ----
// start = first occurrence of needle[0]; greedy in-order scan; end = 1 + last occurrence of needle[n-1]
template <class A, class P>
FRZ_SCAN_FN bool window_k0(const A& a, const P& p, int len, int* ostart, int* oend) {
    if (len == 0) return false;
    int pos = 0, start = 0, q = 0;
    for (int i = 0; i < p.n; i++) {
        Probe pr = probe_of(p, i);
        q = find_first(a, pr.om, pr.tg, pos, len);
        if (q < 0) return false;
        if (i == 0) start = q;
        pos = q + 1;
    }
    Probe last = probe_of(p, p.n - 1);
    *ostart = start;
    *oend = 1 + find_last2(a, last.om, last.tg, last.om, last.tg, q, len);
    return true;
}

// find_end_pos_with_typos (src/prefilter/algo/ascii_typos.rs:375-397): 1 + last occurrence of any of
// the last (k+1) needle bytes, else len.  Chunk-independent.
template <class A, class P>
FRZ_SCAN_FN int end_pos_with_typos(const A& a, const P& p, int len, int k) {
    int best = -1;
    int first = p.n - 1 - k;
    for (int i = first; i < p.n; i += 2) {
        Probe p1 = probe_of(p, i);
        Probe p2 = probe_of(p, i + 1 < p.n ? i + 1 : i);
        int q = find_last2(a, p1.om, p1.tg, p2.om, p2.tg, best < 0 ? 0 : best, len);
        if (q > best) best = q;
    }
    return best < 0 ? len : best + 1;
}

// ---- match_haystack_1_typo (src/prefilter/algo/ascii_typos.rs:15-110), chunk-emulating ----
// Both paths' chunk masks are always suffixes [pos, chunk_end) of the chunk, so a path is the pair
// (needle index, position) and `first_path_chunk_mask > second_path_chunk_mask` ⇔ pf < ps.
template <class A, class P>
FRZ_SCAN_FN bool window_k1(const A& a, const P& p, int len, int* ostart, int* oend) {
    const int n = p.n;
    if (n <= 1) { *ostart = 0; *oend = len; return true; }
    if (len == 0) return false;
    int f = 0, s = 1;
    int ms = 0x7fffffff;
    const int L = p.pf_lanes;
    for (int cs = 0; cs < len; cs += L) {
        const int ce = min(cs + L, len);
        int pf = cs, ps = cs;
        bool f_dead = false, s_dead = false;  // path already failed to find its byte in [pos, ce)
        for (;;) {
            bool adv = false;
            int cand = f + 1;
            if (cand > s) {
                if (cand == n) goto found;
                s = cand; ps = pf; s_dead = false;
            } else if (cand == s && pf < ps) {
                ps = pf; s_dead = false;
            }
            if (!f_dead) {
                Probe pr = probe_of(p, f);
                int q = find_first(a, pr.om, pr.tg, pf, ce);
                if (q >= 0) { ms = min(ms, q); f++; pf = q + 1; adv = true; }
                else f_dead = true;
            }
            if (!s_dead) {
                Probe pr = probe_of(p, s);
                int q = find_first(a, pr.om, pr.tg, ps, ce);
                if (q >= 0) {
                    ms = min(ms, q); s++;
                    if (s >= n) goto found;
                    ps = q + 1; adv = true;
                } else s_dead = true;
            }
            if (!adv) break;
        }
    }
    return false;
found:
    *ostart = ms;
    *oend = end_pos_with_typos(a, p, len, 1);
    return true;
}

// ---- match_haystack_many_typos_impl (ascii_typos.rs:254-360); also used for k == 2 ----
// NOTE the 2-typo specialisation (ascii_typos.rs:113-251) advances each path on its OWN first hit,
// the N-typo version advances all paths on the single lowest hit; they are distinct algorithms.
template <class A, class P>
FRZ_SCAN_FN bool window_k2(const A& a, const P& p, int len, int* ostart, int* oend) {
    const int n = p.n;
    if (n <= 2) { *ostart = 0; *oend = len; return true; }
    if (len == 0) return false;
    int idx[3] = {0, 1, 2};
    int ms = 0x7fffffff;
    const int L = p.pf_lanes;
    for (int cs = 0; cs < len; cs += L) {
        const int ce = min(cs + L, len);
        int pos[3] = {cs, cs, cs};
        for (;;) {
            bool adv = false;
#pragma unroll
            for (int k = 1; k < 3; k++) {
                int cand = idx[k - 1] + 1;
                if (cand > idx[k]) {
                    if (cand == n) goto found;
                    idx[k] = cand; pos[k] = pos[k - 1];
                } else if (cand == idx[k] && pos[k - 1] < pos[k]) {
                    pos[k] = pos[k - 1];
                }
            }
#pragma unroll
            for (int k = 0; k < 3; k++) {
                Probe pr = probe_of(p, idx[k]);
                int q = find_first(a, pr.om, pr.tg, pos[k], ce);
                if (q >= 0) {
                    ms = min(ms, q); idx[k]++;
                    if (k > 0 && idx[k] >= n) goto found;
                    pos[k] = q + 1; adv = true;
                }
            }
            if (!adv) break;
        }
    }
    return false;
found:
    *ostart = ms;
    *oend = end_pos_with_typos(a, p, len, 2);
    return true;
}

constexpr int kMaxPaths = 16;  // FRZ_T_MANY supports max_typos <= 15 on the GPU path

template <class A, class P>
FRZ_SCAN_FN bool window_many(const A& a, const P& p, int len, int* ostart, int* oend) {
    const int n = p.n, k = p.max_typos;
    if (n <= k) { *ostart = 0; *oend = len; return true; }
    if (len == 0) return false;
    const int paths = k + 1;
    int idx[kMaxPaths];
    for (int i = 0; i < paths; i++) idx[i] = 0;
    int ms = 0x7fffffff;
    const int L = p.pf_lanes;
    for (int cs = 0; cs < len; cs += L) {
        const int ce = min(cs + L, len);
        int pos = cs;  // one shared chunk mask (ascii_typos.rs:286,350)
        for (;;) {
            for (int j = 1; j < paths; j++) {
                int cand = idx[j - 1] + 1;
                if (cand > idx[j]) {
                    if (cand == n) goto found;
                    idx[j] = cand;
                }
            }
            // lowest hit over all paths
            int hit = 0x7fffffff;
            for (int j = 0; j < paths; j++) {
                Probe pr = probe_of(p, idx[j]);
                int q = find_first(a, pr.om, pr.tg, pos, min(ce, hit == 0x7fffffff ? ce : hit + 1));
                if (q >= 0 && q < hit) hit = q;
            }
            if (hit == 0x7fffffff) break;
            ms = min(ms, hit);
            uint32_t hb = a.word(hit >> 2) >> ((hit & 3) * 8) & 0xff;
            for (int j = 0; j < paths; j++) {
                int i = idx[j];
                if (((hb | p.om[i]) & 0xff) != p.tg[i]) continue;
                idx[j] = i + 1;
                if (idx[j] == n) goto found;
            }
            pos = hit + 1;
        }
    }
    return false;
found:
    *ostart = ms;
    *oend = end_pos_with_typos(a, p, len, k);
    return true;
}

// ---- literal matcher, ASCII path (src/literal/algo.rs:159-255) ----
FRZ_SCAN_INL bool lit_is_delim(uint32_t b) {
    bool alnum = (b - '0' <= 9u) || (b - 'a' <= 25u) || (b - 'A' <= 25u);
    return b <= 127 && !alnum;
}
template <class A>
FRZ_SCAN_INL uint32_t byte_at(const A& a, int i) { return (a.word(i >> 2) >> ((i & 3) * 8)) & 0xff; }

template <class A, class P>
FRZ_SCAN_FN bool lit_matches_at(const A& a, const P& p, int pos) {
    for (int k = 0; k < p.n; k++) {
        uint32_t b = byte_at(a, pos + k);
        if (b != p.c[k] && b != p.flip[k]) return false;
    }
    return true;
}
template <class A, class P>
FRZ_SCAN_FN uint32_t lit_score_at(const A& a, const P& p, int len, int pos) {
    uint32_t score = 0;
    uint32_t prev = pos > 0 ? byte_at(a, pos - 1) : 0;
    for (int k = 0; k < p.n; k++) {
        int st = pos + k;
        uint32_t b = byte_at(a, st);
        uint32_t sc = p.raw_match;
        if (b == p.c[k]) sc += p.raw_case;
        if (st == 0) sc += p.raw_prefix;
        else {
            if (b - 'A' <= 25u && prev - 'a' <= 25u) sc += p.raw_cap;
            if (lit_is_delim(prev) && !lit_is_delim(b)) sc += p.raw_delim;
        }
        score += sc;
        prev = b;
    }
    if (pos == 0 && p.n == len) score += p.exact_bonus;
    return score & 0xffff;
}
// returns true on match; *opos, *oscore
template <class A, class P>
FRZ_SCAN_FN bool lit_find(const A& a, const P& p, int len, int* opos, uint32_t* oscore) {
    const int n = p.n;
    if (len < n) return false;
    switch (p.matching) {
        case FRZ_MATCHING_EXACT:
            if (len != n || !lit_matches_at(a, p, 0)) return false;
            *opos = 0; *oscore = lit_score_at(a, p, len, 0); return true;
        case FRZ_MATCHING_PREFIX:
            if (!lit_matches_at(a, p, 0)) return false;
            *opos = 0; *oscore = lit_score_at(a, p, len, 0); return true;
        case FRZ_MATCHING_SUFFIX:
            if (!lit_matches_at(a, p, len - n)) return false;
            *opos = len - n; *oscore = lit_score_at(a, p, len, len - n); return true;
        default: {  // SUBSTRING: best score, earliest on ties (find_substring :262-313)
            bool have = false;
            Probe p0 = probe_of(p, 0);
            int from = 0;
            const int last_start = len - n + 1;
            for (;;) {
                int q = find_first(a, p0.om, p0.tg, from, last_start);
                if (q < 0) break;
                if (lit_matches_at(a, p, q)) {
                    uint32_t sc = lit_score_at(a, p, len, q);
                    if (!have || sc > *oscore) { have = true; *opos = q; *oscore = sc; }
                }
                from = q + 1;
            }
            return have;
        }
    }
}

}  // namespace frzpf
