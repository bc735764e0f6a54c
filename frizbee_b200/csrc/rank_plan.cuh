// rank_plan.cuh — the key rules of frz_attr_rank (DESIGN.md §4.17): the 64-bit chunk a row's key gives a refinement
// round, the sort key of a round, and the step from one round's chunk to the next round's place in the key tuple.  Shared
// by the kernels (rank.cu, and the LSD sort's RankKey in sort.cu), the host driver (host.cu) and a CPU build
// (tests/harness/rank_harness.cpp), so the CPU tests run exactly what the kernels run.
//
// The ranked rows are refined most-significant chunk first.  A segment is a run of rows whose tuples agree on every chunk
// read so far; it sits at the positions [seg, seg + size) of the final order, so its first position is its id.  Each
// round gives every row of a segment of more than one row the next chunk of its key tuple, sorts those rows by (segment,
// chunk) and splits every segment where the chunk changes.  Every chunk's ascending unsigned order is its key's order:
//   attribute key   ~frz_order_attr_key(v, !desc): the value's order, reversed by desc, null (all ones) last;
//   text key        kFrzRankChunkBytes bytes from the segment's byte offset, big-endian, then the number of them the
//                   text still has (0 .. 7) in the low byte.  Bytes past the end read as 0, so a text that ends inside
//                   the chunk orders before every longer one with the same bytes, NUL included: either a byte differs,
//                   or the counts do.  A count of 7 means the text may go on; below 7 the text has ended.
//                   desc complements the chunk.
// Where a key ends for a whole segment (an attribute key, or a text that ended) the segment moves to the next key; after
// the last key it is finished, as is every segment of one row.
//
// A segment of a text key first skips the common prefix of its rows (rank.cu compares every row with one row of the
// segment, 16 bytes per load, frz_rank_diff16), so the rounds do not grow with the length of a shared prefix.
#pragma once
#include <stdint.h>

#include "order_plan.cuh"

#if defined(__CUDACC__)
#define FRZ_RK_HD __host__ __device__ __forceinline__
#else
#define FRZ_RK_HD inline
#endif

constexpr uint32_t kFrzRankMaxKeys = 4;           // FRZ_RANK_MAX_KEYS
constexpr uint32_t kFrzRankChunkBytes = 7;        // text bytes per chunk
constexpr uint32_t kFrzRankNone = 0xFFFFFFFFu;    // the segment of a row that is not ranked
constexpr uint32_t kFrzRankOffBits = 24;          // a place in the tuple: key << 24 | byte offset (haystacks < 4 MiB)
constexpr uint32_t kFrzRankOffMask = (1u << kFrzRankOffBits) - 1;

FRZ_RK_HD uint32_t frz_rank_at(uint32_t key, uint32_t off) { return key << kFrzRankOffBits | off; }
FRZ_RK_HD uint32_t frz_rank_at_key(uint32_t at) { return at >> kFrzRankOffBits; }
FRZ_RK_HD uint32_t frz_rank_at_off(uint32_t at) { return at & kFrzRankOffMask; }

// byte b as fold_case compares it: A-Z as a-z
FRZ_RK_HD uint32_t frz_rank_fold_byte(uint32_t b) { return b - 'A' < 26u ? b | 0x20u : b; }

// the four bytes of x folded at once
FRZ_RK_HD uint32_t frz_rank_fold4(uint32_t x) {
    const uint32_t low7 = x & 0x7F7F7F7Fu;
    const uint32_t ge_a = low7 + 0x3F3F3F3Fu;   // high bit: the low 7 bits are >= 'A'
    const uint32_t gt_z = low7 + 0x25252525u;   // high bit: the low 7 bits are > 'Z'
    return x | ((ge_a & ~gt_z & ~x & 0x80808080u) >> 2);
}

// the chunk of an attribute value
FRZ_RK_HD uint64_t frz_rank_attr_chunk(int64_t v, bool desc) { return ~frz_order_attr_key(v, !desc); }

// The chunk of a text of len bytes at byte offset off (<= len); hay(i) is byte i of the text.
template <class Hay>
FRZ_RK_HD uint64_t frz_rank_text_chunk(const Hay& hay, uint32_t len, uint32_t off, bool fold, bool desc) {
    const uint32_t left = len - off < kFrzRankChunkBytes ? len - off : kFrzRankChunkBytes;
    uint64_t c = 0;
    for (uint32_t j = 0; j < kFrzRankChunkBytes; j++) {
        const uint32_t b = j < left ? (uint32_t)hay((int)(off + j)) : 0u;
        c = c << 8 | (fold ? frz_rank_fold_byte(b) : b);
    }
    c = c << 8 | left;
    return desc ? ~c : c;
}

// the key ends with this chunk for every row that has it: an attribute key, or a text that ended inside the chunk
FRZ_RK_HD bool frz_rank_chunk_ends(uint64_t chunk, bool text, bool desc) {
    return !text || ((desc ? ~chunk : chunk) & 0xFFu) < kFrzRankChunkBytes;
}

// The place after a chunk of key tuple place `at` (the segment's key and byte offset, the skipped prefix included) that
// ends or not, with n_keys keys: false when the tuple is used up, else true and the next place in *next.
FRZ_RK_HD bool frz_rank_next(uint32_t at, bool ends, uint32_t n_keys, uint32_t* next) {
    const uint32_t key = frz_rank_at_key(at);
    if (!ends) {
        *next = at + kFrzRankChunkBytes;
        return true;
    }
    if (key + 1 >= n_keys) return false;
    *next = frz_rank_at(key + 1, 0);
    return true;
}

// The sort key of a round, as an order key (order_plan.cuh) whose DESCENDING order is the ascending order of (seg, chunk):
// bits [64, 96) hold ~seg and [0, 64) ~chunk; the top 16 bits are zero.  The LSD sort of sort.cu visits only the digits in
// which two keys differ (frz_order_digits).
FRZ_RK_HD FrzOrderKey frz_rank_sort_key(uint32_t seg, uint64_t chunk) {
    const uint64_t c = ~chunk;
    FrzOrderKey k;
    k.hi = (uint64_t)(uint32_t)~seg << 16 | c >> 48;
    k.lo = c & ((1ull << 48) - 1);
    return k;
}
FRZ_RK_HD uint32_t frz_rank_key_seg(const FrzOrderKey& k) { return ~(uint32_t)(k.hi >> 16); }
FRZ_RK_HD bool frz_rank_key_eq(const FrzOrderKey& a, const FrzOrderKey& b) { return a.hi == b.hi && a.lo == b.lo; }

FRZ_RK_HD uint32_t frz_rank_ctz(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __ffs(x) - 1;
#else
    return __builtin_ctz(x);
#endif
}

// The first byte in which two 16-byte units differ (fold: A-Z as a-z), little-endian words; 16 when none does.
FRZ_RK_HD uint32_t frz_rank_diff16(const uint32_t* a, const uint32_t* b, bool fold) {
    for (uint32_t w = 0; w < 4; w++) {
        const uint32_t x = fold ? frz_rank_fold4(a[w]) ^ frz_rank_fold4(b[w]) : a[w] ^ b[w];
        if (x) return 4 * w + (frz_rank_ctz(x) >> 3);
    }
    return 16;
}

// The common prefix of two texts of len_a and len_b bytes from byte offset off (<= both lengths), bytes compared as
// fold says, reading whole 16-byte units: unit(t, u) is unit u of text t (0 or 1) as four little-endian words.
template <class Unit>
FRZ_RK_HD uint32_t frz_rank_common(const Unit& unit, uint32_t len_a, uint32_t len_b, uint32_t off, bool fold) {
    const uint32_t lim = len_a < len_b ? len_a : len_b;
    for (uint32_t u = off >> 4; u * 16 < lim; u++) {
        uint32_t a[4], b[4];
        unit(0, u, a);
        unit(1, u, b);
        if (u == off >> 4)   // the bytes before off: a takes b's
            for (uint32_t w = 0; w < 4; w++) {
                const uint32_t skip = off & 15, lo = 4 * w;
                const uint32_t keep = skip >= lo + 4 ? 0u : skip <= lo ? ~0u : ~0u << ((skip - lo) * 8);
                a[w] = (a[w] & keep) | (b[w] & ~keep);
            }
        const uint32_t d = frz_rank_diff16(a, b, fold);
        if (d < 16) return (u * 16 + d < lim ? u * 16 + d : lim) - off;
    }
    return lim - off;
}
