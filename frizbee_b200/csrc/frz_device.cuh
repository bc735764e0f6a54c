// frz_device.cuh — data layout shared by the kernels and the host runtime.
//
// HBM layout of a packed corpus (DESIGN.md §3):
//   * haystacks are taken in input order in TILES of FRZ_TILE = 1024;
//   * inside a tile the haystacks are stably sorted by their 16-byte unit count
//     (length bucketing) and laid out in GROUPS of 32 slots — one slot per warp lane;
//   * a group is stored SLOT-MAJOR: slot s of the group owns the `gunits` consecutive 16-byte units
//     [abs_off + s * gunits, abs_off + (s + 1) * gunits) — one haystack is one contiguous, 16-byte aligned
//     run of bytes, so the 48-64 bytes of a prefilter candidate or a Smith-Waterman window are ONE or TWO
//     64-byte DRAM accesses.  (Rounds 1-2a interleaved the units of the 32 slots, which coalesces a warp that
//     streams every haystack; since the signature index nothing streams them any more, and a scattered
//     candidate cost four 64-byte accesses for its four units.)
//   * `gunits` = the longest haystack of the group (zero padded); after bucketing almost every group is
//     uniform, so padding is the 16-byte rounding only.
//   Per slot: one u32 of metadata (len << 10 | index-within-tile).  Per group: 16 bytes.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define FRZ_TILE 1024          // haystacks per tile
#define FRZ_TILE_SHIFT 10
#define FRZ_GROUP 32           // slots per group (= warp)
#define FRZ_GROUPS_PER_TILE (FRZ_TILE / FRZ_GROUP)
#define FRZ_UNIT 16            // bytes per unit
// Longest haystack, in bytes (4 MiB - 2).  Slot meta keeps len in 22 bits; a length of (1 << 22) - 1 at local index 1023
// would encode as 0xFFFFFFFF, the unused-slot sentinel below, so the longest length stops one short of the field's maximum.
#define FRZ_MAX_HAY_LEN ((1u << 22) - 2)
#define FRZ_INVALID_SLOT 0xFFFFFFFFu      // slot meta of an unused slot (last tile)
#define FRZ_MAX_NEEDLE 64      // needle bytes whose per-position data lives in FrzPatternDev (the constant bank)
#define FRZ_LONG_NEEDLE 1024   // longest byte-path needle: 65..1024 bytes read FrzNeedleTab (longer → FRZ_ERR_UNSUPPORTED)
#define FRZ_SW_MAX_WINDOW 1024 // src/smith_waterman/algo/mod.rs:18 (MAX_HAYSTACK_LEN)

// Per-position data of a needle of FRZ_MAX_NEEDLE + 1 .. FRZ_LONG_NEEDLE bytes (the byte path's case_needle pairs and word
// probes, as in FrzPatternDev).  Device-resident, owned by the matcher; the long-needle kernels stage it in shared memory.
struct __align__(16) FrzNeedleTab {
    uint8_t c[FRZ_LONG_NEEDLE];
    uint8_t flip[FRZ_LONG_NEEDLE];
    uint8_t om[FRZ_LONG_NEEDLE];
    uint8_t tg[FRZ_LONG_NEEDLE];
};

struct __align__(16) FrzGroupDesc {
    uint64_t abs_off;   // first unit of the group, in 16-byte units from the start of the packed data
    uint32_t unit_off;  // same, relative to the tile's data base
    uint32_t gunits;    // units per slot in this group
};
// first unit (index into the packed data, 16-byte units) of slot `s` (0..31) of a group; unit k of the slot follows at + k
#if defined(__CUDACC__)
__host__ __device__
#endif
inline uint64_t frz_slot_unit0(const FrzGroupDesc& gd, uint32_t s) { return gd.abs_off + (uint64_t)s * gd.gunits; }

// Device view of a packed corpus.
struct FrzCorpusView {
    const uint4* data;            // packed units
    const uint64_t* tile_base;    // [n_tiles] first unit index (16-byte units) of each tile
    const FrzGroupDesc* groups;   // [n_tiles * 32]
    const uint32_t* slot_meta;    // [n_tiles * 1024]  len << 10 | local index, or FRZ_INVALID_SLOT
    const uint16_t* slot_of;      // [n_tiles * 1024]  inverse permutation: local index → slot
    const uint2* slot_sig;        // [n_tiles * 1024]  byte-class signature of the slot's haystack (frz_sig_bucket): .x = classes
                                  //                   that occur, .y = classes that occur at least twice
    uint64_t n;                   // haystacks
    uint32_t n_tiles;
    uint32_t max_gunits;          // longest haystack in 16-byte units
};

// typo-mode keys (src/matcher/algo.rs:6-7, src/matcher/mod.rs:58-73)
enum { FRZ_T_0 = 0, FRZ_T_1 = 1, FRZ_T_2 = 2, FRZ_T_MANY = 3, FRZ_T_NONE = 4, FRZ_T_LITERAL = 5 };

// One compiled pattern as the kernels see it (passed by value as a kernel parameter →
// constant bank, ~600 bytes).
struct FrzPatternDev {
    // case_needle pairs (src/prefilter/mod.rs:49-65)
    uint8_t c[FRZ_MAX_NEEDLE];
    uint8_t flip[FRZ_MAX_NEEDLE];
    // word-parallel probe: byte b matches needle[i] ⇔ ((b | om[i]) == tg[i]); om = 0x20 for a
    // case-insensitive letter, else 0
    uint8_t om[FRZ_MAX_NEEDLE];
    uint8_t tg[FRZ_MAX_NEEDLE];
    int32_t n;              // needle bytes
    int32_t typo_mode;      // FRZ_T_*
    int32_t max_typos;      // runtime budget for FRZ_T_MANY
    int32_t min_hay_len;    // src/matcher/algo.rs:62-65
    int32_t pf_lanes;       // prefilter chunk width being emulated: 16 / 32 / 64
    int32_t sw_lanes;       // Smith-Waterman chunk width being emulated: 8 / 16 / 32 / 64
    int32_t score_bits;     // 8 or 16 (reference backend family)
    int32_t wrap8;          // 1 → emulate u8 wrap-around explicitly (no-wrap bound not provable)
    int32_t col_classes;    // 1 → windows <= 64 may use the column-limited SW classes (no wrap, no NUL in the needle)
    int32_t matching;       // FRZ_MATCHING_*
    int32_t case_sensitive;
    // scoring constants as the reference splats them (u8 truncated in the u8 family;
    // src/smith_waterman/algo/ascii.rs:35-46)
    int32_t gap_extend;     // gap_extend_penalty
    int32_t gap_open_x;     // gap_open_penalty -sat gap_extend_penalty
    int32_t match_x;        // match_score +sat mismatch_penalty
    int32_t mismatch;
    int32_t case_bonus;
    int32_t cap_bonus;
    int32_t delim_bonus;
    int32_t prefix_bonus;
    int32_t exact_bonus;    // full u16
    // pre-splatted 16x2 constants for the register SW kernel (read straight from the constant bank)
    uint32_t k_pen_a[6];    // -(s * gap_extend)               for s = 1,2,4,8,16,32
    uint32_t k_pen_b[6];    // -(s * gap_extend + gap_open_x)
    uint32_t k_neg_mis, k_ex_add, k_up_plain, k_up_open, k_case, k_cap, k_delim, k_base;
    uint32_t om16[FRZ_MAX_NEEDLE], tg16[FRZ_MAX_NEEDLE], c16[FRZ_MAX_NEEDLE];
    // distinct needle bytes (either-case classes) for the occurrence-mask prefilter
    int32_t n_distinct;                 // 0 → too many distinct bytes, use the scanning fallback
    uint8_t dc_om[16], dc_tg[16];       // probe of distinct class d
    uint8_t cid[FRZ_MAX_NEEDLE];        // needle index → distinct class
    // phase-A signature test (necessary condition, host-chosen): a haystack can only pass the prefilter when at most
    // `sig_k` needle bytes have no partner in it, so  popc(sig_need1 & ~sig.x) + popc(sig_need2 & ~sig.y) <= sig_k
    int32_t sig_on;                     // 0 → no test (NO_PREFILTER): every length-gated haystack is a candidate
    int32_t sig_k;
    uint32_t sig_need1, sig_need2;      // byte classes the needle holds at least once / at least twice
    // untruncated scoring for the literal matcher / greedy fallback (u16 arithmetic)
    int32_t raw_match, raw_mismatch, raw_gap_open, raw_gap_extend, raw_prefix, raw_cap, raw_case, raw_delim;
    // (n > FRZ_MAX_NEEDLE: the arrays above hold the first FRZ_MAX_NEEDLE positions; the long-needle kernels take the
    // whole FrzNeedleTab as a kernel argument of their own, so that this struct, and with it the constant-bank offsets of
    // every argument of the short-needle kernels, keeps its size)
};

// Byte class of the signature index (32 classes).  ASCII letters fold case (a needle byte and its case flip share a
// class, so the class test is valid for case-sensitive and case-insensitive needles alike); digits and the remaining
// bytes share a few classes each (a coarser class only weakens the test, never invalidates it).
#if defined(__CUDACC__)
#define FRZ_DEV_HD __host__ __device__
#else
#define FRZ_DEV_HD
#endif
FRZ_DEV_HD inline uint32_t frz_sig_bucket(uint32_t b) {
    const uint32_t t = (b | 0x20u) - 'a';
    if (t < 26u) return t;
    const uint32_t d = b - '0';
    if (d < 10u) return 26u + d % 3u;
    return 29u + (b + (b >> 5)) % 3u;
}
// one more haystack byte: p1 = classes seen, p2 = classes seen at least twice
FRZ_DEV_HD inline void frz_sig_add(uint32_t& p1, uint32_t& p2, uint32_t byte) {
    const uint32_t bit = 1u << frz_sig_bucket(byte);
    p2 |= p1 & bit;
    p1 |= bit;
}
// lower bound of the number of needle bytes without a partner in the haystack <= typo budget?
FRZ_DEV_HD inline bool frz_sig_pass(uint32_t need1, uint32_t need2, int k, uint32_t p1, uint32_t p2) {
#if defined(__CUDA_ARCH__)
    return __popc(need1 & ~p1) + __popc(need2 & ~p2) <= k;
#else
    return __builtin_popcount(need1 & ~p1) + __builtin_popcount(need2 & ~p2) <= k;
#endif
}

// Survivor of the prefilter, input of the Smith-Waterman stage (16 bytes).
// A prefilter survivor.  Two layouts share the 16 bytes:
//   generic class / literal:  slot_rank = slot | li << 10;  start, end | (end == len) << 31   (literal: score, exact)
//   window classes (<= 128):  slot_rank = slot | li << 10 | W << 20 | (end == len) << 28 | (start == 0) << 29
//                             start = low 32 bits of the unit index of the window's first 16-byte unit (lane-resolved)
//                             end   = high 8 bits of that index | (window start & 15) << 8
// li = index of the haystack inside its tile (its rank in index order).
struct __align__(16) FrzSurvivor {
    uint32_t tile;      // tile index
    uint32_t slot_rank;
    uint32_t start;
    uint32_t end;
};

// SW work classes (which kernel variant scores the window).  Windows of <= 64 bytes are split further by
// the number of DP columns that can influence the score, min(W + needle_len, ceil(W / LANES) * LANES)
// (sw.cu): CC40/48/56 evaluate only that many of the reference's 64 columns.
enum {
    FRZ_C_CC40 = 0, FRZ_C_CC48 = 1, FRZ_C_CC56 = 2, FRZ_C_COLS64 = 3,
    FRZ_C_COLS128 = 4, FRZ_C_GENERIC = 5, FRZ_N_CLASSES = 6
};
struct FrzSurvLists {
    FrzSurvivor* p[FRZ_N_CLASSES];
};

struct __align__(8) FrzMatchDev {  // == frz_match
    uint32_t index;
    uint16_t score;
    uint8_t exact;
    uint8_t pad;
};

// Per-call scratch counters (device), zeroed before each call.
struct FrzCounters {
    unsigned long long class_count[FRZ_N_CLASSES];  // survivors per SW class
    unsigned long long total;                       // total matches (after scan)
    unsigned int max_score;
    unsigned int error;                             // sticky device-side error flags
    unsigned int sw_next;                           // next 32-survivor work item of the SW kernel
    unsigned int pad_;
    unsigned long long cand_count;                  // candidate records written by k_sig_scan
    unsigned int pf_next;                           // (spare)
    unsigned int pad2_;
};

#define FRZ_DEVERR_SURVIVOR_OVERFLOW 1u

#if defined(__CUDACC__)   // device-only helpers (the structs above are shared with host-side test builds)
__device__ __forceinline__ uint32_t frz_lane() { return threadIdx.x & 31; }

// Programmatic dependent launch (frz_launch_dependent).  A kernel launched that way can be scheduled before the kernel
// ahead of it on the stream has finished, so it calls frz_wait_prior_grid() before its first global memory access:
// the wait returns once every prior grid has completed and its writes are visible (it is a no-op in a normal launch).
// Because every dependent kernel waits before touching memory, a kernel may let its dependent be scheduled at any point
// (frz_allow_dependent_launch): that only moves the dependent's launch and block scheduling under this kernel's tail.
__device__ __forceinline__ void frz_wait_prior_grid() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void frz_allow_dependent_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Byte accessor of one packed haystack for the per-thread correctness paths (unicode.cu, k_match_indices):
// `base` is the pointer to unit 0 of the slot (its units are contiguous), `shift` the window start.
struct FrzPackedHay {
    const uint4* base;
    int shift;
    __device__ __forceinline__ uint8_t operator()(int i) const {
        const uint32_t j = (uint32_t)(i + shift);
        return (uint8_t)((reinterpret_cast<const uint32_t*>(base)[j >> 2] >> ((j & 3) * 8)) & 0xff);
    }
};

// address of unit k of (tile, slot)
__device__ __forceinline__ const uint4* frz_unit_ptr(const FrzCorpusView& cv, uint32_t tile, uint32_t slot, uint32_t k) {
    const FrzGroupDesc gd = cv.groups[tile * FRZ_GROUPS_PER_TILE + (slot >> 5)];
    return cv.data + frz_slot_unit0(gd, slot & 31) + k;
}
#endif  // __CUDACC__
