// where_plan.cuh — the row rule of frz_subset_where (DESIGN.md §4.14).  Shared by the device kernels (where.cu), the host
// call (host.cu) and a CPU build (tests/harness/where_harness.cpp).
//
// Index i < n is a member of the filled subset when it is a member of the base (when there is one) and every clause holds
// for v, i's value in the clause's attribute (null past the attribute's array).  A clause tests lo <= v <= hi, or, with set
// values, whether v is one of them (binary search in the clause's sorted, de-duplicated values); a negated clause holds
// where that test fails.  A null value fails every clause, negated or not.
//
// The fill writes the bitmap word by word (32 consecutive indices), counts the members of each chunk of kFrzWhereChunk
// indices, scans the counts, and expands each word into ascending member positions at its chunk's base.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define FRZ_WP_HD __host__ __device__ __forceinline__
#else
#define FRZ_WP_HD inline
#endif

#include <algorithm>
#include <vector>

constexpr int64_t kFrzAttrNull = INT64_MIN;          // FRZ_ATTR_NULL
constexpr uint32_t kFrzWhereMaxClauses = 8;          // FRZ_WHERE_MAX_CLAUSES
constexpr uint32_t kFrzWhereMaxIn = 4096;            // FRZ_WHERE_MAX_IN
constexpr uint32_t kFrzWhereChunkWords = 32;         // bitmap words per scanned chunk
constexpr uint64_t kFrzWhereChunk = kFrzWhereChunkWords * 32;   // indices per scanned chunk

// One clause on the device.
struct FrzWhereClauseDev {
    const int64_t* values;   // the attribute: values[i] for i < n_values; null past it
    uint64_t n_values;
    int64_t lo, hi;          // range clause (n_in == 0)
    uint32_t in_off, n_in;   // set clause (n_in > 0): its sorted distinct values at sets[in_off .. in_off + n_in)
    uint32_t negate;
    uint32_t pad_;
};

// One fill: the clauses, the base, and the outputs.
struct FrzWhereDev {
    FrzWhereClauseDev clauses[kFrzWhereMaxClauses];
    const int64_t* sets;     // [n_sets] every set clause's values
    const uint32_t* base;    // has_base: the base subset's bitmap over [0, n_base)
    uint32_t* bits;          // out: ceil(n / 32) words, bits at and past n zero (may be `base`: each word is read, then written)
    uint32_t* chunk_count;   // out: members per chunk of kFrzWhereChunk indices
    uint64_t n;              // the corpus's length
    uint64_t n_base;
    uint32_t n_clauses;
    uint32_t n_sets;
    uint32_t has_base;
    uint32_t pad_;
};

FRZ_WP_HD uint32_t frz_where_popc(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __popc(x);
#else
    return (uint32_t)__builtin_popcount(x);
#endif
}

// i's value in the clause's attribute
FRZ_WP_HD int64_t frz_where_value(const FrzWhereClauseDev& c, uint64_t i) { return i < c.n_values ? c.values[i] : kFrzAttrNull; }

// v is one of set[0 .. n) (sorted, distinct)
FRZ_WP_HD bool frz_where_in(const int64_t* set, uint32_t n, int64_t v) {
    uint32_t lo = 0, hi = n;   // the first element >= v is in [lo, hi]
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (set[mid] < v) lo = mid + 1;
        else hi = mid;
    }
    return lo < n && set[lo] == v;
}

// the clause holds for value v (sets: the fill's set values)
FRZ_WP_HD bool frz_where_holds(const FrzWhereClauseDev& c, const int64_t* sets, int64_t v) {
    if (v == kFrzAttrNull) return false;
    const bool t = c.n_in ? frz_where_in(sets + c.in_off, c.n_in, v) : (c.lo <= v && v <= c.hi);
    return t != (c.negate != 0);
}

// i is below n and, with a base, a member of it (base_word: the base's word i / 32, read only below n_base)
FRZ_WP_HD bool frz_where_in_base(const FrzWhereDev& w, uint32_t base_word, uint64_t i) {
    return i < w.n && (!w.has_base || (i < w.n_base && ((base_word >> (i & 31)) & 1u)));
}

// the members of `word` below bit `bit`: the offset of that bit's member within the word's members
FRZ_WP_HD uint32_t frz_where_rank(uint32_t word, uint32_t bit) { return frz_where_popc(word & ((1u << bit) - 1u)); }

// (host) Appends in[0 .. n) sorted and de-duplicated to `sets`; returns how many it appended (their offset is the old size).
inline uint32_t frz_where_pack_set(const int64_t* in, uint64_t n, std::vector<int64_t>& sets) {
    const size_t off = sets.size();
    sets.insert(sets.end(), in, in + n);
    std::sort(sets.begin() + off, sets.end());
    sets.erase(std::unique(sets.begin() + off, sets.end()), sets.end());
    return (uint32_t)(sets.size() - off);
}
