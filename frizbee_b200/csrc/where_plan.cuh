// where_plan.cuh — the row rule of frz_subset_where and frz_subset_where_batch (DESIGN.md §4.14).  Shared by the device
// kernels (where.cu), the host calls (host.cu) and CPU builds (tests/harness/where_harness.cpp, where_batch_harness.cpp).
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

#include "frz_hd.cuh"

#include <algorithm>
#include <unordered_map>
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

FRZ_HD uint32_t frz_where_popc(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __popc(x);
#else
    return (uint32_t)__builtin_popcount(x);
#endif
}

// i's value in the clause's attribute
FRZ_HD int64_t frz_where_value(const FrzWhereClauseDev& c, uint64_t i) { return i < c.n_values ? c.values[i] : kFrzAttrNull; }

// v is one of set[0 .. n) (sorted, distinct)
FRZ_HD bool frz_where_in(const int64_t* set, uint32_t n, int64_t v) {
    uint32_t lo = 0, hi = n;   // the first element >= v is in [lo, hi]
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (set[mid] < v) lo = mid + 1;
        else hi = mid;
    }
    return lo < n && set[lo] == v;
}

// the clause holds for value v (sets: the fill's set values)
FRZ_HD bool frz_where_holds(const FrzWhereClauseDev& c, const int64_t* sets, int64_t v) {
    if (v == kFrzAttrNull) return false;
    const bool t = c.n_in ? frz_where_in(sets + c.in_off, c.n_in, v) : (c.lo <= v && v <= c.hi);
    return t != (c.negate != 0);
}

// i is below n and, with a base, a member of it (base_word: the base's word i / 32, read only below n_base)
FRZ_HD bool frz_where_in_base(const FrzWhereDev& w, uint32_t base_word, uint64_t i) {
    return i < w.n && (!w.has_base || (i < w.n_base && ((base_word >> (i & 31)) & 1u)));
}

// the members of `word` below bit `bit`: the offset of that bit's member within the word's members
FRZ_HD uint32_t frz_where_rank(uint32_t word, uint32_t bit) { return frz_where_popc(word & ((1u << bit) - 1u)); }

// (host) Appends in[0 .. n) sorted and de-duplicated to `sets`; returns how many it appended (their offset is the old size).
inline uint32_t frz_where_pack_set(const int64_t* in, uint64_t n, std::vector<int64_t>& sets) {
    const size_t off = sets.size();
    sets.insert(sets.end(), in, in + n);
    std::sort(sets.begin() + off, sets.end());
    sets.erase(std::unique(sets.begin() + off, sets.end()), sets.end());
    return (uint32_t)(sets.size() - off);
}

// ---------------------------------------------------------------------------------- batched fills
// frz_subset_where_batch fills q subsets of one corpus in one pass over the attribute values.  The call's distinct
// attributes form one table, in order of first appearance; each clause refers to its attribute by its place there.  A
// block of k_where_batch takes a chunk of kFrzWhereChunk indices, stages the chunk's values of the table's first
// kFrzWhereBatchStaged attributes in shared memory once (null past an attribute's array, as frz_where_value reads it),
// and then writes every query's bitmap words of that chunk, reading the staged values from shared memory and any other
// attribute's from global memory.  Query j's row rule is the single fill's: frz_where_in_base, then frz_where_holds per
// clause, with its set values at sets[set0 ..).
constexpr uint32_t kFrzWhereBatchStaged = 4;   // attributes staged per chunk (8 KB of shared memory each)

// One distinct attribute of a batched fill.
struct FrzWhereBatchAttr {
    const int64_t* values;   // values[i] for i < n_values; null past it
    uint64_t n_values;
};

// One clause of a batched fill: the single fill's clause (values / n_values those of attribute `attr`, in_off relative to
// its query's set0) and its attribute's place in the call's table.
struct FrzWhereBatchClause {
    FrzWhereClauseDev rule;
    uint32_t attr;
    uint32_t pad_;
};

// One query of a batched fill.  The packer sets clause0, n_clauses and set0; the call sets the rest.
struct FrzWhereBatchQuery {
    uint32_t clause0, n_clauses;   // its clauses: clauses[clause0 .. clause0 + n_clauses)
    uint64_t set0;                 // its set values: sets[set0 ..)
    const uint32_t* base;          // has_base: the base's bitmap over [0, n_base)
    uint64_t n_base;
    uint32_t has_base;
    uint32_t pad_;
    uint32_t* bits;                // out: ceil(n / 32) words (may be `base`: each word is read, then written)
    uint32_t* chunk_count;         // out: members per chunk
    uint64_t* chunk_base;          // out: their exclusive scan
    uint32_t* members;             // out: the member list (set after the member count is read back)
};

// One batched fill.
struct FrzWhereBatchDev {
    const FrzWhereBatchAttr* attrs;      // [n_attrs]
    const FrzWhereBatchClause* clauses;
    const FrzWhereBatchQuery* queries;   // [q]
    const int64_t* sets;
    uint64_t n;                          // the corpus's length
    uint32_t q;
    uint32_t n_staged;                   // min(n_attrs, kFrzWhereBatchStaged)
};

// i's value in attribute a
FRZ_HD int64_t frz_where_attr_value(const FrzWhereBatchAttr& a, uint64_t i) { return i < a.n_values ? a.values[i] : kFrzAttrNull; }

// i's value for clause c in a chunk starting at index i0: from `staged` (the chunk's values of the first n_staged
// attributes, kFrzWhereChunk each) when c's attribute is staged, else from the attribute
FRZ_HD int64_t frz_where_batch_value(const FrzWhereBatchClause& c, const int64_t* staged, uint32_t n_staged, uint64_t i0, uint64_t i) {
    return c.attr < n_staged ? staged[(uint64_t)c.attr * kFrzWhereChunk + (i - i0)] : frz_where_value(c.rule, i);
}

// query qr keeps index i (see frz_where_batch_value; base_word: its base's word i / 32, read only below n_base)
FRZ_HD bool frz_where_batch_row(const FrzWhereBatchDev& b, const FrzWhereBatchQuery& qr, const int64_t* staged, uint64_t i0,
                                uint32_t base_word, uint64_t i) {
    bool keep = i < b.n && (!qr.has_base || (i < qr.n_base && ((base_word >> (i & 31)) & 1u)));   // frz_where_in_base
    for (uint32_t c = 0; c < qr.n_clauses; c++) {
        const FrzWhereBatchClause& cl = b.clauses[qr.clause0 + c];
        keep = frz_where_holds(cl.rule, b.sets + qr.set0, frz_where_batch_value(cl, staged, b.n_staged, i0, i)) && keep;
    }
    return keep;
}

// (host) The staged form of a batched fill, built from the ABI's arguments.
struct FrzWhereBatchPlan {
    std::vector<FrzWhereBatchAttr> attrs;        // the distinct attributes, in order of first appearance
    std::vector<FrzWhereBatchClause> clauses;    // query by query, each query's in its order
    std::vector<FrzWhereBatchQuery> queries;
    std::vector<int64_t> sets;                   // query by query, each clause's values sorted and de-duplicated
    uint32_t n_staged() const { return (uint32_t)std::min<size_t>(attrs.size(), kFrzWhereBatchStaged); }
};

// (host) Packs q queries: query j's clauses are clauses[o_j .. o_j + n_clauses[j]), o_j the sum of the earlier counts.
// Clause has frz_where_clause's fields; attr_of(clause.attr) gives the attribute's FrzWhereBatchAttr, and attributes are
// told apart by their handle.
template <class Clause, class AttrOf>
inline void frz_where_batch_pack(const Clause* clauses, const uint64_t* n_clauses, uint64_t q, AttrOf attr_of, FrzWhereBatchPlan& p) {
    p.attrs.clear();
    p.clauses.clear();
    p.queries.assign(q, FrzWhereBatchQuery{});
    p.sets.clear();
    std::unordered_map<const void*, uint32_t> place;
    uint64_t o = 0;
    for (uint64_t j = 0; j < q; j++) {
        FrzWhereBatchQuery& qr = p.queries[j];
        qr.clause0 = (uint32_t)p.clauses.size();
        qr.n_clauses = (uint32_t)n_clauses[j];
        qr.set0 = p.sets.size();
        for (uint64_t c = 0; c < n_clauses[j]; c++) {
            const Clause& cl = clauses[o + c];
            const auto at = place.emplace(static_cast<const void*>(cl.attr), (uint32_t)p.attrs.size());
            if (at.second) p.attrs.push_back(attr_of(cl.attr));
            FrzWhereBatchClause d = {};
            d.attr = at.first->second;
            d.rule.values = p.attrs[d.attr].values;
            d.rule.n_values = p.attrs[d.attr].n_values;
            d.rule.lo = cl.lo;
            d.rule.hi = cl.hi;
            d.rule.in_off = (uint32_t)(p.sets.size() - qr.set0);
            d.rule.n_in = cl.n_in ? frz_where_pack_set(cl.in, cl.n_in, p.sets) : 0;
            d.rule.negate = cl.negate != 0;
            p.clauses.push_back(d);
        }
        o += n_clauses[j];
    }
}
