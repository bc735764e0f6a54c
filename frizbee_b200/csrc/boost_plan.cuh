// boost_plan.cuh — the row rule of frz_boost_where and frz_boost_where_batch (DESIGN.md §4.18).  Shared by the device
// kernel (boost_where.cu), the host calls (host.cu) and a CPU build (tests/harness/boost_where_harness.cpp).
//
// Query j's value of index i < n is clamp(base_i + the sum of the adds of its rules whose clause holds for i) to int16,
// the sum in int32; base_i is 0 without a base and past the base's values.  A rule's clause is frz_subset_where's, so the
// rule reuses the batched plan of where_plan.cuh: the call's distinct attributes form one table, each rule's clause refers
// to its attribute by its place there, and a block stages the chunk's values of the table's first kFrzWhereBatchStaged
// attributes in shared memory once for every query.  The packer groups each query's rules by attribute, so a row reads
// each attribute of its query once however many rules test it (a recency ladder over one timestamp: one value per row).
#pragma once
#include "where_plan.cuh"

constexpr uint32_t kFrzBoostMaxRules = 8;    // FRZ_BOOST_MAX_RULES
constexpr int32_t kFrzBoostMaxAdd = 65535;   // |add| of a rule: 8 of them and a base stay far inside int32

// One query of a boost fill.  The packer sets rule0, n_rules and set0; the call sets the rest.
struct FrzBoostQuery {
    uint32_t rule0, n_rules;   // its rules: clauses[rule0 ..) and adds[rule0 ..), grouped by attribute
    uint64_t set0;             // its set values: sets[set0 ..)
    const int16_t* base;       // the base's values [0, n_base); 0 past them (n_base == 0 without a base)
    uint64_t n_base;
    int16_t* out;              // out: n values (may be `base`: each value is read, then written)
};

// One boost fill of q queries over one corpus.
struct FrzBoostBatchDev {
    const FrzWhereBatchAttr* attrs;       // [n_attrs]
    const FrzWhereBatchClause* clauses;   // rule r's clause
    const int32_t* adds;                  // rule r's add
    const FrzBoostQuery* queries;         // [q]
    const int64_t* sets;
    int32_t* max;                         // [q] out: max(0, the query's largest value); 0 before the fill
    uint64_t n;                           // the corpus's length
    uint32_t q;
    uint32_t n_staged;                    // min(n_attrs, kFrzWhereBatchStaged)
};

// The sum of query qr's adds over its rules whose clause holds for a row.  value(clause) gives the row's value in the
// clause's attribute; it is called once per run of rules over one attribute.
template <class Value>
FRZ_HD int32_t frz_boost_rules_sum(const FrzBoostBatchDev& b, const FrzBoostQuery& qr, Value value) {
    int32_t sum = 0;
    int64_t v = 0;
    uint32_t at = UINT32_MAX;
    for (uint32_t r = 0; r < qr.n_rules; r++) {
        const FrzWhereBatchClause& cl = b.clauses[qr.rule0 + r];
        if (cl.attr != at) {
            at = cl.attr;
            v = value(cl);
        }
        if (frz_where_holds(cl.rule, b.sets + qr.set0, v)) sum += b.adds[qr.rule0 + r];
    }
    return sum;
}

FRZ_HD int16_t frz_boost_clamp(int32_t x) { return (int16_t)(x < -32768 ? -32768 : x > 32767 ? 32767 : x); }

// query qr's value of index i < n in a chunk starting at i0 (staged: as frz_where_batch_value reads it)
FRZ_HD int16_t frz_boost_row(const FrzBoostBatchDev& b, const FrzBoostQuery& qr, const int64_t* staged, uint64_t i0, uint64_t i) {
    const int32_t base = i < qr.n_base ? qr.base[i] : 0;
    return frz_boost_clamp(base + frz_boost_rules_sum(b, qr, [&](const FrzWhereBatchClause& c) {
               return frz_where_batch_value(c, staged, b.n_staged, i0, i);
           }));
}

// (host) The staged form of a boost fill: the batched plan of the rules' clauses, and each rule's add.
struct FrzBoostPlan {
    FrzWhereBatchPlan where;             // its clauses are the rules', each query's grouped by attribute
    std::vector<int32_t> adds;           // [clause] that rule's add
    std::vector<FrzBoostQuery> queries;
};

// (host) Packs q queries: query j's rules are rules[o_j .. o_j + n_rules[j]), o_j the sum of the earlier counts.  Rule has
// frz_boost_rule's fields (`when`, `add`); attr_of is frz_where_batch_pack's.  Each query's rules are reordered so that
// rules over one attribute are adjacent, the attributes in order of first appearance and the rules of one attribute in
// their order; a sum does not depend on the order of its terms.
template <class Rule, class AttrOf>
inline void frz_boost_pack(const Rule* rules, const uint64_t* n_rules, uint64_t q, AttrOf attr_of, FrzBoostPlan& p) {
    using Clause = decltype(rules->when);
    std::vector<Clause> when;
    p.adds.clear();
    uint64_t o = 0;
    for (uint64_t j = 0; j < q; j++) {
        const uint64_t n = n_rules[j];
        std::vector<bool> taken(n, false);
        for (uint64_t r = 0; r < n; r++) {
            if (taken[r]) continue;
            for (uint64_t s = r; s < n; s++)
                if (!taken[s] && rules[o + s].when.attr == rules[o + r].when.attr) {
                    taken[s] = true;
                    when.push_back(rules[o + s].when);
                    p.adds.push_back(rules[o + s].add);
                }
        }
        o += n;
    }
    frz_where_batch_pack(when.data(), n_rules, q, attr_of, p.where);
    p.queries.assign(q, FrzBoostQuery{});
    for (uint64_t j = 0; j < q; j++) {
        p.queries[j].rule0 = p.where.queries[j].clause0;
        p.queries[j].n_rules = p.where.queries[j].n_clauses;
        p.queries[j].set0 = p.where.queries[j].set0;
    }
}
