// CPU build of frizbee_b200/csrc/boost_plan.cuh: the packer of frz_boost_where / frz_boost_where_batch (the batched
// plan of the rules' clauses, grouped by attribute, and their adds) and k_boost_where's row rule over staged chunks,
// through the header's own functions (tests/test_boost_where_host.py).
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../frizbee_b200/csrc/boost_plan.cuh"
#include "../../include/frz_cuda.h"

namespace {
// attribute handles are the addresses of FrzWhereBatchAttr records (the stand-in attributes)
FrzWhereBatchAttr attr_of(const frz_attr* a) { return *reinterpret_cast<const FrzWhereBatchAttr*>(a); }
FrzBoostPlan g_plan;
}  // namespace

// frz_boost_pack over ABI rules; the plan stays here for h_boost_plan.  Returns the number of distinct attributes.
extern "C" uint64_t h_boost_pack(const frz_boost_rule* rules, const uint64_t* n_rules, uint64_t q) {
    frz_boost_pack(rules, n_rules, q, attr_of, g_plan);
    return g_plan.where.attrs.size();
}

// sizes[0..4) = attributes, rules, set values, staged attributes; then the plan's arrays (each may be NULL)
extern "C" void h_boost_plan(uint64_t* sizes, FrzWhereBatchAttr* attrs, FrzWhereBatchClause* clauses, int32_t* adds,
                             FrzBoostQuery* queries, int64_t* sets) {
    const FrzWhereBatchPlan& w = g_plan.where;
    sizes[0] = w.attrs.size();
    sizes[1] = w.clauses.size();
    sizes[2] = w.sets.size();
    sizes[3] = w.n_staged();
    if (attrs) memcpy(attrs, w.attrs.data(), w.attrs.size() * sizeof(FrzWhereBatchAttr));
    if (clauses) memcpy(clauses, w.clauses.data(), w.clauses.size() * sizeof(FrzWhereBatchClause));
    if (adds) memcpy(adds, g_plan.adds.data(), g_plan.adds.size() * sizeof(int32_t));
    if (queries) memcpy(queries, g_plan.queries.data(), g_plan.queries.size() * sizeof(FrzBoostQuery));
    if (sets) memcpy(sets, w.sets.data(), w.sets.size() * sizeof(int64_t));
}

// The whole fill of q queries over n rows as k_boost_where computes it: pack, then per chunk stage the staged attributes'
// values and write every query's rows with frz_boost_row, its maximum folded from 0.  outs[j] may be bases[j] (in place).
// loads[j]: how many attribute values query j's rule sum read over all rows.
extern "C" void h_boost_fill(const frz_boost_rule* rules, const uint64_t* n_rules, uint64_t q, uint64_t n, const int16_t* const* bases,
                             const uint64_t* n_bases, int16_t* const* outs, int32_t* maxima, uint64_t* loads) {
    frz_boost_pack(rules, n_rules, q, attr_of, g_plan);
    for (uint64_t j = 0; j < q; j++) {
        g_plan.queries[j].base = bases ? bases[j] : nullptr;
        g_plan.queries[j].n_base = bases && bases[j] ? n_bases[j] : 0;
        g_plan.queries[j].out = outs[j];
    }
    const FrzWhereBatchPlan& w = g_plan.where;
    std::vector<int32_t> max(q, 0);
    FrzBoostBatchDev b = {w.attrs.data(), w.clauses.data(), g_plan.adds.data(), g_plan.queries.data(), w.sets.data(), max.data(),
                          n, (uint32_t)q, w.n_staged()};
    std::vector<int64_t> staged((size_t)b.n_staged * kFrzWhereChunk);
    for (uint64_t j = 0; j < q; j++) loads[j] = 0;
    for (uint64_t i0 = 0; i0 < n; i0 += kFrzWhereChunk) {
        for (uint32_t t = 0; t < staged.size(); t++) staged[t] = frz_where_attr_value(b.attrs[t / kFrzWhereChunk], i0 + t % kFrzWhereChunk);
        for (uint64_t j = 0; j < q; j++) {
            const FrzBoostQuery& qr = b.queries[j];
            for (uint64_t i = i0; i < n && i < i0 + kFrzWhereChunk; i++) {
                frz_boost_rules_sum(b, qr, [&](const FrzWhereBatchClause&) { return (int64_t)++loads[j]; });
                const int16_t v = frz_boost_row(b, qr, staged.data(), i0, i);
                qr.out[i] = v;
                max[j] = std::max<int32_t>(max[j], v);
            }
        }
    }
    for (uint64_t j = 0; j < q; j++) maxima[j] = max[j];
}
