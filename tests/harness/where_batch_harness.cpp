// CPU build of the batched-fill part of frizbee_b200/csrc/where_plan.cuh: the packer of frz_subset_where_batch (the
// call's distinct-attribute table, the clauses as references into it, every query's set values) and k_where_batch's
// staged word rule, through the header's own functions (tests/test_where_batch_host.py).
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../frizbee_b200/csrc/where_plan.cuh"
#include "../../include/frz_cuda.h"

// frz_where_batch_pack over ABI clauses whose attr handles point at FrzWhereBatchAttr records (the stand-in attributes);
// the plan stays here for h_where_batch_plan.  Returns the number of distinct attributes.
static FrzWhereBatchPlan g_plan;
extern "C" uint64_t h_where_batch_pack(const frz_where_clause* clauses, const uint64_t* n_clauses, uint64_t q) {
    frz_where_batch_pack(clauses, n_clauses, q, [](const frz_attr* a) { return *reinterpret_cast<const FrzWhereBatchAttr*>(a); }, g_plan);
    return g_plan.attrs.size();
}

// sizes[0..4) = attributes, clauses, set values, staged attributes; then the plan's arrays (each may be NULL)
extern "C" void h_where_batch_plan(uint64_t* sizes, FrzWhereBatchAttr* attrs, FrzWhereBatchClause* clauses, FrzWhereBatchQuery* queries,
                                   int64_t* sets) {
    sizes[0] = g_plan.attrs.size();
    sizes[1] = g_plan.clauses.size();
    sizes[2] = g_plan.sets.size();
    sizes[3] = g_plan.n_staged();
    if (attrs) memcpy(attrs, g_plan.attrs.data(), g_plan.attrs.size() * sizeof(FrzWhereBatchAttr));
    if (clauses) memcpy(clauses, g_plan.clauses.data(), g_plan.clauses.size() * sizeof(FrzWhereBatchClause));
    if (queries) memcpy(queries, g_plan.queries.data(), g_plan.queries.size() * sizeof(FrzWhereBatchQuery));
    if (sets) memcpy(sets, g_plan.sets.data(), g_plan.sets.size() * sizeof(int64_t));
}

// k_where_batch's word `word` of query j: the chunk's values of the staged attributes as the block stages them, the base
// word as the warp reads it, and the ballot of the 32 lanes' frz_where_batch_row
extern "C" uint32_t h_where_batch_word(const FrzWhereBatchDev* b, uint32_t j, uint64_t word) {
    const uint64_t chunk = word / kFrzWhereChunkWords, i0 = chunk * kFrzWhereChunk;
    std::vector<int64_t> staged((size_t)b->n_staged * kFrzWhereChunk);
    for (uint32_t t = 0; t < staged.size(); t++) staged[t] = frz_where_attr_value(b->attrs[t / kFrzWhereChunk], i0 + t % kFrzWhereChunk);
    const FrzWhereBatchQuery& qr = b->queries[j];
    const uint32_t base_word = qr.has_base && word * 32 < qr.n_base ? qr.base[word] : 0u;
    uint32_t w = 0;
    for (uint32_t lane = 0; lane < 32; lane++) w |= (uint32_t)frz_where_batch_row(*b, qr, staged.data(), i0, base_word, word * 32 + lane) << lane;
    return w;
}
