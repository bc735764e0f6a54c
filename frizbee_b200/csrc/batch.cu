// batch.cu — the last stage of a batched top-K sub-batch (frz_match_list_batch, DESIGN.md §4.11): every query's first
// min(k, total) rows out of its index-ordered list, in one launch of one block per query.  The position arithmetic is
// batch_plan.cuh's (shared with the CPU tests).
#include "frz_device.cuh"

#include "batch_collapse_plan.cuh"
#include "batch_plan.cuh"
#include "frz_host.h"

namespace {

constexpr int kTopThreads = 1024;
static_assert(kFrzBatchMaxK <= kTopThreads, "one kept row per thread in the sort");

// exclusive count of the block's threads before this one with `f` set, and the block's count in *all (every thread)
__device__ __forceinline__ uint32_t block_excl_count(bool f, uint32_t* warp_cnt, uint32_t* all) {
    const uint32_t lane = frz_lane(), warp = threadIdx.x >> 5;
    const uint32_t ballot = __ballot_sync(0xffffffffu, f);
    if (lane == 0) warp_cnt[warp] = __popc(ballot);
    __syncthreads();
    uint32_t before = 0, sum = 0;
    for (uint32_t w = 0; w < blockDim.x / 32; w++) {
        const uint32_t c = warp_cnt[w];
        before += w < warp ? c : 0;
        sum += c;
    }
    __syncthreads();   // warp_cnt is reused by the next call
    *all = sum;
    return before + __popc(ballot & ((1u << lane) - 1));
}

// the sum of every thread's v (every thread)
__device__ __forceinline__ uint64_t block_sum(uint32_t v, uint32_t* warp_cnt) {
    v = __reduce_add_sync(0xffffffffu, v);
    if (frz_lane() == 0) warp_cnt[threadIdx.x >> 5] = v;
    __syncthreads();
    uint64_t sum = 0;
    for (uint32_t w = 0; w < blockDim.x / 32; w++) sum += warp_cnt[w];
    __syncthreads();   // warp_cnt is reused by the next call
    return sum;
}

// The key source of k_batch_top: which rows of a query's list are its rows, and the 16-bit value they are ordered by.
// ScoreKey (frz_match_list_batch_top): every row, by score under the score strategies.
struct ScoreKey {
    static constexpr bool kScoped = false;
    struct Query {};
    __device__ __forceinline__ Query query(uint32_t) const { return Query(); }
    __device__ __forceinline__ static bool by_value(const Query&, bool by_score) { return by_score; }
    __device__ __forceinline__ static bool member(const Query&, const FrzMatchDev*) { return true; }
    __device__ __forceinline__ static uint32_t value(const Query&, const FrzMatchDev* m) { return m->score; }
};
// ScopedKey (frz_match_list_batch): a scoped query's rows are its subset's members; a ranked query is ordered by
// clamp(score + boost[index], 0, 65535) under every strategy.  The rows themselves keep their raw scores.
struct ScopedKey {
    static constexpr bool kScoped = true;
    const FrzBatchScope* scopes;   // [j]
    using Query = FrzBatchScope;
    __device__ __forceinline__ Query query(uint32_t j) const { return scopes[j]; }
    __device__ __forceinline__ static bool by_value(const Query& q, bool by_score) { return q.ranked || by_score; }
    __device__ __forceinline__ static bool member(const Query& q, const FrzMatchDev* m) {
        return !q.scoped || frz_batch_member(q.bits, q.n_bits, m->index);
    }
    __device__ __forceinline__ static uint32_t value(const Query& q, const FrzMatchDev* m) {
        if (!q.ranked) return m->score;
        const uint32_t i = m->index;
        return frz_batch_ranked_value(m->score, i < q.n_boost ? (int32_t)__ldg(q.boost + i) : 0);
    }
};

// CollapsedKey (frz_match_list_batch_collapsed): a grouped query's rows are the members of its subset that its collapse
// keeps (frz_collapse_keep, after the rounds of collapse.cu); its total is their number, |C|.  Value and order are
// ScopedKey's.  A query without groups is answered as under ScopedKey.
struct CollapsedKey {
    static constexpr bool kScoped = true;
    FrzBatchTables t;
    const FrzMatchDev* lists;
    uint64_t list_stride;
    struct Query {
        FrzBatchScope s;
        FrzBatchCollapse c;
        const uint32_t* counts;    // the query's count table
        const uint8_t* taken;      // [list row]
        const FrzMatchDev* list;
        bool scoped;               // its rows are a filter of its list: a subset, or groups with a cap
    };
    __device__ __forceinline__ Query query(uint32_t j) const {
        Query q;
        q.s = t.scopes[j];
        q.c = t.cols[j];
        q.counts = t.counts + q.c.table;
        q.taken = t.taken + j * list_stride;
        q.list = lists + j * list_stride;
        q.scoped = q.s.scoped || (q.c.ids && frz_batch_collapse_rounds(q.c.per_group) > 0);
        return q;
    }
    __device__ __forceinline__ static bool by_value(const Query& q, bool by_score) { return ScopedKey::by_value(q.s, by_score); }
    __device__ __forceinline__ static bool member(const Query& q, const FrzMatchDev* m) {
        if (!ScopedKey::member(q.s, m)) return false;
        if (!q.c.ids) return true;
        const uint32_t g = frz_collapse_group(q.c.ids, q.c.n_ids, m->index);
        return frz_collapse_keep(g, g == kFrzGroupNone ? 0u : q.counts[g], q.c.per_group, q.taken[m - q.list] != 0);
    }
    __device__ __forceinline__ static uint32_t value(const Query& q, const FrzMatchDev* m) { return ScopedKey::value(q.s, m); }
};

template <class Key>
__global__ void __launch_bounds__(kTopThreads) k_batch_top(const FrzBatchDev b, uint32_t k, FrzMatchDev* __restrict__ rows,
                                                           unsigned long long* __restrict__ totals, const Key key) {
    __shared__ uint32_t hist[kFrzBatchBins];
    __shared__ uint64_t keys[kFrzBatchMaxK];
    __shared__ uint32_t warp_cnt[32];
    __shared__ int hi_bin;
    __shared__ unsigned long long above_hi;
    __shared__ FrzBatchCut cut;
    const uint32_t j = blockIdx.x;
    const uint64_t n_list = b.ctr[j].total;   // the list's length; `total` counts the query's rows in it
    const unsigned int err = b.ctr[j].error;
    const typename Key::Query kq = key.query(j);
    const FrzMatchDev* __restrict__ list = b.lists + j * b.list_stride;
    uint64_t total = n_list;
    if constexpr (Key::kScoped) {
        if (!err && kq.scoped) {
            uint32_t c = 0;
            for (uint64_t i = threadIdx.x; i < n_list; i += blockDim.x) c += Key::member(kq, list + i);
            total = block_sum(c, warp_cnt);
        }
    }
    if (threadIdx.x == 0) totals[j] = err ? kFrzBatchOverflow : total;
    const uint32_t n_rows = (uint32_t)frz_batch_rows(k, total);
    if (err || n_rows == 0) return;   // an overflowed sub-batch is run again query by query
    FrzMatchDev* __restrict__ out = rows + frz_batch_row0(j, k);
    if (!Key::by_value(kq, b.by_score[j])) {   // index order: the list's head
        if constexpr (Key::kScoped) {
            if (kq.scoped) {   // its members' head
                uint32_t kept = 0;
                for (uint64_t base = 0; base < n_list && kept < n_rows; base += blockDim.x) {
                    const uint64_t i = base + threadIdx.x;
                    const bool in = i < n_list && Key::member(kq, list + i);
                    uint32_t n_in = 0;
                    const uint32_t pos = kept + block_excl_count(in, warp_cnt, &n_in);
                    if (in && pos < n_rows) out[pos] = list[i];
                    kept += n_in;
                }
                return;
            }
        }
        for (uint32_t i = threadIdx.x; i < n_rows; i += blockDim.x) out[i] = list[i];
        return;
    }
    // the cut: high value byte, then low value byte within the selected high bin
    for (uint32_t i = threadIdx.x; i < kFrzBatchBins; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (uint64_t i = threadIdx.x; i < n_list; i += blockDim.x)
        if (Key::member(kq, list + i)) atomicAdd(&hist[Key::value(kq, list + i) >> 8], 1u);
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t a = 0;
        hi_bin = frz_batch_cut_hi(hist, n_rows, &a);
        above_hi = a;
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < kFrzBatchBins; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const uint32_t hb = (uint32_t)hi_bin;
    for (uint64_t i = threadIdx.x; i < n_list; i += blockDim.x) {
        if (!Key::member(kq, list + i)) continue;
        const uint32_t s = Key::value(kq, list + i);
        if ((s >> 8) == hb) atomicAdd(&hist[s & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) cut = frz_batch_cut_lo(hist, hi_bin, above_hi, n_rows);
    __syncthreads();
    const FrzBatchCut c = cut;
    // the kept rows, in list order
    uint64_t eq_base = 0;
    uint32_t kept = 0;
    for (uint64_t base = 0; base < n_list && kept < n_rows; base += blockDim.x) {
        const uint64_t i = base + threadIdx.x;
        const bool valid = i < n_list && Key::member(kq, list + i);
        const uint32_t s = valid ? Key::value(kq, list + i) : 0u;
        uint32_t n_eq = 0, n_keep = 0;
        const uint32_t eq_before = block_excl_count(valid && s == c.threshold, warp_cnt, &n_eq);
        const bool keep = valid && frz_batch_keep(s, c, eq_base + eq_before);
        const uint32_t pos = kept + block_excl_count(keep, warp_cnt, &n_keep);
        if (keep) keys[pos] = frz_batch_key(s, (uint32_t)i);
        eq_base += n_eq;
        kept += n_keep;
    }
    // bitonic sort of the kept keys (padded to a power of two)
    uint32_t p2 = 1;
    while (p2 < n_rows) p2 <<= 1;
    for (uint32_t i = n_rows + threadIdx.x; i < p2; i += blockDim.x) keys[i] = ~0ull;
    __syncthreads();
    for (uint32_t size = 2; size <= p2; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            const uint32_t i = threadIdx.x, partner = i ^ stride;
            if (i < p2 && partner > i) {
                const uint64_t x = keys[i], y = keys[partner];
                if ((x > y) == ((i & size) == 0)) { keys[i] = y; keys[partner] = x; }
            }
            __syncthreads();
        }
    }
    for (uint32_t i = threadIdx.x; i < n_rows; i += blockDim.x) out[i] = list[frz_batch_key_pos(keys[i])];
}

}  // namespace

frz_status frz_launch_batch_top(const FrzBatchDev& b, const FrzBatchScope* scopes, uint32_t nq, uint32_t k, FrzMatchDev* rows,
                                unsigned long long* totals, cudaStream_t stream, FrzLaunchStats* st) {
    if (nq == 0) return FRZ_OK;
    if (k > kFrzBatchMaxK) return frz_fail(FRZ_ERR_INVALID_ARG, "batched top-K serves k <= %u", kFrzBatchMaxK);
    if (scopes) k_batch_top<<<nq, kTopThreads, 0, stream>>>(b, k, rows, totals, ScopedKey{scopes});
    else k_batch_top<<<nq, kTopThreads, 0, stream>>>(b, k, rows, totals, ScoreKey());
    FRZ_CUDA_TRY(cudaGetLastError());
    if (st) st->launches++;
    return FRZ_OK;
}

frz_status frz_launch_batch_top_collapsed(const FrzBatchDev& b, const FrzBatchTables& t, uint32_t nq, uint32_t k, FrzMatchDev* rows,
                                          unsigned long long* totals, cudaStream_t stream, FrzLaunchStats* st) {
    if (nq == 0) return FRZ_OK;
    if (k > kFrzBatchMaxK) return frz_fail(FRZ_ERR_INVALID_ARG, "batched top-K serves k <= %u", kFrzBatchMaxK);
    k_batch_top<<<nq, kTopThreads, 0, stream>>>(b, k, rows, totals, CollapsedKey{t, b.lists, b.list_stride});
    FRZ_CUDA_TRY(cudaGetLastError());
    st->launches++;
    return FRZ_OK;
}
