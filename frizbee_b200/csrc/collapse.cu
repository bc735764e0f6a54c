// collapse.cu — the per-group count and the rounds of the collapsed call (frz_match_list_collapsed, DESIGN.md §4.12), of
// the ordered collapsed calls (frz_match_list_ordered_collapsed, frz_match_list_columns_ordered, §4.15.1), and of the
// batched collapsed call's sub-batches (frz_match_list_batch_collapsed, §4.11).  The row rule is collapse_plan.cuh's;
// host.cu compacts the kept rows and sorts them, or k_batch_top<CollapsedKey> (batch.cu) cuts them per query, or for the
// batched ordered call's sub-batches (frz_match_list_batch_ordered) the rounds run on the order key and the batched select
// (order.cu) orders the kept rows.
#include "batch_collapse_plan.cuh"
#include "batch_order_plan.cuh"
#include "collapse_plan.cuh"
#include "frz_host.h"

namespace {

constexpr int kCollapseBlock = 256;
constexpr unsigned kFullWarp = 0xffffffffu;

__device__ __forceinline__ uint64_t row_key(const FrzCollapseDev& c, const FrzMatchDev& r) {
    const int32_t b = c.order == FRZ_COLLAPSE_BY_KEY && r.index < c.n_boost ? (int32_t)c.boost[r.index] : 0;
    return frz_collapse_key(c.order, c.reversed != 0, r.score, b, r.index);
}

// The three kernels walk the list warp by warp (row i0 + lane, i0 warp-uniform), so every lane of a warp reaches the warp
// intrinsics together; lanes past the list's end hold no group.

// counts[group] += the list's rows in it; taken[i] = 0.  A warp adds once per distinct group among its lanes, so a group
// holding every row costs one atomic per warp.
__global__ void __launch_bounds__(kCollapseBlock) k_collapse_count(FrzCollapseDev c, const FrzMatchDev* __restrict__ list,
                                                                  const unsigned long long* __restrict__ n_ptr) {
    const unsigned long long n = *n_ptr;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < n; i0 += stride) {
        const uint64_t i = i0 + lane;
        uint32_t g = kFrzGroupNone;
        if (i < n) {
            g = frz_collapse_group(c.ids, c.n_ids, list[i].index);
            c.taken[i] = 0;
        }
        const uint32_t peers = __match_any_sync(kFullWarp, g);
        if (g != kFrzGroupNone && lane == (uint32_t)__ffs(peers) - 1) atomicAdd(&c.counts[g], (uint32_t)__popc(peers));
    }
}

// One round, first half: best[group] = the largest entry among the group's contenders.  A warp whose lanes all contend for
// one group reduces in registers and makes one atomic; an atomic that cannot raise the entry is skipped.
__global__ void __launch_bounds__(kCollapseBlock) k_collapse_max(FrzCollapseDev c, const FrzMatchDev* __restrict__ list,
                                                                const unsigned long long* __restrict__ n_ptr) {
    const unsigned long long n = *n_ptr;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < n; i0 += stride) {
        const uint64_t i = i0 + lane;
        uint32_t g = kFrzGroupNone;
        unsigned long long e = 0;
        if (i < n) {
            const FrzMatchDev r = list[i];
            const uint32_t rg = frz_collapse_group(c.ids, c.n_ids, r.index);
            if (rg != kFrzGroupNone && frz_collapse_contends(rg, c.counts[rg], c.per_group, c.taken[i] != 0)) {
                g = rg;
                e = frz_collapse_entry(row_key(c, r));
            }
        }
        const uint32_t peers = __match_any_sync(kFullWarp, g);
        if (g != kFrzGroupNone && peers == kFullWarp) {   // warp-uniform: every lane contends for g
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) e = max(e, __shfl_xor_sync(kFullWarp, e, d));
            if (lane == 0 && e > __ldcg(&c.best[g])) atomicMax(&c.best[g], e);
        } else if (g != kFrzGroupNone && e > __ldcg(&c.best[g])) {
            atomicMax(&c.best[g], e);
        }
    }
}

// One round, second half: the contender whose entry is the max is taken, and resets the entry for the next round.
__global__ void __launch_bounds__(kCollapseBlock) k_collapse_take(FrzCollapseDev c, const FrzMatchDev* __restrict__ list,
                                                                 const unsigned long long* __restrict__ n_ptr) {
    const unsigned long long n = *n_ptr;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const FrzMatchDev r = list[i];
        const uint32_t g = frz_collapse_group(c.ids, c.n_ids, r.index);
        if (g == kFrzGroupNone || !frz_collapse_contends(g, c.counts[g], c.per_group, c.taken[i] != 0)) continue;
        if (frz_collapse_entry(row_key(c, r)) == __ldcg(&c.best[g])) {
            c.taken[i] = 1;
            c.best[g] = 0;
        }
    }
}

// The rounds on the order key (frz_match_list_ordered_collapsed, the ordered column call): the three steps of
// collapse_plan.cuh's two-step max, one kernel each.  keys[i] is list row i's FrzOrderKey (k_order_keys, in list order), read
// as one 16-byte load; c.best is the best_hi table.  The max kernels keep k_collapse_max's warp-uniform register reduction
// and its skip of an atomic that cannot raise the entry.
__device__ __forceinline__ FrzOrderKey load_key(const FrzOrderKey* __restrict__ keys, uint64_t i) {
    const ulonglong2 v = __ldg(reinterpret_cast<const ulonglong2*>(keys) + i);
    return FrzOrderKey{v.x, v.y};
}

__device__ __forceinline__ void warp_max_into(unsigned long long* table, uint32_t g, unsigned long long e, uint32_t lane) {
    const uint32_t peers = __match_any_sync(kFullWarp, g);
    if (g != kFrzGroupNone && peers == kFullWarp) {   // warp-uniform: every lane contends for g
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) e = max(e, __shfl_xor_sync(kFullWarp, e, d));
        if (lane == 0 && e > __ldcg(&table[g])) atomicMax(&table[g], e);
    } else if (g != kFrzGroupNone && e > __ldcg(&table[g])) {
        atomicMax(&table[g], e);
    }
}

// Step 1: best_hi[group] = the largest hi among the group's contenders.
__global__ void __launch_bounds__(kCollapseBlock) k_collapse_max_hi(FrzCollapseDev c, const FrzMatchDev* __restrict__ list,
                                                                   const FrzOrderKey* __restrict__ keys,
                                                                   const unsigned long long* __restrict__ n_ptr) {
    const unsigned long long n = *n_ptr;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < n; i0 += stride) {
        const uint64_t i = i0 + lane;
        uint32_t g = kFrzGroupNone;
        unsigned long long e = 0;
        if (i < n) {
            const uint32_t rg = frz_collapse_group(c.ids, c.n_ids, list[i].index);
            if (rg != kFrzGroupNone && frz_collapse_contends(rg, c.counts[rg], c.per_group, c.taken[i] != 0)) {
                g = rg;
                e = frz_collapse_hi_entry(load_key(keys, i));
            }
        }
        warp_max_into(c.best, g, e, lane);
    }
}

// Step 2: best_lo[group] = the largest lo + 1 among the contenders whose hi is best_hi[group].
__global__ void __launch_bounds__(kCollapseBlock) k_collapse_max_lo(FrzCollapseDev c, const FrzMatchDev* __restrict__ list,
                                                                   const FrzOrderKey* __restrict__ keys, unsigned long long* best_lo,
                                                                   const unsigned long long* __restrict__ n_ptr) {
    const unsigned long long n = *n_ptr;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < n; i0 += stride) {
        const uint64_t i = i0 + lane;
        uint32_t g = kFrzGroupNone;
        unsigned long long e = 0;
        if (i < n) {
            const uint32_t rg = frz_collapse_group(c.ids, c.n_ids, list[i].index);
            if (rg != kFrzGroupNone && frz_collapse_contends(rg, c.counts[rg], c.per_group, c.taken[i] != 0)) {
                g = rg;
                e = frz_collapse_lo_entry(load_key(keys, i), __ldcg(&c.best[rg]));
            }
        }
        warp_max_into(best_lo, g, e, lane);
    }
}

// Step 3: the contender whose lo + 1 is best_lo[group] is taken, and resets both entries for the next round.
__global__ void __launch_bounds__(kCollapseBlock) k_collapse_take_key(FrzCollapseDev c, const FrzMatchDev* __restrict__ list,
                                                                     const FrzOrderKey* __restrict__ keys, unsigned long long* best_lo,
                                                                     const unsigned long long* __restrict__ n_ptr) {
    const unsigned long long n = *n_ptr;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t g = frz_collapse_group(c.ids, c.n_ids, list[i].index);
        if (g == kFrzGroupNone || !frz_collapse_contends(g, c.counts[g], c.per_group, c.taken[i] != 0)) continue;
        if (frz_collapse_key_takes(load_key(keys, i), __ldcg(&best_lo[g]))) {
            c.taken[i] = 1;
            c.best[g] = 0;
            best_lo[g] = 0;
        }
    }
}

// The batched passes (frz_match_list_batch_collapsed): block row blockIdx.y walks query j = blockIdx.y's list as the kernels
// above walk one list, over the rows that are members of its subset (non-members are in the list: the subset is applied
// late), with its own tables.  A query without groups, with its device error set, or past its rounds leaves at once.
struct BatchQuery {
    FrzBatchCollapse c;
    FrzBatchScope s;
    const FrzMatchDev* list;
    uint8_t* taken;
    unsigned long long n;
    uint8_t reversed;
};
__device__ __forceinline__ bool batch_query(const FrzBatchDev& b, const FrzBatchTables& t, uint32_t j, BatchQuery* q) {
    q->c = t.cols[j];
    if (!q->c.ids || b.ctr[j].error) return false;
    q->s = t.scopes[j];
    q->list = b.lists + j * b.list_stride;
    q->taken = t.taken + j * b.list_stride;
    q->n = b.ctr[j].total;
    q->reversed = b.reversed[j];
    return true;
}
// the group of a list row, kFrzGroupNone for a row in no group or not a member of the query's subset
__device__ __forceinline__ uint32_t batch_group(const BatchQuery& q, uint32_t index) {
    if (q.s.scoped && !frz_batch_member(q.s.bits, q.s.n_bits, index)) return kFrzGroupNone;
    return frz_collapse_group(q.c.ids, q.c.n_ids, index);
}
__device__ __forceinline__ uint64_t batch_entry(const BatchQuery& q, const FrzMatchDev& r) {
    const int32_t b = q.c.order == FRZ_COLLAPSE_BY_KEY && r.index < q.s.n_boost ? (int32_t)q.s.boost[r.index] : 0;
    return frz_collapse_entry(frz_collapse_key(q.c.order, q.reversed != 0, r.score, b, r.index));
}

__global__ void __launch_bounds__(kCollapseBlock) k_batch_collapse_count(const FrzBatchDev b, const FrzBatchTables t) {
    BatchQuery q;
    if (!batch_query(b, t, blockIdx.y, &q)) return;
    uint32_t* counts = t.counts + q.c.table;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < q.n; i0 += stride) {
        const uint64_t i = i0 + lane;
        uint32_t g = kFrzGroupNone;
        if (i < q.n) {
            g = batch_group(q, q.list[i].index);
            q.taken[i] = 0;
        }
        const uint32_t peers = __match_any_sync(kFullWarp, g);
        if (g != kFrzGroupNone && lane == (uint32_t)__ffs(peers) - 1) atomicAdd(&counts[g], (uint32_t)__popc(peers));
    }
}

__global__ void __launch_bounds__(kCollapseBlock) k_batch_collapse_max(const FrzBatchDev b, const FrzBatchTables t, uint32_t round) {
    BatchQuery q;
    if (!batch_query(b, t, blockIdx.y, &q) || !frz_batch_collapse_in_round(q.c.per_group, round)) return;
    const uint32_t* counts = t.counts + q.c.table;
    unsigned long long* best = t.best + q.c.table;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < q.n; i0 += stride) {
        const uint64_t i = i0 + lane;
        uint32_t g = kFrzGroupNone;
        unsigned long long e = 0;
        if (i < q.n) {
            const FrzMatchDev r = q.list[i];
            const uint32_t rg = batch_group(q, r.index);
            if (rg != kFrzGroupNone && frz_collapse_contends(rg, counts[rg], q.c.per_group, q.taken[i] != 0)) {
                g = rg;
                e = batch_entry(q, r);
            }
        }
        const uint32_t peers = __match_any_sync(kFullWarp, g);
        if (g != kFrzGroupNone && peers == kFullWarp) {   // warp-uniform: every lane contends for g
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) e = max(e, __shfl_xor_sync(kFullWarp, e, d));
            if (lane == 0 && e > __ldcg(&best[g])) atomicMax(&best[g], e);
        } else if (g != kFrzGroupNone && e > __ldcg(&best[g])) {
            atomicMax(&best[g], e);
        }
    }
}

__global__ void __launch_bounds__(kCollapseBlock) k_batch_collapse_take(const FrzBatchDev b, const FrzBatchTables t, uint32_t round) {
    BatchQuery q;
    if (!batch_query(b, t, blockIdx.y, &q) || !frz_batch_collapse_in_round(q.c.per_group, round)) return;
    const uint32_t* counts = t.counts + q.c.table;
    unsigned long long* best = t.best + q.c.table;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < q.n; i += (uint64_t)gridDim.x * blockDim.x) {
        const FrzMatchDev r = q.list[i];
        const uint32_t g = batch_group(q, r.index);
        if (g == kFrzGroupNone || !frz_collapse_contends(g, counts[g], q.c.per_group, q.taken[i] != 0)) continue;
        if (batch_entry(q, r) == __ldcg(&best[g])) {
            q.taken[i] = 1;
            best[g] = 0;
        }
    }
}

// The batched rounds on the order key (frz_match_list_batch_ordered): k_collapse_max_hi / _max_lo / _take_key per query,
// over its members, with its keys (k_batch_order_keys), its best table as best_hi and its best_lo table.
__global__ void __launch_bounds__(kCollapseBlock) k_batch_collapse_max_hi(const FrzBatchDev b, const FrzBatchTables t,
                                                                         const FrzBatchOrderDev o, uint32_t round) {
    BatchQuery q;
    if (!batch_query(b, t, blockIdx.y, &q) || !frz_batch_collapse_in_round(q.c.per_group, round)) return;
    const uint32_t* counts = t.counts + q.c.table;
    unsigned long long* best_hi = t.best + q.c.table;
    const FrzOrderKey* keys = o.keys + frz_batch_order_keys_at(blockIdx.y, b.list_stride);
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < q.n; i0 += stride) {
        const uint64_t i = i0 + lane;
        uint32_t g = kFrzGroupNone;
        unsigned long long e = 0;
        if (i < q.n) {
            const uint32_t rg = batch_group(q, q.list[i].index);
            if (rg != kFrzGroupNone && frz_collapse_contends(rg, counts[rg], q.c.per_group, q.taken[i] != 0)) {
                g = rg;
                e = frz_collapse_hi_entry(load_key(keys, i));
            }
        }
        warp_max_into(best_hi, g, e, lane);
    }
}

__global__ void __launch_bounds__(kCollapseBlock) k_batch_collapse_max_lo(const FrzBatchDev b, const FrzBatchTables t,
                                                                         const FrzBatchOrderDev o, uint32_t round) {
    BatchQuery q;
    if (!batch_query(b, t, blockIdx.y, &q) || !frz_batch_collapse_in_round(q.c.per_group, round)) return;
    const uint32_t* counts = t.counts + q.c.table;
    const unsigned long long* best_hi = t.best + q.c.table;
    unsigned long long* best_lo = o.best_lo + q.c.table;
    const FrzOrderKey* keys = o.keys + frz_batch_order_keys_at(blockIdx.y, b.list_stride);
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < q.n; i0 += stride) {
        const uint64_t i = i0 + lane;
        uint32_t g = kFrzGroupNone;
        unsigned long long e = 0;
        if (i < q.n) {
            const uint32_t rg = batch_group(q, q.list[i].index);
            if (rg != kFrzGroupNone && frz_collapse_contends(rg, counts[rg], q.c.per_group, q.taken[i] != 0)) {
                g = rg;
                e = frz_collapse_lo_entry(load_key(keys, i), __ldcg(&best_hi[rg]));
            }
        }
        warp_max_into(best_lo, g, e, lane);
    }
}

__global__ void __launch_bounds__(kCollapseBlock) k_batch_collapse_take_key(const FrzBatchDev b, const FrzBatchTables t,
                                                                           const FrzBatchOrderDev o, uint32_t round) {
    BatchQuery q;
    if (!batch_query(b, t, blockIdx.y, &q) || !frz_batch_collapse_in_round(q.c.per_group, round)) return;
    const uint32_t* counts = t.counts + q.c.table;
    unsigned long long* best_hi = t.best + q.c.table;
    unsigned long long* best_lo = o.best_lo + q.c.table;
    const FrzOrderKey* keys = o.keys + frz_batch_order_keys_at(blockIdx.y, b.list_stride);
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < q.n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t g = batch_group(q, q.list[i].index);
        if (g == kFrzGroupNone || !frz_collapse_contends(g, counts[g], q.c.per_group, q.taken[i] != 0)) continue;
        if (frz_collapse_key_takes(load_key(keys, i), __ldcg(&best_lo[g]))) {
            q.taken[i] = 1;
            best_hi[g] = 0;
            best_lo[g] = 0;
        }
    }
}

}  // namespace

frz_status frz_launch_batch_collapse(const FrzBatchDev& b, const FrzBatchTables& t, uint32_t nq, uint32_t rounds, cudaStream_t stream,
                                     FrzLaunchStats* st) {
    if (nq == 0) return FRZ_OK;
    // as many blocks in all as the single-query passes over one list of list_stride rows
    const uint32_t gx = (uint32_t)std::max<uint64_t>(1, (uint64_t)grid_for(b.list_stride, kCollapseBlock) / nq);
    const dim3 grid(gx, nq);
    k_batch_collapse_count<<<grid, kCollapseBlock, 0, stream>>>(b, t);
    for (uint32_t r = 0; r < rounds; r++) {
        k_batch_collapse_max<<<grid, kCollapseBlock, 0, stream>>>(b, t, r);
        k_batch_collapse_take<<<grid, kCollapseBlock, 0, stream>>>(b, t, r);
    }
    st->launches += 1 + 2 * (uint64_t)rounds;
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

frz_status frz_launch_batch_collapse_by_key(const FrzBatchDev& b, const FrzBatchTables& t, const FrzBatchOrderDev& o, uint32_t nq,
                                            uint32_t rounds, cudaStream_t stream, FrzLaunchStats* st) {
    if (nq == 0) return FRZ_OK;
    const uint32_t gx = (uint32_t)std::max<uint64_t>(1, (uint64_t)grid_for(b.list_stride, kCollapseBlock) / nq);
    const dim3 grid(gx, nq);
    k_batch_collapse_count<<<grid, kCollapseBlock, 0, stream>>>(b, t);
    for (uint32_t r = 0; r < rounds; r++) {
        k_batch_collapse_max_hi<<<grid, kCollapseBlock, 0, stream>>>(b, t, o, r);
        k_batch_collapse_max_lo<<<grid, kCollapseBlock, 0, stream>>>(b, t, o, r);
        k_batch_collapse_take_key<<<grid, kCollapseBlock, 0, stream>>>(b, t, o, r);
    }
    st->launches += 1 + 3 * (uint64_t)rounds;
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

frz_status frz_launch_collapse(const FrzCollapseDev& c, const FrzMatchDev* list, const unsigned long long* n_ptr, uint64_t n_cap,
                               uint64_t n_groups, uint32_t rounds, cudaStream_t stream, FrzLaunchStats* st) {
    FRZ_CUDA_TRY(cudaMemsetAsync(c.counts, 0, n_groups * sizeof(uint32_t), stream));
    const int grid = grid_for(n_cap, kCollapseBlock);
    k_collapse_count<<<grid, kCollapseBlock, 0, stream>>>(c, list, n_ptr);
    for (uint32_t r = 0; r < rounds; r++) {
        k_collapse_max<<<grid, kCollapseBlock, 0, stream>>>(c, list, n_ptr);
        k_collapse_take<<<grid, kCollapseBlock, 0, stream>>>(c, list, n_ptr);
    }
    st->launches += 1 + 2 * (uint64_t)rounds;
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

frz_status frz_launch_collapse_by_key(const FrzCollapseDev& c, unsigned long long* best_lo, const FrzOrderKey* keys,
                                      const FrzMatchDev* list, const unsigned long long* n_ptr, uint64_t n_cap, uint64_t n_groups,
                                      uint32_t rounds, cudaStream_t stream, FrzLaunchStats* st) {
    FRZ_CUDA_TRY(cudaMemsetAsync(c.counts, 0, n_groups * sizeof(uint32_t), stream));
    const int grid = grid_for(n_cap, kCollapseBlock);
    k_collapse_count<<<grid, kCollapseBlock, 0, stream>>>(c, list, n_ptr);
    for (uint32_t r = 0; r < rounds; r++) {
        k_collapse_max_hi<<<grid, kCollapseBlock, 0, stream>>>(c, list, keys, n_ptr);
        k_collapse_max_lo<<<grid, kCollapseBlock, 0, stream>>>(c, list, keys, best_lo, n_ptr);
        k_collapse_take_key<<<grid, kCollapseBlock, 0, stream>>>(c, list, keys, best_lo, n_ptr);
    }
    st->launches += 1 + 3 * (uint64_t)rounds;
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}
