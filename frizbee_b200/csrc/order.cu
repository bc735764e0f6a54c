// order.cu — the ordered call's kernels (frz_match_list_ordered, DESIGN.md §4.15): the order keys, the MSB-first radix
// select over them, and the one-block sort of a small selection.  The key and the pick rule are order_plan.cuh's; host.cu
// runs the steps, and a large selection is sorted by the histogram-kernel sort with OrderKey digits (sort.cu).
//
//   k_order_keys        the key of every list row, in list order, and the OR of the keys and of their complements
//   k_order_pass        one select pass: compact the previous pass's candidates by its pick (selected rows to the selection
//                       list, the pick's bucket to the next candidates), histogram this pass's digit over the new
//                       candidates, and in the last block to finish, pick (frz_order_pick); a pass after the selection is
//                       complete returns at once
//   k_order_sort_block  at most kFrzOrderBlockRows selected rows: a bitonic sort in shared memory, then the first `limit`
//   k_order_gather      a larger selection's rows into a list for the multi-block sort
// The batched ordered call's sub-batches (frz_match_list_batch_ordered, DESIGN.md §4.11) run the same select and sort per
// query, one launch over the sub-batch's queries each (order_pass and order_sort_block are shared):
//   k_batch_order_keys     every list row's key
//   k_batch_order_members  the query's rows (its subset's members, kept by its collapse) → its first candidate list, and
//                          the masks of their keys
//   k_batch_order_pass     pass p: the query's p-th varying digit
//   k_batch_order_sort     one block per query: the sort, its first rows and its total
#include "batch_order_plan.cuh"
#include "frz_host.h"
#include "order_plan.cuh"

namespace {

constexpr int kOrderBlock = 256;   // == kFrzOrderBins: a pass's last block handles one bin per thread
static_assert(kOrderBlock == (int)kFrzOrderBins, "one bin per thread");
constexpr int kSortBlockThreads = 1024;
constexpr unsigned kFullWarp = 0xffffffffu;

__device__ __forceinline__ unsigned long long warp_or(unsigned long long x) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x |= __shfl_xor_sync(kFullWarp, x, o);
    return x;
}

__global__ void __launch_bounds__(kOrderBlock) k_order_keys(const FrzMatchDev* __restrict__ list, const unsigned long long* __restrict__ n_ptr,
                                                            const __grid_constant__ FrzOrderDev o, FrzOrderKey* __restrict__ keys,
                                                            FrzOrderState* __restrict__ st) {
    const unsigned long long n = *n_ptr;
    unsigned long long or_hi = 0, or_lo = 0, nor_hi = 0, nor_lo = 0;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const FrzMatchDev m = list[i];
        const FrzOrderKey k = frz_order_row_key(o, m.index, m.score);
        keys[i] = k;
        or_hi |= k.hi;
        or_lo |= k.lo;
        nor_hi |= ~k.hi;
        nor_lo |= ~k.lo & ((1ull << 48) - 1);
    }
    // one set of atomics per block: every block ORs into the same four words
    __shared__ unsigned long long s_or[kOrderBlock / 32][4];
    const uint32_t warp = threadIdx.x >> 5;
    or_hi = warp_or(or_hi);
    or_lo = warp_or(or_lo);
    nor_hi = warp_or(nor_hi);
    nor_lo = warp_or(nor_lo);
    if ((threadIdx.x & 31) == 0) {
        s_or[warp][0] = or_hi;
        s_or[warp][1] = or_lo;
        s_or[warp][2] = nor_hi;
        s_or[warp][3] = nor_lo;
    }
    __syncthreads();
    if (threadIdx.x < 4) {
        unsigned long long x = 0;
        for (uint32_t w = 0; w < kOrderBlock / 32; w++) x |= s_or[w][threadIdx.x];
        if (x) atomicOr(&st->vary_hi + threadIdx.x, x);   // vary_hi, vary_lo, flip_hi, flip_lo in turn
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) st->n = n;
}

// Appends the rows of the warp whose `want` is set to list[*count ..] (one atomic per warp); every lane must call it.
__device__ __forceinline__ void warp_append(bool want, uint32_t pos, unsigned long long* count, uint32_t* list) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t b = __ballot_sync(kFullWarp, want);
    if (!b) return;
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(count, (unsigned long long)__popc(b));
    base = __shfl_sync(kFullWarp, base, 0);
    if (want) list[base + __popc(b & ((1u << lane) - 1))] = pos;
}

// Pass p of the select (host.cu launches passes 0 .. P, P being the number of digits visited), once the select is known to
// be unfinished.  Pass 0 histograms digit `shift` over every row; pass p > 0 compacts the candidates of pass p - 1 (cand_in,
// or every row for p == 1) by its pick at `prev_shift`, and unless that pick took its bucket whole (or p == P: no digit
// left), histograms digit `shift` over the rows it keeps.  "Every row" is positions 0 .. st->n, or first_in[0 .. st->n)
// when first_in is given.  fit: frz_order_pick's.  h and is_last: the block's shared histogram and flag.
__device__ __forceinline__ void order_pass(const FrzOrderKey* __restrict__ keys, FrzOrderState* st, uint32_t* __restrict__ hist,
                                           const uint32_t* __restrict__ first_in, const uint32_t* __restrict__ cand_in,
                                           uint32_t* __restrict__ cand_out, uint32_t* __restrict__ sel, uint32_t p, uint32_t prev_shift,
                                           uint32_t shift, uint32_t has_digit, uint64_t need0, uint64_t fit, uint32_t* h, bool* is_last) {
    h[threadIdx.x] = 0;
    __syncthreads();
    const bool first = p == 0;
    const uint32_t bucket = first ? 0u : st->bucket;
    const bool take = !first && st->take != 0;
    const bool count = has_digit && !take;
    const unsigned long long n = p <= 1 ? st->n : st->n_cand[(p - 1) & 1];
    unsigned long long* n_out = &st->n_cand[p & 1];
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    // warp-uniform trips: every lane takes part in the appends' ballots
    const unsigned long long start = (unsigned long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u);
    for (unsigned long long i0 = start; i0 < n; i0 += stride) {
        const unsigned long long i = i0 + (threadIdx.x & 31);
        const bool valid = i < n;
        uint32_t pos = 0;
        FrzOrderKey k = {0, 0};
        if (valid) {
            pos = p <= 1 ? (first_in ? first_in[i] : (uint32_t)i) : cand_in[i];
            k = keys[pos];
        }
        bool keep = valid, selected = false;
        if (!first && valid) {
            const uint32_t d = frz_order_digit(k, prev_shift);
            keep = d == bucket && !take;
            selected = d > bucket || (d == bucket && take);
        }
        if (!first) {   // (warp-uniform)
            warp_append(selected, pos, &st->n_sel, sel);
            warp_append(keep && count, pos, n_out, cand_out);
        }
        if (keep && count) atomicAdd(&h[frz_order_digit(k, shift)], 1u);
    }
    __syncthreads();
    if (count && h[threadIdx.x]) atomicAdd(&hist[threadIdx.x], h[threadIdx.x]);
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) *is_last = atomicAdd(&st->done_blocks, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!*is_last) return;
    __threadfence();
    if (!count) {   // the selection is complete
        if (threadIdx.x == 0) {
            st->finished = 1;
            st->done_blocks = 0;
        }
        return;
    }
    h[threadIdx.x] = __ldcg(&hist[threadIdx.x]);
    hist[threadIdx.x] = 0;   // zero for the next pass and the next call
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned long long need = first ? need0 : st->need;
        const FrzOrderPick pk = frz_order_pick(h, need, __ldcg(&st->n_sel), fit);
        st->bucket = pk.bucket;
        st->take = pk.take;
        st->need = need - pk.above;
        st->n_cand[(p + 1) & 1] = 0;   // the next pass's output (this pass's input is consumed)
        st->done_blocks = 0;
    }
}

__global__ void __launch_bounds__(kOrderBlock) k_order_pass(const FrzOrderKey* __restrict__ keys, FrzOrderState* st,
                                                            uint32_t* __restrict__ hist, const uint32_t* __restrict__ cand_in,
                                                            uint32_t* __restrict__ cand_out, uint32_t* __restrict__ sel, uint32_t p,
                                                            uint32_t prev_shift, uint32_t shift, uint32_t has_digit, uint64_t need0,
                                                            uint64_t fit) {
    __shared__ uint32_t h[kFrzOrderBins];
    __shared__ bool is_last;
    frz_wait_prior_grid();   // the keys and the state come from the kernels ahead
    if (*(volatile unsigned int*)&st->finished) return;
    frz_allow_dependent_launch();
    order_pass(keys, st, hist, nullptr, cand_in, cand_out, sel, p, prev_shift, shift, has_digit, need0, fit, h, &is_last);
}

// One block: the n selected rows (positions sel[0 .. n), or every row 0 .. n when sel is null; n <= kFrzOrderBlockRows),
// sorted by descending key in shared memory (bitonic), and the first `limit` written to out as whole list records.
// smem: kFrzOrderBlockRows * 20 bytes.
__device__ __forceinline__ void order_sort_block(const FrzMatchDev* __restrict__ list, const FrzOrderKey* __restrict__ keys,
                                                 const uint32_t* __restrict__ sel, uint32_t n, uint32_t limit,
                                                 FrzMatchDev* __restrict__ out, unsigned long long* smem) {
    unsigned long long* s_hi = smem;
    unsigned long long* s_lo = s_hi + kFrzOrderBlockRows;
    uint32_t* s_pos = reinterpret_cast<uint32_t*>(s_lo + kFrzOrderBlockRows);
    constexpr uint32_t kPad = 0xFFFFFFFFu;   // a slot past the selection: behind every row
    uint32_t n2 = 1;
    while (n2 < n) n2 <<= 1;
    for (uint32_t j = threadIdx.x; j < n2; j += blockDim.x) {
        uint32_t pos = kPad;
        FrzOrderKey k = {0, 0};
        if (j < n) {
            pos = sel ? sel[j] : j;
            k = keys[pos];
        }
        s_hi[j] = k.hi;
        s_lo[j] = k.lo;
        s_pos[j] = pos;
    }
    __syncthreads();
    for (uint32_t size = 2; size <= n2; size <<= 1) {
        for (uint32_t half = size >> 1; half > 0; half >>= 1) {
            for (uint32_t t = threadIdx.x; t < n2 / 2; t += blockDim.x) {
                const uint32_t i = 2 * t - (t & (half - 1)), j = i + half;
                const FrzOrderKey a = {s_hi[i], s_lo[i]}, b = {s_hi[j], s_lo[j]};
                const bool a_ahead = s_pos[i] != kPad && (s_pos[j] == kPad || frz_order_ahead(a, b));
                const bool b_ahead = s_pos[j] != kPad && (s_pos[i] == kPad || frz_order_ahead(b, a));
                // the block of `size` at i is sorted ahead-first when (i & size) == 0, behind-first otherwise
                if ((i & size) == 0 ? b_ahead : a_ahead) {
                    s_hi[i] = b.hi; s_lo[i] = b.lo;
                    s_hi[j] = a.hi; s_lo[j] = a.lo;
                    const uint32_t q = s_pos[i];
                    s_pos[i] = s_pos[j];
                    s_pos[j] = q;
                }
            }
            __syncthreads();
        }
    }
    const uint32_t m = min(n, limit);
    for (uint32_t r = threadIdx.x; r < m; r += blockDim.x) out[r] = list[s_pos[r]];
}

// One block: the selected rows (positions sel[0 .. *n_ptr), or every row 0 .. *n_ptr when sel is null), sorted, the first
// `limit` → out (order_sort_block)
__global__ void __launch_bounds__(kSortBlockThreads) k_order_sort_block(const FrzMatchDev* __restrict__ list,
                                                                        const FrzOrderKey* __restrict__ keys,
                                                                        const uint32_t* __restrict__ sel,
                                                                        const unsigned long long* __restrict__ n_ptr, uint32_t limit,
                                                                        FrzMatchDev* __restrict__ out) {
    extern __shared__ unsigned long long smem[];
    frz_wait_prior_grid();   // the selection and the keys come from the kernels ahead
    const uint32_t n = (uint32_t)min(*n_ptr, (unsigned long long)kFrzOrderBlockRows);
    order_sort_block(list, keys, sel, n, limit, out, smem);
}

__global__ void __launch_bounds__(kOrderBlock) k_order_gather(const FrzMatchDev* __restrict__ list, const uint32_t* __restrict__ sel,
                                                              const unsigned long long* __restrict__ n_ptr, FrzMatchDev* __restrict__ out) {
    frz_wait_prior_grid();   // the selection comes from the passes
    const unsigned long long n = *n_ptr;
    for (unsigned long long j = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (unsigned long long)gridDim.x * blockDim.x)
        out[j] = list[sel[j]];
}

// The batched ordered call's sub-batches (frz_match_list_batch_ordered; the per-query arithmetic is
// batch_order_plan.cuh's): block row blockIdx.y is query j = blockIdx.y, with its own keys, rows, state and histogram.  A
// query whose sticky device error is set leaves at once; the sort then reports kFrzBatchOverflow.

// Every list row's key (k_order_keys without the masks: they are taken over the query's rows only)
__global__ void __launch_bounds__(kOrderBlock) k_batch_order_keys(const FrzBatchDev b, const FrzBatchOrderDev o) {
    const uint32_t j = blockIdx.y;
    if (b.ctr[j].error) return;
    const unsigned long long n = b.ctr[j].total;
    const FrzOrderDev od = o.ords[j];
    const FrzMatchDev* __restrict__ list = b.lists + j * b.list_stride;
    FrzOrderKey* __restrict__ keys = o.keys + frz_batch_order_keys_at(j, b.list_stride);
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const FrzMatchDev m = list[i];
        keys[i] = frz_order_row_key(od, m.index, m.score);
    }
}

// The query's rows (frz_batch_order_member) → its first candidate list, their number → st->n, and the OR of their keys
// and of their complements → the state's masks
__global__ void __launch_bounds__(kOrderBlock) k_batch_order_members(const FrzBatchDev b, const FrzBatchTables t, const FrzBatchOrderDev o) {
    __shared__ unsigned long long s_or[kOrderBlock / 32][4];
    const uint32_t j = blockIdx.y;
    if (b.ctr[j].error) return;
    const unsigned long long n = b.ctr[j].total;
    const FrzBatchScope s = t.scopes[j];
    FrzBatchCollapse c = {};
    if (t.cols) c = t.cols[j];
    const uint32_t* counts = c.ids ? t.counts + c.table : nullptr;
    const uint8_t* taken = t.taken + j * b.list_stride;   // (read for a grouped query only)
    const FrzMatchDev* __restrict__ list = b.lists + j * b.list_stride;
    const FrzOrderKey* __restrict__ keys = o.keys + frz_batch_order_keys_at(j, b.list_stride);
    uint32_t* rows = o.cand + frz_batch_order_cand_at(j, b.list_stride);
    FrzOrderState* st = o.st + j;
    unsigned long long or_hi = 0, or_lo = 0, nor_hi = 0, nor_lo = 0;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    // warp-uniform trips: every lane takes part in the append's ballot
    for (unsigned long long i0 = (unsigned long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < n; i0 += stride) {
        const unsigned long long i = i0 + (threadIdx.x & 31);
        bool in = false;
        if (i < n) {
            in = frz_batch_order_member(s.scoped ? s.bits : nullptr, s.n_bits, c.ids, c.n_ids, counts, c.per_group, c.ids && taken[i],
                                        list[i].index);
            if (in) {
                const FrzOrderKey k = keys[i];
                or_hi |= k.hi;
                or_lo |= k.lo;
                nor_hi |= ~k.hi;
                nor_lo |= ~k.lo & ((1ull << 48) - 1);
            }
        }
        warp_append(in, (uint32_t)i, &st->n, rows);
    }
    const uint32_t warp = threadIdx.x >> 5;
    or_hi = warp_or(or_hi);
    or_lo = warp_or(or_lo);
    nor_hi = warp_or(nor_hi);
    nor_lo = warp_or(nor_lo);
    if ((threadIdx.x & 31) == 0) {
        s_or[warp][0] = or_hi;
        s_or[warp][1] = or_lo;
        s_or[warp][2] = nor_hi;
        s_or[warp][3] = nor_lo;
    }
    __syncthreads();
    if (threadIdx.x < 4) {
        unsigned long long x = 0;
        for (uint32_t w = 0; w < kOrderBlock / 32; w++) x |= s_or[w][threadIdx.x];
        if (x) atomicOr(&st->vary_hi + threadIdx.x, x);   // vary_hi, vary_lo, flip_hi, flip_lo in turn
    }
}

// Pass p of every query's select (order_pass): its p-th varying digit, from its own masks.  A query whose rows fit the
// block sort, or with k = 0, has nothing to select; one that has finished, or has fewer digits, leaves at once.
__global__ void __launch_bounds__(kOrderBlock) k_batch_order_pass(const FrzBatchDev b, const FrzBatchOrderDev o, uint32_t k, uint32_t p) {
    __shared__ uint32_t h[kFrzOrderBins];
    __shared__ bool is_last;
    frz_wait_prior_grid();   // the rows and the state come from the kernels ahead
    const uint32_t j = blockIdx.y;
    FrzOrderState* st = o.st + j;
    if (b.ctr[j].error || *(volatile unsigned int*)&st->finished) return;
    frz_allow_dependent_launch();
    const unsigned long long n = st->n;
    if (k == 0 || frz_batch_order_whole(n)) return;
    const FrzOrderKey vary = frz_batch_order_vary(*st);
    uint32_t prev = 0, cur = 0;
    if (p > 0 && !frz_batch_order_shift(vary, p - 1, &prev)) return;
    const bool has_digit = frz_batch_order_shift(vary, p, &cur);
    uint32_t* cand = o.cand + frz_batch_order_cand_at(j, b.list_stride);
    order_pass(o.keys + frz_batch_order_keys_at(j, b.list_stride), st, o.hist + frz_batch_order_hist_at(j), cand,
               cand + (uint64_t)((p + 1) & 1) * b.list_stride, cand + (uint64_t)(p & 1) * b.list_stride, o.sel + frz_batch_order_sel_at(j),
               p, prev, cur, has_digit, min(n, (unsigned long long)k), kFrzOrderBlockRows, h, &is_last);
}

// One block per query: its rows (all of them when they fit, else the selection) sorted, the first min(k, total) → rows +
// frz_batch_row0(j, k), and its total → totals[j]
__global__ void __launch_bounds__(kSortBlockThreads) k_batch_order_sort(const FrzBatchDev b, const FrzBatchOrderDev o, uint32_t k,
                                                                        FrzMatchDev* __restrict__ rows,
                                                                        unsigned long long* __restrict__ totals) {
    extern __shared__ unsigned long long smem[];
    frz_wait_prior_grid();   // the selection comes from the passes
    const uint32_t j = blockIdx.x;
    const bool err = b.ctr[j].error != 0;
    const FrzOrderState* st = o.st + j;
    const unsigned long long n = st->n;
    if (threadIdx.x == 0) totals[j] = err ? kFrzBatchOverflow : n;
    if (err || k == 0 || n == 0) return;   // an overflowed sub-batch is run again query by query
    const bool whole = frz_batch_order_whole(n);
    const uint32_t* sel = whole ? o.cand + frz_batch_order_cand_at(j, b.list_stride) : o.sel + frz_batch_order_sel_at(j);
    const uint32_t n_sel = (uint32_t)min(whole ? n : st->n_sel, (unsigned long long)kFrzOrderBlockRows);
    order_sort_block(b.lists + j * b.list_stride, o.keys + frz_batch_order_keys_at(j, b.list_stride), sel, n_sel, k,
                     rows + frz_batch_row0(j, k), smem);
}

}  // namespace

frz_status frz_launch_order_keys(const FrzMatchDev* list, const unsigned long long* n_ptr, uint64_t n_cap, const FrzOrderDev& o,
                                 FrzOrderKey* keys, FrzOrderState* st, cudaStream_t stream, FrzLaunchStats* ls) {
    FRZ_CUDA_TRY(cudaMemsetAsync(st, 0, sizeof(FrzOrderState), stream));
    const int grid = std::min(grid_for(n_cap, kOrderBlock), frz_sm_count() * 4);
    k_order_keys<<<grid, kOrderBlock, 0, stream>>>(list, n_ptr, o, keys, st);
    FRZ_CUDA_TRY(cudaGetLastError());
    ls->launches++;
    return FRZ_OK;
}

frz_status frz_launch_order_select(const FrzOrderKey* keys, FrzOrderState* st, uint32_t* hist, uint32_t* cand, uint32_t* sel,
                                   uint64_t n, uint64_t need, const uint32_t* shifts, uint32_t n_shifts, uint64_t fit,
                                   cudaStream_t stream, FrzLaunchStats* ls) {
    const int grid = (int)std::max<uint64_t>(1, std::min<uint64_t>((n + kOrderBlock - 1) / kOrderBlock, (uint64_t)frz_sm_count() * 4));
    for (uint32_t p = 0; p <= n_shifts; p++) {
        const uint32_t prev = p ? shifts[p - 1] : 0u, cur = p < n_shifts ? shifts[p] : 0u;
        uint32_t* c_in = cand + (uint64_t)((p + 1) & 1) * n;   // pass p reads what pass p - 1 wrote
        uint32_t* c_out = cand + (uint64_t)(p & 1) * n;
        FRZ_CUDA_TRY(frz_launch_dependent(k_order_pass, grid, kOrderBlock, 0, stream, keys, st, hist, c_in, c_out, sel, p, prev, cur,
                                          (uint32_t)(p < n_shifts), need, fit));
    }
    ls->launches += n_shifts + 1;
    return FRZ_OK;
}

frz_status frz_launch_order_sort_block(const FrzMatchDev* list, const FrzOrderKey* keys, const uint32_t* sel,
                                       const unsigned long long* n_ptr, uint32_t limit, FrzMatchDev* out, cudaStream_t stream,
                                       FrzLaunchStats* ls) {
    constexpr size_t smem = (size_t)kFrzOrderBlockRows * (2 * sizeof(unsigned long long) + sizeof(uint32_t));
    FRZ_CUDA_TRY(cudaFuncSetAttribute(k_order_sort_block, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    FRZ_CUDA_TRY(frz_launch_dependent(k_order_sort_block, 1, kSortBlockThreads, smem, stream, list, keys, sel, n_ptr, limit, out));
    ls->launches++;
    return FRZ_OK;
}

frz_status frz_launch_order_gather(const FrzMatchDev* list, const uint32_t* sel, const unsigned long long* n_ptr, uint64_t n_cap,
                                   FrzMatchDev* out, cudaStream_t stream, FrzLaunchStats* ls) {
    FRZ_CUDA_TRY(frz_launch_dependent(k_order_gather, grid_for(n_cap, kOrderBlock), kOrderBlock, 0, stream, list, sel, n_ptr, out));
    ls->launches++;
    return FRZ_OK;
}

frz_status frz_launch_batch_order_keys(const FrzBatchDev& b, const FrzBatchOrderDev& o, uint32_t nq, cudaStream_t stream, FrzLaunchStats* st) {
    if (nq == 0) return FRZ_OK;
    const dim3 grid((uint32_t)std::max<uint64_t>(1, (uint64_t)grid_for(b.list_stride, kOrderBlock) / nq), nq);
    k_batch_order_keys<<<grid, kOrderBlock, 0, stream>>>(b, o);
    FRZ_CUDA_TRY(cudaGetLastError());
    st->launches++;
    return FRZ_OK;
}

frz_status frz_launch_batch_order_top(const FrzBatchDev& b, const FrzBatchTables& t, const FrzBatchOrderDev& o, uint32_t nq, uint32_t k,
                                      FrzMatchDev* rows, unsigned long long* totals, cudaStream_t stream, FrzLaunchStats* st) {
    if (nq == 0) return FRZ_OK;
    if (k > kFrzBatchMaxK) return frz_fail(FRZ_ERR_INVALID_ARG, "batched top-K serves k <= %u", kFrzBatchMaxK);
    // as many blocks in all as the single-query passes over one list of list_stride rows
    const dim3 grid((uint32_t)std::max<uint64_t>(1, (uint64_t)grid_for(b.list_stride, kOrderBlock) / nq), nq);
    k_batch_order_members<<<grid, kOrderBlock, 0, stream>>>(b, t, o);
    FRZ_CUDA_TRY(cudaGetLastError());
    for (uint32_t p = 0; p < kFrzBatchOrderPasses; p++)
        FRZ_CUDA_TRY(frz_launch_dependent(k_batch_order_pass, grid, kOrderBlock, 0, stream, b, o, k, p));
    constexpr size_t smem = (size_t)kFrzOrderBlockRows * (2 * sizeof(unsigned long long) + sizeof(uint32_t));
    FRZ_CUDA_TRY(cudaFuncSetAttribute(k_batch_order_sort, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    FRZ_CUDA_TRY(frz_launch_dependent(k_batch_order_sort, nq, kSortBlockThreads, smem, stream, b, o, k, rows, totals));
    st->launches += 2 + kFrzBatchOrderPasses;
    return FRZ_OK;
}
