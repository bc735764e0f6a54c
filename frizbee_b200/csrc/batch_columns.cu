// batch_columns.cu — the join of a batched column call's sub-batch (frz_match_list_batch_columns, DESIGN.md §4.13).  Each
// column's batched stages leave one index-ordered list per query that has a pattern in it; k_batch_columns_fold folds
// them into per-query, per-row accumulators, and k_batch_columns_count / k_batch_columns_emit compact the rows that
// matched every column into each query's list, which k_batch_top (and, for grouped queries, the batched collapse) then
// cut as in frz_match_list_batch_collapsed.  The per-row rule is batch_columns_plan.cuh's.
#include "frz_device.cuh"

#include "batch_columns_plan.cuh"
#include "frz_host.h"

namespace {

constexpr int kFoldThreads = 256;
constexpr int kJoinThreads = FRZ_TILE;   // one tile of rows per block: the tile counts and bases of the batched stages

// row i's slot in the column is in use (it was not removed)
__device__ __forceinline__ bool row_live(const uint32_t* __restrict__ slot_meta, const uint16_t* __restrict__ slot_of, uint64_t i) {
    return slot_meta[(i & ~(uint64_t)(FRZ_TILE - 1)) + slot_of[i]] != FRZ_INVALID_SLOT;
}

// Block row blockIdx.y folds column c for query j = blockIdx.y: its list in the column's stages (b, slot f.slot), or the
// rows live in the column.  A query whose list overflowed marks its error word and folds nothing.
__global__ void __launch_bounds__(kFoldThreads) k_batch_columns_fold(const FrzBatchDev b, const FrzBatchColumnsDev d,
                                                                     const uint32_t* __restrict__ slot_meta,
                                                                     const uint16_t* __restrict__ slot_of, uint32_t c) {
    const uint32_t j = blockIdx.y;
    const FrzColumnFold f = d.fold[(uint64_t)c * gridDim.y + j];
    if (f.slot == kFrzColumnSkip) return;
    uint32_t* __restrict__ acc = d.acc + j * b.list_stride;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f.slot == kFrzColumnLive) {
        for (uint64_t i = i0; i < d.n_rows; i += stride)
            if (row_live(slot_meta, slot_of, i)) acc[i] = frz_columns_fold(acc[i], f.pass, 0, 0);
        return;
    }
    const FrzCounters& ctr = b.ctr[f.slot];
    if (ctr.error) {
        if (i0 == 0) d.err[j] = ctr.error;
        return;
    }
    const uint64_t n = ctr.total;
    const FrzMatchDev* __restrict__ list = b.lists + f.slot * b.list_stride;
    for (uint64_t i = i0; i < n; i += stride) {
        const FrzMatchDev r = list[i];
        acc[r.index] = frz_columns_fold(acc[r.index], f.pass, r.score, r.exact);
    }
}

// Block (t, j): query j's matches among the rows of tile t → b.tile_count[j][t]; block (0, j) also sets query j's error.
__global__ void __launch_bounds__(kJoinThreads) k_batch_columns_count(const FrzBatchDev b, const FrzBatchColumnsDev d, uint32_t n_tiles) {
    const uint32_t j = blockIdx.y, t = blockIdx.x;
    const uint64_t i = (uint64_t)t * FRZ_TILE + threadIdx.x;
    const bool keep = i < d.n_rows && frz_columns_matched(d.acc[j * b.list_stride + i], d.need[j]);
    const int n = __syncthreads_count(keep);
    if (threadIdx.x == 0) {
        b.tile_count[(uint64_t)j * n_tiles + t] = (uint32_t)n;
        if (t == 0) b.ctr[j].error = d.err[j];
    }
}

// Block (t, j): query j's matches among the rows of tile t → their records in b.lists[j], index order (reversed under the
// *_DESC strategies) from the tile's base.
__global__ void __launch_bounds__(kJoinThreads) k_batch_columns_emit(const FrzBatchDev b, const FrzBatchColumnsDev d, uint32_t n_tiles) {
    __shared__ uint32_t warp_cnt[kJoinThreads / 32];
    const uint32_t j = blockIdx.y, t = blockIdx.x;
    const uint32_t lane = frz_lane(), warp = threadIdx.x >> 5;
    const uint64_t i = (uint64_t)t * FRZ_TILE + threadIdx.x;
    const uint32_t a = i < d.n_rows ? d.acc[j * b.list_stride + i] : 0u;
    const bool keep = i < d.n_rows && frz_columns_matched(a, d.need[j]);
    const uint32_t ballot = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_cnt[warp] = __popc(ballot);
    __syncthreads();
    if (!keep) return;
    uint32_t before = __popc(ballot & ((1u << lane) - 1));
    for (uint32_t w = 0; w < warp; w++) before += warp_cnt[w];
    const uint64_t p = b.tile_out_base[(uint64_t)j * n_tiles + t] + before;
    FrzMatchDev r;
    r.index = (uint32_t)i;
    r.score = (uint16_t)frz_columns_score(a);
    r.exact = (uint8_t)frz_columns_exact(a);
    r.pad = 0;
    b.lists[j * b.list_stride + frz_columns_pos(p, b.ctr[j].total, b.reversed[j] != 0)] = r;
}

}  // namespace

frz_status frz_launch_batch_columns_fold(const FrzBatchDev& b, const FrzBatchColumnsDev& d, const FrzCorpusView& cv, uint32_t c,
                                         uint32_t nq, cudaStream_t stream, FrzLaunchStats* st) {
    if (nq == 0 || d.n_rows == 0) return FRZ_OK;
    // as many blocks in all as one pass over a list of n_rows rows
    const uint32_t gx = (uint32_t)std::max<uint64_t>(1, (uint64_t)grid_for(d.n_rows, kFoldThreads) / nq);
    k_batch_columns_fold<<<dim3(gx, nq), kFoldThreads, 0, stream>>>(b, d, cv.slot_meta, cv.slot_of, c);
    FRZ_CUDA_TRY(cudaGetLastError());
    st->launches++;
    return FRZ_OK;
}

frz_status frz_launch_batch_columns_join(const FrzBatchDev& b, const FrzBatchColumnsDev& d, uint32_t n_tiles, uint32_t nq,
                                         cudaStream_t stream, FrzLaunchStats* st) {
    if (nq == 0) return FRZ_OK;
    if (n_tiles) k_batch_columns_count<<<dim3(n_tiles, nq), kJoinThreads, 0, stream>>>(b, d, n_tiles);
    FRZ_CUDA_TRY(cudaGetLastError());
    FRZ_TRY(frz_launch_tile_scan_batch(b, n_tiles, nq, stream, st));
    if (n_tiles) k_batch_columns_emit<<<dim3(n_tiles, nq), kJoinThreads, 0, stream>>>(b, d, n_tiles);
    FRZ_CUDA_TRY(cudaGetLastError());
    st->launches += n_tiles ? 2 : 0;
    return FRZ_OK;
}
