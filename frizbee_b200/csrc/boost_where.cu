// boost_where.cu — the fill of frz_boost_where and frz_boost_where_batch (DESIGN.md §4.18): every query's boost values
// and their maximum from its rules and its base.  The row rule is boost_plan.cuh's; host.cu owns the boosts and reads the
// maxima back.  The single call is the batch of one.
#include "frz_host.h"
#include "boost_plan.cuh"

namespace {

constexpr int kBoostBlock = 256;
constexpr uint32_t kBoostWarps = kBoostBlock / 32;
constexpr uint32_t kBoostRound = 32;   // queries whose maxima a block gathers per round
constexpr unsigned kFullWarp = 0xffffffffu;

// Block (x, y) walks chunks of kFrzWhereChunk indices along x.  For each it stages the chunk's values of the staged
// attributes in shared memory (k_where_batch's staging), then writes the chunk's values of queries [y * per_block, ...):
// per query, thread t takes indices t, t + 256, t + 512 and t + 768 of the chunk, so each warp's int16 stores are
// coalesced.  A warp's maximum of a round of kBoostRound queries meets the other warps' in shared memory, and one thread
// per query folds the block's maximum into b.max with one atomicMax (none when it is at most 0, the cell's start).
__global__ void __launch_bounds__(kBoostBlock) k_boost_where(const __grid_constant__ FrzBoostBatchDev b, uint32_t per_block) {
    extern __shared__ int64_t s_vals[];   // [n_staged][kFrzWhereChunk]
    __shared__ int32_t s_max[kBoostWarps][kBoostRound];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t n_chunks = (b.n + kFrzWhereChunk - 1) / kFrzWhereChunk;
    const uint32_t j0 = blockIdx.y * per_block, j1 = min(b.q, j0 + per_block);
    for (uint64_t chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x) {
        const uint64_t i0 = chunk * kFrzWhereChunk;
        for (uint32_t t = threadIdx.x; t < b.n_staged * (uint32_t)kFrzWhereChunk; t += blockDim.x)
            s_vals[t] = frz_where_attr_value(b.attrs[t / kFrzWhereChunk], i0 + t % kFrzWhereChunk);
        __syncthreads();
        for (uint32_t r0 = j0; r0 < j1; r0 += kBoostRound) {
            const uint32_t r1 = min(j1, r0 + kBoostRound);
            for (uint32_t j = r0; j < r1; j++) {
                const FrzBoostQuery& qr = b.queries[j];
                int32_t m = 0;
#pragma unroll
                for (uint32_t k = 0; k < kFrzWhereChunk / kBoostBlock; k++) {
                    const uint64_t i = i0 + k * kBoostBlock + threadIdx.x;
                    if (i < b.n) {
                        const int16_t v = frz_boost_row(b, qr, s_vals, i0, i);
                        qr.out[i] = v;
                        m = max(m, (int32_t)v);
                    }
                }
                m = __reduce_max_sync(kFullWarp, m);
                if (lane == 0) s_max[warp][j - r0] = m;
            }
            __syncthreads();
            if (threadIdx.x < r1 - r0) {
                int32_t t = 0;
                for (uint32_t w = 0; w < kBoostWarps; w++) t = max(t, s_max[w][threadIdx.x]);
                if (t > 0) atomicMax(b.max + r0 + threadIdx.x, t);
            }
            __syncthreads();
        }
    }
}

}  // namespace

frz_status frz_launch_boost_where(const FrzBoostBatchDev& b, cudaStream_t stream) {
    const uint64_t n_chunks = (b.n + kFrzWhereChunk - 1) / kFrzWhereChunk;
    if (n_chunks == 0 || b.q == 0) return FRZ_OK;
    // Few chunks leave SMs idle: split the queries over y until about four blocks per SM are in flight (as k_where_batch).
    const uint64_t target = (uint64_t)frz_sm_count() * 4;
    const uint64_t ys = std::min<uint64_t>(b.q, std::max<uint64_t>(1, (target + n_chunks - 1) / n_chunks));
    const uint32_t per_block = (uint32_t)((b.q + ys - 1) / ys);
    const dim3 grid((unsigned)std::min<uint64_t>(n_chunks, (uint64_t)frz_sm_count() * 8), (b.q + per_block - 1) / per_block);
    k_boost_where<<<grid, kBoostBlock, b.n_staged * kFrzWhereChunk * sizeof(int64_t), stream>>>(b, per_block);
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}
