// where.cu — the fill of frz_subset_where (DESIGN.md §4.14): the bitmap and per-chunk member counts from the clauses, and
// the member list from the bitmap; and the same two steps for every query of frz_subset_where_batch at once.  The row rule
// is where_plan.cuh's; host.cu scans the chunk counts (k_scan_blocks, k_scan_blocks_batch) between the two kernels and
// owns the subsets.
#include "frz_host.h"
#include "where_plan.cuh"

namespace {

constexpr int kWhereBlock = 256;
constexpr uint32_t kWhereWarps = kWhereBlock / 32;
constexpr unsigned kFullWarp = 0xffffffffu;

// One warp per bitmap word: lane l tests index 32 * word + l, each clause a coalesced 8-byte load per lane, and the ballot
// is the word.  A block walks whole chunks (its warps take consecutive words) and writes each chunk's member count.  The
// set values are staged in shared memory once per block.  A word of `base` is read before the same warp writes `bits`, so
// the two may be one array.
__global__ void __launch_bounds__(kWhereBlock) k_where(const __grid_constant__ FrzWhereDev w) {
    extern __shared__ int64_t s_sets[];
    __shared__ uint32_t s_cnt[kWhereWarps];
    for (uint32_t j = threadIdx.x; j < w.n_sets; j += blockDim.x) s_sets[j] = w.sets[j];
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t n_words = (w.n + 31) / 32, n_chunks = (w.n + kFrzWhereChunk - 1) / kFrzWhereChunk;
    for (uint64_t chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x) {
        uint32_t cnt = 0;
#pragma unroll
        for (uint32_t k = 0; k < kFrzWhereChunkWords / kWhereWarps; k++) {
            const uint64_t word = chunk * kFrzWhereChunkWords + k * kWhereWarps + warp;
            if (word >= n_words) break;   // warp-uniform
            const uint64_t i = word * 32 + lane;
            const uint32_t base_word = w.has_base && word * 32 < w.n_base ? w.base[word] : 0u;
            bool keep = frz_where_in_base(w, base_word, i);
#pragma unroll
            for (uint32_t c = 0; c < kFrzWhereMaxClauses; c++)   // every clause's load is issued, whatever the others give
                if (c < w.n_clauses) keep = frz_where_holds(w.clauses[c], s_sets, frz_where_value(w.clauses[c], i)) && keep;
            const uint32_t b = __ballot_sync(kFullWarp, keep);
            if (lane == 0) w.bits[word] = b;
            cnt += __popc(b);
        }
        if (lane == 0) s_cnt[warp] = cnt;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t t = 0;
            for (uint32_t j = 0; j < kWhereWarps; j++) t += s_cnt[j];
            w.chunk_count[chunk] = t;
        }
        __syncthreads();
    }
}

// One warp per chunk: lane l holds the chunk's word l, a warp scan gives each word's first member slot, and the warp then
// writes the words' members one word at a time, lane l storing bit l's index (coalesced, ascending).  The grid's warps
// take the chunks in turn along x.
__device__ __forceinline__ void where_members(const uint32_t* __restrict__ bits, uint64_t n, const uint64_t* __restrict__ chunk_base,
                                              uint32_t* __restrict__ members) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n_words = (n + 31) / 32, n_chunks = (n + kFrzWhereChunk - 1) / kFrzWhereChunk;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
    for (uint64_t chunk = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; chunk < n_chunks; chunk += warps) {
        const uint64_t word = chunk * kFrzWhereChunkWords + lane;
        const uint32_t x = word < n_words ? bits[word] : 0u;
        const uint32_t c = __popc(x);
        uint32_t incl = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(kFullWarp, incl, d);
            if (lane >= (uint32_t)d) incl += y;
        }
        const uint32_t excl = incl - c;
        const uint64_t base = chunk_base[chunk];
        for (uint32_t t = 0; t < kFrzWhereChunkWords; t++) {
            const uint32_t xt = __shfl_sync(kFullWarp, x, t);
            const uint32_t et = __shfl_sync(kFullWarp, excl, t);
            if ((xt >> lane) & 1u)
                members[base + et + frz_where_rank(xt, lane)] = (uint32_t)((chunk * kFrzWhereChunkWords + t) * 32 + lane);
        }
    }
}

__global__ void __launch_bounds__(kWhereBlock) k_where_members(const uint32_t* __restrict__ bits, uint64_t n,
                                                               const uint64_t* __restrict__ chunk_base, uint32_t* __restrict__ members) {
    where_members(bits, n, chunk_base, members);
}

constexpr uint32_t kWhereBatchRound = 32;   // queries whose chunk counts a block gathers per round

// k_where for many queries (where_plan.cuh, "batched fills").  Block (x, y) walks chunks along x; for each it stages the
// chunk's values of the staged attributes in shared memory, then writes the words of queries [y * per_block, ...) of
// that chunk: per query, warp w takes words w, w + 8, w + 16 and w + 24 as k_where does.  The warps' counts of a round of
// kWhereBatchRound queries meet in shared memory, and one thread per query writes its chunk count.
__global__ void __launch_bounds__(kWhereBlock) k_where_batch(const __grid_constant__ FrzWhereBatchDev b, uint32_t per_block) {
    extern __shared__ int64_t s_vals[];   // [n_staged][kFrzWhereChunk]
    __shared__ uint32_t s_cnt[kWhereWarps][kWhereBatchRound];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t n_words = (b.n + 31) / 32, n_chunks = (b.n + kFrzWhereChunk - 1) / kFrzWhereChunk;
    const uint32_t j0 = blockIdx.y * per_block, j1 = min(b.q, j0 + per_block);
    for (uint64_t chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x) {
        const uint64_t i0 = chunk * kFrzWhereChunk;
        for (uint32_t t = threadIdx.x; t < b.n_staged * (uint32_t)kFrzWhereChunk; t += blockDim.x)
            s_vals[t] = frz_where_attr_value(b.attrs[t / kFrzWhereChunk], i0 + t % kFrzWhereChunk);
        __syncthreads();
        for (uint32_t r0 = j0; r0 < j1; r0 += kWhereBatchRound) {
            const uint32_t r1 = min(j1, r0 + kWhereBatchRound);
            for (uint32_t j = r0; j < r1; j++) {
                const FrzWhereBatchQuery& qr = b.queries[j];
                uint32_t cnt = 0;
#pragma unroll
                for (uint32_t k = 0; k < kFrzWhereChunkWords / kWhereWarps; k++) {
                    const uint64_t word = chunk * kFrzWhereChunkWords + k * kWhereWarps + warp;
                    if (word >= n_words) break;   // warp-uniform
                    const uint64_t i = word * 32 + lane;
                    const uint32_t base_word = qr.has_base && word * 32 < qr.n_base ? qr.base[word] : 0u;
                    const uint32_t w = __ballot_sync(kFullWarp, frz_where_batch_row(b, qr, s_vals, i0, base_word, i));
                    if (lane == 0) qr.bits[word] = w;
                    cnt += __popc(w);
                }
                if (lane == 0) s_cnt[warp][j - r0] = cnt;
            }
            __syncthreads();
            if (threadIdx.x < r1 - r0) {
                uint32_t t = 0;
                for (uint32_t w = 0; w < kWhereWarps; w++) t += s_cnt[w][threadIdx.x];
                b.queries[r0 + threadIdx.x].chunk_count[chunk] = t;
            }
            __syncthreads();
        }
    }
}

// k_where_members for many queries: grid row y writes the lists of queries y, y + gridDim.y, ... (those with members).
__global__ void __launch_bounds__(kWhereBlock) k_where_members_batch(const FrzWhereBatchQuery* __restrict__ queries,
                                                                     const unsigned long long* __restrict__ totals, uint64_t n, uint32_t q) {
    for (uint32_t j = blockIdx.y; j < q; j += gridDim.y)
        if (totals[j]) where_members(queries[j].bits, n, queries[j].chunk_base, queries[j].members);
}

}  // namespace

frz_status frz_launch_where(const FrzWhereDev& w, cudaStream_t stream) {
    const uint64_t n_chunks = (w.n + kFrzWhereChunk - 1) / kFrzWhereChunk;
    if (n_chunks == 0) return FRZ_OK;
    const int grid = (int)std::min<uint64_t>(n_chunks, (uint64_t)frz_sm_count() * 8);
    k_where<<<grid, kWhereBlock, w.n_sets * sizeof(int64_t), stream>>>(w);
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

frz_status frz_launch_where_members(const uint32_t* bits, uint64_t n, const uint64_t* chunk_base, uint32_t* members, cudaStream_t stream) {
    const uint64_t n_chunks = (n + kFrzWhereChunk - 1) / kFrzWhereChunk;
    if (n_chunks == 0) return FRZ_OK;
    const int grid = (int)std::min<uint64_t>((n_chunks + kWhereWarps - 1) / kWhereWarps, (uint64_t)frz_sm_count() * 8);
    k_where_members<<<grid, kWhereBlock, 0, stream>>>(bits, n, chunk_base, members);
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

frz_status frz_launch_where_batch(const FrzWhereBatchDev& b, cudaStream_t stream) {
    const uint64_t n_chunks = (b.n + kFrzWhereChunk - 1) / kFrzWhereChunk;
    if (n_chunks == 0 || b.q == 0) return FRZ_OK;
    // Few chunks leave SMs idle: split the queries over y until about four blocks per SM are in flight.
    const uint64_t target = (uint64_t)frz_sm_count() * 4;
    const uint64_t ys = std::min<uint64_t>(b.q, std::max<uint64_t>(1, (target + n_chunks - 1) / n_chunks));
    const uint32_t per_block = (uint32_t)((b.q + ys - 1) / ys);
    const dim3 grid((unsigned)std::min<uint64_t>(n_chunks, (uint64_t)frz_sm_count() * 8), (b.q + per_block - 1) / per_block);
    k_where_batch<<<grid, kWhereBlock, b.n_staged * kFrzWhereChunk * sizeof(int64_t), stream>>>(b, per_block);
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

frz_status frz_launch_where_members_batch(const FrzWhereBatchQuery* queries, const unsigned long long* totals, uint64_t n, uint32_t q,
                                          cudaStream_t stream) {
    const uint64_t n_chunks = (n + kFrzWhereChunk - 1) / kFrzWhereChunk;
    if (n_chunks == 0 || q == 0) return FRZ_OK;
    const uint64_t x = std::min<uint64_t>((n_chunks + kWhereWarps - 1) / kWhereWarps,
                                          std::max<uint64_t>(1, (uint64_t)frz_sm_count() * 8 / q));
    const dim3 grid((unsigned)x, (unsigned)std::min<uint32_t>(q, 65535));
    k_where_members_batch<<<grid, kWhereBlock, 0, stream>>>(queries, totals, n, q);
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}
