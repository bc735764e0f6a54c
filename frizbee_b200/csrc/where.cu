// where.cu — the fill of frz_subset_where (DESIGN.md §4.14): the bitmap and per-chunk member counts from the clauses, and
// the member list from the bitmap.  The row rule is where_plan.cuh's; host.cu scans the chunk counts (k_scan_blocks) between
// the two kernels and owns the subset.
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
// writes the words' members one word at a time, lane l storing bit l's index (coalesced, ascending).
__global__ void __launch_bounds__(kWhereBlock) k_where_members(const uint32_t* __restrict__ bits, uint64_t n,
                                                               const uint64_t* __restrict__ chunk_base, uint32_t* __restrict__ members) {
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
