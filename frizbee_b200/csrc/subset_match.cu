// subset_match.cu — the fold of frz_subset_match (DESIGN.md §4.19): one step per compiled pattern folds the pattern's
// prefilter survivor bitmap into the subset's bitmap, and the last step writes the chunk counts that host.cu's common
// fill tail scans.  The per-word rule is subset_match_plan.cuh's.
#include "frz_host.h"
#include "subset_match_plan.cuh"

namespace {

constexpr int kFoldBlock = 256;
constexpr unsigned kFullWarp = 0xffffffffu;
static_assert(kFrzWhereChunk == FRZ_TILE, "a chunk of the fold is one tile of slot metadata");

// One warp per chunk of kFrzWhereChunk indices (one tile): lane l owns the chunk's word l, so every array is read and
// written 128 bytes per warp.  Without a survivor bitmap the step starts from T's live rows: 32 ballots over the chunk's
// indices, word t landing in lane t.  A word of `base` is read before the same lane writes `bits`, so the two may be one
// array.
__global__ void __launch_bounds__(kFoldBlock) k_subset_fold(const __grid_constant__ FrzSubsetFoldDev f) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n_words = (f.n + 31) / 32, n_chunks = (f.n + kFrzWhereChunk - 1) / kFrzWhereChunk;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
    for (uint64_t chunk = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; chunk < n_chunks; chunk += warps) {
        const uint64_t word = chunk * kFrzWhereChunkWords + lane;
        uint32_t surv = 0;
        if (f.surv) {
            surv = word < n_words ? f.surv[word] : 0u;
        } else {
            for (uint32_t t = 0; t < kFrzWhereChunkWords; t++) {
                const uint64_t i = (chunk * kFrzWhereChunkWords + t) * 32 + lane;
                const bool live = i < f.n && f.slot_meta[chunk * kFrzWhereChunk + f.slot_of[i]] != FRZ_INVALID_SLOT;
                const uint32_t b = __ballot_sync(kFullWarp, live);
                if (lane == t) surv = b;
            }
        }
        uint32_t x = 0;
        if (word < n_words) {
            const uint32_t base_word = f.has_base && word * 32 < f.n_base ? f.base[word] : 0u;
            const uint32_t cur = f.op == kFrzFoldFirst ? 0u : f.bits[word];
            x = frz_fold_word(f.op, cur, surv, frz_fold_base(f.has_base, base_word, word, f.n_base), frz_fold_below(word, f.n));
            f.bits[word] = x;
        }
        if (f.chunk_count) {
            uint32_t c = __popc(x);
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(kFullWarp, c, d);
            if (lane == 0) f.chunk_count[chunk] = c;
        }
    }
}

}  // namespace

frz_status frz_launch_subset_fold(const FrzSubsetFoldDev& f, cudaStream_t stream) {
    const uint64_t n_chunks = (f.n + kFrzWhereChunk - 1) / kFrzWhereChunk;
    if (n_chunks == 0) return FRZ_OK;
    constexpr uint32_t warps = kFoldBlock / 32;
    const int grid = (int)std::min<uint64_t>((n_chunks + warps - 1) / warps, (uint64_t)frz_sm_count() * 8);
    k_subset_fold<<<grid, kFoldBlock, 0, stream>>>(f);
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}
