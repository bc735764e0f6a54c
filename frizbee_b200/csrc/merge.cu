// merge.cu — k_merge_matches_by (src/k_merge.rs:90-131) on the device, for frz_merge_runs_device and parallel.cu.  The
// position arithmetic is merge_plan.cuh.
#include <string.h>

#include <algorithm>
#include <mutex>

#include "frz_device.cuh"
#include "frz_host.h"
#include "merge_plan.cuh"

namespace {
// Run metadata travels BY VALUE as a kernel parameter: no staging buffer, so back-to-back merges with different counts
// cannot race and the entry point needs no per-call H2D copy.
struct MergeMeta {
    uint64_t counts[FRZ_MERGE_MAX_RUNS];   // valid entries of run r
    uint64_t total;
};

__global__ void k_gather_runs(const FrzMatchDev* runs, uint64_t stride, const __grid_constant__ MergeMeta meta, int n_runs,
                              int reverse_runs, FrzMatchDev* out, unsigned long long* d_total) {
    if (blockIdx.x == 0 && threadIdx.x == 0 && d_total) *d_total = meta.total;
    uint64_t base = 0;   // of the k-th run in merge order
    for (int k = 0; k < n_runs; k++) {
        const int src_run = frzmerge::run_at(k, n_runs, reverse_runs != 0);
        const FrzMatchDev* src = runs + (uint64_t)src_run * stride;
        const uint64_t cnt = meta.counts[src_run];
        for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += (uint64_t)gridDim.x * blockDim.x)
            out[base + i] = src[i];
        base += cnt;
    }
}

// ---- score-sorted runs, without comparing heads: gt by binary search, pos0 from gt, one scatter pass (gridDim.y = one
// row of blocks per run, so every run streams at full width).  No concatenation, no re-sort.
constexpr int kMergeMaxBins = 4096;

__global__ void k_merge_bounds(const FrzMatchDev* __restrict__ runs, uint64_t stride, const __grid_constant__ MergeMeta meta,
                               int n_runs, int bins, uint32_t* __restrict__ tables) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_runs * bins) return;
    const int r = t / bins;
    const uint32_t s = (uint32_t)(t - r * bins);
    const FrzMatchDev* run = runs + (uint64_t)r * stride;
    uint64_t lo = 0, hi = meta.counts[r];   // first index whose score <= s
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if (run[mid].score > s) lo = mid + 1; else hi = mid;
    }
    tables[frzmerge::table_row(r, bins) + bins + s] = (uint32_t)lo;
}

__global__ void k_merge_bases(uint32_t* __restrict__ tables, const __grid_constant__ MergeMeta meta, int n_runs, int bins,
                              int reverse_runs) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= bins) return;
    frzmerge::block_bases<uint32_t>(
        s, n_runs, reverse_runs != 0, [&](int r, int b) { return tables[frzmerge::table_row(r, bins) + bins + b]; },
        [&](int r) { return (uint32_t)meta.counts[r]; },
        [&](int r, uint32_t pos0, uint32_t, uint32_t) { tables[frzmerge::table_row(r, bins) + s] = pos0; return true; });
}

__global__ void __launch_bounds__(256) k_merge_scatter(const FrzMatchDev* __restrict__ src, const __grid_constant__ FrzMergePieces pieces,
                                                       const uint32_t* __restrict__ tables, int bins, FrzMatchDev* __restrict__ out) {
    const int q = blockIdx.y;
    const FrzMatchDev* piece = src + pieces.src[q];
    const uint32_t n = pieces.n[q], a = pieces.a[q];
    const uint32_t* row = tables + frzmerge::table_row(q, bins);   // pos0[s] = row[s], gt[s] = row[bins + s]
    const uint32_t step = gridDim.x * blockDim.x;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i = n - i > step ? i + step : n) {   // i + step may pass 2^32
        const FrzMatchDev m = piece[i];
        const uint32_t s = frzmerge::bin_of(m.score, bins);
        out[row[s] + (a + i - row[bins + s]) - pieces.lo] = m;
    }
}
}  // namespace

frz_status frz_launch_merge_scatter(const FrzMatchDev* src, const FrzMergePieces& pieces, int n_runs, const uint32_t* tables, int bins,
                                    int blocks_per_sm, FrzMatchDev* out, cudaStream_t stream) {
    uint64_t longest = 0;
    for (int q = 0; q < n_runs; q++) longest = std::max<uint64_t>(longest, pieces.n[q]);
    if (longest == 0) return FRZ_OK;
    const dim3 grid((unsigned)std::max<uint64_t>(1, std::min<uint64_t>((longest + 255) / 256, frz_sm_count() * blocks_per_sm / n_runs + 1)),
                    (unsigned)n_runs);
    k_merge_scatter<<<grid, 256, 0, stream>>>(src, pieces, tables, bins, out);
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

// k_merge_matches_by on `stream` with caller-owned scratch (one per concurrent user; grow-only).  Without a usable score
// bound: the runs concatenated in merge order and stable-sorted by score (ties resolve by index: shards are index-ordered).
frz_status frz_merge_runs_ex(FrzMergeScratch& ms, const FrzMatchDev* runs, uint64_t run_stride, const uint64_t* run_counts_host,
                             int n_runs, uint8_t sort, uint32_t score_bound_in, FrzMatchDev* d_out, cudaStream_t stream) {
    if (!runs || !run_counts_host || !d_out || n_runs <= 0 || n_runs > FRZ_MERGE_MAX_RUNS) return frz_fail(FRZ_ERR_INVALID_ARG, "bad argument");
    const bool reversed = sort == FRZ_SORT_INDEX_DESC || sort == FRZ_SORT_SCORE_THEN_INDEX_DESC;
    const bool by_score = sort == FRZ_SORT_SCORE_THEN_INDEX_ASC || sort == FRZ_SORT_SCORE_THEN_INDEX_DESC;
    const uint32_t score_bound = score_bound_in ? score_bound_in : 0xFFFF;
    MergeMeta meta;
    memset(&meta, 0, sizeof meta);
    uint64_t total = 0;
    for (int r = 0; r < n_runs; r++) {
        meta.counts[r] = run_counts_host[r];
        total += run_counts_host[r];
    }
    meta.total = total;
    if (!ms.d_total.get()) {   // first use, all or nothing: a failed set-up leaves the scratch empty
        FrzMergeScratch fresh;
        FRZ_TRY(frz_sort_hist_alloc(fresh.sort.hist));
        FRZ_TRY(fresh.tables.reserve((size_t)2 * FRZ_MERGE_MAX_RUNS * kMergeMaxBins));
        FRZ_TRY(fresh.d_total.reserve(1));
        ms = std::move(fresh);
    }
    const int bins = (int)std::min<uint32_t>(score_bound, 0xFFFFu) + 1;
    if (total == 0) return FRZ_OK;
    if (by_score && bins <= kMergeMaxBins && total <= 0xFFFFFFFFull) {
        uint32_t* tables = ms.tables.get();
        k_merge_bounds<<<(n_runs * bins + 255) / 256, 256, 0, stream>>>(runs, run_stride, meta, n_runs, bins, tables);
        k_merge_bases<<<(bins + 127) / 128, 128, 0, stream>>>(tables, meta, n_runs, bins, reversed ? 1 : 0);
        FrzMergePieces pieces{};
        for (int r = 0; r < n_runs; r++) {
            pieces.src[r] = (uint64_t)r * run_stride;
            pieces.n[r] = (uint32_t)run_counts_host[r];
        }
        return frz_launch_merge_scatter(runs, pieces, n_runs, tables, bins, 8, d_out, stream);   // asynchronous on `stream`
    }
    if (by_score) {
        FRZ_TRY(ms.cat.reserve(total, total + total / 4 + 1024));
        FRZ_TRY(ms.tmp.reserve(total, total + total / 4 + 1024));
    }
    FrzMatchDev* dst = by_score ? ms.cat.get() : d_out;
    k_gather_runs<<<grid_for(total / n_runs + 1, 256), 256, 0, stream>>>(runs, run_stride, meta, n_runs, reversed ? 1 : 0, dst, ms.d_total.get());
    if (by_score) FRZ_TRY(frz_launch_sort_by_score_dev(ms.cat.get(), ms.tmp.get(), d_out, ms.d_total.get(), score_bound, ms.sort, stream, nullptr));
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;  // asynchronous on `stream`
}

extern "C" frz_status frz_merge_runs_device(const frz_match* d_runs, uint64_t run_stride, const uint64_t* run_counts_host,
                                            int n_runs, uint8_t sort, uint32_t score_bound_in, frz_match* d_out, int device, void* stream_) {
    FRZ_TRY(frz_ensure_device(device));
    if (device >= 64) return frz_fail(FRZ_ERR_INVALID_ARG, "device index too large");
    // grow-only per-device scratch (tables only: the run metadata travels as kernel parameters).  Calls for one device
    // must be stream-ordered with each other, as documented in the header.  Never destroyed: its destructors would run
    // at process exit, when the CUDA runtime may already be gone.
    static FrzMergeScratch* const scratch = new FrzMergeScratch[64];
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    return frz_merge_runs_ex(scratch[device], reinterpret_cast<const FrzMatchDev*>(d_runs), run_stride, run_counts_host, n_runs, sort,
                             score_bound_in, reinterpret_cast<FrzMatchDev*>(d_out), (cudaStream_t)stream_);
}
