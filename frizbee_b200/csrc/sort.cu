// sort.cu — stable descending-score sort of index-ordered matches.
//
// Reference replaced: radix_sort_matches (src/sort.rs:6-40): a stable 2-pass LSD radix sort on the
// u16 score of a list that is already in index order, giving (score desc, index asc).  Any stable
// sort by descending score yields the identical sequence; here it is a counting sort whose digit is
// the whole score when the score bound allows it (one pass), else the reference's two 8-bit passes.
//
//   k_sort_hist     each "virtual warp" owns a contiguous segment and counts its digits in smem
//   k_sort_scan_rows per-digit exclusive prefix over the segments; its last block adds the descending exclusive prefix
//                   over the digits (digit_base)
//   k_sort_scatter  each virtual warp re-walks its segment IN ORDER, 32 elements at a time;
//                   __match_any_sync gives the in-warp stable rank, a per-warp counter array the rest
//
// The fused single-pass sort (frz_sort_fused_prepare / frz_launch_sort_fused) has no histogram kernel: the scoring kernels
// count every match they emit into FrzScoreHist (per score digit, per 2048-element segment of its index-ordered position),
// k_sort_scan_rows scans that histogram (and re-zeroes it), and k_sort_scatter_seg places one segment per block.
//
// The element count lives in device memory (it is produced by the previous stage), so the whole
// match_list pipeline runs without a host round trip until the final copy-out.
//
// Top-K calls (frz_match_list_top): the final scatter of every sort takes a limit and stores only the positions below it —
// every element's final position is known before its store, so the first `limit` elements of the sorted list are exactly
// the ones written.  Full sorts pass kFrzNoLimit.
#include "frz_device.cuh"
#include "frz_host.h"

#include <algorithm>

namespace {

constexpr int kSortBlocks = 288;              // ~2 blocks per SM
constexpr int kSortWarps = 8;
constexpr int kV = kSortBlocks * kSortWarps;  // 2304 virtual warps = segments: the in-order walk of a segment is latency-bound, so
                                              // more, shorter segments are faster (1024 segments: 22 us scatter at 750 k matches)
static_assert(kV % 128 == 0, "k_sort_scan_rows reads a digit row as 32 lanes x uint4");
constexpr int kMaxBins = 1024;

__device__ __forceinline__ void segment_of(unsigned long long n, int v, unsigned long long* lo, unsigned long long* hi) {
    unsigned long long seg = (n + kV - 1) / kV;
    seg = (seg + 31) & ~31ull;
    unsigned long long a = seg * v;
    *lo = a < n ? a : n;
    unsigned long long b = a + seg;
    *hi = b < n ? b : n;
}

__device__ __forceinline__ uint32_t digit_of(const FrzMatchDev& m, int shift, uint32_t mask) {
    return ((uint32_t)m.score >> shift) & mask;
}

__global__ void __launch_bounds__(kSortWarps * 32) k_sort_hist(const FrzMatchDev* __restrict__ in,
                                                               const unsigned long long* __restrict__ n_ptr, int shift,
                                                               int bins, uint32_t* __restrict__ hist) {
    extern __shared__ uint32_t sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t* cnt = sm + warp * bins;
    for (int d = lane; d < bins; d += 32) cnt[d] = 0;
    __syncwarp();
    const int v = blockIdx.x * kSortWarps + warp;
    unsigned long long lo, hi;
    segment_of(*n_ptr, v, &lo, &hi);
    const uint32_t mask = (uint32_t)bins - 1;
    // four loads in flight per lane: the walk is latency-bound (one 256-byte line per trip)
    unsigned long long i = lo + lane;
    for (; i + 96 < hi; i += 128) {
        const FrzMatchDev a = in[i], b = in[i + 32], c = in[i + 64], d = in[i + 96];
        atomicAdd(&cnt[digit_of(a, shift, mask)], 1u);
        atomicAdd(&cnt[digit_of(b, shift, mask)], 1u);
        atomicAdd(&cnt[digit_of(c, shift, mask)], 1u);
        atomicAdd(&cnt[digit_of(d, shift, mask)], 1u);
    }
    for (; i < hi; i += 32) atomicAdd(&cnt[digit_of(in[i], shift, mask)], 1u);
    __syncwarp();
    for (int d = lane; d < bins; d += 32) hist[(size_t)d * kV + v] = cnt[d];
}

// hist[d][v] → exclusive prefix over v into pref[d][v], one warp per digit row; totals[d] = row sum.  A row holds `stride`
// words of which the first `count` are used: count = kV for k_sort_hist's segments, or (n_ptr) the number of
// 2^kFrzSortSegShift-element segments of the list, read at run time.  ZERO: the words read are zeroed again (the fused
// histogram is left clean for the next call).  A lane owns 4 * U contiguous entries of a 128 * U-entry chunk; U = kV / 128
// covers k_sort_hist's rows in one chunk with all loads in flight.  The LAST block to finish (device counter,
// self-resetting) then turns the row totals into digit_base[d] = #elements with digit > d (descending exclusive prefix over
// the digits) — one launch instead of two.
template <int U, bool ZERO>
__global__ void __launch_bounds__(256) k_sort_scan_rows(uint32_t* __restrict__ hist, uint32_t* __restrict__ pref, uint32_t stride,
                                                        const unsigned long long* __restrict__ n_ptr, int bins,
                                                        uint32_t* __restrict__ totals, uint32_t* __restrict__ digit_base,
                                                        unsigned int* __restrict__ done_counter) {
    __shared__ bool is_last;
    __shared__ uint32_t wsum[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int d = blockIdx.x * 8 + warp;
    if (d < bins) {
        const uint32_t count = n_ptr ? (uint32_t)((*n_ptr + (1ull << kFrzSortSegShift) - 1) >> kFrzSortSegShift) : (uint32_t)kV;
        uint4* row = reinterpret_cast<uint4*>(hist + (size_t)d * stride);
        uint4* prow = reinterpret_cast<uint4*>(pref + (size_t)d * stride);
        uint32_t carry = 0;
        for (uint32_t c0 = 0; c0 < count; c0 += 128 * U) {
            const uint32_t q0 = (c0 >> 2) + lane * U;   // this lane's first uint4 of the chunk
            uint4 v[U];
            uint32_t s = 0;
#pragma unroll
            for (int k = 0; k < U; k++) {
                v[k] = make_uint4(0, 0, 0, 0);
                if ((q0 + k) * 4 < count) v[k] = row[q0 + k];
                s += v[k].x + v[k].y + v[k].z + v[k].w;
            }
            uint32_t x = s;
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
                if (lane >= o) x += y;
            }
            uint32_t run = carry + x - s;
#pragma unroll
            for (int k = 0; k < U; k++) {
                if ((q0 + k) * 4 >= count) break;
                uint4 o4;
                o4.x = run; run += v[k].x;
                o4.y = run; run += v[k].y;
                o4.z = run; run += v[k].z;
                o4.w = run; run += v[k].w;
                prow[q0 + k] = o4;
                if (ZERO) row[q0 + k] = make_uint4(0, 0, 0, 0);
            }
            carry += __shfl_sync(0xffffffffu, x, 31);
        }
        if (lane == 0) totals[d] = carry;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = atomicAdd(done_counter, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    // digit_base over bins <= 1024 entries: thread t owns the PERT digits t*PERT .. of the DESCENDING sequence
    const int PERT = (bins + 255) / 256;
    uint32_t loc[4] = {0, 0, 0, 0}, sum = 0;
    for (int k = 0; k < PERT; k++) {
        const int t = threadIdx.x * PERT + k;
        loc[k] = t < bins ? __ldcg(&totals[bins - 1 - t]) : 0u;
        sum += loc[k];
    }
    uint32_t x = sum;
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < 8 ? wsum[lane] : 0u, xs = w;
        for (int o = 1; o < 8; o <<= 1) {
            uint32_t y = __shfl_up_sync(0xffffffffu, xs, o);
            if (lane >= o) xs += y;
        }
        if (lane < 8) wsum[lane] = xs - w;
    }
    __syncthreads();
    uint32_t run = wsum[warp] + x - sum;
    for (int k = 0; k < PERT; k++) {
        const int t = threadIdx.x * PERT + k;
        if (t < bins) digit_base[bins - 1 - t] = run;
        run += loc[k];
    }
    if (threadIdx.x == 0) *done_counter = 0;   // ready for the next pass
}

__global__ void __launch_bounds__(kSortWarps * 32) k_sort_scatter(const FrzMatchDev* __restrict__ in, FrzMatchDev* __restrict__ out,
                                                                  const unsigned long long* __restrict__ n_ptr, int shift, int bins,
                                                                  const uint32_t* __restrict__ hist,
                                                                  const uint32_t* __restrict__ digit_base, uint32_t limit) {
    extern __shared__ uint32_t sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t* cnt = sm + warp * bins;
    const int v = blockIdx.x * kSortWarps + warp;
    for (int d = lane; d < bins; d += 32) cnt[d] = digit_base[d] + hist[(size_t)d * kV + v];
    __syncwarp();
    unsigned long long lo, hi;
    segment_of(*n_ptr, v, &lo, &hi);
    const uint32_t mask = (uint32_t)bins - 1;
    // the element of the NEXT trip is loaded before this trip's rank / counter chain (software pipelining: the walk has
    // to stay in order for stability, so the only parallelism inside a segment is load-ahead)
    FrzMatchDev nxt;
    nxt.index = 0; nxt.score = 0; nxt.exact = 0; nxt.pad = 0;
    if (lo + lane < hi) nxt = in[lo + lane];
    for (unsigned long long base = lo; base < hi; base += 32) {
        const unsigned long long i = base + lane;
        const bool valid = i < hi;
        const FrzMatchDev m = nxt;
        if (i + 32 < hi) nxt = in[i + 32];
        uint32_t d = (uint32_t)bins + lane;  // sentinel: matches nobody
        if (valid) d = digit_of(m, shift, mask);
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        const uint32_t rank = __popc(peers & ((1u << lane) - 1));
        uint32_t pos = 0;
        if (valid) pos = cnt[d] + rank;
        __syncwarp();
        if (valid && rank == 0) cnt[d] += __popc(peers);
        __syncwarp();
        if (valid && pos < limit) out[pos] = m;
    }
}

// The fused single-pass scatter: one block per 2^kFrzSortSegShift-element segment of the list (a persistent grid strides over
// the segments).  Warp w owns the segment's w-th run of kSegRounds * 32 elements and loads all of it at once (coalesced, every
// load in flight).  It ranks its run stably, 32 elements per round: __match_any_sync gives the rank inside the round, and the
// round's leader of each digit adds the round's count to the warp's digit counter in shared memory, whose old value it
// broadcasts.  A per-digit exclusive prefix over the warps, plus digit_base[d] + pref[d][segment] (the scoring kernels'
// histogram, scanned), then gives every element its final position: (score desc, index asc) exactly.
constexpr int kSegThreads = 256;
constexpr int kSegWarps = kSegThreads / 32;
constexpr int kSegRounds = (1 << kFrzSortSegShift) / kSegThreads;   // elements per lane
static_assert(kSegRounds * kSegThreads == (1 << kFrzSortSegShift), "a segment is a whole number of block-wide rounds");

__global__ void __launch_bounds__(kSegThreads) k_sort_scatter_seg(const FrzMatchDev* __restrict__ in, FrzMatchDev* __restrict__ out,
                                                                  const unsigned long long* __restrict__ n_ptr, int bins,
                                                                  const uint32_t* __restrict__ pref, uint32_t stride,
                                                                  const uint32_t* __restrict__ digit_base, uint32_t limit) {
    extern __shared__ uint32_t sm[];   // [kSegWarps][bins]: per-warp digit counters, then each warp's output base per digit
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t* cnt = sm + warp * bins;
    const unsigned long long n = *n_ptr;
    const uint32_t nseg = (uint32_t)((n + (1ull << kFrzSortSegShift) - 1) >> kFrzSortSegShift);
    const uint32_t mask = (uint32_t)bins - 1;
    const uint32_t lt = (1u << lane) - 1;
    for (uint32_t seg = blockIdx.x; seg < nseg; seg += gridDim.x) {
        for (int d = threadIdx.x; d < kSegWarps * bins; d += kSegThreads) sm[d] = 0;
        const unsigned long long first = ((unsigned long long)seg << kFrzSortSegShift) + warp * (kSegRounds * 32) + lane;
        FrzMatchDev m[kSegRounds];
#pragma unroll
        for (int r = 0; r < kSegRounds; r++) {
            m[r].index = 0; m[r].score = 0; m[r].exact = 0; m[r].pad = 0;
            if (first + r * 32 < n) m[r] = in[first + r * 32];
        }
        __syncthreads();
        uint32_t rank[kSegRounds];
#pragma unroll
        for (int r = 0; r < kSegRounds; r++) {
            const bool valid = first + r * 32 < n;
            const uint32_t d = valid ? (uint32_t)m[r].score & mask : (uint32_t)bins + lane;   // sentinel: matches nobody
            const uint32_t peers = __match_any_sync(0xffffffffu, d);
            const int leader = __ffs(peers) - 1;
            uint32_t old = 0;
            if (valid && lane == leader) old = atomicAdd(&cnt[d], (uint32_t)__popc(peers));
            rank[r] = __shfl_sync(0xffffffffu, old, leader) + __popc(peers & lt);
        }
        __syncthreads();
        // per digit: exclusive prefix over the warps, offset by where the digit's run of this segment starts in the output
        for (int d = threadIdx.x; d < bins; d += kSegThreads) {
            uint32_t tot = 0;
#pragma unroll
            for (int w = 0; w < kSegWarps; w++) tot += sm[w * bins + d];
            uint32_t run = tot ? digit_base[d] + pref[(size_t)d * stride + seg] : 0u;
#pragma unroll
            for (int w = 0; w < kSegWarps; w++) {
                const uint32_t c = sm[w * bins + d];
                sm[w * bins + d] = run;
                run += c;
            }
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < kSegRounds; r++)
            if (first + r * 32 < n) {
                const uint32_t pos = cnt[(uint32_t)m[r].score & mask] + rank[r];
                if (pos < limit) out[pos] = m[r];
            }
        __syncthreads();   // the counters are reset for the next segment
    }
}

}  // namespace

// n_ptr: device pointer to the element count.  score_bound: host-known upper bound of any score.
frz_status frz_launch_sort_by_score_dev(const FrzMatchDev* d_in, FrzMatchDev* d_tmp, FrzMatchDev* d_out,
                                        const unsigned long long* n_ptr, uint32_t score_bound, FrzWorkspace& ws,
                                        cudaStream_t stream, FrzLaunchStats* st, uint32_t limit) {
    auto pass = [&](const FrzMatchDev* src, FrzMatchDev* dst, int shift, int bins, uint32_t keep) -> frz_status {
        const size_t smem = (size_t)kSortWarps * bins * sizeof(uint32_t);
        k_sort_hist<<<kSortBlocks, kSortWarps * 32, smem, stream>>>(src, n_ptr, shift, bins, ws.sort_hist);
        uint32_t* totals = ws.sort_hist + (size_t)kMaxBins * kV;
        uint32_t* digit_base = totals + kMaxBins;
        unsigned int* done_counter = reinterpret_cast<unsigned int*>(digit_base + kMaxBins);   // zeroed at allocation, self-resetting
        k_sort_scan_rows<kV / 128, false><<<(bins + 7) / 8, 256, 0, stream>>>(ws.sort_hist, ws.sort_hist, kV, nullptr, bins, totals,
                                                                               digit_base, done_counter);
        if (ws.arm_table_ev && ws.table_ev) {   // digit_base is final: the multi-GPU layer publishes it while the scatter runs
            FRZ_CUDA_TRY(cudaEventRecord(ws.table_ev, stream));
            ws.table_ev_recorded = true;
        }
        k_sort_scatter<<<kSortBlocks, kSortWarps * 32, smem, stream>>>(src, dst, n_ptr, shift, bins, ws.sort_hist, digit_base, keep);
        FRZ_CUDA_TRY(cudaGetLastError());
        if (st) st->launches += 3;
        return FRZ_OK;
    };
    if (score_bound < 256) return pass(d_in, d_out, 0, 256, limit);
    if (score_bound < 512) return pass(d_in, d_out, 0, 512, limit);
    if (score_bound < 1024) return pass(d_in, d_out, 0, 1024, limit);
    // the reference's two 8-bit LSD passes (src/sort.rs:8-39); only the second one knows final positions
    FRZ_TRY(pass(d_in, d_tmp, 0, 256, kFrzNoLimit));
    return pass(d_tmp, d_out, 8, 256, limit);
}

size_t frz_sort_hist_words() { return (size_t)kMaxBins * kV + 2 * kMaxBins + 4; }   // + the pass-completion counter (must start at zero)
// allocates the sort scratch on the current device (the completion counter of k_sort_scan_rows starts at zero)
frz_status frz_sort_hist_alloc(uint32_t** out) {
    FRZ_CUDA_TRY(cudaMalloc(out, frz_sort_hist_words() * sizeof(uint32_t)));
    FRZ_CUDA_TRY(cudaMemset(*out + (size_t)kMaxBins * kV + 2 * kMaxBins, 0, 4 * sizeof(uint32_t)));
    return FRZ_OK;
}

// digit_base[d] of the LAST pass run on this workspace = number of elements whose digit is greater than d.  After a
// single-pass sort (score bound < 1024) that is, per score s, how many matches of the run score higher than s — the table
// the multi-GPU slice exchange needs (parallel.cu) — so nobody has to binary-search the sorted run for it.
const uint32_t* frz_sort_digit_base(const FrzWorkspace& ws) { return ws.sort_hist ? ws.sort_hist + (size_t)kMaxBins * kV + kMaxBins : nullptr; }
int frz_sort_single_pass_bins(uint32_t score_bound) { return score_bound < 256 ? 256 : score_bound < 512 ? 512 : score_bound < 1024 ? 1024 : 0; }

// fused_hist holds the counts ([bins][stride]) and then the scan's prefix rows (same shape).  The counts are zero between
// calls (the scan re-zeroes every word the scoring kernels can have touched), so only growth, a new layout reaching past
// the words known to be zero, or a call that stopped between scoring and scan costs a memset.
frz_status frz_sort_fused_prepare(FrzWorkspace& ws, uint64_t n_cap, uint32_t score_bound, cudaStream_t stream, FrzScoreHist* out) {
    const int bins = frz_sort_single_pass_bins(score_bound);
    if (bins == 0) return frz_fail(FRZ_ERR_INVALID_ARG, "fused sort needs a score bound below 1024 (got %u)", score_bound);
    const uint64_t segs = (n_cap + (1ull << kFrzSortSegShift) - 1) >> kFrzSortSegShift;
    const uint64_t stride = std::max<uint64_t>((segs + 3) & ~3ull, 4);
    const uint64_t words = (uint64_t)bins * stride;
    if (ws.fused_hist_cap < 2 * words) {
        cudaFree(ws.fused_hist);
        ws.fused_hist = nullptr; ws.fused_hist_cap = 0; ws.fused_clean_words = 0;
        FRZ_CUDA_TRY(cudaMalloc(&ws.fused_hist, 2 * words * sizeof(uint32_t)));
        ws.fused_hist_cap = 2 * words;
    }
    if (ws.fused_hist_dirty || ws.fused_clean_words < words)
        FRZ_CUDA_TRY(cudaMemsetAsync(ws.fused_hist, 0, words * sizeof(uint32_t), stream));
    ws.fused_clean_words = words;   // the prefix rows are written right behind the counts
    ws.fused_hist_dirty = true;
    out->counts = ws.fused_hist;
    out->stride = (uint32_t)stride;
    out->mask = (uint32_t)bins - 1;
    return FRZ_OK;
}

frz_status frz_launch_sort_fused(const FrzMatchDev* d_in, FrzMatchDev* d_out, const unsigned long long* n_ptr, const FrzScoreHist& h,
                                 FrzWorkspace& ws, cudaStream_t stream, FrzLaunchStats* st, uint32_t limit) {
    const int bins = (int)h.mask + 1;
    uint32_t* pref = h.counts + (size_t)bins * h.stride;
    uint32_t* totals = ws.sort_hist + (size_t)kMaxBins * kV;
    uint32_t* digit_base = totals + kMaxBins;
    unsigned int* done_counter = reinterpret_cast<unsigned int*>(digit_base + kMaxBins);
    k_sort_scan_rows<4, true><<<(bins + 7) / 8, 256, 0, stream>>>(h.counts, pref, h.stride, n_ptr, bins, totals, digit_base, done_counter);
    FRZ_CUDA_TRY(cudaGetLastError());
    ws.fused_hist_dirty = false;
    if (ws.arm_table_ev && ws.table_ev) {   // digit_base is final: the multi-GPU layer publishes it while the scatter runs
        FRZ_CUDA_TRY(cudaEventRecord(ws.table_ev, stream));
        ws.table_ev_recorded = true;
    }
    const size_t smem = (size_t)kSegWarps * bins * sizeof(uint32_t);
    const int grid = (int)std::max<uint32_t>(1, std::min<uint32_t>(h.stride, (uint32_t)frz_sm_count() * 4));
    k_sort_scatter_seg<<<grid, kSegThreads, smem, stream>>>(d_in, d_out, n_ptr, bins, pref, h.stride, digit_base, limit);
    FRZ_CUDA_TRY(cudaGetLastError());
    if (st) st->launches += 2;
    return FRZ_OK;
}
