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
// k_sort_scan_rows scans that histogram (and re-zeroes it), and k_sort_scatter_seg sorts one segment per block and writes
// it out as whole score runs.  Both are launched dependent (frz_launch_dependent): each waits for the kernel ahead of it
// before its first memory access.  The multi-GPU table event recorded between them still marks the scan's completion: an
// event orders like any stream operation, and the scatter after it starts early only behind a kernel.
//
// The element count lives in device memory (it is produced by the previous stage), so the whole
// match_list pipeline runs without a host round trip until the final copy-out.
//
// Top-K calls (frz_match_list_top): the final scatter of every sort takes a limit and stores only the positions below it —
// every element's final position is known before its store, so the first `limit` elements of the sorted list are exactly
// the ones written.  Full sorts pass kFrzNoLimit.
//
// Ranked calls (frz_match_list_ranked) sort by a key in place of the score: k_sort_hist and k_sort_scatter take the digit
// source as a template parameter (ScoreKey, BoostKey), and frz_launch_sort_by_key_dev runs the same one- or two-pass
// histogram-kernel sort on clamp(score + boost[index], 0, 65535).  The elements keep their raw scores.
//
// The ordered call's multi-block sort (frz_match_list_ordered, DESIGN.md §4.15) runs the same 8-bit passes, least
// significant first, over the digits of its 112-bit order key (OrderKey), skipping digits no two rows differ in.
#include "frz_device.cuh"
#include "frz_host.h"
#include "order_plan.cuh"

#include <algorithm>

#include <cub/block/block_radix_sort.cuh>

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

// The digit source of k_sort_hist / k_sort_scatter: the 16-bit key an element is sorted by.  Either way the element itself
// is moved unchanged.
struct ScoreKey {   // the score sort
    __device__ __forceinline__ uint32_t operator()(const FrzMatchDev& m) const { return m.score; }
};
struct BoostKey {   // the ranked sort: clamp(score + boost[index], 0, 65535), boost 0 at and past index n
    const int16_t* boost;
    uint32_t n;
    __device__ __forceinline__ uint32_t operator()(const FrzMatchDev& m) const {
        const int b = m.index < n ? (int)__ldg(boost + m.index) : 0;
        return (uint32_t)min(max((int)m.score + b, 0), 0xFFFF);
    }
};

template <class Key>
__device__ __forceinline__ uint32_t digit_of(const FrzMatchDev& m, int shift, uint32_t mask, const Key& key) {
    return (key(m) >> shift) & mask;
}

template <class Key>
__global__ void __launch_bounds__(kSortWarps * 32) k_sort_hist(const FrzMatchDev* __restrict__ in,
                                                               const unsigned long long* __restrict__ n_ptr, int shift,
                                                               int bins, uint32_t* __restrict__ hist, Key key) {
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
        atomicAdd(&cnt[digit_of(a, shift, mask, key)], 1u);
        atomicAdd(&cnt[digit_of(b, shift, mask, key)], 1u);
        atomicAdd(&cnt[digit_of(c, shift, mask, key)], 1u);
        atomicAdd(&cnt[digit_of(d, shift, mask, key)], 1u);
    }
    for (; i < hi; i += 32) atomicAdd(&cnt[digit_of(in[i], shift, mask, key)], 1u);
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
    frz_wait_prior_grid();   // the histogram and the count come from the scoring kernels
    frz_allow_dependent_launch();
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

template <class Key>
__global__ void __launch_bounds__(kSortWarps * 32) k_sort_scatter(const FrzMatchDev* __restrict__ in, FrzMatchDev* __restrict__ out,
                                                                  const unsigned long long* __restrict__ n_ptr, int shift, int bins,
                                                                  const uint32_t* __restrict__ hist,
                                                                  const uint32_t* __restrict__ digit_base, uint32_t limit, Key key) {
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
        if (valid) d = digit_of(m, shift, mask, key);
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
// the segments).  The block sorts its segment in shared memory and writes it out as whole digit runs:
//   1. load: thread t loads the segment's elements t*8 .. t*8+7 (the blocked order cub's stable sort ranks by) and stages
//      them in shared memory;
//   2. sort: the key of element p is ((bins-1 - digit) << 11) | p, sorted by cub::BlockRadixSort over the digit bits only.
//      The sort is stable, so every digit run keeps index order, and the low 11 bits carry the element's position;
//   3. runs: rank r of the sorted segment starts a run where its digit differs from rank r-1's; that rank stores
//      off[d] = digit_base[d] + pref[d][segment] - r, so the element of rank r goes to off[d] + r;
//   4. store: thread t writes ranks t, t+256, ... (striped), so consecutive threads write consecutive addresses of a run.
// Elements past the end of the list (last segment) get digit 0's key: they sort behind every real digit-0 element (their
// positions are larger) and so take exactly the ranks >= the segment's element count, which are not stored.
constexpr int kSegThreads = 256;
constexpr int kSegItems = (1 << kFrzSortSegShift) / kSegThreads;   // elements per thread
static_assert(kSegItems * kSegThreads == (1 << kFrzSortSegShift), "a segment is a whole number of block-wide rounds");
static_assert(kSegItems % 2 == 0, "the blocked load moves two elements per 16-byte load");
using SegSort = cub::BlockRadixSort<uint32_t, kSegThreads, kSegItems>;

__global__ void __launch_bounds__(kSegThreads) k_sort_scatter_seg(const FrzMatchDev* __restrict__ in, FrzMatchDev* __restrict__ out,
                                                                  const unsigned long long* __restrict__ n_ptr, int bins,
                                                                  const uint32_t* __restrict__ pref, uint32_t stride,
                                                                  const uint32_t* __restrict__ digit_base, uint32_t limit) {
    constexpr int kSeg = 1 << kFrzSortSegShift;
    __shared__ union {
        typename SegSort::TempStorage sort;
        uint16_t digit[kSeg];   // digit of each sorted rank (after the sort)
    } tmp;
    __shared__ uint2 elem[kSeg];         // the segment, index order
    __shared__ uint32_t off[kMaxBins];   // per digit present in the segment: output position of rank 0 of its run
    frz_wait_prior_grid();   // pref and digit_base come from k_sort_scan_rows
    const unsigned long long n = *n_ptr;
    const uint32_t nseg = (uint32_t)((n + kSeg - 1) >> kFrzSortSegShift);
    const uint32_t mask = (uint32_t)bins - 1;
    const int end_bit = kFrzSortSegShift + 32 - __clz(mask);   // bins is a power of two
    const int t = threadIdx.x;
    for (uint32_t seg = blockIdx.x; seg < nseg; seg += gridDim.x) {
        const unsigned long long seg0 = (unsigned long long)seg << kFrzSortSegShift;
        const uint32_t cnt = (uint32_t)min(n - seg0, (unsigned long long)kSeg);
        const uint4* src = reinterpret_cast<const uint4*>(in + seg0) + t * (kSegItems / 2);
        uint32_t key[kSegItems];
#pragma unroll
        for (int j = 0; j < kSegItems / 2; j++) {
            const uint32_t p = t * kSegItems + 2 * j;
            uint4 v = make_uint4(0, 0, 0, 0);
            if (p + 1 < cnt) v = src[j];
            else if (p < cnt) { const uint2 h = *reinterpret_cast<const uint2*>(src + j); v.x = h.x; v.y = h.y; }
            reinterpret_cast<uint4*>(elem)[p >> 1] = v;
            // FrzMatchDev word 1: score in the low 16 bits
            key[2 * j] = ((mask - (v.y & mask)) << kFrzSortSegShift) | p;
            key[2 * j + 1] = ((mask - (v.w & mask)) << kFrzSortSegShift) | (p + 1);
        }
        // past the end: digit 0 (above), sorted behind every real element of that digit
        SegSort(tmp.sort).SortBlockedToStriped(key, kFrzSortSegShift, end_bit);
        __syncthreads();   // the sort's storage becomes the digit array
#pragma unroll
        for (int j = 0; j < kSegItems; j++) tmp.digit[t + j * kSegThreads] = (uint16_t)(mask - (key[j] >> kFrzSortSegShift));
        __syncthreads();
#pragma unroll
        for (int j = 0; j < kSegItems; j++) {
            const uint32_t r = t + j * kSegThreads;
            const uint32_t d = tmp.digit[r];
            if (r < cnt && (r == 0 || tmp.digit[r - 1] != d)) off[d] = digit_base[d] + pref[(size_t)d * stride + seg] - r;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < kSegItems; j++) {
            const uint32_t r = t + j * kSegThreads;
            if (r < cnt) {
                const uint32_t pos = off[mask - (key[j] >> kFrzSortSegShift)] + r;
                if (pos < limit) reinterpret_cast<uint2*>(out)[pos] = elem[key[j] & (kSeg - 1)];
            }
        }
        __syncthreads();   // elem, off and the sort storage are reused by the next segment
    }
}

// One histogram-kernel pass: the list at src scattered to dst, stably by descending digit (Key >> shift) & (bins - 1).
// Only the positions below `keep` are stored.
template <class Key>
frz_status sort_pass(const FrzMatchDev* src, FrzMatchDev* dst, const unsigned long long* n_ptr, int shift, int bins, uint32_t keep,
                     Key key, FrzSortScratch& ss, cudaStream_t stream, FrzLaunchStats* st) {
    uint32_t* const hist = ss.hist.get();
    const size_t smem = (size_t)kSortWarps * bins * sizeof(uint32_t);
    k_sort_hist<<<kSortBlocks, kSortWarps * 32, smem, stream>>>(src, n_ptr, shift, bins, hist, key);
    uint32_t* totals = hist + (size_t)kMaxBins * kV;
    uint32_t* digit_base = totals + kMaxBins;
    unsigned int* done_counter = reinterpret_cast<unsigned int*>(digit_base + kMaxBins);   // zeroed at allocation, self-resetting
    k_sort_scan_rows<kV / 128, false><<<(bins + 7) / 8, 256, 0, stream>>>(hist, hist, kV, nullptr, bins, totals,
                                                                           digit_base, done_counter);
    if (ss.arm_table_ev && ss.table_ev) {   // digit_base is final: the multi-GPU layer publishes it while the scatter runs
        FRZ_CUDA_TRY(cudaEventRecord(ss.table_ev.get(), stream));
        ss.table_ev_recorded = true;
    }
    k_sort_scatter<<<kSortBlocks, kSortWarps * 32, smem, stream>>>(src, dst, n_ptr, shift, bins, hist, digit_base, keep, key);
    FRZ_CUDA_TRY(cudaGetLastError());
    if (st) st->launches += 3;
    return FRZ_OK;
}

// The histogram-kernel sort of the list at d_in by descending Key (stable): one pass when the key bound allows it, else
// the reference's two 8-bit LSD passes.  n_ptr: device pointer to the element count.  bound: host-known upper bound of
// any key.
template <class Key>
frz_status launch_sort_dev(const FrzMatchDev* d_in, FrzMatchDev* d_tmp, FrzMatchDev* d_out, const unsigned long long* n_ptr,
                           uint32_t bound, Key key, FrzSortScratch& ss, cudaStream_t stream, FrzLaunchStats* st, uint32_t limit) {
    auto pass = [&](const FrzMatchDev* src, FrzMatchDev* dst, int shift, int bins, uint32_t keep) -> frz_status {
        return sort_pass(src, dst, n_ptr, shift, bins, keep, key, ss, stream, st);
    };
    if (bound < 256) return pass(d_in, d_out, 0, 256, limit);
    if (bound < 512) return pass(d_in, d_out, 0, 512, limit);
    if (bound < 1024) return pass(d_in, d_out, 0, 1024, limit);
    // the reference's two 8-bit LSD passes (src/sort.rs:8-39); only the second one knows final positions
    FRZ_TRY(pass(d_in, d_tmp, 0, 256, kFrzNoLimit));
    return pass(d_tmp, d_out, 8, 256, limit);
}

// The digit source of the ordered call's sort (frz_match_list_ordered): digit `shift` of the row's order key
// (order_plan.cuh), recomputed from the record, its attribute value and its boost.
struct OrderKey {
    FrzOrderDev o;
    uint32_t shift;
    __device__ __forceinline__ uint32_t operator()(const FrzMatchDev& m) const {
        return frz_order_digit(frz_order_row_key(o, m.index, m.score), shift);
    }
};

}  // namespace

frz_status frz_launch_sort_by_score_dev(const FrzMatchDev* d_in, FrzMatchDev* d_tmp, FrzMatchDev* d_out,
                                        const unsigned long long* n_ptr, uint32_t score_bound, FrzSortScratch& ss,
                                        cudaStream_t stream, FrzLaunchStats* st, uint32_t limit) {
    return launch_sort_dev(d_in, d_tmp, d_out, n_ptr, score_bound, ScoreKey(), ss, stream, st, limit);
}

frz_status frz_launch_sort_by_key_dev(const FrzMatchDev* d_in, FrzMatchDev* d_tmp, FrzMatchDev* d_out,
                                      const unsigned long long* n_ptr, const int16_t* boost, uint32_t n_boost, uint32_t key_bound,
                                      FrzSortScratch& ss, cudaStream_t stream, FrzLaunchStats* st, uint32_t limit) {
    return launch_sort_dev(d_in, d_tmp, d_out, n_ptr, key_bound, BoostKey{boost, n_boost}, ss, stream, st, limit);
}

frz_status frz_launch_sort_by_order_dev(const FrzMatchDev* d_in, FrzMatchDev* d_tmp, FrzMatchDev* d_out, const unsigned long long* n_ptr,
                                        const FrzOrderDev& o, const uint32_t* shifts, uint32_t n_shifts, FrzSortScratch& ss,
                                        cudaStream_t stream, FrzLaunchStats* st, uint32_t limit) {
    if (n_shifts == 0) return frz_fail(FRZ_ERR_INVALID_ARG, "an ordered sort needs a digit");
    const FrzMatchDev* src = d_in;
    for (uint32_t i = 0; i < n_shifts; i++) {   // least significant digit first; the last pass lands in d_out
        FrzMatchDev* dst = (n_shifts - 1 - i) % 2 == 0 ? d_out : d_tmp;
        FRZ_TRY(sort_pass(src, dst, n_ptr, 0, (int)kFrzOrderBins, i + 1 == n_shifts ? limit : kFrzNoLimit,
                          OrderKey{o, shifts[n_shifts - 1 - i]}, ss, stream, st));
        src = dst;
    }
    return FRZ_OK;
}

// allocates the sort scratch on the current device: counts, totals, digit_base + the pass-completion counter of
// k_sort_scan_rows, which must start at zero
frz_status frz_sort_hist_alloc(FrzDevArray<uint32_t>& out) {
    FRZ_TRY(out.reserve((size_t)kMaxBins * kV + 2 * kMaxBins + 4));
    FRZ_CUDA_TRY(cudaMemset(out.get() + (size_t)kMaxBins * kV + 2 * kMaxBins, 0, 4 * sizeof(uint32_t)));
    return FRZ_OK;
}

// digit_base[d] of the LAST pass run with this scratch = number of elements whose digit is greater than d.  After a
// single-pass sort (score bound < 1024) that is, per score s, how many matches of the run score higher than s — the table
// the multi-GPU slice exchange needs (parallel.cu) — so nobody has to binary-search the sorted run for it.
const uint32_t* frz_sort_digit_base(const FrzSortScratch& ss) { return ss.hist.get() ? ss.hist.get() + (size_t)kMaxBins * kV + kMaxBins : nullptr; }
int frz_sort_single_pass_bins(uint32_t score_bound) { return score_bound < 256 ? 256 : score_bound < 512 ? 512 : score_bound < 1024 ? 1024 : 0; }

// ss.fused holds the counts ([bins][stride]) and then the scan's prefix rows (same shape).  The counts are zero between
// calls (the scan re-zeroes every word the scoring kernels can have touched), so only growth, a new layout reaching past
// the words known to be zero, or a call that stopped between scoring and scan costs a memset.
frz_status frz_sort_fused_prepare(FrzSortScratch& ss, uint64_t n_cap, uint32_t score_bound, cudaStream_t stream, FrzScoreHist* out) {
    const int bins = frz_sort_single_pass_bins(score_bound);
    if (bins == 0) return frz_fail(FRZ_ERR_INVALID_ARG, "fused sort needs a score bound below 1024 (got %u)", score_bound);
    const uint64_t segs = (n_cap + (1ull << kFrzSortSegShift) - 1) >> kFrzSortSegShift;
    const uint64_t stride = std::max<uint64_t>((segs + 3) & ~3ull, 4);
    const uint64_t words = (uint64_t)bins * stride;
    if (ss.fused.cap() < 2 * words) {
        ss.fused_clean_words = 0;
        FRZ_TRY(ss.fused.reserve(2 * words));
    }
    if (ss.fused_dirty || ss.fused_clean_words < words)
        FRZ_CUDA_TRY(cudaMemsetAsync(ss.fused.get(), 0, words * sizeof(uint32_t), stream));
    ss.fused_clean_words = words;   // the prefix rows are written right behind the counts
    ss.fused_dirty = true;
    out->counts = ss.fused.get();
    out->stride = (uint32_t)stride;
    out->mask = (uint32_t)bins - 1;
    return FRZ_OK;
}

frz_status frz_launch_sort_fused(const FrzMatchDev* d_in, FrzMatchDev* d_out, const unsigned long long* n_ptr, const FrzScoreHist& h,
                                 FrzSortScratch& ss, cudaStream_t stream, FrzLaunchStats* st, uint32_t limit) {
    const int bins = (int)h.mask + 1;
    uint32_t* pref = h.counts + (size_t)bins * h.stride;
    uint32_t* totals = ss.hist.get() + (size_t)kMaxBins * kV;
    uint32_t* digit_base = totals + kMaxBins;
    unsigned int* done_counter = reinterpret_cast<unsigned int*>(digit_base + kMaxBins);
    FRZ_CUDA_TRY(frz_launch_dependent(k_sort_scan_rows<4, true>, (bins + 7) / 8, 256, 0, stream, h.counts, pref, h.stride, n_ptr, bins,
                                      totals, digit_base, done_counter));
    ss.fused_dirty = false;
    if (ss.arm_table_ev && ss.table_ev) {   // digit_base is final: the multi-GPU layer publishes it while the scatter runs
        FRZ_CUDA_TRY(cudaEventRecord(ss.table_ev.get(), stream));
        ss.table_ev_recorded = true;
    }
    const int grid = (int)std::max<uint32_t>(1, std::min<uint32_t>(h.stride, (uint32_t)frz_sm_count() * 4));
    FRZ_CUDA_TRY(frz_launch_dependent(k_sort_scatter_seg, grid, kSegThreads, 0, stream, d_in, d_out, n_ptr, bins, pref, h.stride,
                                      digit_base, limit));
    if (st) st->launches += 2;
    return FRZ_OK;
}
