// frz_host.h — internal host-side declarations shared by the .cu translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <atomic>
#include <memory>
#include <string>
#include <vector>

#include "../../include/frz_cuda.h"
#include "frz_device.cuh"
#include "order_plan.cuh"
#include "unicode_path.cuh"

frz_status frz_fail(frz_status s, const char* fmt, ...);
// Argument checks of the entry points (host.cu), with their status codes and messages.
frz_status frz_ensure_device(int device);                                  // a valid device, made current
frz_status frz_check_offset_width(int offset_width);                       // Arrow offsets of 4 or 8 bytes
frz_status frz_check_index_range(uint64_t n, uint32_t index_offset);       // the indices of n rows from index_offset fit in u32
inline int frz_current_device() { int d = 0; cudaGetDevice(&d); return d; }
// SMs of the current device (cached per device): persistent grids and grid caps are multiples of it
inline int frz_sm_count() {
    static int count_dev[64] = {};
    const int d = frz_current_device();
    int& c = count_dev[d & 63];
    if (c <= 0 && (cudaDeviceGetAttribute(&c, cudaDevAttrMultiProcessorCount, d) != cudaSuccess || c <= 0)) c = 132;   // H100 SXM
    return c;
}
// a grid of `block`-thread blocks over n items, at most 16 blocks per SM
inline int grid_for(uint64_t n, int block) {
    return (int)std::max<uint64_t>(1, std::min<uint64_t>((n + block - 1) / block, (uint64_t)frz_sm_count() * 16));
}

// Launches `k` with programmatic stream serialization: its blocks may be scheduled while the kernel ahead of it on the
// stream drains its tail (and run before it completes when that kernel calls frz_allow_dependent_launch).  `k` must call
// frz_wait_prior_grid() before its first global memory access (frz_device.cuh).  Any other stream operation ahead of it
// (a copy, a memset, an event record) orders it as a normal launch would.
template <typename... KArgs, typename... Args>
inline cudaError_t frz_launch_dependent(void (*k)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, k, std::forward<Args>(args)...);
}

#define FRZ_CUDA_TRY(expr)                                                                         \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            cudaGetLastError();                                                                    \
            return frz_fail(_e == cudaErrorMemoryAllocation ? FRZ_ERR_OOM : FRZ_ERR_CUDA,          \
                            "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
        }                                                                                          \
    } while (0)

#define FRZ_TRY(expr)                         \
    do {                                      \
        frz_status _s = (expr);               \
        if (_s != FRZ_OK) return _s;          \
    } while (0)

// ------------------------------------------------------------------------------------------ owners
// The only place the library frees CUDA memory, events and streams.  Every buffer, event and stream is held by one of
// these move-only types, so error paths and device switches release what they own without a hand-written list.

// Bytes held by all device FrzDevArrays (frz_debug_device_bytes).
inline std::atomic<uint64_t> g_frz_device_bytes{0};
// Their high-water mark since the last frz_debug_device_bytes_peak(reset != 0).
inline std::atomic<uint64_t> g_frz_device_bytes_peak{0};

// A grow-only array of T on one device (Pinned: in page-locked host memory).  It remembers the device it was allocated on
// and frees the block there; an empty array makes no CUDA call, so host-only users never touch the runtime.
template <typename T, bool Pinned = false>
class FrzDevArray {
public:
    FrzDevArray() = default;
    FrzDevArray(FrzDevArray&& o) noexcept : p_(o.p_), cap_(o.cap_), dev_(o.dev_) { o.p_ = nullptr; o.cap_ = 0; }
    FrzDevArray& operator=(FrzDevArray&& o) noexcept {
        if (this != &o) {
            reset();
            p_ = o.p_; cap_ = o.cap_; dev_ = o.dev_;
            o.p_ = nullptr; o.cap_ = 0;
        }
        return *this;
    }
    FrzDevArray(const FrzDevArray&) = delete;
    FrzDevArray& operator=(const FrzDevArray&) = delete;
    ~FrzDevArray() { reset(); }

    T* get() const { return p_; }
    uint64_t cap() const { return cap_; }   // in elements
    int device() const { return dev_; }
    // cap() >= need afterwards.  Growing frees the old block first (its contents are dropped, so the peak stays one block)
    // and then allocates `want` (>= need) elements on the current device.
    frz_status reserve(uint64_t need, uint64_t want) {
        if (cap_ >= need) return FRZ_OK;
        reset();
        void* p = nullptr;
        FRZ_CUDA_TRY(Pinned ? cudaMallocHost(&p, want * sizeof(T)) : cudaMalloc(&p, want * sizeof(T)));
        cudaGetDevice(&dev_);
        p_ = static_cast<T*>(p);
        cap_ = want;
        if (!Pinned) {
            const uint64_t now = g_frz_device_bytes += cap_ * sizeof(T);
            uint64_t peak = g_frz_device_bytes_peak.load();
            while (now > peak && !g_frz_device_bytes_peak.compare_exchange_weak(peak, now)) {}
        }
        return FRZ_OK;
    }
    frz_status reserve(uint64_t n) { return reserve(n, n); }
    // frees the block on its own device; the calling thread's current device is left as it was
    void reset() {
        if (!p_) return;
        int cur = dev_;
        cudaGetDevice(&cur);
        if (cur != dev_) cudaSetDevice(dev_);
        if (Pinned) cudaFreeHost(p_);
        else { cudaFree(p_); g_frz_device_bytes -= cap_ * sizeof(T); }
        if (cur != dev_) cudaSetDevice(cur);
        p_ = nullptr;
        cap_ = 0;
    }

private:
    T* p_ = nullptr;
    uint64_t cap_ = 0;
    int dev_ = -1;
};
template <typename T>
using FrzPinnedArray = FrzDevArray<T, true>;

struct FrzEventDeleter { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
struct FrzStreamDeleter { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
using FrzEvent = std::unique_ptr<CUevent_st, FrzEventDeleter>;
using FrzStream = std::unique_ptr<CUstream_st, FrzStreamDeleter>;
inline frz_status frz_event_create(FrzEvent& out, unsigned flags) {
    cudaEvent_t e = nullptr;
    FRZ_CUDA_TRY(cudaEventCreateWithFlags(&e, flags));
    out.reset(e);
    return FRZ_OK;
}
inline frz_status frz_stream_create(FrzStream& out, unsigned flags) {
    cudaStream_t s = nullptr;
    FRZ_CUDA_TRY(cudaStreamCreateWithFlags(&s, flags));
    out.reset(s);
    return FRZ_OK;
}

// Owned device buffers of a packed corpus.
struct FrzCorpusStorage {
    // grow-only, reused by the end-to-end path (no cudaMalloc/cudaFree per call); tile_base.cap() is the tile capacity
    FrzDevArray<uint4> data;
    FrzDevArray<uint64_t> tile_base;
    FrzDevArray<FrzGroupDesc> groups;
    FrzDevArray<uint32_t> slot_meta;
    FrzDevArray<uint16_t> slot_of;
    FrzDevArray<uint2> slot_sig;
    FrzDevArray<uint64_t> scratch_tile_units;  // [tile capacity] + 2 words (total, error)
    uint64_t n = 0;
    uint32_t n_tiles = 0;
    uint64_t total_units = 0;  // end of the arena: units [0, total_units) are written
    uint64_t total_bytes = 0;  // sum of the live haystacks' lengths
    uint32_t max_gunits = 0;   // longest haystack of the corpus in 16-byte units (never below the truth)
    uint64_t n_removed = 0;    // haystacks whose slot is FRZ_INVALID_SLOT (frz_corpus_remove); matching filters only when > 0
    uint64_t dead_units = 0;   // arena units no tile points at any more (left behind by re-packed tiles)
    int device = 0;

    FrzCorpusView view() const {
        FrzCorpusView v;
        v.data = data.get();
        v.tile_base = tile_base.get();
        v.groups = groups.get();
        v.slot_meta = slot_meta.get();
        v.slot_of = slot_of.get();
        v.slot_sig = slot_sig.get();
        v.n = n;
        v.n_tiles = n_tiles;
        v.max_gunits = max_gunits;
        return v;
    }
};

// Staging arena + copy stream of the streamed ingest (pack.cu): grow-only, reused across calls.
struct FrzIngest {
    static constexpr int kMaxChunks = 32;
    static constexpr uint64_t kMinChunkBytes = 8ull << 20;
    FrzDevArray<uint8_t> d_bytes;
    FrzDevArray<uint8_t> d_offsets;
    FrzStream copy_stream;            // non-blocking: overlaps the (legacy default) compute stream
    FrzEvent ev[kMaxChunks + 1];      // [c] chunk c landed; [kMaxChunks] offsets landed / arena free
    frz_status reserve(uint64_t bytes, uint64_t offset_bytes);
};

struct frz_corpus {
    FrzCorpusStorage st;
    std::unique_ptr<FrzIngest> ingest;   // created by the first frz_corpus_append / _remove / _replace, kept for the next ones
    // metadata of the tiles a frz_corpus_replace re-packs (grow-only; a replace releases it, and the ingest staging, once
    // they pass 64 MiB)
    std::unique_ptr<FrzCorpusStorage> edit_tiles;
    // pinned staging of frz_match_list_batch (patterns up, rows and counts down), grow-only
    mutable FrzPinnedArray<uint8_t> batch_stage;
    // device staging of frz_subset_where_batch (attributes, clauses, queries, set values, member counts), grow-only
    mutable FrzDevArray<uint8_t> where_stage;
};

// pack.cu
frz_status frz_pack_corpus_device(const uint8_t* d_bytes, const void* d_offsets, int offset_width, uint64_t n, uint64_t total_bytes,
                                  cudaStream_t stream, FrzCorpusStorage* out);
frz_status frz_append_host(FrzIngest& ing, const uint8_t* h_bytes, const void* h_offsets, int offset_width, uint64_t n_new,
                           cudaStream_t stream, FrzCorpusStorage* st);
// In-place edits (the arguments are checked by the callers in host.cu, before anything changes).  Synchronous.
frz_status frz_remove_host(FrzIngest& ing, const uint32_t* which, uint64_t n, cudaStream_t stream, FrzCorpusStorage* st);
frz_status frz_replace_host(FrzIngest& ing, FrzCorpusStorage& scratch, const uint32_t* which, uint64_t n, const uint8_t* h_bytes,
                            const void* h_offsets, int offset_width, cudaStream_t stream, FrzCorpusStorage* st);
// `after_chunk` (optional) is called on the host right after the pack kernels of tiles [t0, t1) have been enqueued on
// `stream` (chunks arrive in tile order; `last` marks the final one): the caller may enqueue work on those tiles at once.
typedef frz_status (*FrzChunkFn)(void* ctx, uint32_t t0, uint32_t t1, bool last);
frz_status frz_ingest_host(FrzIngest& ing, const uint8_t* h_bytes, const void* h_offsets, int offset_width, uint64_t n,
                           cudaStream_t stream, FrzCorpusStorage* out, FrzChunkFn after_chunk = nullptr, void* ctx = nullptr);

// Score histogram that the scoring kernels (sw.cu) accumulate as they emit, for the single-pass score sort (sort.cu):
// counts[d * stride + s] = matches with score digit d whose index-ordered position lies in segment s = pos >> kFrzSortSegShift.
// counts == nullptr: no histogram is wanted.
constexpr int kFrzSortSegShift = 11;   // 2048-element segments
struct FrzScoreHist {
    uint32_t* counts = nullptr;
    uint32_t stride = 0;   // words per digit row: segments of the largest possible list, rounded up to a multiple of 4
    uint32_t mask = 0;     // bins - 1
};

// Scratch of the score sorts (sort.cu), one per concurrent user.
struct FrzSortScratch {
    FrzDevArray<uint32_t> hist;             // frz_sort_hist_alloc: per-segment digit counts, totals, digit_base, pass counter
    FrzDevArray<uint32_t> fused;            // FrzScoreHist counts, then the per-segment prefix rows the sort's scan writes
    uint64_t fused_clean_words = 0;         // leading words of `fused` known to be zero (the scan re-zeroes what it reads)
    bool fused_dirty = false;               // counts were handed to the scoring kernels, their scan was not enqueued yet
    FrzEvent table_ev;                      // recorded right after the sort's scan kernel: the per-score table is final there,
    bool arm_table_ev = false;              //   one kernel (the scatter) before the run itself (shard calls arm it)
    bool table_ev_recorded = false;
};

// Per-matcher device workspace (grown on demand, reused across calls).  Everything in it lives on `device`; moving to
// another device is a move-assignment from a fresh workspace.
struct FrzWorkspace {
    int device = -1;
    FrzDevArray<FrzCounters> counters;
    FrzPinnedArray<FrzCounters> h_counters;          // host mirror
    FrzDevArray<unsigned long long> stream_total;    // [0] running match count of a streamed call (tile-scan carry), [1] spare count slot
    FrzDevArray<FrzSurvivor> survivors[FRZ_N_CLASSES];
    FrzSurvLists lists() const { FrzSurvLists l; for (int c = 0; c < FRZ_N_CLASSES; c++) l.p[c] = survivors[c].get(); return l; }
    uint64_t survivor_cap() const { return survivors[0].cap(); }   // per class
    FrzDevArray<uint32_t> surv_bitmap;      // [n_tiles * 32] survivor bits by index-within-tile
    FrzDevArray<uint16_t> word_prefix;      // [n_tiles * 32] exclusive popcount prefix of surv_bitmap words
    FrzDevArray<uint32_t> tile_count;       // [n_tiles] matches per tile
    FrzDevArray<uint64_t> tile_out_base;    // [n_tiles] exclusive scan of tile_count
    FrzDevArray<FrzMatchDev> matches_a;     // index-ordered matches
    FrzDevArray<FrzMatchDev> matches_b;     // sort ping-pong / final
    FrzDevArray<FrzMatchDev> multi_a;       // multi-pattern candidate ping-pong / two-pass sort scratch
    FrzDevArray<FrzMatchDev> multi_b;
    FrzSortScratch sort;
    FrzDevArray<uint4> cand_list;           // k_sig_scan → k_window candidate records (16 bytes each)
    FrzDevArray<uint32_t> retain_cnt;       // multi-pattern stable compaction scratch
    FrzDevArray<uint64_t> retain_base;
    FrzDevArray<uint8_t> retain_keep;
    FrzDevArray<uint16_t> unicode_scratch;  // unicode.cu: per-thread row state of the per-scalar Smith-Waterman
    FrzDevArray<uint32_t> subset_meta;      // [n_tiles * 1024] slot metadata of a subset call: non-members are unused slots
    FrzDevArray<FrzMatchDev> subset_list;   // [2 * members] list-form subset call: member records, then the live ones compacted
    FrzDevArray<uint32_t> collapse_counts;  // [n_groups] collapsed call: the list's rows per group
    FrzDevArray<unsigned long long> collapse_best;  // [n_groups] its round table, all zero between calls
    FrzDevArray<unsigned long long> collapse_best_lo;  // [n_groups] the second table of rounds on the order key, zero too
    FrzDevArray<uint8_t> collapse_taken;    // [corpus length] its rows taken in a round
    FrzDevArray<FrzOrderKey> order_keys;    // [list rows] ordered call: the order key of each list row
    FrzDevArray<uint32_t> order_cand;       // [2 * list rows] its select's candidate positions (two pass parities)
    FrzDevArray<uint32_t> order_sel;        // [list rows] its selected positions
    FrzDevArray<uint32_t> order_hist;       // [kFrzOrderBins] a select pass's digit counts, zero between passes
    FrzDevArray<FrzOrderState> order_state;
    FrzPinnedArray<FrzOrderState> h_order_state;
    FrzEvent ev[4];                         // call start, scan done, scoring done, call end
    bool ev_rec[4] = {false, false, false, false};  // recorded during the current call
};

// kernels (prefilter.cu / sw.cu / sort.cu) — all asynchronous on `stream`
struct FrzLaunchStats {
    uint64_t launches = 0;
};

// ntab: the needle's FrzNeedleTab (device) when pat.n > FRZ_MAX_NEEDLE, else unused
frz_status frz_launch_prefilter(const FrzCorpusView& cv, const FrzPatternDev& pat, FrzWorkspace& ws, cudaStream_t stream,
                                FrzLaunchStats* st, const FrzNeedleTab* ntab = nullptr);
frz_status frz_launch_sig_scan(const FrzCorpusView& cv, const FrzPatternDev& pat, FrzWorkspace& ws, cudaStream_t stream,
                               FrzLaunchStats* st);
// member_only: only the survivor bitmap (frz_subset_match): no Smith-Waterman, exact check or survivor records
frz_status frz_launch_unicode(const FrzCorpusView& cv, const FrzPatternDev& pat, const FrzUNeedle& un, const FrzUScoring& usc,
                              const FrzMatchDev* cand, uint64_t n_cand, uint32_t index_offset, FrzWorkspace& ws,
                              cudaStream_t stream, FrzLaunchStats* st, bool member_only = false);
frz_status frz_launch_match_indices(const FrzCorpusView& cv, const FrzPatternDev& pat, const FrzUNeedle& un, const FrzUScoring& usc,
                                    bool unicode, const uint32_t* d_which, uint64_t n, FrzMatchDev* d_matches, uint32_t* d_idx,
                                    uint32_t stride, uint32_t* d_cnt, uint16_t* d_scratch, uint64_t scratch_stride, uint32_t threads,
                                    cudaStream_t stream);
frz_status frz_launch_prefilter_list(const FrzCorpusView& cv, const FrzPatternDev& pat, const FrzMatchDev* cand,
                                     uint64_t n_cand, uint32_t index_offset, FrzWorkspace& ws, cudaStream_t stream,
                                     FrzLaunchStats* st, const FrzNeedleTab* ntab = nullptr);
frz_status frz_launch_tile_scan(const FrzCorpusView& cv, FrzWorkspace& ws, cudaStream_t stream, FrzLaunchStats* st,
                                unsigned long long* carry = nullptr);
// hist.counts != nullptr: every emitted match also counts itself into `hist` (see FrzScoreHist)
frz_status frz_launch_sw(const FrzCorpusView& cv, const FrzPatternDev& pat, uint32_t index_offset, bool reversed,
                         FrzWorkspace& ws, FrzMatchDev* d_out, cudaStream_t stream, FrzLaunchStats* st,
                         const FrzScoreHist& hist = FrzScoreHist(), const FrzNeedleTab* ntab = nullptr);
// "no limit" for the sorts' `limit` argument: every position of a list is below it (lists hold at most 2^32 - 1 matches)
constexpr uint32_t kFrzNoLimit = 0xFFFFFFFFu;
// stable sort by descending score; the element count is read from device memory (*n_ptr).
// d_tmp is only used when score_bound >= 1024 (two 8-bit passes); result always lands in d_out.
// limit: only the sorted positions below it are stored (top-K calls); kFrzNoLimit sorts the whole list.
frz_status frz_launch_sort_by_score_dev(const FrzMatchDev* d_in, FrzMatchDev* d_tmp, FrzMatchDev* d_out,
                                        const unsigned long long* n_ptr, uint32_t score_bound, FrzSortScratch& ss,
                                        cudaStream_t stream, FrzLaunchStats* st, uint32_t limit = kFrzNoLimit);
// The same sort by descending key = clamp(score + boost[index], 0, 65535), boost 0 at indices >= n_boost (ranked calls).
// key_bound: host-known upper bound of any key; d_tmp is used when it is >= 1024.
frz_status frz_launch_sort_by_key_dev(const FrzMatchDev* d_in, FrzMatchDev* d_tmp, FrzMatchDev* d_out,
                                      const unsigned long long* n_ptr, const int16_t* boost, uint32_t n_boost, uint32_t key_bound,
                                      FrzSortScratch& ss, cudaStream_t stream, FrzLaunchStats* st, uint32_t limit = kFrzNoLimit);
frz_status frz_sort_hist_alloc(FrzDevArray<uint32_t>& out);
const uint32_t* frz_sort_digit_base(const FrzSortScratch& ss);
int frz_sort_single_pass_bins(uint32_t score_bound);   // bins of the single-pass sort for this bound, 0 = two passes
// The fused single-pass sort: the scoring kernels build the histogram (frz_launch_sw with `hist`), so the sort is a scan
// and a block-per-segment scatter.  prepare: sizes and zeroes the histogram for lists of up to n_cap matches whose scores
// are below score_bound (< 1024).  The sort reads the count at *n_ptr and leaves the histogram zeroed for the next call.
frz_status frz_sort_fused_prepare(FrzSortScratch& ss, uint64_t n_cap, uint32_t score_bound, cudaStream_t stream, FrzScoreHist* out);
frz_status frz_launch_sort_fused(const FrzMatchDev* d_in, FrzMatchDev* d_out, const unsigned long long* n_ptr, const FrzScoreHist& hist,
                                 FrzSortScratch& ss, cudaStream_t stream, FrzLaunchStats* st, uint32_t limit = kFrzNoLimit);

// One sub-batch of frz_match_list_batch_top (host.cu, DESIGN.md §4.11) on the device.  Query j (0 <= j < the sub-batch's
// size) owns slice j of every array; its kernels see exactly the buffers a single-query call's kernels see.  A batched
// launch covers a group of queries (FrzBatchGroup, a kernel argument): block row blockIdx.y runs query grp.j[blockIdx.y].
constexpr uint32_t kFrzBatchMaxSub = 64;   // queries of one sub-batch
struct FrzBatchGroup {
    uint16_t j[kFrzBatchMaxSub];
};
struct FrzBatchDev {
    const FrzPatternDev* pats;        // [j] compiled pattern
    const uint8_t* reversed;          // [j] 1: the list is written in descending index order (the *_DESC strategies)
    const uint8_t* by_score;          // [j] 1: the rows are ordered by score (the ScoreThenIndex strategies)
    FrzSurvivor* surv;                // [j][class][surv_cap]
    unsigned long long surv_cap;      // per query and class
    FrzCounters* ctr;                 // [j]
    uint32_t* surv_bitmap;            // [j][n_tiles * 32]
    uint16_t* word_prefix;            // [j][n_tiles * 32]
    uint32_t* tile_count;             // [j][n_tiles]
    uint64_t* tile_out_base;          // [j][n_tiles]
    FrzMatchDev* lists;               // [j][list_stride] index-ordered matches
    uint64_t list_stride;
};
#if defined(__CUDACC__)
__device__ __forceinline__ FrzSurvLists frz_batch_lists(const FrzBatchDev& b, uint32_t j) {
    FrzSurvLists l;
    for (int c = 0; c < FRZ_N_CLASSES; c++) l.p[c] = b.surv + ((uint64_t)j * FRZ_N_CLASSES + c) * b.surv_cap;
    return l;
}
// the block's copy of query j's pattern (call before the block's first barrier, then __syncthreads)
__device__ __forceinline__ void frz_batch_stage_pattern(const FrzBatchDev& b, uint32_t j, FrzPatternDev* pat_s) {
    static_assert(sizeof(FrzPatternDev) % 4 == 0, "pattern words");
    const uint32_t* src = reinterpret_cast<const uint32_t*>(b.pats + j);
    uint32_t* dst = reinterpret_cast<uint32_t*>(pat_s);
    for (uint32_t i = threadIdx.x; i < sizeof(FrzPatternDev) / 4; i += blockDim.x) dst[i] = src[i];
}
#endif
// Stages of a sub-batch, all asynchronous on `stream`.  h_pats: host copies of the nq patterns (they choose the kernel
// variants).  prefilter.cu: one k_scan_window_batch launch per typo mode present (the counters and bitmaps must be zeroed), then the
// per-query tile ranks and scans
frz_status frz_launch_prefilter_batch(const FrzCorpusView& cv, const FrzBatchDev& b, const FrzPatternDev* h_pats, uint32_t nq,
                                      cudaStream_t stream, FrzLaunchStats* st);
// sw.cu: the scoring classes of frz_launch_sw, one launch per kernel variant present
frz_status frz_launch_sw_batch(const FrzCorpusView& cv, const FrzBatchDev& b, const FrzPatternDev* h_pats, uint32_t nq,
                               cudaStream_t stream, FrzLaunchStats* st);
// The subset and boost of one query of frz_match_list_batch (host.cu), read by k_batch_top<ScopedKey> (batch.cu).  A query
// without either has scoped = ranked = 0 and is answered as by frz_match_list_batch_top.
struct FrzBatchScope {
    const uint32_t* bits;    // scoped: the subset's bitmap over [0, n_bits) (frz_batch_member)
    const int16_t* boost;    // ranked: boost[index] for index < n_boost, 0 past it
    uint64_t n_bits;
    uint32_t n_boost;
    uint8_t scoped;          // 1: only the subset's members are rows of the query
    uint8_t ranked;          // 1: the rows are ordered by clamp(score + boost[index], 0, 65535) under every strategy
    uint8_t pad[2];
};
// batch.cu: per query, its first min(k, total) rows → rows[j * k ...] and its total → totals[j], or kFrzBatchOverflow
// there when its sticky device error is set (k <= kFrzBatchMaxK).  scopes: nullptr, or the nq queries' FrzBatchScope
// records on the device (a sub-batch with a scoped or ranked query).
frz_status frz_launch_batch_top(const FrzBatchDev& b, const FrzBatchScope* scopes, uint32_t nq, uint32_t k, FrzMatchDev* rows,
                                unsigned long long* totals, cudaStream_t stream, FrzLaunchStats* st);

// The groups of a sub-batch of frz_match_list_batch_collapsed (host.cu; the per-query arithmetic is batch_collapse_plan.cuh's).
struct FrzBatchCollapse;
struct FrzBatchTables {
    const FrzBatchCollapse* cols;   // [j] the query's groups (ids == nullptr: none), on the device
    const FrzBatchScope* scopes;    // [j] its subset and boost
    uint32_t* counts;               // [slot][n_groups_max] the list's member rows per group
    unsigned long long* best;       // [slot][n_groups_max] a round's max entry; zero between rounds and calls
    uint8_t* taken;                 // [j][list_stride] the list's rows taken in a round
};
// collapse.cu: the count pass over every grouped query's list (counts must be zero), then `rounds` rounds of a max pass and
// a take pass, each one launch over the nq queries.  A query with its sticky device error set is skipped.
frz_status frz_launch_batch_collapse(const FrzBatchDev& b, const FrzBatchTables& t, uint32_t nq, uint32_t rounds, cudaStream_t stream,
                                     FrzLaunchStats* st);
// batch.cu: frz_launch_batch_top whose rows are, for a grouped query, the kept rows of its collapse (k_batch_top<CollapsedKey>)
frz_status frz_launch_batch_top_collapsed(const FrzBatchDev& b, const FrzBatchTables& t, uint32_t nq, uint32_t k, FrzMatchDev* rows,
                                          unsigned long long* totals, cudaStream_t stream, FrzLaunchStats* st);

// The ordering of a sub-batch of frz_match_list_batch_ordered (host.cu; the per-query arithmetic is batch_order_plan.cuh's).
// Every query of such a sub-batch is ordered.
struct FrzBatchOrderDev {
    const FrzOrderDev* ords;        // [j] the query's attribute, boost, order and direction, on the device
    FrzOrderKey* keys;              // [j][list_stride] its list rows' keys
    uint32_t* cand;                 // [j][2][list_stride] its rows, then the select's candidates
    uint32_t* sel;                  // [j][kFrzOrderBlockRows] the selection
    FrzOrderState* st;              // [j] zero before the key kernel
    uint32_t* hist;                 // [j][kFrzOrderBins] zero
    unsigned long long* best_lo;    // [slot][n_groups_max] with grouped queries: zero between rounds and calls
};
// order.cu: every query's keys (k_batch_order_keys), one launch over the nq queries
frz_status frz_launch_batch_order_keys(const FrzBatchDev& b, const FrzBatchOrderDev& o, uint32_t nq, cudaStream_t stream, FrzLaunchStats* st);
// collapse.cu: frz_launch_batch_collapse with rounds on the order keys (collapse_plan.cuh's two-step max, three passes per round)
frz_status frz_launch_batch_collapse_by_key(const FrzBatchDev& b, const FrzBatchTables& t, const FrzBatchOrderDev& o, uint32_t nq,
                                            uint32_t rounds, cudaStream_t stream, FrzLaunchStats* st);
// order.cu: every query's rows (t: the groups, or t.cols == nullptr when no query of the sub-batch has any), their select
// and their sort: its first min(k, total) rows in order → rows[j * k ...] and its total → totals[j], or kFrzBatchOverflow
// there when its sticky device error is set (k <= kFrzBatchMaxK)
frz_status frz_launch_batch_order_top(const FrzBatchDev& b, const FrzBatchTables& t, const FrzBatchOrderDev& o, uint32_t nq, uint32_t k,
                                      FrzMatchDev* rows, unsigned long long* totals, cudaStream_t stream, FrzLaunchStats* st);

// The join of a sub-batch of frz_match_list_batch_columns (host.cu; the per-row rule is batch_columns_plan.cuh's).
struct FrzColumnFold;
struct FrzBatchColumnsDev {
    uint32_t* acc;                 // [j][list_stride] the query's accumulator per row (zero before the first fold)
    uint32_t* err;                 // [j] the sticky device error of the query's column stages (zero before the first fold)
    const FrzColumnFold* fold;     // [c][nq] how query j folds column c
    const uint8_t* need;           // [j] the columns query j folds
    uint64_t n_rows;
};
// prefilter.cu: k_tile_scan_batch alone (tile_out_base and ctr[j].total from tile_count, for the nq queries)
frz_status frz_launch_tile_scan_batch(const FrzBatchDev& b, uint32_t n_tiles, uint32_t nq, cudaStream_t stream, FrzLaunchStats* st);
// batch_columns.cu: fold column c into every query's accumulator, from the lists its batched stages left in b's slots (cv:
// the column, for the rows live in it), one launch over the nq queries
frz_status frz_launch_batch_columns_fold(const FrzBatchDev& b, const FrzBatchColumnsDev& d, const FrzCorpusView& cv, uint32_t c,
                                         uint32_t nq, cudaStream_t stream, FrzLaunchStats* st);
// batch_columns.cu: every query's rows that matched each column it folds → b.lists[j] (index order, reversed when
// b.reversed[j]), their number → b.ctr[j].total and its error word → b.ctr[j].error: the list k_batch_top cuts
frz_status frz_launch_batch_columns_join(const FrzBatchDev& b, const FrzBatchColumnsDev& d, uint32_t n_tiles, uint32_t nq,
                                         cudaStream_t stream, FrzLaunchStats* st);

// The groups of a collapsed call on the device (frz_match_list_collapsed, host.cu; the rule is collapse_plan.cuh's).
struct FrzCollapseDev {
    const uint32_t* ids;         // group of index i < n_ids (frz_groups); indices past it are in no group
    const int16_t* boost;        // FRZ_COLLAPSE_BY_KEY: boost[index] for index < n_boost, 0 past it
    uint32_t* counts;            // [n_groups] rows of the list per group
    unsigned long long* best;    // [n_groups] a round's max entry (frz_collapse_entry); zero between rounds and calls
    uint8_t* taken;              // [list rows] taken in a round
    uint64_t n_ids;
    uint32_t n_boost;
    uint32_t per_group;          // 1..32 (0xFFFFFFFF: no cap, every count fits)
    uint8_t order;               // FrzCollapseOrder
    uint8_t reversed;            // 1: the *_DESC strategies
};
// collapse.cu: counts = zero, then the count pass over the list (its length at *n_ptr, at most n_cap rows), then `rounds`
// rounds (a max pass and a take pass each).  c.best must be zero on entry; it is zero again when the rounds have run.
frz_status frz_launch_collapse(const FrzCollapseDev& c, const FrzMatchDev* list, const unsigned long long* n_ptr, uint64_t n_cap,
                               uint64_t n_groups, uint32_t rounds, cudaStream_t stream, FrzLaunchStats* st);
// collapse.cu: frz_launch_collapse with rounds on the order key (collapse_plan.cuh's two-step max): keys[i] is list row i's
// FrzOrderKey, c.best is the best_hi table and best_lo the second one ([n_groups] each, zero on entry and again after the
// rounds); c.boost and c.order are not read.  Each round is three passes.
frz_status frz_launch_collapse_by_key(const FrzCollapseDev& c, unsigned long long* best_lo, const FrzOrderKey* keys,
                                      const FrzMatchDev* list, const unsigned long long* n_ptr, uint64_t n_cap, uint64_t n_groups,
                                      uint32_t rounds, cudaStream_t stream, FrzLaunchStats* st);

// The fill of frz_subset_where (host.cu; the rule and FrzWhereDev are where_plan.cuh's).
struct FrzWhereDev;
// where.cu: w.bits and w.chunk_count from the clauses and the base (k_where)
frz_status frz_launch_where(const FrzWhereDev& w, cudaStream_t stream);
// where.cu: the members of bits[0 .. ceil(n / 32)) in ascending order, chunk c's from members[chunk_base[c]] (k_where_members)
frz_status frz_launch_where_members(const uint32_t* bits, uint64_t n, const uint64_t* chunk_base, uint32_t* members, cudaStream_t stream);
// frz_subset_where_batch (host.cu; FrzWhereBatchDev is where_plan.cuh's)
struct FrzWhereBatchDev;
struct FrzWhereBatchQuery;
// where.cu: every query's bits and chunk counts (k_where_batch)
frz_status frz_launch_where_batch(const FrzWhereBatchDev& b, cudaStream_t stream);
// where.cu: the member list of every query j with totals[j] > 0 (k_where_members_batch)
frz_status frz_launch_where_members_batch(const FrzWhereBatchQuery* queries, const unsigned long long* totals, uint64_t n, uint32_t q,
                                          cudaStream_t stream);

// frz_subset_match (host.cu; FrzSubsetFoldDev is subset_match_plan.cuh's)
struct FrzSubsetFoldDev;
// subset_match.cu: one fold step into f.bits, and the chunk counts when f.chunk_count is set (k_subset_fold)
frz_status frz_launch_subset_fold(const FrzSubsetFoldDev& f, cudaStream_t stream);

// frz_boost_where and frz_boost_where_batch (host.cu; FrzBoostBatchDev is boost_plan.cuh's)
struct FrzBoostBatchDev;
// boost_where.cu: every query's values and b.max (k_boost_where)
frz_status frz_launch_boost_where(const FrzBoostBatchDev& b, cudaStream_t stream);

// The ordered call (host.cu, DESIGN.md §4.15; the key and the pick are order_plan.cuh's), all asynchronous on `stream`.
// order.cu: zero *st, then the key of each of the *n_ptr list rows (n_cap bounds it) → keys, and st's n and bit masks
frz_status frz_launch_order_keys(const FrzMatchDev* list, const unsigned long long* n_ptr, uint64_t n_cap, const FrzOrderDev& o,
                                 FrzOrderKey* keys, FrzOrderState* st, cudaStream_t stream, FrzLaunchStats* ls);
// order.cu: the select of the `need` rows of largest key among the n = st->n list rows, over the digits shifts[0 ..
// n_shifts) (most significant first; frz_order_digits), as frz_order_pick with `fit`: their positions → sel, their number
// → st->n_sel.  hist: zero; cand: 2 * n entries.
frz_status frz_launch_order_select(const FrzOrderKey* keys, FrzOrderState* st, uint32_t* hist, uint32_t* cand, uint32_t* sel,
                                   uint64_t n, uint64_t need, const uint32_t* shifts, uint32_t n_shifts, uint64_t fit,
                                   cudaStream_t stream, FrzLaunchStats* ls);
// order.cu: the *n_ptr (<= kFrzOrderBlockRows) rows at positions sel[..] of list (sel null: positions 0 ..) sorted by key
// in one block; the first `limit` → out
frz_status frz_launch_order_sort_block(const FrzMatchDev* list, const FrzOrderKey* keys, const uint32_t* sel,
                                       const unsigned long long* n_ptr, uint32_t limit, FrzMatchDev* out, cudaStream_t stream,
                                       FrzLaunchStats* ls);
// order.cu: out[j] = list[sel[j]] for j < *n_ptr (<= n_cap)
frz_status frz_launch_order_gather(const FrzMatchDev* list, const uint32_t* sel, const unsigned long long* n_ptr, uint64_t n_cap,
                                   FrzMatchDev* out, cudaStream_t stream, FrzLaunchStats* ls);
// sort.cu: the *n_ptr rows at d_in sorted by descending order key, LSD over shifts[0 .. n_shifts) in reverse (n_shifts >= 1,
// every digit in which two rows differ); the first `limit` land in d_out.  d_tmp: scratch of the same size.
frz_status frz_launch_sort_by_order_dev(const FrzMatchDev* d_in, FrzMatchDev* d_tmp, FrzMatchDev* d_out, const unsigned long long* n_ptr,
                                        const FrzOrderDev& o, const uint32_t* shifts, uint32_t n_shifts, FrzSortScratch& ss,
                                        cudaStream_t stream, FrzLaunchStats* st, uint32_t limit = kFrzNoLimit);

// The fill of frz_attr_rank (host.cu, DESIGN.md §4.17; the key rules are rank_plan.cuh's).  A segment is a run of rows
// whose tuples agree so far, named by its first position in the final order.
struct FrzRankKeyDev {
    FrzCorpusView text;          // a text key: the corpus whose haystacks are the key
    const int64_t* values;       // an attribute key: values[i] for i < n_values, null past them
    uint64_t n_values;
    uint32_t is_text;
    uint32_t desc;
    uint32_t fold;
    uint32_t pad_;
};
struct FrzRankDev {
    FrzRankKeyDev keys[4];       // FRZ_RANK_MAX_KEYS
    uint32_t n_keys;
    uint32_t any_text;
    uint64_t n;                  // rows of C
    const uint32_t* slot_meta;   // C's slots: the rows live in C
    const uint16_t* slot_of;
    uint32_t* seg_of;            // [n] the row's segment, kFrzRankNone: not ranked
    uint32_t* at_row;            // [n] the place in the tuple (rank_plan.cuh) of the row's chunk this round
    FrzOrderKey* keys_row;       // [n] the row's sort key this round (frz_rank_sort_key)
    uint2* segs;                 // [n] by segment: one of its rows, and the place of its next chunk
    uint32_t* skip;              // [n] by segment: the bytes its rows share from that place (text keys), kFrzRankNone: unknown
    uint32_t* heads;             // [ceil(n / 32)] bit p: a finished segment starts at position p
    unsigned long long* state;   // rows of the list of even rounds, of odd rounds, then the OR of the keys (hi, lo) and of
                                 // their complements (hi, lo)
};
// rank.cu, all asynchronous on `stream`.  init: the ranked rows → list (their number → state[0], which must be zero),
// seg_of, the first segment.  round: the rows' skips (text keys) and chunks, *n_ptr listed rows (<= n_cap); state[2 ..
// 6) must be zero.  split: the sorted rows' new segments; the rows still to refine → next, their number → *n_next (zero).
frz_status frz_launch_rank_init(const FrzRankDev& d, FrzMatchDev* list, cudaStream_t stream);
frz_status frz_launch_rank_round(const FrzRankDev& d, const FrzMatchDev* list, const unsigned long long* n_ptr, uint64_t n_cap,
                                 cudaStream_t stream);
frz_status frz_launch_rank_split(const FrzRankDev& d, const FrzMatchDev* sorted, const unsigned long long* n_ptr, uint64_t n_cap,
                                 FrzMatchDev* next, unsigned long long* n_next, cudaStream_t stream);
// rank.cu: per 1024 positions of the m ranked rows, the heads before each bitmap word (word_pref) and their total
// (chunk_count); then, with chunk_base the exclusive scan of chunk_count, value[i] for the n rows of C
frz_status frz_launch_rank_heads(const uint32_t* heads, uint64_t m, uint32_t* word_pref, uint32_t* chunk_count, cudaStream_t stream);
frz_status frz_launch_rank_write(const uint32_t* seg_of, uint64_t n, const uint32_t* heads, const uint32_t* word_pref,
                                 const uint64_t* chunk_base, int64_t* values, cudaStream_t stream);
// sort.cu: frz_launch_sort_by_order_dev for a round of frz_attr_rank: the *n_ptr rows at d_in (index = row) sorted by
// descending keys[row], LSD over shifts[0 .. n_shifts) in reverse (n_shifts >= 1)
frz_status frz_launch_sort_by_rank_dev(const FrzMatchDev* d_in, FrzMatchDev* d_tmp, FrzMatchDev* d_out, const unsigned long long* n_ptr,
                                       const FrzOrderKey* keys, const uint32_t* shifts, uint32_t n_shifts, FrzSortScratch& ss,
                                       cudaStream_t stream, FrzLaunchStats* st);

// k-way merge of per-shard runs (merge.cu) with caller-owned scratch — one per concurrent user (parallel.cu: one per rank)
#define FRZ_MERGE_MAX_RUNS 64
struct FrzMergeScratch {
    FrzSortScratch sort;                      // of the concatenate-and-sort fallback
    FrzDevArray<uint32_t> tables;             // pos0 / gt tables of the scatter merge (merge_plan.cuh)
    FrzDevArray<FrzMatchDev> cat;
    FrzDevArray<FrzMatchDev> tmp;
    FrzDevArray<unsigned long long> d_total;
};
frz_status frz_merge_runs_ex(FrzMergeScratch& ms, const FrzMatchDev* runs, uint64_t run_stride, const uint64_t* run_counts_host,
                             int n_runs, uint8_t sort, uint32_t score_bound, FrzMatchDev* d_out, cudaStream_t stream);
// The merge's scatter over one piece per run (k_merge_scatter): piece q is run q's elements [a[q], a[q] + n[q]) at src + src[q],
// stored at their merged positions minus lo.  The whole merge passes whole runs and lo = 0, the slice exchange its pieces.
struct FrzMergePieces {
    uint64_t src[FRZ_MERGE_MAX_RUNS];
    uint32_t n[FRZ_MERGE_MAX_RUNS];
    uint32_t a[FRZ_MERGE_MAX_RUNS];
    uint32_t lo;
};
frz_status frz_launch_merge_scatter(const FrzMatchDev* src, const FrzMergePieces& pieces, int n_runs, const uint32_t* tables, int bins,
                                    int blocks_per_sm, FrzMatchDev* out, cudaStream_t stream);

// Matcher internals the multi-GPU layer needs (host.cu)
uint64_t frz_matcher_epoch(const frz_matcher* m);                  // changes whenever the compiled patterns change
uint8_t frz_matcher_sort(const frz_matcher* m);
// After a match_list / shard call: the per-score "how many matches score higher" table of the run just produced (device
// pointer, valid until the next call on m) and its length; bins = 0 when the run was not ordered by a single-pass score sort.
const uint32_t* frz_matcher_last_sort_table(const frz_matcher* m, int* bins);
// event recorded when that table became final (before the sort's scatter kernel), or nullptr
cudaEvent_t frz_matcher_table_event(const frz_matcher* m);
// host Arrow buffers → the matcher's reusable packed corpus (the ingest half of frz_match_list_host_arrow)
frz_status frz_matcher_ingest_e2e(frz_matcher* m, const uint8_t* bytes, const void* offsets, int offset_width, uint64_t n, int device,
                                  const frz_corpus** out);
// frz_match_shard_device that writes only the first `limit` elements of the run (top-K calls; *d_count is the full count)
frz_status frz_match_shard_device_top(frz_matcher* m, const frz_corpus* shard, uint32_t index_offset, frz_match* d_out, uint64_t cap,
                                      uint64_t* d_count, void* stream, uint32_t limit);
// frz_matcher_ingest_e2e + frz_match_shard_device in one pass: the match pipeline runs over consecutive tile ranges as their
// H2D chunks land (prefilter → scan with carry → scoring append to one list), only the sort waits for the last chunk.
frz_status frz_match_shard_streamed(frz_matcher* m, const uint8_t* bytes, const void* offsets, int offset_width, uint64_t n, int device,
                                    uint32_t index_offset, frz_match* d_out, uint64_t cap, uint64_t* d_count, void* stream);
