// frz_host.h — internal host-side declarations shared by the .cu translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/frz_cuda.h"
#include "frz_device.cuh"
#include "unicode_path.cuh"

frz_status frz_fail(frz_status s, const char* fmt, ...);
inline int frz_current_device() { int d = 0; cudaGetDevice(&d); return d; }
// SMs of the current device (cached per device): persistent grids and grid caps are multiples of it
inline int frz_sm_count() {
    static int count_dev[64] = {};
    const int d = frz_current_device();
    int& c = count_dev[d & 63];
    if (c <= 0 && (cudaDeviceGetAttribute(&c, cudaDevAttrMultiProcessorCount, d) != cudaSuccess || c <= 0)) c = 132;   // H100 SXM
    return c;
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

// Owned device buffers of a packed corpus.
struct FrzCorpusStorage {
    uint4* data = nullptr;
    uint64_t* tile_base = nullptr;
    FrzGroupDesc* groups = nullptr;
    uint32_t* slot_meta = nullptr;
    uint16_t* slot_of = nullptr;
    uint2* slot_sig = nullptr;
    uint64_t n = 0;
    uint32_t n_tiles = 0;
    uint64_t total_units = 0;
    uint64_t total_bytes = 0;
    uint32_t max_gunits = 0;   // longest haystack of the corpus in 16-byte units
    int device = 0;
    // capacities (grow-only reuse by the end-to-end path: no cudaMalloc/cudaFree per call)
    uint32_t cap_tiles = 0;
    uint64_t cap_units = 0;
    uint64_t* scratch_tile_units = nullptr;  // [cap_tiles] + 2 words (total, error)

    FrzCorpusView view() const {
        FrzCorpusView v;
        v.data = data;
        v.tile_base = tile_base;
        v.groups = groups;
        v.slot_meta = slot_meta;
        v.slot_of = slot_of;
        v.slot_sig = slot_sig;
        v.n = n;
        v.n_tiles = n_tiles;
        v.max_gunits = max_gunits;
        return v;
    }
    void release() {
        cudaFree(data); cudaFree(tile_base); cudaFree(groups); cudaFree(slot_meta); cudaFree(slot_of); cudaFree(slot_sig); cudaFree(scratch_tile_units);
        data = nullptr; tile_base = nullptr; groups = nullptr; slot_meta = nullptr; slot_of = nullptr; slot_sig = nullptr; scratch_tile_units = nullptr;
        cap_tiles = 0; cap_units = 0;
    }
};

struct FrzIngest;
struct frz_corpus {
    FrzCorpusStorage st;
    FrzIngest* ingest = nullptr;   // created by the first frz_corpus_append, kept for the next ones
};

// Staging arena + copy stream of the streamed ingest (pack.cu): grow-only, reused across calls.
struct FrzIngest {
    static constexpr int kMaxChunks = 32;
    static constexpr uint64_t kMinChunkBytes = 8ull << 20;
    uint8_t* d_bytes = nullptr;
    uint64_t bytes_cap = 0;
    void* d_offsets = nullptr;
    uint64_t offsets_cap = 0;             // bytes
    cudaStream_t copy_stream = nullptr;   // non-blocking: overlaps the (legacy default) compute stream
    cudaEvent_t ev[kMaxChunks + 1] = {};  // [c] chunk c landed; [kMaxChunks] offsets landed / arena free
    frz_status reserve(uint64_t bytes, uint64_t offset_bytes);
    void release();
};

// pack.cu
frz_status frz_pack_corpus_device(const uint8_t* d_bytes, const void* d_offsets, int offset_width, uint64_t n, uint64_t total_bytes,
                                  cudaStream_t stream, FrzCorpusStorage* out);
frz_status frz_append_host(FrzIngest& ing, const uint8_t* h_bytes, const void* h_offsets, int offset_width, uint64_t n_new,
                           cudaStream_t stream, FrzCorpusStorage* st);
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

// Per-matcher device workspace (grown on demand, reused across calls).
struct FrzWorkspace {
    int device = -1;
    FrzCounters* counters = nullptr;        // device
    FrzCounters* h_counters = nullptr;      // pinned host mirror
    unsigned long long* stream_total = nullptr;   // device: running match count of a streamed call (tile-scan carry)
    FrzSurvivor* survivors[FRZ_N_CLASSES] = {};
    FrzSurvLists lists() const { FrzSurvLists l; for (int c = 0; c < FRZ_N_CLASSES; c++) l.p[c] = survivors[c]; return l; }
    uint64_t survivor_cap = 0;              // per class
    uint32_t* surv_bitmap = nullptr;        // [n_tiles * 32] survivor bits by index-within-tile
    uint16_t* word_prefix = nullptr;        // [n_tiles * 32] exclusive popcount prefix of surv_bitmap words
    uint32_t* tile_count = nullptr;         // [n_tiles] matches per tile
    uint64_t* tile_out_base = nullptr;      // [n_tiles] exclusive scan of tile_count
    uint32_t tiles_cap = 0;
    FrzMatchDev* matches_a = nullptr;       // index-ordered matches
    FrzMatchDev* matches_b = nullptr;       // sort ping-pong / final
    uint64_t match_cap = 0;
    uint32_t* sort_hist = nullptr;          // [256 * n_sort_blocks]
    uint64_t sort_hist_cap = 0;
    uint32_t* fused_hist = nullptr;         // FrzScoreHist counts, then the per-segment prefix rows the sort's scan writes
    uint64_t fused_hist_cap = 0;            // in words
    uint64_t fused_clean_words = 0;         // leading words of fused_hist known to be zero (the scan re-zeroes what it reads)
    bool fused_hist_dirty = false;          // counts were handed to the scoring kernels, their scan was not enqueued yet
    void* cand_list = nullptr;              // k_sig_scan → k_window candidate records (16 bytes each)
    uint64_t cand_cap = 0;                  // in records
    uint32_t* retain_cnt = nullptr;         // multi-pattern stable compaction scratch
    uint64_t* retain_base = nullptr;
    uint8_t* retain_keep = nullptr;
    uint64_t retain_cap = 0;
    uint16_t* unicode_scratch = nullptr;    // unicode.cu: per-thread row state of the per-scalar Smith-Waterman
    uint64_t unicode_scratch_cap = 0;       // in uint16 elements
    cudaEvent_t table_ev = nullptr;         // recorded right after the sort's scan kernel: the per-score table is final there,
    bool arm_table_ev = false;              //   one kernel (the scatter) before the run itself (shard calls arm it)
    bool table_ev_recorded = false;
    cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    bool ev_rec[6] = {false, false, false, false, false, false};  // recorded during the current call
    void release();
};

// kernels (prefilter.cu / sw.cu / sort.cu) — all asynchronous on `stream`
struct FrzLaunchStats {
    uint64_t launches = 0;
};

frz_status frz_launch_prefilter(const FrzCorpusView& cv, const FrzPatternDev& pat, FrzWorkspace& ws, cudaStream_t stream,
                                FrzLaunchStats* st);
frz_status frz_launch_sig_scan(const FrzCorpusView& cv, const FrzPatternDev& pat, FrzWorkspace& ws, cudaStream_t stream,
                               FrzLaunchStats* st);
frz_status frz_launch_unicode(const FrzCorpusView& cv, const FrzPatternDev& pat, const FrzUNeedle& un, const FrzUScoring& usc,
                              const FrzMatchDev* cand, uint64_t n_cand, uint32_t index_offset, FrzWorkspace& ws,
                              cudaStream_t stream, FrzLaunchStats* st);
frz_status frz_launch_match_indices(const FrzCorpusView& cv, const FrzPatternDev& pat, const FrzUNeedle& un, const FrzUScoring& usc,
                                    bool unicode, const uint32_t* d_which, uint64_t n, FrzMatchDev* d_matches, uint32_t* d_idx,
                                    uint32_t stride, uint32_t* d_cnt, uint16_t* d_scratch, uint64_t scratch_stride, uint32_t threads,
                                    cudaStream_t stream);
frz_status frz_launch_prefilter_list(const FrzCorpusView& cv, const FrzPatternDev& pat, const FrzMatchDev* cand,
                                     uint64_t n_cand, uint32_t index_offset, FrzWorkspace& ws, cudaStream_t stream,
                                     FrzLaunchStats* st);
frz_status frz_launch_tile_scan(const FrzCorpusView& cv, FrzWorkspace& ws, cudaStream_t stream, FrzLaunchStats* st,
                                unsigned long long* carry = nullptr);
// hist.counts != nullptr: every emitted match also counts itself into `hist` (see FrzScoreHist)
frz_status frz_launch_sw(const FrzCorpusView& cv, const FrzPatternDev& pat, uint32_t index_offset, bool reversed,
                         FrzWorkspace& ws, FrzMatchDev* d_out, cudaStream_t stream, FrzLaunchStats* st,
                         const FrzScoreHist& hist = FrzScoreHist());
// "no limit" for the sorts' `limit` argument: every position of a list is below it (lists hold at most 2^32 - 1 matches)
constexpr uint32_t kFrzNoLimit = 0xFFFFFFFFu;
// stable sort by descending score; the element count is read from device memory (*n_ptr).
// d_tmp is only used when score_bound >= 1024 (two 8-bit passes); result always lands in d_out.
// limit: only the sorted positions below it are stored (top-K calls); kFrzNoLimit sorts the whole list.
frz_status frz_launch_sort_by_score_dev(const FrzMatchDev* d_in, FrzMatchDev* d_tmp, FrzMatchDev* d_out,
                                        const unsigned long long* n_ptr, uint32_t score_bound, FrzWorkspace& ws,
                                        cudaStream_t stream, FrzLaunchStats* st, uint32_t limit = kFrzNoLimit);
size_t frz_sort_hist_words();
frz_status frz_sort_hist_alloc(uint32_t** out);
const uint32_t* frz_sort_digit_base(const FrzWorkspace& ws);
int frz_sort_single_pass_bins(uint32_t score_bound);   // bins of the single-pass sort for this bound, 0 = two passes
// The fused single-pass sort: the scoring kernels build the histogram (frz_launch_sw with `hist`), so the sort is a scan
// and a block-per-segment scatter.  prepare: sizes and zeroes the histogram for lists of up to n_cap matches whose scores
// are below score_bound (< 1024).  The sort reads the count at *n_ptr and leaves the histogram zeroed for the next call.
frz_status frz_sort_fused_prepare(FrzWorkspace& ws, uint64_t n_cap, uint32_t score_bound, cudaStream_t stream, FrzScoreHist* out);
frz_status frz_launch_sort_fused(const FrzMatchDev* d_in, FrzMatchDev* d_out, const unsigned long long* n_ptr, const FrzScoreHist& hist,
                                 FrzWorkspace& ws, cudaStream_t stream, FrzLaunchStats* st, uint32_t limit = kFrzNoLimit);

// k-way merge of per-shard runs (host.cu) with caller-owned scratch — one per concurrent user (parallel.cu: one per rank)
#define FRZ_MERGE_MAX_RUNS 64
struct FrzMergeScratch {
    uint32_t* hist = nullptr;      // sort scratch of the concatenate-and-sort fallback
    uint32_t* tables = nullptr;    // gt / pos0 tables of the scatter merge
    FrzMatchDev* cat = nullptr;
    FrzMatchDev* tmp = nullptr;
    unsigned long long* d_total = nullptr;
    uint64_t cap = 0;
    int device = -1;
    void release();
};
frz_status frz_merge_runs_ex(FrzMergeScratch& ms, const FrzMatchDev* runs, uint64_t run_stride, const uint64_t* run_counts_host,
                             int n_runs, uint8_t sort, uint32_t score_bound, FrzMatchDev* d_out, cudaStream_t stream);

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
