// sw.cu — stage 2 of match_list: affine-gap Smith-Waterman score of each surviving window,
// exact flag, and the Match record written straight to its index-ordered position.
//
// Reference path replaced: MatcherImpl::smith_waterman_one (src/matcher/algo.rs:229-263) →
// SmithWaterman<B>::score_haystack (src/smith_waterman/algo/ascii.rs:10-158) with
// propagate_{8,16,32,64}_lane (src/smith_waterman/algo/ascii_gap.rs:11-105).
//
// One window per thread.  The score row lives in registers as packed signed 16-bit cells
// (2 per register) and every recurrence step is one Hopper DPX instruction:
//     diag        max(prev_shifted + delta, 0)                 VIADDMNMX.S16x2.RELU
//     up ⊔ diag   max(prev + up_pen, diag, 0)                  VIADDMNMX.S16x2.RELU
//     gap step    max(row_shifted_by_s + pen_s, row, 0)        VIADDMNMX.S16x2.RELU
// (u8x4 SIMD-in-register intrinsics compile to 5-8 instruction emulations on sm_90a; the 16x2
// DPX forms are single instructions — see DESIGN.md §4.2.)
//
// The reference's result depends on its SIMD width: the horizontal gap propagation is a log-step
// doubling scan over LANES-cell chunks.  The kernel is templated on that LANES and evaluates the
// matrix row-major (bit-identical to the reference's chunk-major order: every (row, chunk) block
// depends only on (row-1, chunk), the last lane of (row-1, chunk-1) and (row, chunk-1)).
// Lanes past the end of the window hold zero bytes and are scanned and max-ed like real lanes,
// exactly as in the reference (zero-filled tail loads, src/smith_waterman/backend/scalar.rs:78-85).
//
// u8 and u16 reference families share this kernel: u8 cell values are exact in 16-bit lanes as
// long as no u8 add can wrap; when the host cannot prove that (pat.wrap8) the WRAP8 variant
// re-applies the 8-bit wrap after every add.
#include "frz_device.cuh"
#include <cuda_pipeline.h>
#include <stdlib.h>

#include "frz_host.h"
#include "sw_core.cuh"
#include "sw_generic.cuh"

namespace {

using namespace frzsw;
template <int LANES, bool WRAP8>
constexpr int kSw64MinBlocks = kSw64RowsInSmem<LANES, WRAP8> ? 3 : 2;

struct FrzRankView {
    const uint64_t* tile_out_base;
    const uint32_t* surv_bitmap;
    const uint16_t* word_prefix;
};
FrzRankView rank_view(const FrzWorkspace& ws) { return FrzRankView{ws.tile_out_base, ws.surv_bitmap, ws.word_prefix}; }


// decoded window record (FrzSurvivor, window-class layout)
struct WindowRec {
    uint64_t addr;      // unit index of the first unit of the window
    uint32_t startlo;   // window start inside that unit
    int W;
    bool start0, full_end;
};
__device__ __forceinline__ WindowRec decode_window(const FrzSurvivor& rec) {
    WindowRec r;
    r.addr = ((uint64_t)(rec.end & 0xffu) << 32) | rec.start;
    r.startlo = (rec.end >> 8) & 15u;
    r.W = (int)((rec.slot_rank >> 20) & 0xffu);
    r.full_end = ((rec.slot_rank >> 28) & 1u) != 0;
    r.start0 = ((rec.slot_rank >> 29) & 1u) != 0;
    return r;
}
__device__ __forceinline__ int window_units(const WindowRec& r) { return r.W > 0 ? (int)((r.startlo + r.W - 1) >> 4) + 1 : 0; }


// Output position of a survivor: its tile's base + its rank among the tile's survivors in index order (from
// the survivor bitmap).  Independent of the score, so callers request it before the DP and use it after.
__device__ __forceinline__ uint64_t match_position(const FrzSurvivor& rec, bool reversed, const FrzRankView& rv,
                                                   const FrzCounters* __restrict__ ctr) {
    const uint32_t li = (rec.slot_rank >> 10) & 0x3ff;
    const uint64_t wi = (uint64_t)rec.tile * 32 + (li >> 5);
    const uint32_t rank = rv.word_prefix[wi] + __popc(rv.surv_bitmap[wi] & ((1u << (li & 31)) - 1));
    uint64_t pos = rv.tile_out_base[rec.tile] + rank;
    if (reversed) pos = ctr->total - 1 - pos;
    return pos;
}
__device__ __forceinline__ void store_match(const FrzSurvivor& rec, uint64_t pos, uint32_t score, bool exact, uint32_t index_offset,
                                            FrzMatchDev* __restrict__ out) {
    const uint32_t li = (rec.slot_rank >> 10) & 0x3ff;
    FrzMatchDev m;
    m.index = index_offset + rec.tile * FRZ_TILE + li;
    m.score = (uint16_t)score;
    m.exact = exact ? 1 : 0;
    m.pad = 0;
    out[pos] = m;
}
__device__ __forceinline__ void emit_match(const FrzSurvivor& rec, uint32_t score, bool exact, uint32_t index_offset,
                                           bool reversed, const FrzRankView& rv,
                                           const FrzCounters* __restrict__ ctr, FrzMatchDev* __restrict__ out) {
    store_match(rec, match_position(rec, reversed, rv, ctr), score, exact, index_offset, out);
}

// One survivor whose window units are in registers: score it, write the Match at its index-ordered position.
template <int LANES, int COLS, bool WRAP8, int CC, int VAR = 0>
__device__ __forceinline__ uint32_t score_window(const FrzPatternDev& pat, const FrzSurvivor& rec, const WindowRec& wr,
                                                 const uint4 (&u)[(CC + 15) / 16 + 1], const FrzRankView& rv,
                                                 const FrzCounters* __restrict__ ctr, uint32_t index_offset, int reversed,
                                                 FrzMatchDev* __restrict__ out, uint32_t* sw_smem) {
    const uint64_t pos = match_position(rec, reversed != 0, rv, ctr);   // loads overlap the DP
    uint32_t hw[CC / 4];
    window_from_units<CC>(u, wr.startlo, wr.W, hw);
    uint32_t score = SwCore<LANES, COLS, WRAP8, VAR, CC>::run(hw, wr.W, pat, wr.start0, sw_smem);
    bool exact = wr.start0 && wr.full_end && window_equals_needle(hw, wr.W, pat);
    if (exact) score = (score + pat.exact_bonus) & 0xffffu;
    store_match(rec, pos, score, exact, index_offset, out);
    return score;
}

// Same, loading the units straight from the packed corpus.
template <int LANES, int COLS, bool WRAP8, int CC, int VAR = 0>
__device__ __forceinline__ uint32_t score_survivor(const FrzCorpusView& cv, const FrzPatternDev& pat, const FrzSurvivor& rec,
                                                   const FrzRankView& rv, const FrzCounters* __restrict__ ctr, uint32_t index_offset,
                                                   int reversed, FrzMatchDev* __restrict__ out, uint32_t* sw_smem) {
    constexpr int NU = (CC + 15) / 16 + 1;
    const WindowRec wr = decode_window(rec);
    const int nu = window_units(wr);
    const uint4* base = cv.data + wr.addr;
    uint4 u[NU];
#pragma unroll
    for (int k = 0; k < NU; k++) {
        u[k] = make_uint4(0, 0, 0, 0);
        if (k < nu) u[k] = __ldg(base + k);
    }
    return score_window<LANES, COLS, WRAP8, CC, VAR>(pat, rec, wr, u, rv, ctr, index_offset, reversed, out, sw_smem);
}

// Windows of 65..128 bytes: one window per thread, score rows in shared memory, survivors strided over a
// persistent grid.
template <int LANES, int COLS, bool WRAP8, int VAR = 0>
__global__ void __launch_bounds__(kSwThreads) k_sw(const FrzCorpusView cv, const __grid_constant__ FrzPatternDev pat,
                                                   const FrzSurvivor* __restrict__ surv, unsigned long long surv_cap, int cls,
                                                   const FrzRankView rv, FrzCounters* __restrict__ ctr,
                                                   uint32_t index_offset, int reversed, FrzMatchDev* __restrict__ out) {
    extern __shared__ __align__(16) uint32_t sw_smem[];
    const unsigned long long count = min(ctr->class_count[cls], surv_cap);
    uint32_t local_max = 0;
    for (unsigned long long j = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; j < count;
         j += (unsigned long long)gridDim.x * blockDim.x) {
        const FrzSurvivor rec = surv[j];
        local_max = max(local_max, score_survivor<LANES, COLS, WRAP8, COLS, VAR>(cv, pat, rec, rv, ctr, index_offset, reversed, out, sw_smem));
    }
    local_max = __reduce_max_sync(0xffffffffu, local_max);
    if (frz_lane() == 0 && local_max) atomicMax(&ctr->max_score, local_max);
}

// Windows of <= 64 bytes: the four column classes (CC64 first: longest items first) share one persistent
// kernel.  A work item is 32 consecutive survivors of one class; warps claim items from a device counter, so
// the load balances itself and the only tail is the last item of each warp.
//
// The kernel is issue-bound (three warps per scheduler for LANES 64), so every exposed load latency costs: the loop is
// software-pipelined two items deep.  While item i is being scored, item i+1's window units travel
// global → shared with cp.async (no registers held) and item i+2's records are in flight.
constexpr int kSw64Units = 5;  // 16-byte units a <= 64-byte window can straddle
struct Sw64Stage {
    uint4 units[kSw64Units][kSwThreads];  // [k][thread]: conflict-free 16-byte columns
};

template <int LANES, bool WRAP8, int VAR = 0>
__global__ void __launch_bounds__(kSwThreads, (kSw64MinBlocks<LANES, WRAP8>)) k_sw64(const FrzCorpusView cv, const __grid_constant__ FrzPatternDev pat,
                                                     const FrzSurvLists lists, unsigned long long surv_cap,
                                                     const FrzRankView rv, FrzCounters* __restrict__ ctr,
                                                     uint32_t index_offset, int reversed, FrzMatchDev* __restrict__ out) {
    __shared__ Sw64Stage stage;
    __shared__ __align__(16) uint32_t rows_smem[kSw64RowsInSmem<LANES, WRAP8> ? 2 * 32 * kSwThreads : 1];
    const uint32_t lane = frz_lane();
    unsigned long long cnt[4];
    uint32_t items_end[4];   // cumulative item counts in processing order CC64, CC56, CC48, CC40
    {
        uint32_t acc = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            cnt[k] = min(ctr->class_count[FRZ_C_COLS64 - k], surv_cap);
            acc += (uint32_t)((cnt[k] + 31) >> 5);
            items_end[k] = acc;
        }
    }
    const uint32_t n_items = items_end[3];
    const uint32_t opaque_zero = ctr->pad_;   // always 0 (the counters are zeroed before every call)
    // work-item claim, split so that the atomic's round trip overlaps a whole DP: `claim_issue` returns lane 0's
    // raw ticket (other lanes: garbage) and `claim_get` broadcasts it one iteration later
    auto claim_issue = [&]() {
        uint32_t t = 0xFFFFFFFFu;
        // ptxas rewrites an atomic add on a warp-uniform address into its warp-aggregated form, whose trailing
        // SHFL waits for the atomic right here.  Offsetting the address by tid.x * (a zero it cannot see through)
        // makes the address formally lane-dependent: the atomic is left alone and its result stays in flight.
        if (lane == 0)
            asm volatile("{ .reg .u32 x; .reg .u64 a, o;\n"
                         "  mov.u32 x, %%tid.x; mul.lo.u32 x, x, %2; mul.wide.u32 o, x, 4; add.u64 a, %1, o;\n"
                         "  atom.global.add.u32 %0, [a], 1; }"
                         : "=r"(t) : "l"(&ctr->sw_next), "r"(opaque_zero) : "memory");
        return t;
    };
    auto claim_get = [&](uint32_t ticket) { return __shfl_sync(0xffffffffu, ticket, 0); };
    auto class_of = [&](uint32_t item) { return item < items_end[0] ? 0 : item < items_end[1] ? 1 : item < items_end[2] ? 2 : 3; };
    // this lane's record of `item` (tile = 0xFFFFFFFF when the lane has none)
    auto load_rec = [&](uint32_t item) {
        FrzSurvivor rec;
        rec.tile = 0xFFFFFFFFu; rec.slot_rank = 0; rec.start = 0; rec.end = 0;
        if (item < n_items) {
            const int k = class_of(item);
            const uint32_t first = k == 0 ? 0u : k == 1 ? items_end[0] : k == 2 ? items_end[1] : items_end[2];
            const unsigned long long cnt_k = k == 0 ? cnt[0] : k == 1 ? cnt[1] : k == 2 ? cnt[2] : cnt[3];
            const unsigned long long j = (unsigned long long)(item - first) * 32 + lane;
            const FrzSurvivor* list = k == 0 ? lists.p[FRZ_C_COLS64] : k == 1 ? lists.p[FRZ_C_CC56] : k == 2 ? lists.p[FRZ_C_CC48] : lists.p[FRZ_C_CC40];
            if (j < cnt_k) rec = list[j];
        }
        return rec;
    };
    // stage the window units of `rec` into this thread's shared-memory column
    auto stage_units = [&](const FrzSurvivor& rec) {
        if (rec.tile != 0xFFFFFFFFu) {
            const WindowRec wr = decode_window(rec);
            const int nu = window_units(wr);
            const uint4* base = cv.data + wr.addr;
#pragma unroll
            for (int k = 0; k < kSw64Units; k++)
                if (k < nu) __pipeline_memcpy_async(&stage.units[k][threadIdx.x], base + k, 16);
        }
        __pipeline_commit();
    };

    uint32_t local_max = 0;
    // pipeline: item0 = being scored (units staged), item1 = records in registers, item2 = ticket in flight
    uint32_t item0 = claim_get(claim_issue()), item1 = claim_get(claim_issue());
    uint32_t ticket2 = claim_issue();
    FrzSurvivor rec0 = load_rec(item0);
    stage_units(rec0);
    FrzSurvivor rec1 = load_rec(item1);
    while (item0 < n_items) {
        // units of item0 have landed → registers
        __pipeline_wait_prior(0);
        const WindowRec wr = decode_window(rec0);
        const int nu = window_units(wr);
        uint4 u[kSw64Units];
#pragma unroll
        for (int k = 0; k < kSw64Units; k++) {
            u[k] = make_uint4(0, 0, 0, 0);
            if (k < nu && rec0.tile != 0xFFFFFFFFu) u[k] = stage.units[k][threadIdx.x];
        }
        // next item's units start moving; the ticket taken one iteration ago becomes item2, whose records are
        // requested now; a new ticket is taken for the iteration after
        stage_units(rec1);
        const uint32_t item2 = claim_get(ticket2);
        ticket2 = claim_issue();
        const FrzSurvivor rec2 = load_rec(item2);
        if (rec0.tile != 0xFFFFFFFFu) {
            const int k = class_of(item0);
            uint32_t sc;
            if (k == 0) {
                sc = score_window<LANES, 64, WRAP8, 64, VAR>(pat, rec0, wr, u, rv, ctr, index_offset, reversed, out, rows_smem);
            } else if (k == 1) {
                sc = score_window<LANES, 64, WRAP8, 56, VAR>(pat, rec0, wr, u, rv, ctr, index_offset, reversed, out, rows_smem);
            } else if (k == 2) {
                const uint4 (&u4)[4] = reinterpret_cast<const uint4 (&)[4]>(u);
                sc = score_window<LANES, 64, WRAP8, 48, VAR>(pat, rec0, wr, u4, rv, ctr, index_offset, reversed, out, rows_smem);
            } else {
                const uint4 (&u4)[4] = reinterpret_cast<const uint4 (&)[4]>(u);
                sc = score_window<LANES, 64, WRAP8, 40, VAR>(pat, rec0, wr, u4, rv, ctr, index_offset, reversed, out, rows_smem);
            }
            local_max = max(local_max, sc);
        }
        item0 = item1; rec0 = rec1;
        item1 = item2; rec1 = rec2;
    }
    __pipeline_wait_prior(0);
    local_max = __reduce_max_sync(0xffffffffu, local_max);
    if (lane == 0 && local_max) atomicMax(&ctr->max_score, local_max);
}

// ---- generic fallback: windows of 129..1024 bytes (row-major, local-memory rows) and the greedy scorer for
// ---- windows > 1024 (sw_generic.cuh).  One window per thread.
__device__ __forceinline__ uint32_t hay_byte(const uint4* base, uint32_t i) {
    return (reinterpret_cast<const uint32_t*>(base)[i >> 2] >> ((i & 3) * 8)) & 0xff;
}
// byte i of the window that starts at byte `start` of the haystack at `base`
struct GenericHay {
    const uint4* base;
    uint32_t start;
    __device__ __forceinline__ uint32_t operator()(int i) const { return hay_byte(base, start + i); }
};

__global__ void __launch_bounds__(64) k_sw_generic(const FrzCorpusView cv, const __grid_constant__ FrzPatternDev pat,
                                                   const FrzSurvivor* __restrict__ surv, unsigned long long surv_cap, int cls,
                                                   const FrzRankView rv, FrzCounters* __restrict__ ctr,
                                                   uint32_t index_offset, int reversed, FrzMatchDev* __restrict__ out) {
    const unsigned long long count = min(ctr->class_count[cls], surv_cap);
    uint32_t local_max = 0;
    for (unsigned long long j = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; j < count;
         j += (unsigned long long)gridDim.x * blockDim.x) {
        const FrzSurvivor rec = surv[j];
        const uint32_t slot = rec.slot_rank & 0x3ff;
        const uint32_t start = rec.start, end = rec.end & 0x7fffffffu;
        const bool full_end = (rec.end >> 31) != 0;
        const int W = (int)(end - start);
        const uint4* base = frz_unit_ptr(cv, rec.tile, slot, 0);
        const bool include_prefix = start == 0;
        const GenericHay hay{base, start};
        uint32_t score;
        if (W > FRZ_SW_MAX_WINDOW) {
            int g = greedy_score(hay, W, pat, include_prefix);
            score = g < 0 ? 0u : (uint32_t)g;
        } else {
            score = generic_score(hay, W, pat, include_prefix);
        }
        bool exact = false;
        if (start == 0 && full_end && W == pat.n) {
            exact = true;
            for (int k = 0; k < pat.n; k++) exact = exact && hay_byte(base, k) == pat.c[k];
        }
        if (exact) score = (score + pat.exact_bonus) & 0xffffu;
        emit_match(rec, score, exact, index_offset, reversed != 0, rv, ctr, out);
        local_max = max(local_max, score);
    }
    if (local_max) atomicMax(&ctr->max_score, local_max);
}

// literal patterns: the prefilter stage already produced (score, exact); just place the match
__global__ void __launch_bounds__(256) k_emit_literal(const FrzSurvivor* __restrict__ surv, unsigned long long surv_cap,
                                                      const FrzRankView rv, FrzCounters* __restrict__ ctr,
                                                      uint32_t index_offset, int reversed, FrzMatchDev* __restrict__ out) {
    const unsigned long long count = min(ctr->class_count[FRZ_C_COLS64], surv_cap);
    uint32_t local_max = 0;
    for (unsigned long long j = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; j < count;
         j += (unsigned long long)gridDim.x * blockDim.x) {
        const FrzSurvivor rec = surv[j];
        emit_match(rec, rec.start, rec.end != 0, index_offset, reversed != 0, rv, ctr, out);
        local_max = max(local_max, rec.start);
    }
    if (local_max) atomicMax(&ctr->max_score, local_max);
}

template <int LANES>
frz_status launch_sw_lanes(const FrzCorpusView& cv, const FrzPatternDev& pat, uint32_t index_offset, bool reversed,
                           FrzWorkspace& ws, FrzMatchDev* d_out, cudaStream_t stream) {
    // persistent grids: a multiple of the SM count
    const int blocks = frz_sm_count() * 2;
    const int rev = reversed ? 1 : 0;
    // VAR 8: the per-column bonus is classified on the packed window bytes (SwCore) rather than per 16-bit lane.
    // kSwVarLanePen: gap_extend == 0 < gap_open_x, whose penalties the default IMAD form gets wrong (SwCore).
    const bool lane_pen = !pat.wrap8 && pat.gap_extend == 0 && pat.gap_open_x > 0;
    if (pat.wrap8)
        k_sw64<LANES, true><<<frz_sm_count() * kSw64MinBlocks<LANES, true>, kSwThreads, 0, stream>>>(
            cv, pat, ws.lists(), ws.survivor_cap, rank_view(ws), ws.counters, index_offset, rev, d_out);
    else if (lane_pen)
        k_sw64<LANES, false, 8 | kSwVarLanePen><<<frz_sm_count() * kSw64MinBlocks<LANES, false>, kSwThreads, 0, stream>>>(
            cv, pat, ws.lists(), ws.survivor_cap, rank_view(ws), ws.counters, index_offset, rev, d_out);
    else
        k_sw64<LANES, false, 8><<<frz_sm_count() * kSw64MinBlocks<LANES, false>, kSwThreads, 0, stream>>>(
            cv, pat, ws.lists(), ws.survivor_cap, rank_view(ws), ws.counters, index_offset, rev, d_out);
    // windows of 65..128 bytes only exist when some haystack of the corpus is longer than 64 bytes (recorded at pack time)
    if (cv.max_gunits <= 4) { FRZ_CUDA_TRY(cudaGetLastError()); return FRZ_OK; }
    const size_t smem = SwCore<LANES, 128, false>::smem_bytes;
    static bool attr_set_dev[64] = {};   // function attributes are per device
    bool& attr_set = attr_set_dev[frz_current_device() & 63];
    if (!attr_set) {
        FRZ_CUDA_TRY(cudaFuncSetAttribute(k_sw<LANES, 128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        FRZ_CUDA_TRY(cudaFuncSetAttribute(k_sw<LANES, 128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        FRZ_CUDA_TRY(cudaFuncSetAttribute(k_sw<LANES, 128, false, kSwVarLanePen>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set = true;
    }
    if (pat.wrap8)
        k_sw<LANES, 128, true><<<blocks, kSwThreads, smem, stream>>>(cv, pat, ws.survivors[FRZ_C_COLS128], ws.survivor_cap, FRZ_C_COLS128,
                                                                    rank_view(ws), ws.counters, index_offset, rev, d_out);
    else if (lane_pen)
        k_sw<LANES, 128, false, kSwVarLanePen><<<blocks, kSwThreads, smem, stream>>>(cv, pat, ws.survivors[FRZ_C_COLS128], ws.survivor_cap,
                                                                                  FRZ_C_COLS128, rank_view(ws), ws.counters, index_offset,
                                                                                  rev, d_out);
    else
        k_sw<LANES, 128, false><<<blocks, kSwThreads, smem, stream>>>(cv, pat, ws.survivors[FRZ_C_COLS128], ws.survivor_cap, FRZ_C_COLS128,
                                                                     rank_view(ws), ws.counters, index_offset, rev, d_out);
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

}  // namespace

frz_status frz_launch_sw(const FrzCorpusView& cv, const FrzPatternDev& pat, uint32_t index_offset, bool reversed,
                         FrzWorkspace& ws, FrzMatchDev* d_out, cudaStream_t stream, FrzLaunchStats* st) {
    if (cv.n_tiles == 0) return FRZ_OK;
    if (pat.typo_mode == FRZ_T_LITERAL) {
        k_emit_literal<<<frz_sm_count() * 4, 256, 0, stream>>>(ws.survivors[FRZ_C_COLS64], ws.survivor_cap, rank_view(ws), ws.counters,
                                                           index_offset, reversed ? 1 : 0, d_out);
        FRZ_CUDA_TRY(cudaGetLastError());
        if (st) st->launches++;
        return FRZ_OK;
    }
    switch (pat.sw_lanes) {
        case 64: FRZ_TRY(launch_sw_lanes<64>(cv, pat, index_offset, reversed, ws, d_out, stream)); break;
        case 32: FRZ_TRY(launch_sw_lanes<32>(cv, pat, index_offset, reversed, ws, d_out, stream)); break;
        case 16: FRZ_TRY(launch_sw_lanes<16>(cv, pat, index_offset, reversed, ws, d_out, stream)); break;
        case 8: FRZ_TRY(launch_sw_lanes<8>(cv, pat, index_offset, reversed, ws, d_out, stream)); break;
        default: return frz_fail(FRZ_ERR_INVALID_ARG, "unsupported lane count %d", pat.sw_lanes);
    }
    if (cv.max_gunits > 8) {   // windows > 128 bytes need a haystack > 128 bytes
        k_sw_generic<<<frz_sm_count() * 2, 64, 0, stream>>>(cv, pat, ws.survivors[FRZ_C_GENERIC], ws.survivor_cap, FRZ_C_GENERIC, rank_view(ws),
                                                        ws.counters, index_offset, reversed ? 1 : 0, d_out);
    }
    FRZ_CUDA_TRY(cudaGetLastError());
    if (st) st->launches += 1 + (cv.max_gunits > 4 ? 1 : 0) + (cv.max_gunits > 8 ? 1 : 0);
    return FRZ_OK;
}
