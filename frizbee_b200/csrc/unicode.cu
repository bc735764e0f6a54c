// unicode.cu — the unicode-needle path on the packed corpus (SURVEY.md §8(f) rank 4).
//
// Reference replaced: MatcherImpl::match_list_into_impl with UNICODE = true (src/matcher/algo.rs:78-103):
// length gate → Prefilter::match_haystack_unicode* → trim_haystack → SmithWaterman::score_haystack_unicode →
// exact flag; and LiteralImpl::match_list_impl::<true> (src/literal/algo.rs:84-116) for the literal modes.
// The algorithms are in unicode_path.cuh (shared with the CPU test build); this file is the kernel around them.
// Two stages, like the byte path: the streaming SIGNATURE scan (prefilter.cu: k_sig_scan, 12 bytes per haystack) rejects
// every haystack that cannot hold the needle's ASCII scalars up to the typo budget without reading its bytes — the
// signature classes fold ASCII case, and a needle's ASCII scalars can only be matched by the same ASCII letter in
// either case, so the byte-path argument (DESIGN.md §3) carries over with the non-ASCII scalars simply not counted
// (host.cu: compile_pattern) — and k_unicode then takes the surviving CANDIDATE RECORDS, one thread per candidate,
// through prefilter → trim → per-scalar Smith-Waterman and emits a literal-style survivor record (score, exact), which
// the common tail (tile rank/scan → k_emit_literal → sort) places in index order.  The per-candidate code is the
// restated reference (local arrays, one global scratch row block per thread), not a register-row kernel.
#include "frz_device.cuh"
#include "frz_host.h"
#include "unicode_path.cuh"

namespace {

constexpr int kUThreads = 128;

using PackedHay = FrzPackedHay;

__global__ void __launch_bounds__(kUThreads) k_unicode(const FrzCorpusView cv, const __grid_constant__ FrzPatternDev pat,
                                                       const __grid_constant__ FrzUNeedle un, const FrzUScoring usc,
                                                       const FrzMatchDev* __restrict__ cand, unsigned long long n_cand,
                                                       const uint4* __restrict__ recs, unsigned long long recs_cap,
                                                       uint32_t index_offset, const FrzSurvLists lists, unsigned long long surv_cap,
                                                       uint32_t* __restrict__ surv_bitmap, FrzCounters* __restrict__ ctr,
                                                       uint16_t* __restrict__ scratch, uint32_t scratch_stride) {
    const unsigned long long tid = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long nthreads = (unsigned long long)gridDim.x * blockDim.x;
    uint16_t* my_scratch = scratch + tid * scratch_stride;
    // work list: the candidate records of k_sig_scan (whole-corpus call), or a match list (multi-pattern candidate mode)
    const unsigned long long total = cand ? n_cand : min(ctr->cand_count, recs_cap);
    const int max_typos = pat.typo_mode == FRZ_T_NONE ? -1 : pat.typo_mode == FRZ_T_0 ? 0 : pat.typo_mode == FRZ_T_1 ? 1
                        : pat.typo_mode == FRZ_T_2 ? 2 : pat.max_typos;
    for (unsigned long long j = tid; j < total; j += nthreads) {
        uint32_t tile, slot, meta;
        const uint4* unit0;
        if (cand) {   // candidate-list mode (multi-pattern, src/matcher/multi.rs:108-120)
            const uint32_t idx = cand[j].index - index_offset;
            tile = idx >> FRZ_TILE_SHIFT;
            slot = cv.slot_of[idx];
            meta = cv.slot_meta[(uint64_t)tile * FRZ_TILE + slot];
            if (meta == FRZ_INVALID_SLOT) continue;
            const FrzGroupDesc gd = cv.groups[tile * FRZ_GROUPS_PER_TILE + (slot >> 5)];
            unit0 = cv.data + frz_slot_unit0(gd, slot & 31);
        } else {      // a candidate record: {tile << 10 | slot, len << 10 | index-in-tile, unit index of the slot's unit 0}
            const uint4 r = recs[j];
            tile = r.x >> FRZ_TILE_SHIFT;
            slot = r.x & (FRZ_TILE - 1);
            meta = r.y;
            unit0 = cv.data + (((unsigned long long)r.w << 32) | r.z);
        }
        const int len = (int)(meta >> FRZ_TILE_SHIFT);
        const uint32_t li = meta & (FRZ_TILE - 1);
        const PackedHay hay{unit0, 0};
        bool ok = false, exact = false;
        uint32_t score = 0;
        if (pat.matching != FRZ_MATCHING_FUZZY) {
            int pos = 0;
            ok = frzu::lit_find(un, usc, hay, len, pat.matching, &pos, &score);
            exact = ok && pos == 0 && un.nbytes == len;
        } else if (len >= pat.min_hay_len) {
            int start = 0, end = len;
            ok = frzu::prefilter(un, hay, len, pat.pf_lanes, max_typos, &start, &end);
            if (ok) {
                start = start > 0 ? start - 1 : 0;   // trim_haystack (src/matcher/algo.rs:331-338)
                const int W = end - start;
                const PackedHay win{hay.base, start};
                score = frzu::sw_score(un, usc, win, W, start == 0, pat.sw_lanes, pat.score_bits == 8, my_scratch);
                exact = start == 0 && end == len && W == un.nbytes;   // include_exact && needle bytes == haystack
                for (int k = 0; exact && k < W; k++) exact = win(k) == un.c[k];
                if (exact) score = (score + (uint32_t)usc.exact_bonus) & 0xffffu;
            }
        }
        if (!ok) continue;
        FrzSurvivor rec;
        rec.tile = tile;
        rec.slot_rank = slot | (li << 10);
        rec.start = score;            // literal-style record: (score, exact)
        rec.end = exact ? 1u : 0u;
        atomicOr(&surv_bitmap[(uint64_t)tile * 32 + (li >> 5)], 1u << (li & 31));
        const unsigned long long pos = atomicAdd(&ctr->class_count[FRZ_C_COLS64], 1ull);
        if (pos < surv_cap) lists.p[FRZ_C_COLS64][pos] = rec;
        else atomicOr(&ctr->error, FRZ_DEVERR_SURVIVOR_OVERFLOW);
    }
}

}  // namespace

frz_status frz_launch_unicode(const FrzCorpusView& cv, const FrzPatternDev& pat, const FrzUNeedle& un, const FrzUScoring& usc,
                              const FrzMatchDev* cand, uint64_t n_cand, uint32_t index_offset, FrzWorkspace& ws,
                              cudaStream_t stream, FrzLaunchStats* st) {
    if (cv.n_tiles == 0) return FRZ_OK;
    FRZ_CUDA_TRY(cudaMemsetAsync(ws.surv_bitmap.get(), 0, (size_t)cv.n_tiles * 32 * sizeof(uint32_t), stream));
    if (cand && n_cand == 0) return FRZ_OK;
    if (!cand) FRZ_TRY(frz_launch_sig_scan(cv, pat, ws, stream, st));   // length gate + signature test → candidate records
    const int sms = frz_sm_count();
    const uint64_t work = cand ? n_cand : (uint64_t)cv.n_tiles * FRZ_TILE;
    const uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)sms * 4, (work + kUThreads - 1) / kUThreads));
    // per-thread Smith-Waterman row state: previous-chunk rows + pending-gap-open vectors of every needle scalar
    const uint32_t stride = 2u * (uint32_t)(un.n + 1) * (uint32_t)pat.sw_lanes;
    const uint64_t need = (uint64_t)grid * kUThreads * stride;
    FRZ_TRY(ws.unicode_scratch.reserve(need));
    k_unicode<<<grid, kUThreads, 0, stream>>>(cv, pat, un, usc, cand, n_cand, ws.cand_list.get(), ws.cand_list.cap(),
                                              index_offset, ws.lists(), ws.survivor_cap(),
                                              ws.surv_bitmap.get(), ws.counters.get(), ws.unicode_scratch.get(), stride);
    FRZ_CUDA_TRY(cudaGetLastError());
    if (st) st->launches++;
    return FRZ_OK;
}
