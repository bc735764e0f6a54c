// prefilter.cu — stage 1 of match_list: length gate → ordered char-mask prefilter → window trim
// → survivor records.
//
// Reference path replaced (per haystack, src/matcher/algo.rs:85-100):
//     if len >= min_haystack_len { (matched,start,end) = prefilter_haystack(..); trim_haystack(..) }
// with Prefilter::match_haystack (src/prefilter/algo/ascii.rs:6-54), match_haystack_1_typo /
// _2_typos / _many_typos (src/prefilter/algo/ascii_typos.rs:15-360) and trim_haystack
// (src/matcher/algo.rs:331-338).  Literal modes (src/literal/algo.rs:234-255) are decided here too.
//
// Structure (persistent, warp-autonomous, no block barriers — the first version synchronised a
// block per tile and spent most of its issue slots waiting at barriers):
//   phase A  warp per group, lane per haystack: length gate + the byte-class SIGNATURE test (8 bytes per
//            haystack, written at pack time — pack.cu: k_pack_sig): "at most k needle bytes lack a partner
//            in this haystack", a necessary condition of every prefilter of the reference.  The haystack bytes
//            are not read for rejected haystacks.  Passing lanes queue in the warp's shared-memory ring.
//            (Rounds 1's phase A streamed every haystack byte through word-parallel probes: 0.35 of the HBM
//            roofline, ALU-issue-bound; the signature test reads 12 bytes per haystack instead of len + 8.)
//   phase B  whenever 32 candidates are queued: lane per candidate, the exact reference window
//            (chunk-emulating for k >= 1) from occurrence masks of the candidate's bytes, all lanes busy.
//   emit     survivors go to per-SW-class lists (warp-aggregated atomics) and set their bit in a
//            per-tile bitmap; k_tile_rank turns the bitmap into index-order ranks so that the
//            scoring stage can write each match straight to its index-ordered position.
#include "frz_device.cuh"
#include <cuda_pipeline.h>
#include <algorithm>
#include <type_traits>

#include "frz_host.h"
#include "indices_path.cuh"
#include "prefilter_masks.cuh"
#include "prefilter_scan.cuh"

namespace {

using namespace frzpf;

constexpr int kThreads = 128;
constexpr int kWarps = kThreads / 32;

struct GlobalAcc {
    const uint4* base;  // unit 0 of this slot; its units (and so its bytes) are contiguous
    __device__ __forceinline__ uint32_t word(uint32_t w) const { return reinterpret_cast<const uint32_t*>(base)[w]; }
};


// the block's copy of the table (first 4 * n bytes of `tab_s`); call before the block's first barrier
__device__ __forceinline__ LongPat stage_long_pat(const FrzPatternDev& p, const FrzNeedleTab* __restrict__ ntab, uint8_t* tab_s) {
    const int n = p.n;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        tab_s[i] = ntab->c[i];
        tab_s[n + i] = ntab->flip[i];
        tab_s[2 * n + i] = ntab->om[i];
        tab_s[3 * n + i] = ntab->tg[i];
    }
    LongPat l;
    l.c = tab_s; l.flip = tab_s + n; l.om = tab_s + 2 * n; l.tg = tab_s + 3 * n;
    l.n = n; l.pf_lanes = p.pf_lanes; l.sw_lanes = p.sw_lanes; l.max_typos = p.max_typos; l.matching = p.matching;
    l.col_classes = p.col_classes; l.n_distinct = 0;
    l.raw_match = p.raw_match; l.raw_case = p.raw_case; l.raw_prefix = p.raw_prefix; l.raw_cap = p.raw_cap;
    l.raw_delim = p.raw_delim; l.exact_bonus = p.exact_bonus;
    return l;
}
constexpr size_t kLongPatSmem = 4 * FRZ_LONG_NEEDLE;



struct OccTable {
    uint2 occ[kMaxDistinct][32];             // per-lane occurrence masks of the distinct needle byte classes
};

template <class P>
__device__ __forceinline__ int sw_class_of(int window, const P& pat) {
    if (window > 128) return FRZ_C_GENERIC;
    if (window > 64) return FRZ_C_COLS128;
    if (!pat.col_classes) return FRZ_C_COLS64;
    // columns whose cells can reach the score: the window, needle_len diagonal steps past its end, and never
    // more than the chunks the reference evaluates
    const int chunk_cols = (window + pat.sw_lanes - 1) / pat.sw_lanes * pat.sw_lanes;
    const int need = min(window + pat.n, chunk_cols);
    // four classes: two (48 / 64) were slower (the extra columns cost more than the smaller kernel saves)
    return need <= 40 ? FRZ_C_CC40 : need <= 48 ? FRZ_C_CC48 : need <= 56 ? FRZ_C_CC56 : FRZ_C_COLS64;
}

// Exact window of one queued candidate (phase B) + survivor emission.  All 32 lanes of the warp call
// this together (`active` lanes have an entry); emission uses warp-aggregated atomics.
// One candidate as phase B sees it.  `units` is where the mask builders read the haystack's 16-byte units from (unit k at
// units + k): the packed corpus itself, or this lane's row of a shared-memory stage filled by cp.async.
struct Cand {
    uint32_t tile, slot, li;   // li = index of the haystack inside its tile
    int len;
    const uint4* base;         // unit 0 of the slot in the packed corpus
    const uint4* units;
};
// resolves (tile, slot) through the group descriptor and the slot metadata (candidate lists of the multi-pattern path)
__device__ __forceinline__ Cand resolve_cand(const FrzCorpusView& cv, uint32_t tile, uint32_t slot, int len) {
    Cand c;
    c.tile = tile; c.slot = slot; c.len = len;
    const FrzGroupDesc gd = cv.groups[tile * FRZ_GROUPS_PER_TILE + (slot >> 5)];
    c.base = cv.data + frz_slot_unit0(gd, slot & 31);
    c.units = c.base;
    c.li = cv.slot_meta[(uint64_t)tile * FRZ_TILE + slot] & (FRZ_TILE - 1);
    return c;
}

// what process_candidate found for one lane's candidate, on its way to the per-class survivor lists
struct Emit {
    FrzSurvivor rec;
    unsigned long long base_raw;   // leader lanes: the reserved list position (result of the atomic, may still be in flight)
    uint32_t peers;                // lanes of the warp with the same SW class
    int cls;
    bool ok;
};

template <int MODE, class P>
__device__ __forceinline__ void process_candidate(const FrzCorpusView& cv, const P& pat, const uint8_t* __restrict__ cid_s,
                                                  uint2 (*occ)[32], const Cand& cd, bool active,
                                                  uint32_t* __restrict__ surv_bitmap, Emit* out, bool single_chunk = false) {
    bool ok = false;
    int cls = 0;
    FrzSurvivor rec;
    rec.tile = 0; rec.slot_rank = 0; rec.start = 0; rec.end = 0;
    const uint32_t tile = cd.tile, slot = cd.slot;
    const int len = active ? cd.len : 0;
    GlobalAcc ga{active ? cd.base : nullptr};
    const uint4* units = active ? cd.units : nullptr;
    // warp-wide occurrence-mask windows (uniform code) for the 0- and 1-typo modes
    bool flat_done = false, flat_ok = false;
    int flat_start = 0, flat_end = 0;
    if constexpr (std::is_same<P, FrzPatternDev>::value) {   // (long needles take the scanning forms)
    if ((MODE == FRZ_T_0 || MODE == FRZ_T_1) && pat.n_distinct > 0) {
        if (single_chunk) {   // warp-uniform: corpus of <= 64-byte haystacks at the 64-lane width (prefilter_masks.cuh)
            if (MODE == FRZ_T_0) flat_ok = masks_k0_single(units, pat, occ, len, active, &flat_start, &flat_end);
            else flat_ok = masks_k1_single(units, pat, occ, len, active, &flat_start, &flat_end);
        } else {
            if (MODE == FRZ_T_0) flat_ok = masks_k0(units, pat, cid_s, occ, len, active, &flat_start, &flat_end);
            else flat_ok = masks_k1(units, pat, cid_s, occ, len, active, &flat_start, &flat_end);
        }
        flat_done = true;
    }
    // 2-typo / N-typo trackers on the same occurrence masks (prefilter_masks.cuh: masks_paths<3>, masks_many).  An order of
    // magnitude faster than the scanning forms window_k2 / window_many at k = 2 and k = 3.  The scanning forms remain for needles with > 16 distinct byte classes.
    if ((MODE == FRZ_T_2 || MODE == FRZ_T_MANY) && pat.n_distinct > 0) {
        if (MODE == FRZ_T_2) flat_ok = masks_paths<3>(units, pat, cid_s, occ, len, active, &flat_start, &flat_end);
        else flat_ok = masks_many(units, pat, cid_s, occ, len, active, &flat_start, &flat_end);
        flat_done = true;
    }
    }
    if (active) {
        const uint32_t li = cd.li;
        int start = 0, end = len;
        uint32_t lit_score = 0;
        if (flat_done) { ok = flat_ok; start = flat_start; end = flat_end; }
        else if (MODE == FRZ_T_0) ok = window_k0(ga, pat, len, &start, &end);
        else if (MODE == FRZ_T_1) ok = window_k1(ga, pat, len, &start, &end);
        else if (MODE == FRZ_T_2) ok = window_k2(ga, pat, len, &start, &end);
        else if (MODE == FRZ_T_MANY) ok = window_many(ga, pat, len, &start, &end);
        else if (MODE == FRZ_T_LITERAL) {
            int pos = 0;
            ok = lit_find(ga, pat, len, &pos, &lit_score);
            start = pos; end = pos + pat.n;
        } else ok = true;  // FRZ_T_NONE: NO_PREFILTER (src/matcher/algo.rs:178)
        if (ok) {
            rec.tile = tile;
            rec.slot_rank = slot | (li << 10);
            if (MODE == FRZ_T_LITERAL) {
                // literal matches are final: carry (score, exact) through start/end
                cls = FRZ_C_COLS64;
                rec.start = lit_score;
                rec.end = (start == 0 && pat.n == len) ? 1u : 0u;
            } else {
                start = start > 0 ? start - 1 : 0;  // trim_haystack (src/matcher/algo.rs:331-338)
                cls = sw_class_of(end - start, pat);
                if (cls < FRZ_C_GENERIC) {
                    // window record (frz_device.cuh): everything the SW kernel needs, including the address of the
                    // window's first 16-byte unit, so that it never touches the group descriptors
                    const uint64_t addr = (uint64_t)(ga.base - cv.data) + (uint64_t)(start >> 4);
                    rec.slot_rank |= (uint32_t)(end - start) << 20 | (uint32_t)(end == len) << 28 | (uint32_t)(start == 0) << 29;
                    rec.start = (uint32_t)addr;
                    rec.end = (uint32_t)(addr >> 32) | ((uint32_t)start & 15u) << 8;
                } else {
                    rec.start = (uint32_t)start;
                    rec.end = (uint32_t)end | ((uint32_t)(end == len) << 31);
                }
            }
            atomicOr(&surv_bitmap[(uint64_t)tile * 32 + (li >> 5)], 1u << (li & 31));
        }
    }
    out->rec = rec;
    out->ok = ok;
    out->cls = cls;
}

// Survivor emission, split in two so that the round trip of the list-space atomic overlaps the NEXT item's work:
//   emit_request  the lowest lane of every SW class present reserves list slots for its peers (one atomic per class);
//                 the result stays in flight
//   emit_commit   (one item later) broadcast of the reserved base, then the 16-byte record stores
__device__ __forceinline__ void emit_request(Emit& e, FrzCounters* __restrict__ ctr) {
    const uint32_t lane = frz_lane();
    e.peers = __match_any_sync(0xffffffffu, e.ok ? e.cls : -1);
    e.base_raw = 0;
    if (e.ok && (int)lane == __ffs(e.peers) - 1)
        e.base_raw = atomicAdd(&ctr->class_count[e.cls], (unsigned long long)__popc(e.peers));
}
__device__ __forceinline__ void emit_commit(const Emit& e, const FrzSurvLists& lists, unsigned long long surv_cap,
                                            FrzCounters* __restrict__ ctr) {
    if (!__any_sync(0xffffffffu, e.ok)) return;
    const uint32_t lane = frz_lane();
    const unsigned long long base = __shfl_sync(0xffffffffu, e.base_raw, __ffs(e.peers) - 1);
    if (e.ok) {
        const unsigned long long pos = base + __popc(e.peers & ((1u << lane) - 1));
        if (pos < surv_cap) lists.p[e.cls][pos] = e.rec;
        else atomicOr(&ctr->error, FRZ_DEVERR_SURVIVOR_OVERFLOW);
    }
}

// ================================================================================================================
// k_sig_scan — the streaming signature scan alone: the unicode path's first stage (k_scan_window scans the same way on
// the byte path).  Lane per FOUR consecutive haystacks: one 16-byte load of their lengths and
// two 16-byte loads of their byte-class signatures (written at pack time, pack.cu: k_pack_sig) decide "can this
// haystack hold the needle up to the typo budget?" (two POPCs each).  The haystack bytes themselves are never touched
// here: a rejected haystack costs 12 bytes of HBM traffic instead of len + 8.  Survivors of the test become 16-byte
// candidate records {tile << 10 | slot, len << 10 | index-in-tile, address of unit 0}: the group descriptor is resolved
// here (four contiguous 16-byte descriptors per trip, L2-resident), so the consumer starts its unit loads straight from the
// record.  Warp-autonomous: a per-warp ring in shared memory collects candidates, every 32 are flushed with ONE atomic
// and one coalesced 512-byte store.  Small (about 40 registers): 12 blocks per SM keep enough bytes in flight to stream
// at HBM speed.
constexpr int kScanThreads = 128;
constexpr int kScanWarps = kScanThreads / 32;
constexpr int kScanRing = 256;   // entries per warp: up to 31 left over + up to 128 new per trip

struct __align__(16) CandRec {
    uint32_t tile_slot;   // tile << 10 | slot
    uint32_t meta;        // len << 10 | index inside the tile
    uint64_t unit0;       // unit index (16-byte units from the start of the packed data) of the slot's unit 0
};

// ---- TMA staging (cp.async.bulk, 1-D) of the phase-A arrays ---------------------------------------------------------
// The metadata, signature and group-descriptor arrays are contiguous, so a warp's next 128-slot chunk is three bulk
// copies (512 + 1024 + 64 bytes) that complete on the warp's OWN mbarrier: warp-autonomous, no block barrier, and the
// bytes in flight hold no registers (a register prefetch pays 14 registers per chunk in flight, and ptxas sinks such loads
// towards their use).  Three stages per warp.
constexpr int kScanStages = 3;
struct __align__(16) ScanStage {
    uint32_t meta[128];
    uint2 sig[128];
    FrzGroupDesc desc[4];
};
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

__global__ void __launch_bounds__(kScanThreads, 6) k_sig_scan(const FrzCorpusView cv, int use_sig, uint32_t need1, uint32_t need2,
                                                              int sig_k, int min_len, CandRec* __restrict__ cand,
                                                              unsigned long long cand_cap, FrzCounters* __restrict__ ctr) {
    extern __shared__ __align__(16) unsigned char scan_smem[];
    const uint32_t lane = frz_lane(), warp = threadIdx.x >> 5;
    CandRec* ring = reinterpret_cast<CandRec*>(scan_smem) + (size_t)warp * kScanRing;
    const uint32_t n_warps = gridDim.x * kScanWarps;
    const uint32_t total_chunks = cv.n_tiles * (FRZ_TILE / 128);   // 128 slots (4 groups) per chunk
    uint32_t head = 0, count = 0;
    // ---- candidate ring → global list, in two steps so that the atomic's round trip overlaps the next chunk:
    //      flush_request reserves list space for the 32 oldest entries (they stay in the ring), flush_commit stores them
    unsigned long long pend_base = 0;
    uint32_t pend_head = 0, pend_n = 0;
    auto flush_commit = [&]() {
        if (pend_n == 0) return;
        const unsigned long long base = __shfl_sync(0xffffffffu, pend_base, 0);
        if (lane < pend_n) {
            const unsigned long long pos = base + lane;
            if (pos < cand_cap) reinterpret_cast<uint4*>(cand)[pos] = reinterpret_cast<const uint4*>(ring)[(pend_head + lane) & (kScanRing - 1)];
            else atomicOr(&ctr->error, FRZ_DEVERR_SURVIVOR_OVERFLOW);
        }
        pend_n = 0;
    };
    auto flush_request = [&](uint32_t n_out) {
        flush_commit();   // at most one reservation in flight
        if (lane == 0) pend_base = atomicAdd(&ctr->cand_count, (unsigned long long)n_out);
        pend_head = head;
        pend_n = n_out;
        head = (head + n_out) & (kScanRing - 1);
        count -= n_out;
    };
    // length gate + signature test of one slot; passing lanes append their record to the ring
    auto test_slot = [&](uint32_t m, uint32_t p1, uint32_t p2, uint32_t slot_global, unsigned long long unit0) {
        bool pass = m != FRZ_INVALID_SLOT && (int)(m >> FRZ_TILE_SHIFT) >= min_len;
        if (use_sig) pass = pass && frz_sig_pass(need1, need2, sig_k, p1, p2);
        const uint32_t ballot = __ballot_sync(0xffffffffu, pass);
        if (pass)   // one 16-byte shared-memory store (a CandRec, field by field)
            reinterpret_cast<uint4*>(ring)[(head + count + __popc(ballot & ((1u << lane) - 1))) & (kScanRing - 1)] =
                make_uint4(slot_global, m, (uint32_t)unit0, (uint32_t)(unit0 >> 32));
        count += __popc(ballot);
    };
    // one chunk = 128 consecutive slots (4 groups): lane L owns slots 4L .. 4L+3, all in group L / 8 of the chunk
    auto process = [&](uint32_t idx, const uint4& meta, const uint4& sig0, const uint4& sig1, unsigned long long grp_off, uint32_t gunits) {
        const uint32_t slot_g = idx * 128 + lane * 4;                   // == tile << 10 | slot of this lane's first slot
        const unsigned long long unit0 = grp_off + (unsigned long long)((lane * 4) & 31) * gunits;   // unit 0 of that slot (slot-major group)
        test_slot(meta.x, sig0.x, sig0.y, slot_g, unit0);
        test_slot(meta.y, sig0.z, sig0.w, slot_g + 1, unit0 + gunits);
        test_slot(meta.z, sig1.x, sig1.y, slot_g + 2, unit0 + 2 * gunits);
        test_slot(meta.w, sig1.z, sig1.w, slot_g + 3, unit0 + 3 * gunits);
        __syncwarp();
        flush_commit();                       // the reservation made one chunk ago has arrived
        while (count >= 32) flush_request(32);
        __syncwarp();
    };
    ScanStage* stages = reinterpret_cast<ScanStage*>(scan_smem + sizeof(CandRec) * kScanRing * kScanWarps) + warp * kScanStages;
    uint64_t* bars = reinterpret_cast<uint64_t*>(scan_smem + (sizeof(CandRec) * kScanRing + sizeof(ScanStage) * kScanStages) * kScanWarps) +
                     warp * kScanStages;
    if (lane == 0)
        for (int i = 0; i < kScanStages; i++) mbar_init(&bars[i], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncwarp();
    const uint32_t tx_bytes = (uint32_t)(sizeof(uint32_t) * 128 + sizeof(FrzGroupDesc) * 4) + (use_sig ? (uint32_t)sizeof(uint2) * 128 : 0u);
    uint32_t req = blockIdx.x * kScanWarps + warp;   // next chunk to REQUEST
    auto issue = [&](int st) {
        if (req < total_chunks && lane == 0) {
            const uint64_t slot0 = (uint64_t)req * 128;
            mbar_expect_tx(&bars[st], tx_bytes);
            bulk_g2s(stages[st].meta, cv.slot_meta + slot0, (uint32_t)sizeof(uint32_t) * 128, &bars[st]);
            if (use_sig) bulk_g2s(stages[st].sig, cv.slot_sig + slot0, (uint32_t)sizeof(uint2) * 128, &bars[st]);
            bulk_g2s(stages[st].desc, cv.groups + (size_t)req * 4, (uint32_t)sizeof(FrzGroupDesc) * 4, &bars[st]);
        }
        req += n_warps;
    };
    uint32_t cur = req;
#pragma unroll
    for (int i = 0; i < kScanStages; i++) issue(i);
    int st = 0;
    uint32_t parity = 0;
    while (cur < total_chunks) {
        mbar_wait(&bars[st], parity);
        const uint4 meta = reinterpret_cast<const uint4*>(stages[st].meta)[lane];
        uint4 sig0 = make_uint4(0u, 0u, 0u, 0u), sig1 = sig0;
        if (use_sig) {
            sig0 = reinterpret_cast<const uint4*>(stages[st].sig)[2 * lane];
            sig1 = reinterpret_cast<const uint4*>(stages[st].sig)[2 * lane + 1];
        }
        const unsigned long long grp_off = stages[st].desc[lane >> 3].abs_off;
        const uint32_t grp_units = stages[st].desc[lane >> 3].gunits;
        __syncwarp();
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic reads of the stage before its async refill
        issue(st);
        process(cur, meta, sig0, sig1, grp_off, grp_units);
        cur += n_warps;
        if (++st == kScanStages) { st = 0; parity ^= 1; }
    }
    flush_commit();
    if (count) { flush_request(count); flush_commit(); }
}

// ================================================================================================================
// Stage 1 of the whole-corpus byte path  k_scan_window — the signature scan of k_sig_scan and the exact reference
// window (process_candidate) in one persistent kernel.  The scan keeps HBM busy and leaves the ALUs idle, the window
// machine the other way round; in one kernel an SM's warps do both at once, and the candidates never leave the SM.
// The two jobs run on different warps of a block, so that each runs at its own rate:
//   - the PRODUCER warp (warp 0) walks the block's statically strided 128-slot chunks like k_sig_scan (kProdStages TMA
//     stages on its own mbarriers, each refilled as soon as it has been read) and appends the records of the haystacks
//     that pass the length gate and the signature test to the block's candidate QUEUE: kQueueSlots slots of 32 records,
//     each with a "full" and an "empty" mbarrier.  A full slot is published as one batch; when every slot is taken the
//     producer waits for one to be freed (backpressure, nothing is dropped).  At the end it publishes the last partial
//     batch and one empty batch per window warp as the done marker.
//   - each WINDOW warp claims the next batch (a shared counter), copies its records to registers (lane per candidate) and
//     frees the slot, starts the cp.async copies of their haystack units into one of its two unit stages, and then windows
//     and emits the batch it claimed before — so one batch's units are in flight while the warp runs the other.
// Haystacks of more than four units (staged == false) are read by the mask builders straight from the corpus.
constexpr int kWinWarps = 3;                           // window warps per block, after the producer warp
constexpr int kScanWinThreads = 32 * (1 + kWinWarps);
constexpr int kProdStages = 6;                         // TMA stages of the producer warp
constexpr int kQueueSlots = 8;                         // 32-record batch slots of the candidate queue (a power of two)
// a window warp waits for at most one batch, so batch b's slot was freed by batch b - kQueueSlots before b is claimed
static_assert(kQueueSlots >= kWinWarps && (kQueueSlots & (kQueueSlots - 1)) == 0, "queue slots");
struct WinStage {
    uint4 units[32][5];   // [lane][unit]: the lane's four units contiguous like in the packed corpus; the fifth pads the row
                          // to 80 bytes, which makes the warp's 16-byte accesses bank-conflict-free (rows of 64 would be 4-way)
};
struct __align__(16) ScanWinSmem {   // the block's dynamic shared memory, before the occurrence tables
    ScanStage stage[kProdStages];
    CandRec queue[kQueueSlots * 32];
    WinStage win[kWinWarps][2];
    uint64_t stage_bar[kProdStages];
    uint64_t full_bar[kQueueSlots];    // 32 arrivals (the producer's lanes): the slot holds a batch
    uint64_t empty_bar[kQueueSlots];   // 32 arrivals (the consuming warp's lanes): the slot's records are in registers
    uint32_t queue_n[kQueueSlots];     // records in the slot's batch; 0 = no more batches
    uint32_t next_batch;               // the window warps' claim counter
};
// ScanWinSmem is followed by one occurrence table per window warp (OccTable's layout) of `occ_rows` rows: only the rows
// the mask builders touch, n_distinct (+ n for the single-chunk forms' position masks).
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// The needle as process_candidate reads it: the pattern itself, or (LONG) the block's staged copy of its FrzNeedleTab.
template <bool LONG>
__device__ __forceinline__ std::conditional_t<LONG, LongPat, const FrzPatternDev&> needle_view(const FrzPatternDev& p, const FrzNeedleTab* ntab,
                                                                                                  uint8_t* tab_s) {
    if constexpr (LONG) return stage_long_pat(p, ntab, tab_s);
    else return p;
}

// k_scan_window (needles of up to FRZ_MAX_NEEDLE bytes) and k_scan_window_long (longer needles: the dynamic shared memory
// holds the needle table after ScanWinSmem, where the occurrence tables would be — a long needle has none).
template <int MODE, bool LONG>
__device__ __forceinline__ void scan_window(const FrzCorpusView& cv, const FrzPatternDev& pat, int use_sig, int occ_rows,
                                            const FrzSurvLists& lists, unsigned long long surv_cap,
                                            uint32_t* __restrict__ surv_bitmap, FrzCounters* __restrict__ ctr,
                                            const FrzNeedleTab* ntab) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    frz_allow_dependent_launch();
    const uint32_t lane = frz_lane(), warp = threadIdx.x >> 5;
    ScanWinSmem& sm = *reinterpret_cast<ScanWinSmem*>(smem_raw);
    __shared__ uint8_t cid_s[FRZ_MAX_NEEDLE];
    if (threadIdx.x < FRZ_MAX_NEEDLE) cid_s[threadIdx.x] = pat.cid[threadIdx.x];
    const auto& pv = needle_view<LONG>(pat, ntab, smem_raw + sizeof(ScanWinSmem));
    if (threadIdx.x == 0) {
        for (int i = 0; i < kProdStages; i++) mbar_init(&sm.stage_bar[i], 1);
        for (int i = 0; i < kQueueSlots; i++) {
            mbar_init(&sm.full_bar[i], 32);
            mbar_init(&sm.empty_bar[i], 32);
        }
        sm.next_batch = 0;
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    const uint4 none = make_uint4(0xFFFFFFFFu, 0u, 0u, 0u);
    uint4* queue = reinterpret_cast<uint4*>(sm.queue);
    if (warp == 0) {   // ---- producer
        const uint32_t total_chunks = cv.n_tiles * (FRZ_TILE / 128);   // 128 slots (4 groups) per chunk
        const uint32_t tx_bytes = (uint32_t)(sizeof(uint32_t) * 128 + sizeof(FrzGroupDesc) * 4) + (use_sig ? (uint32_t)sizeof(uint2) * 128 : 0u);
        uint32_t req = blockIdx.x;   // next chunk to REQUEST
        auto issue = [&](int st) {
            if (req < total_chunks && lane == 0) {
                const uint64_t slot0 = (uint64_t)req * 128;
                mbar_expect_tx(&sm.stage_bar[st], tx_bytes);
                bulk_g2s(sm.stage[st].meta, cv.slot_meta + slot0, (uint32_t)sizeof(uint32_t) * 128, &sm.stage_bar[st]);
                if (use_sig) bulk_g2s(sm.stage[st].sig, cv.slot_sig + slot0, (uint32_t)sizeof(uint2) * 128, &sm.stage_bar[st]);
                bulk_g2s(sm.stage[st].desc, cv.groups + (size_t)req * 4, (uint32_t)sizeof(FrzGroupDesc) * 4, &sm.stage_bar[st]);
            }
            req += gridDim.x;
        };
        uint32_t count = 0;       // records appended so far; record r goes to queue[r % (kQueueSlots * 32)], batch r / 32
        uint32_t acquired = 0;    // batches whose slot may be written
        uint32_t published = 0;   // batches handed to the window warps
        auto acquire = [&](uint32_t upto) {   // makes batches < upto writable: batch b reuses the slot of batch b - kQueueSlots
            for (; acquired < upto; acquired++)
                if (acquired >= (uint32_t)kQueueSlots)
                    mbar_wait(&sm.empty_bar[acquired % kQueueSlots], (acquired / kQueueSlots - 1) & 1);
        };
        auto publish = [&](uint32_t n) {   // every lane arrives after its own record stores
            if (lane == 0) sm.queue_n[published % kQueueSlots] = n;
            mbar_arrive(&sm.full_bar[published % kQueueSlots]);
            published++;
        };
        // length gate + signature test of one slot
        auto test_slot = [&](uint32_t m, uint32_t p1, uint32_t p2) {
            bool pass = m != FRZ_INVALID_SLOT && (int)(m >> FRZ_TILE_SHIFT) >= pat.min_hay_len;
            if (use_sig) pass = pass && frz_sig_pass(pat.sig_need1, pat.sig_need2, pat.sig_k, p1, p2);
            return pass;
        };
        // a passing lane appends its record behind the chunk's `before` earlier records
        auto put = [&](uint32_t ballot, uint32_t before, uint32_t m, uint32_t slot_global, unsigned long long unit0) {
            if (ballot >> lane & 1u)
                queue[(count + before + __popc(ballot & ((1u << lane) - 1))) & (kQueueSlots * 32 - 1)] =
                    make_uint4(slot_global, m, (uint32_t)unit0, (uint32_t)(unit0 >> 32));
        };
#pragma unroll
        for (int i = 0; i < kProdStages; i++) issue(i);
        int st = 0;
        uint32_t parity = 0;
        for (uint32_t cur = blockIdx.x; cur < total_chunks; cur += gridDim.x) {
            mbar_wait(&sm.stage_bar[st], parity);
            const uint4 meta = reinterpret_cast<const uint4*>(sm.stage[st].meta)[lane];
            uint4 sig0 = make_uint4(0u, 0u, 0u, 0u), sig1 = sig0;
            if (use_sig) {
                sig0 = reinterpret_cast<const uint4*>(sm.stage[st].sig)[2 * lane];
                sig1 = reinterpret_cast<const uint4*>(sm.stage[st].sig)[2 * lane + 1];
            }
            const unsigned long long grp_off = sm.stage[st].desc[lane >> 3].abs_off;
            const uint32_t gunits = sm.stage[st].desc[lane >> 3].gunits;
            __syncwarp();
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic reads of the stage before its async refill
            issue(st);
            // lane L owns slots 4L .. 4L+3 of the chunk, all in group L / 8
            const uint32_t slot_g = cur * 128 + lane * 4;                   // == tile << 10 | slot of this lane's first slot
            const unsigned long long unit0 = grp_off + (unsigned long long)((lane * 4) & 31) * gunits;   // slot-major group
            // the four tests are independent: one queue acquisition and one publication per chunk
            const uint32_t b0 = __ballot_sync(0xffffffffu, test_slot(meta.x, sig0.x, sig0.y));
            const uint32_t b1 = __ballot_sync(0xffffffffu, test_slot(meta.y, sig0.z, sig0.w));
            const uint32_t b2 = __ballot_sync(0xffffffffu, test_slot(meta.z, sig1.x, sig1.y));
            const uint32_t b3 = __ballot_sync(0xffffffffu, test_slot(meta.w, sig1.z, sig1.w));
            const uint32_t n0 = __popc(b0), n01 = n0 + __popc(b1), n012 = n01 + __popc(b2), n = n012 + __popc(b3);
            if (n) {
                acquire((count + n + 31) / 32);
                put(b0, 0, meta.x, slot_g, unit0);
                put(b1, n0, meta.y, slot_g + 1, unit0 + gunits);
                put(b2, n01, meta.z, slot_g + 2, unit0 + 2 * gunits);
                put(b3, n012, meta.w, slot_g + 3, unit0 + 3 * gunits);
                count += n;
                while (published < count / 32) publish(32);
            }
            if (++st == kProdStages) { st = 0; parity ^= 1; }
        }
        if (count % 32) publish(count % 32);   // partial batch: lanes >= its size are inactive
        for (int w = 0; w < kWinWarps; w++) {  // the done markers: every window warp stops at the first it claims
            acquire(published + 1);
            publish(0);
        }
        return;
    }
    // ---- window warps
    const uint32_t ww = warp - 1;
    uint2 (*occ)[32] = reinterpret_cast<uint2 (*)[32]>(smem_raw + sizeof(ScanWinSmem)) + (size_t)ww * occ_rows;
    const bool staged = cv.max_gunits <= 4;   // every haystack fits the four staged units
    // (single_chunk_ok implies occ_rows > 0.  Testing that kernel argument first keeps the FRZ_T_0 / FRZ_T_1 code that
    // CUDA 12.9's ptxas schedules best: when the first test is on max_gunits, the prefilter stage of the max_typos=1
    // benchmark measured about 4% slower on an H100 SXM at 400 W.)
    const bool single = (MODE == FRZ_T_0 || MODE == FRZ_T_1) && occ_rows > 0 && single_chunk_ok(pat, cv.max_gunits);
    Emit pending;
    pending.ok = false; pending.cls = 0; pending.peers = 0; pending.base_raw = 0;
    pending.rec.tile = 0; pending.rec.slot_rank = 0; pending.rec.start = 0; pending.rec.end = 0;
    // windows and emits one batch: this lane's candidate record (x == 0xFFFFFFFF: none), its units in unit stage `ws`
    auto run_batch = [&](const uint4& batch, int ws) {
        const bool active = batch.x != 0xFFFFFFFFu;
        Cand cd;
        cd.tile = batch.x >> FRZ_TILE_SHIFT;
        cd.slot = batch.x & (FRZ_TILE - 1);
        cd.li = batch.y & (FRZ_TILE - 1);
        cd.len = (int)(batch.y >> FRZ_TILE_SHIFT);
        cd.base = cv.data + (((unsigned long long)batch.w << 32) | batch.z);
        cd.units = staged ? &sm.win[ww][ws].units[lane][0] : cd.base;
        Emit cur;
        process_candidate<MODE>(cv, pv, cid_s, occ, cd, active, surv_bitmap, &cur, single);
        emit_commit(pending, lists, surv_cap, ctr);      // the previous batch's list space has arrived by now
        emit_request(cur, ctr);
        pending = cur;
        __syncwarp();
    };
    uint4 prev = none;   // the claimed batch whose units are in flight
    int prev_ws = -1;
    for (;;) {
        uint32_t b = 0;
        if (lane == 0) b = atomicAdd(&sm.next_batch, 1u);
        b = __shfl_sync(0xffffffffu, b, 0);
        const uint32_t s = b % kQueueSlots;
        mbar_wait(&sm.full_bar[s], (b / kQueueSlots) & 1);
        const uint32_t n = sm.queue_n[s];
        const uint4 batch = lane < n ? queue[s * 32 + lane] : none;
        mbar_arrive(&sm.empty_bar[s]);
        if (n == 0) break;
        const int ws = prev_ws < 0 ? 0 : prev_ws ^ 1;
        if (staged && batch.x != 0xFFFFFFFFu) {
            const int units = ((int)(batch.y >> FRZ_TILE_SHIFT) + 15) >> 4;
            const uint4* base = cv.data + (((unsigned long long)batch.w << 32) | batch.z);
#pragma unroll
            for (int k = 0; k < 4; k++)
                if (k < units) __pipeline_memcpy_async(&sm.win[ww][ws].units[lane][k], base + k, 16);
        }
        __pipeline_commit();
        if (prev_ws >= 0) {
            __pipeline_wait_prior(1);
            __syncwarp();
            run_batch(prev, prev_ws);
        }
        prev = batch;
        prev_ws = ws;
    }
    if (prev_ws >= 0) {
        __pipeline_wait_prior(0);
        __syncwarp();
        run_batch(prev, prev_ws);
    }
    emit_commit(pending, lists, surv_cap, ctr);
}
template <int MODE>
__global__ void __launch_bounds__(kScanWinThreads, 5) k_scan_window(const FrzCorpusView cv, const __grid_constant__ FrzPatternDev pat,
                                                                    int use_sig, int occ_rows, const FrzSurvLists lists,
                                                                    unsigned long long surv_cap, uint32_t* __restrict__ surv_bitmap,
                                                                    FrzCounters* __restrict__ ctr) {
    scan_window<MODE, false>(cv, pat, use_sig, occ_rows, lists, surv_cap, surv_bitmap, ctr, nullptr);
}
template <int MODE>
__global__ void __launch_bounds__(kScanWinThreads, 5) k_scan_window_long(const FrzCorpusView cv, const __grid_constant__ FrzPatternDev pat,
                                                                         int use_sig, int occ_rows, const FrzSurvLists lists,
                                                                         unsigned long long surv_cap, uint32_t* __restrict__ surv_bitmap,
                                                                         FrzCounters* __restrict__ ctr, const FrzNeedleTab* ntab) {
    scan_window<MODE, true>(cv, pat, use_sig, occ_rows, lists, surv_cap, surv_bitmap, ctr, ntab);
}

// k_scan_window over the queries of a batch group (frz_match_list_batch_top): block row y runs query grp.j[y] with the
// buffers of that query, on a copy of its pattern in shared memory.  The dynamic shared memory is sized for the group's
// largest occurrence table.
template <int MODE>
__global__ void __launch_bounds__(kScanWinThreads, 5) k_scan_window_batch(const FrzCorpusView cv, const FrzBatchDev b,
                                                                          const __grid_constant__ FrzBatchGroup grp) {
    __shared__ FrzPatternDev pat_s;
    const uint32_t j = grp.j[blockIdx.y];
    frz_batch_stage_pattern(b, j, &pat_s);
    __syncthreads();
    const int use_sig = pat_s.typo_mode != FRZ_T_NONE && pat_s.sig_on;
    const int occ_rows = pat_s.n_distinct ? min(kMaxDistinct, pat_s.n_distinct + pat_s.n) : 0;
    scan_window<MODE, false>(cv, pat_s, use_sig, occ_rows, frz_batch_lists(b, j), b.surv_cap,
                             b.surv_bitmap + (uint64_t)j * cv.n_tiles * 32, b.ctr + j, nullptr);
}

// k_tile_scan for each query of a sub-batch: block j scans query j's tile counts (a contiguous run of tiles per thread).
__global__ void __launch_bounds__(1024) k_tile_scan_batch(const FrzBatchDev b, uint32_t n) {
    __shared__ uint64_t warp_sum[32];
    const uint32_t j = blockIdx.x;
    const uint32_t* cnt = b.tile_count + (uint64_t)j * n;
    uint64_t* out = b.tile_out_base + (uint64_t)j * n;
    const uint32_t per = (n + blockDim.x - 1) / blockDim.x;
    const uint32_t lo = min(threadIdx.x * per, n), hi = min(lo + per, n);
    uint64_t sum = 0;
    for (uint32_t i = lo; i < hi; i++) sum += cnt[i];
    uint64_t x = sum;
    for (int d = 1; d < 32; d <<= 1) {
        uint64_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (frz_lane() >= (uint32_t)d) x += y;
    }
    if (frz_lane() == 31) warp_sum[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
        uint64_t w = warp_sum[threadIdx.x], xs = w;
        for (int d = 1; d < 32; d <<= 1) {
            uint64_t y = __shfl_up_sync(0xffffffffu, xs, d);
            if (frz_lane() >= (uint32_t)d) xs += y;
        }
        warp_sum[threadIdx.x] = xs - w;
    }
    __syncthreads();
    uint64_t run = warp_sum[threadIdx.x >> 5] + x - sum;
    for (uint32_t i = lo; i < hi; i++) {
        out[i] = run;
        run += cnt[i];
    }
    if (threadIdx.x == blockDim.x - 1) b.ctr[j].total = run;
}

// Candidate-list mode (multi-pattern, src/matcher/multi.rs:108-120): the extra patterns are evaluated only
// on the haystacks that survived the previous patterns.  The list is already compact, so each warp takes 32
// candidates at a time straight to phase B.
template <int MODE>
__global__ void __launch_bounds__(kThreads) k_prefilter_list(const FrzCorpusView cv, const __grid_constant__ FrzPatternDev pat,
                                                             const FrzMatchDev* __restrict__ cand, unsigned long long n_cand,
                                                             uint32_t index_offset,
                                                             const FrzSurvLists lists, unsigned long long surv_cap,
                                                             uint32_t* __restrict__ surv_bitmap, FrzCounters* __restrict__ ctr) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const uint32_t lane = frz_lane(), warp = threadIdx.x >> 5;
    uint2 (*occ)[32] = reinterpret_cast<OccTable*>(smem_raw)[warp].occ;
    __shared__ uint8_t cid_s[FRZ_MAX_NEEDLE];
    if (threadIdx.x < FRZ_MAX_NEEDLE) cid_s[threadIdx.x] = pat.cid[threadIdx.x];
    __syncthreads();
    const unsigned long long n_warps = (unsigned long long)gridDim.x * kWarps;
    for (unsigned long long base = ((unsigned long long)blockIdx.x * kWarps + warp) * 32; base < n_cand; base += n_warps * 32) {
        const unsigned long long i = base + lane;
        bool active = i < n_cand;
        Cand cd;
        cd.tile = 0; cd.slot = 0; cd.li = 0; cd.len = 0; cd.base = nullptr; cd.units = nullptr;
        if (active) {
            const uint32_t idx = cand[i].index - index_offset;
            const uint32_t tile = idx >> FRZ_TILE_SHIFT, li = idx & (FRZ_TILE - 1);
            const uint32_t slot = cv.slot_of[(uint64_t)tile * FRZ_TILE + li];
            const uint32_t len = cv.slot_meta[(uint64_t)tile * FRZ_TILE + slot] >> FRZ_TILE_SHIFT;
            active = (int)len >= pat.min_hay_len;   // length gate (src/matcher/algo.rs:88)
            cd = resolve_cand(cv, tile, slot, (int)len);
        }
        __syncwarp();
        Emit e;
        process_candidate<MODE>(cv, pat, cid_s, occ, cd, active, surv_bitmap, &e);
        emit_request(e, ctr);
        emit_commit(e, lists, surv_cap, ctr);
        __syncwarp();
    }
}
// The same for a long needle: the scanning forms over the block's staged copy of its table (no occurrence tables).
template <int MODE>
__global__ void __launch_bounds__(kThreads) k_prefilter_list_long(const FrzCorpusView cv, const __grid_constant__ FrzPatternDev pat,
                                                                  const FrzMatchDev* __restrict__ cand, unsigned long long n_cand,
                                                                  uint32_t index_offset,
                                                                  const FrzSurvLists lists, unsigned long long surv_cap,
                                                                  uint32_t* __restrict__ surv_bitmap, FrzCounters* __restrict__ ctr,
                                                                  const FrzNeedleTab* __restrict__ ntab) {
    __shared__ __align__(16) uint8_t tab_s[kLongPatSmem];
    const uint32_t lane = frz_lane(), warp = threadIdx.x >> 5;
    const LongPat lp = stage_long_pat(pat, ntab, tab_s);
    __syncthreads();
    const unsigned long long n_warps = (unsigned long long)gridDim.x * kWarps;
    for (unsigned long long base = ((unsigned long long)blockIdx.x * kWarps + warp) * 32; base < n_cand; base += n_warps * 32) {
        const unsigned long long i = base + lane;
        bool active = i < n_cand;
        Cand cd;
        cd.tile = 0; cd.slot = 0; cd.li = 0; cd.len = 0; cd.base = nullptr; cd.units = nullptr;
        if (active) {
            const uint32_t idx = cand[i].index - index_offset;
            const uint32_t tile = idx >> FRZ_TILE_SHIFT, li = idx & (FRZ_TILE - 1);
            const uint32_t slot = cv.slot_of[(uint64_t)tile * FRZ_TILE + li];
            const uint32_t len = cv.slot_meta[(uint64_t)tile * FRZ_TILE + slot] >> FRZ_TILE_SHIFT;
            active = (int)len >= pat.min_hay_len;
            cd = resolve_cand(cv, tile, slot, (int)len);
        }
        __syncwarp();
        Emit e;
        process_candidate<MODE>(cv, lp, nullptr, nullptr, cd, active, surv_bitmap, &e);
        emit_request(e, ctr);
        emit_commit(e, lists, surv_cap, ctr);
        __syncwarp();
    }
}

// Per tile: exclusive prefix popcount of the 32 survivor-bitmap words (→ rank of a survivor among
// its tile's survivors in index order) and the tile's survivor count.  One warp per tile.
__global__ void __launch_bounds__(256) k_tile_rank(const uint32_t* __restrict__ surv_bitmap, uint16_t* __restrict__ word_prefix,
                                                   uint32_t* __restrict__ tile_count, uint32_t n_tiles) {
    frz_wait_prior_grid();
    frz_allow_dependent_launch();
    const uint32_t tile = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = frz_lane();
    if (tile >= n_tiles) return;
    const uint32_t c = __popc(surv_bitmap[(uint64_t)tile * 32 + lane]);
    uint32_t x = c;
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= (uint32_t)d) x += y;
    }
    word_prefix[(uint64_t)tile * 32 + lane] = (uint16_t)(x - c);
    if (lane == 31) tile_count[tile] = x;
}

// exclusive scan of tile_count → tile_out_base; total → counters.total.  One block; every thread owns a CONTIGUOUS run
// of ceil(n / 1024) tiles, so the block makes one pass (two for > 1 M tiles) instead of n / 1024 barrier rounds.
// Up to kTileScanSmem tiles the counts go through shared memory: loaded and stored coalesced, the per-thread runs walk
// shared memory (a run walked in global memory is a chain of dependent loads per thread).  Larger corpora walk the
// global arrays.
// `carry` (optional): the scan starts at *carry and leaves the new total there too — streamed calls (host.cu:
// frz_match_shard_streamed) run the pipeline over consecutive tile ranges and append each range's matches to the same list.
constexpr uint32_t kTileScanSmem = 12224;   // with warp_sum, 48 KB of static shared memory; the sum of the counts (<= 1024 per tile) fits 32 bits
__global__ void __launch_bounds__(1024) k_tile_scan(const uint32_t* __restrict__ tile_count, uint64_t* __restrict__ out,
                                                    uint32_t n, FrzCounters* __restrict__ ctr, unsigned long long* carry) {
    __shared__ uint64_t warp_sum[32];
    __shared__ uint32_t cnt_s[kTileScanSmem];
    frz_wait_prior_grid();
    frz_allow_dependent_launch();
    const bool in_smem = n <= kTileScanSmem;
    if (in_smem) {
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) cnt_s[i] = tile_count[i];
        __syncthreads();
    }
    const uint32_t* cnt = in_smem ? cnt_s : tile_count;
    const uint32_t per = (n + blockDim.x - 1) / blockDim.x;
    const uint32_t lo = min(threadIdx.x * per, n), hi = min(lo + per, n);
    uint64_t sum = 0;
    for (uint32_t i = lo; i < hi; i++) sum += cnt[i];
    uint64_t x = sum;
    for (int d = 1; d < 32; d <<= 1) {
        uint64_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (frz_lane() >= (uint32_t)d) x += y;
    }
    if (frz_lane() == 31) warp_sum[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
        uint64_t w = warp_sum[threadIdx.x], xs = w;
        for (int d = 1; d < 32; d <<= 1) {
            uint64_t y = __shfl_up_sync(0xffffffffu, xs, d);
            if (frz_lane() >= (uint32_t)d) xs += y;
        }
        warp_sum[threadIdx.x] = xs - w;
    }
    __syncthreads();
    const uint64_t start = carry ? *carry : 0ull;
    __syncthreads();                                        // everybody has read the carry before the last thread replaces it
    uint64_t run = start + warp_sum[threadIdx.x >> 5] + x - sum;   // exclusive prefix of this thread's run
    if (in_smem) {   // exclusive prefixes (without the carry) in place, then one coalesced pass
        uint32_t r = (uint32_t)(run - start);
        for (uint32_t i = lo; i < hi; i++) {
            const uint32_t c = cnt_s[i];
            cnt_s[i] = r;
            r += c;
        }
        run = start + r;
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) out[i] = start + cnt_s[i];
    } else {
        for (uint32_t i = lo; i < hi; i++) {
            out[i] = run;
            run += tile_count[i];
        }
    }
    if (threadIdx.x == blockDim.x - 1) {   // the last thread's run ends at n (empty runs carry the total)
        ctr->total = run;
        if (carry) *carry = run;
    }
}

// Matcher::match_list_indices for chosen haystacks (src/matcher/mod.rs:234-262 → match_one_indices_impl,
// src/matcher/algo.rs:138-169, src/literal/algo.rs:134-155).  One thread per requested haystack; the scoring with
// full matrices and the traceback are in indices_path.cuh (shared with the CPU test build), the ASCII windows come
// from the scanning prefilters above.  Not a hot path: the reference documents it as unoptimised too.
__global__ void __launch_bounds__(128) k_match_indices(const FrzCorpusView cv, const __grid_constant__ FrzPatternDev pat,
                                                       const __grid_constant__ FrzUNeedle un, const FrzUScoring usc, int unicode,
                                                       const uint32_t* __restrict__ which, unsigned long long n,
                                                       FrzMatchDev* __restrict__ out_matches, uint32_t* __restrict__ out_idx,
                                                       uint32_t stride, uint32_t* __restrict__ out_cnt,
                                                       uint16_t* __restrict__ scratch, unsigned long long scratch_stride) {
    const unsigned long long tid = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long nthreads = (unsigned long long)gridDim.x * blockDim.x;
    uint16_t* my_scratch = scratch + tid * scratch_stride;
    const int max_typos = pat.typo_mode == FRZ_T_NONE ? -1 : pat.typo_mode == FRZ_T_0 ? 0 : pat.typo_mode == FRZ_T_1 ? 1
                        : pat.typo_mode == FRZ_T_2 ? 2 : pat.max_typos;
    for (unsigned long long j = tid; j < n; j += nthreads) {
        const uint32_t idx = which[j];
        out_cnt[j] = 0xFFFFFFFFu;
        if (idx >= cv.n) continue;
        const uint32_t tile = idx >> FRZ_TILE_SHIFT;
        const uint32_t slot = cv.slot_of[idx];
        const uint32_t meta = cv.slot_meta[(uint64_t)tile * FRZ_TILE + slot];
        if (meta == FRZ_INVALID_SLOT) continue;   // a removed haystack (frz_corpus_remove) matches nothing
        const int len = (int)(meta >> FRZ_TILE_SHIFT);
        const FrzGroupDesc gd = cv.groups[tile * FRZ_GROUPS_PER_TILE + (slot >> 5)];
        const GlobalAcc ga{cv.data + frz_slot_unit0(gd, slot & 31)};
        const FrzPackedHay hay{ga.base, 0};
        uint32_t* my_out = out_idx + j * (unsigned long long)stride;
        uint32_t score = 0;
        bool exact = false;
        int cnt = 0;
        if (pat.matching != FRZ_MATCHING_FUZZY) {
            int pos = 0;
            const bool ok = unicode ? frzu::lit_find(un, usc, hay, len, pat.matching, &pos, &score) : lit_find(ga, pat, len, &pos, &score);
            if (!ok) continue;
            exact = pos == 0 && pat.n == len;
            for (int i = pos + pat.n - 1; i >= pos; i--) { if (cnt < (int)stride) my_out[cnt] = (uint32_t)i; cnt++; }
        } else {
            if (len < pat.min_hay_len) continue;
            int start = 0, end = len;
            bool ok;
            if (unicode) ok = frzu::prefilter(un, hay, len, pat.pf_lanes, max_typos, &start, &end);
            else if (pat.typo_mode == FRZ_T_0) ok = window_k0(ga, pat, len, &start, &end);
            else if (pat.typo_mode == FRZ_T_1) ok = window_k1(ga, pat, len, &start, &end);
            else if (pat.typo_mode == FRZ_T_2) ok = window_k2(ga, pat, len, &start, &end);
            else if (pat.typo_mode == FRZ_T_MANY) ok = window_many(ga, pat, len, &start, &end);
            else ok = true;
            if (!ok) continue;
            start = start > 0 ? start - 1 : 0;   // trim_haystack
            const int W = end - start;
            const FrzPackedHay win{ga.base, start};
            score = frzi::sw_indices(un, unicode != 0, usc, win, W, start, max_typos, pat.sw_lanes, pat.score_bits == 8, my_scratch,
                                     my_out, (int)stride, &cnt);
            exact = start == 0 && end == len && W == pat.n;
            for (int k = 0; exact && k < W; k++) exact = win(k) == pat.c[k];
            if (exact) score = (score + (uint32_t)pat.exact_bonus) & 0xffffu;
        }
        FrzMatchDev m;
        m.index = idx; m.score = (uint16_t)score; m.exact = exact ? 1 : 0; m.pad = 0;
        out_matches[j] = m;
        out_cnt[j] = (uint32_t)cnt;   // untruncated (only the first `stride` offsets were stored)
    }
}

}  // namespace

frz_status frz_launch_prefilter_list(const FrzCorpusView& cv, const FrzPatternDev& pat, const FrzMatchDev* cand,
                                     uint64_t n_cand, uint32_t index_offset, FrzWorkspace& ws, cudaStream_t stream,
                                     FrzLaunchStats* st, const FrzNeedleTab* ntab) {
    if (cv.n_tiles == 0) return FRZ_OK;
    const bool is_long = pat.n > FRZ_MAX_NEEDLE;
    const size_t smem = is_long ? 0 : sizeof(OccTable) * kWarps;
    FRZ_CUDA_TRY(cudaMemsetAsync(ws.surv_bitmap.get(), 0, (size_t)cv.n_tiles * 32 * sizeof(uint32_t), stream));
    if (n_cand == 0) return FRZ_OK;
    const uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)frz_sm_count() * 4, (n_cand + kThreads - 1) / kThreads));
#define FRZ_PFL_LAUNCH(MODE)                                                                                          \
    do {                                                                                                              \
        if (is_long) {                                                                                                \
            k_prefilter_list_long<MODE><<<grid, kThreads, smem, stream>>>(cv, pat, cand, n_cand, index_offset, ws.lists(), \
                                                                          ws.survivor_cap(), ws.surv_bitmap.get(), ws.counters.get(), ntab); \
        } else {                                                                                                      \
            k_prefilter_list<MODE><<<grid, kThreads, smem, stream>>>(cv, pat, cand, n_cand, index_offset, ws.lists(), \
                                                                     ws.survivor_cap(), ws.surv_bitmap.get(), ws.counters.get());   \
        }                                                                                                             \
    } while (0)
    switch (pat.typo_mode) {
        case FRZ_T_0: FRZ_PFL_LAUNCH(FRZ_T_0); break;
        case FRZ_T_1: FRZ_PFL_LAUNCH(FRZ_T_1); break;
        case FRZ_T_2: FRZ_PFL_LAUNCH(FRZ_T_2); break;
        case FRZ_T_MANY: FRZ_PFL_LAUNCH(FRZ_T_MANY); break;
        case FRZ_T_NONE: FRZ_PFL_LAUNCH(FRZ_T_NONE); break;
        case FRZ_T_LITERAL: FRZ_PFL_LAUNCH(FRZ_T_LITERAL); break;
        default: return frz_fail(FRZ_ERR_INVALID_ARG, "bad typo mode %d", pat.typo_mode);
    }
#undef FRZ_PFL_LAUNCH
    FRZ_CUDA_TRY(cudaGetLastError());
    if (st) st->launches++;
    return FRZ_OK;
}

// The streaming signature scan alone over the whole corpus → candidate records in ws.cand_list, their number in
// ws.counters->cand_count, for the unicode path (k_unicode consumes the records).
frz_status frz_launch_sig_scan(const FrzCorpusView& cv, const FrzPatternDev& pat, FrzWorkspace& ws, cudaStream_t stream, FrzLaunchStats* st) {
    if (cv.n_tiles == 0) return FRZ_OK;
    const int sms = frz_sm_count();
    CandRec* cand = reinterpret_cast<CandRec*>(ws.cand_list.get());
    {   // persistent warps, as many blocks as fit
        const uint32_t total_chunks = cv.n_tiles * (FRZ_TILE / 128);
        const int use_sig = pat.typo_mode != FRZ_T_NONE && pat.sig_on;
        const size_t smem = (sizeof(CandRec) * kScanRing + sizeof(ScanStage) * kScanStages + sizeof(uint64_t) * kScanStages) * kScanWarps;
        static int bps_dev[64] = {};
        int& bps = bps_dev[frz_current_device() & 63];
        if (!bps) {
            FRZ_CUDA_TRY(cudaFuncSetAttribute(k_sig_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            FRZ_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_sig_scan, kScanThreads, smem));
            if (bps < 1) bps = 1;
        }
        const uint32_t grid = std::max<uint32_t>(1, std::min<uint32_t>((uint32_t)(sms * bps), (total_chunks + kScanWarps - 1) / kScanWarps));
        k_sig_scan<<<grid, kScanThreads, smem, stream>>>(cv, use_sig, pat.sig_need1, pat.sig_need2, pat.sig_k, pat.min_hay_len, cand,
                                                         ws.cand_list.cap(), ws.counters.get());
    }
    FRZ_CUDA_TRY(cudaGetLastError());
    if (st) st->launches++;
    return FRZ_OK;
}

// Stage 1 of match_list over the whole corpus: k_scan_window (length gate + signature test + exact windows → survivor
// records + per-tile survivor bitmap).
frz_status frz_launch_prefilter(const FrzCorpusView& cv, const FrzPatternDev& pat, FrzWorkspace& ws, cudaStream_t stream,
                                FrzLaunchStats* st, const FrzNeedleTab* ntab) {
    if (cv.n_tiles == 0) return FRZ_OK;
    const int sms = frz_sm_count();
    FRZ_CUDA_TRY(cudaMemsetAsync(ws.surv_bitmap.get(), 0, (size_t)cv.n_tiles * 32 * sizeof(uint32_t), stream));
    const int use_sig = pat.typo_mode != FRZ_T_NONE && pat.sig_on;
    const int occ_rows = pat.n_distinct ? std::min(kMaxDistinct, pat.n_distinct + pat.n) : 0;
    const uint32_t total_chunks = cv.n_tiles * (FRZ_TILE / 128);
    if (pat.n > FRZ_MAX_NEEDLE) {   // long needle (n_distinct 0: no occurrence tables), the table after ScanWinSmem
        const size_t smem = sizeof(ScanWinSmem) + kLongPatSmem;
#define FRZ_PF_LAUNCH_LONG(MODE)                                                                                          \
    do {                                                                                                                 \
        static int bps_dev[64] = {};                                                                                     \
        int& bps = bps_dev[frz_current_device() & 63];                                                                   \
        if (!bps) {                                                                                                      \
            FRZ_CUDA_TRY(cudaFuncSetAttribute(k_scan_window_long<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            FRZ_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_scan_window_long<MODE>, kScanWinThreads, smem)); \
            if (bps < 1) bps = 1;                                                                                        \
        }                                                                                                                \
        const uint32_t grid = std::max<uint32_t>(1, std::min<uint32_t>((uint32_t)(sms * bps), total_chunks));   /* a producer per block */ \
        k_scan_window_long<MODE><<<grid, kScanWinThreads, smem, stream>>>(cv, pat, use_sig, 0, ws.lists(), ws.survivor_cap(),     \
                                                                   ws.surv_bitmap.get(), ws.counters.get(), ntab);                   \
    } while (0)
        switch (pat.typo_mode) {
            case FRZ_T_0: FRZ_PF_LAUNCH_LONG(FRZ_T_0); break;
            case FRZ_T_1: FRZ_PF_LAUNCH_LONG(FRZ_T_1); break;
            case FRZ_T_2: FRZ_PF_LAUNCH_LONG(FRZ_T_2); break;
            case FRZ_T_MANY: FRZ_PF_LAUNCH_LONG(FRZ_T_MANY); break;
            case FRZ_T_NONE: FRZ_PF_LAUNCH_LONG(FRZ_T_NONE); break;
            case FRZ_T_LITERAL: FRZ_PF_LAUNCH_LONG(FRZ_T_LITERAL); break;
            default: return frz_fail(FRZ_ERR_INVALID_ARG, "bad typo mode %d", pat.typo_mode);
        }
#undef FRZ_PF_LAUNCH_LONG
        FRZ_CUDA_TRY(cudaGetLastError());
        if (st) st->launches++;
        return FRZ_OK;
    }
    const size_t smem = sizeof(ScanWinSmem) + sizeof(uint2) * 32 * occ_rows * kWinWarps;
    const size_t smem_max = sizeof(ScanWinSmem) + sizeof(OccTable) * kWinWarps;
#define FRZ_PF_LAUNCH(MODE)                                                                                              \
    do {                                                                                                                 \
        static int bps_dev[64][kMaxDistinct + 1] = {};   /* blocks per SM by device and occurrence-table rows */         \
        int& bps = bps_dev[frz_current_device() & 63][occ_rows];                                                         \
        if (!bps) {                                                                                                      \
            FRZ_CUDA_TRY(cudaFuncSetAttribute(k_scan_window<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max)); \
            FRZ_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_scan_window<MODE>, kScanWinThreads, smem)); \
            if (bps < 1) bps = 1;                                                                                        \
        }                                                                                                                \
        const uint32_t grid = std::max<uint32_t>(1, std::min<uint32_t>((uint32_t)(sms * bps), total_chunks));   /* a producer per block */ \
        k_scan_window<MODE><<<grid, kScanWinThreads, smem, stream>>>(cv, pat, use_sig, occ_rows, ws.lists(), ws.survivor_cap(),   \
                                                              ws.surv_bitmap.get(), ws.counters.get());                              \
    } while (0)
    switch (pat.typo_mode) {
        case FRZ_T_0: FRZ_PF_LAUNCH(FRZ_T_0); break;
        case FRZ_T_1: FRZ_PF_LAUNCH(FRZ_T_1); break;
        case FRZ_T_2: FRZ_PF_LAUNCH(FRZ_T_2); break;
        case FRZ_T_MANY: FRZ_PF_LAUNCH(FRZ_T_MANY); break;
        case FRZ_T_NONE: FRZ_PF_LAUNCH(FRZ_T_NONE); break;
        case FRZ_T_LITERAL: FRZ_PF_LAUNCH(FRZ_T_LITERAL); break;
        default: return frz_fail(FRZ_ERR_INVALID_ARG, "bad typo mode %d", pat.typo_mode);
    }
#undef FRZ_PF_LAUNCH
    FRZ_CUDA_TRY(cudaGetLastError());
    if (st) st->launches++;
    return FRZ_OK;
}

// Stage 1 of a batch sub-batch: one k_scan_window_batch launch per typo mode present, its grid split evenly over the
// mode's queries (as many blocks in all as one single-query launch), then every query's tile ranks (one k_tile_rank over
// the sub-batch's bitmaps, which lie back to back) and tile scans (one k_tile_scan_batch).
frz_status frz_launch_prefilter_batch(const FrzCorpusView& cv, const FrzBatchDev& b, const FrzPatternDev* h_pats, uint32_t nq,
                                      cudaStream_t stream, FrzLaunchStats* st) {
    if (cv.n_tiles == 0 || nq == 0) return FRZ_OK;
    const int sms = frz_sm_count();
    const uint32_t total_chunks = cv.n_tiles * (FRZ_TILE / 128);
    const size_t smem_max = sizeof(ScanWinSmem) + sizeof(OccTable) * kWinWarps;
    for (int mode = FRZ_T_0; mode <= FRZ_T_NONE; mode++) {
        FrzBatchGroup grp;
        uint32_t ng = 0;
        int occ_max = 0;
        for (uint32_t j = 0; j < nq; j++) {
            if (h_pats[j].typo_mode != mode) continue;
            grp.j[ng++] = (uint16_t)j;
            const FrzPatternDev& p = h_pats[j];
            occ_max = std::max(occ_max, p.n_distinct ? std::min(kMaxDistinct, p.n_distinct + p.n) : 0);
        }
        if (ng == 0) continue;
        const size_t smem = sizeof(ScanWinSmem) + sizeof(uint2) * 32 * occ_max * kWinWarps;
#define FRZ_PFB_LAUNCH(MODE)                                                                                             \
    do {                                                                                                                 \
        static int bps_dev[64][kMaxDistinct + 1] = {};                                                                   \
        int& bps = bps_dev[frz_current_device() & 63][occ_max];                                                          \
        if (!bps) {                                                                                                      \
            FRZ_CUDA_TRY(cudaFuncSetAttribute(k_scan_window_batch<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max)); \
            FRZ_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_scan_window_batch<MODE>, kScanWinThreads, smem)); \
            if (bps < 1) bps = 1;                                                                                        \
        }                                                                                                                \
        const uint32_t gx = std::max<uint32_t>(1, std::min<uint32_t>((uint32_t)(sms * bps) / ng, total_chunks));         \
        k_scan_window_batch<MODE><<<dim3(gx, ng), kScanWinThreads, smem, stream>>>(cv, b, grp);                          \
    } while (0)
        switch (mode) {
            case FRZ_T_0: FRZ_PFB_LAUNCH(FRZ_T_0); break;
            case FRZ_T_1: FRZ_PFB_LAUNCH(FRZ_T_1); break;
            case FRZ_T_2: FRZ_PFB_LAUNCH(FRZ_T_2); break;
            case FRZ_T_MANY: FRZ_PFB_LAUNCH(FRZ_T_MANY); break;
            default: FRZ_PFB_LAUNCH(FRZ_T_NONE); break;
        }
#undef FRZ_PFB_LAUNCH
        FRZ_CUDA_TRY(cudaGetLastError());
        if (st) st->launches++;
    }
    const uint32_t tiles = cv.n_tiles * nq;
    k_tile_rank<<<(tiles * 32 + 255) / 256, 256, 0, stream>>>(b.surv_bitmap, b.word_prefix, b.tile_count, tiles);
    k_tile_scan_batch<<<nq, 1024, 0, stream>>>(b, cv.n_tiles);
    FRZ_CUDA_TRY(cudaGetLastError());
    if (st) st->launches += 2;
    return FRZ_OK;
}

frz_status frz_launch_tile_scan_batch(const FrzBatchDev& b, uint32_t n_tiles, uint32_t nq, cudaStream_t stream, FrzLaunchStats* st) {
    if (nq == 0) return FRZ_OK;
    k_tile_scan_batch<<<nq, 1024, 0, stream>>>(b, n_tiles);
    FRZ_CUDA_TRY(cudaGetLastError());
    st->launches++;
    return FRZ_OK;
}

frz_status frz_launch_tile_scan(const FrzCorpusView& cv, FrzWorkspace& ws, cudaStream_t stream, FrzLaunchStats* st,
                                unsigned long long* carry) {
    if (cv.n_tiles) {
        FRZ_CUDA_TRY(frz_launch_dependent(k_tile_rank, (cv.n_tiles * 32 + 255) / 256, 256, 0, stream, ws.surv_bitmap.get(),
                                          ws.word_prefix.get(), ws.tile_count.get(), cv.n_tiles));
        if (st) st->launches++;
    }
    FRZ_CUDA_TRY(frz_launch_dependent(k_tile_scan, 1, 1024, 0, stream, ws.tile_count.get(), ws.tile_out_base.get(), cv.n_tiles,
                                      ws.counters.get(), carry));
    if (st) st->launches++;
    return FRZ_OK;
}

frz_status frz_launch_match_indices(const FrzCorpusView& cv, const FrzPatternDev& pat, const FrzUNeedle& un, const FrzUScoring& usc,
                                    bool unicode, const uint32_t* d_which, uint64_t n, FrzMatchDev* d_matches, uint32_t* d_idx,
                                    uint32_t stride, uint32_t* d_cnt, uint16_t* d_scratch, uint64_t scratch_stride, uint32_t threads,
                                    cudaStream_t stream) {
    if (n == 0) return FRZ_OK;
    const uint32_t grid = (threads + 127) / 128;
    k_match_indices<<<grid, 128, 0, stream>>>(cv, pat, un, usc, unicode ? 1 : 0, d_which, n, d_matches, d_idx, stride, d_cnt,
                                              d_scratch, scratch_stride);
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}
