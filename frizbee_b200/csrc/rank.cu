// rank.cu — the device work of frz_attr_rank (DESIGN.md §4.17).  The key rules are rank_plan.cuh's; host.cu drives the
// rounds, sorts each round's rows with the LSD sort of sort.cu (frz_launch_sort_by_rank_dev) and scans the head counts.
//
//   k_rank_init    the ranked rows (live in C and in every text key's corpus) → the first list, all in segment 0
//   k_rank_skip    a text segment's common prefix from its place: every row against the segment's first row, 16 bytes per
//                  load, the minimum per segment
//   k_rank_chunk   every listed row's chunk and round sort key, and the OR of the keys and of their complements
//   k_rank_split   over the sorted list: each row's new segment, the places of the new segments, the rows still to refine
//                  → the next list, and the first position of every finished segment → the head bitmap
//   k_rank_heads   per 1024 positions: the heads before each bitmap word and their total
//   k_rank_write   value[i] = the number of heads before row i's segment, or FRZ_ATTR_NULL
#include "frz_host.h"
#include "rank_plan.cuh"

namespace {

constexpr int kRankBlock = 256;
constexpr unsigned kFullWarp = 0xffffffffu;

__device__ __forceinline__ bool live_in(const uint32_t* __restrict__ slot_meta, const uint16_t* __restrict__ slot_of, uint64_t i) {
    return slot_meta[(i & ~(uint64_t)(FRZ_TILE - 1)) + slot_of[i]] != FRZ_INVALID_SLOT;
}

// Row i's text in a text key's corpus: its length and its first unit.
struct RankText {
    const uint4* base;
    uint32_t len;
};
__device__ __forceinline__ RankText text_of(const FrzCorpusView& cv, uint32_t i) {
    const uint32_t tile = i >> FRZ_TILE_SHIFT, slot = cv.slot_of[i];
    const uint32_t meta = cv.slot_meta[(uint64_t)tile * FRZ_TILE + slot];
    return RankText{frz_unit_ptr(cv, tile, slot, 0), meta >> 10};
}

// The slot in a list counted at *count of each lane whose `want` is set (one atomic per warp); every lane must call it.
__device__ __forceinline__ uint32_t warp_slot(bool want, unsigned long long* count) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t b = __ballot_sync(kFullWarp, want);
    unsigned long long base = 0;
    if (b && lane == 0) base = atomicAdd(count, (unsigned long long)__popc(b));
    base = __shfl_sync(kFullWarp, base, 0);
    return (uint32_t)(base + __popc(b & ((1u << lane) - 1)));
}

__global__ void __launch_bounds__(kRankBlock) k_rank_init(const __grid_constant__ FrzRankDev d, FrzMatchDev* __restrict__ list) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t b0 = (uint64_t)blockIdx.x * blockDim.x; b0 < d.n; b0 += stride) {   // every lane runs every trip
        const uint64_t i = b0 + threadIdx.x;
        bool ranked = i < d.n && live_in(d.slot_meta, d.slot_of, i);
        for (uint32_t k = 0; k < d.n_keys; k++)
            if (ranked && d.keys[k].is_text) ranked = live_in(d.keys[k].text.slot_meta, d.keys[k].text.slot_of, i);
        const uint32_t p = warp_slot(ranked, &d.state[0]);
        if (ranked) {
            list[p] = FrzMatchDev{(uint32_t)i, 0, 0, 0};
            d.seg_of[i] = 0;
            if (p == 0) {
                d.segs[0] = make_uint2((uint32_t)i, frz_rank_at(0, 0));
                d.skip[0] = kFrzRankNone;
            }
        } else if (i < d.n) {
            d.seg_of[i] = kFrzRankNone;
        }
    }
}

__global__ void __launch_bounds__(kRankBlock) k_rank_skip(const __grid_constant__ FrzRankDev d, const FrzMatchDev* __restrict__ list,
                                                          const unsigned long long* __restrict__ n_ptr) {
    const uint64_t n = *n_ptr, stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t b0 = (uint64_t)blockIdx.x * blockDim.x; b0 < n; b0 += stride) {
        const uint64_t j = b0 + threadIdx.x;
        uint32_t s = 0, common = kFrzRankNone;
        bool text = false;
        if (j < n) {
            const uint32_t row = list[j].index;
            s = d.seg_of[row];
            const uint2 seg = d.segs[s];
            const FrzRankKeyDev& key = d.keys[frz_rank_at_key(seg.y)];
            text = key.is_text != 0;
            if (text && row != seg.x) {
                const RankText a = text_of(key.text, row), b = text_of(key.text, seg.x);
                const auto unit = [&](int t, uint32_t u, uint32_t* w) {
                    const uint4 v = (t ? b.base : a.base)[u];
                    w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
                };
                common = frz_rank_common(unit, a.len, b.len, frz_rank_at_off(seg.y), key.fold != 0);
            }
        }
        const uint32_t mask = __ballot_sync(kFullWarp, text);
        if (text) {   // one atomic per segment present in the warp
            const uint32_t peers = __match_any_sync(mask, s);
            const uint32_t m = __reduce_min_sync(peers, common);
            if ((threadIdx.x & 31) == (uint32_t)__ffs(peers) - 1 && m != kFrzRankNone) atomicMin(&d.skip[s], m);
        }
    }
}

__device__ __forceinline__ unsigned long long warp_or(unsigned long long x) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x |= __shfl_xor_sync(kFullWarp, x, o);
    return x;
}

__global__ void __launch_bounds__(kRankBlock) k_rank_chunk(const __grid_constant__ FrzRankDev d, const FrzMatchDev* __restrict__ list,
                                                           const unsigned long long* __restrict__ n_ptr) {
    const uint64_t n = *n_ptr, stride = (uint64_t)gridDim.x * blockDim.x;
    unsigned long long or_hi = 0, or_lo = 0, nor_hi = 0, nor_lo = 0;
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
        const uint32_t row = list[j].index;
        const uint32_t s = d.seg_of[row];
        uint32_t at = d.segs[s].y;
        const FrzRankKeyDev& key = d.keys[frz_rank_at_key(at)];
        uint64_t chunk;
        if (key.is_text) {
            const uint32_t skip = d.skip[s];
            if (skip != kFrzRankNone) at += skip;
            const RankText t = text_of(key.text, row);
            chunk = frz_rank_text_chunk(FrzPackedHay{t.base, 0}, t.len, frz_rank_at_off(at), key.fold != 0, key.desc != 0);
        } else {
            chunk = frz_rank_attr_chunk(frz_order_value(key.values, key.n_values, row), key.desc != 0);
        }
        const FrzOrderKey k = frz_rank_sort_key(s, chunk);
        d.keys_row[row] = k;
        d.at_row[row] = at;
        or_hi |= k.hi;
        or_lo |= k.lo;
        nor_hi |= ~k.hi;
        nor_lo |= ~k.lo & ((1ull << 48) - 1);
    }
    __shared__ unsigned long long s_or[kRankBlock / 32][4];
    const uint32_t warp = threadIdx.x >> 5;
    or_hi = warp_or(or_hi);
    or_lo = warp_or(or_lo);
    nor_hi = warp_or(nor_hi);
    nor_lo = warp_or(nor_lo);
    if ((threadIdx.x & 31) == 0) {
        s_or[warp][0] = or_hi;
        s_or[warp][1] = or_lo;
        s_or[warp][2] = nor_hi;
        s_or[warp][3] = nor_lo;
    }
    __syncthreads();
    if (threadIdx.x < 4) {
        unsigned long long x = 0;
        for (uint32_t w = 0; w < kRankBlock / 32; w++) x |= s_or[w][threadIdx.x];
        if (x) atomicOr(&d.state[2 + threadIdx.x], x);   // OR of the keys (hi, lo), then of their complements
    }
}

// the first position in [lo, hi) of the sorted list whose key is not ahead of k (the keys descend), or whose segment is not
// below seg when by_seg
__device__ __forceinline__ uint64_t first_not_ahead(const FrzRankDev& d, const FrzMatchDev* list, uint64_t lo, uint64_t hi,
                                                    const FrzOrderKey& k, bool by_seg) {
    const uint32_t seg = frz_rank_key_seg(k);
    while (lo < hi) {
        const uint64_t mid = (lo + hi) / 2;
        const FrzOrderKey m = d.keys_row[list[mid].index];
        if (by_seg ? frz_rank_key_seg(m) < seg : frz_order_ahead(m, k)) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(kRankBlock) k_rank_split(const __grid_constant__ FrzRankDev d, const FrzMatchDev* __restrict__ sorted,
                                                           const unsigned long long* __restrict__ n_ptr, FrzMatchDev* __restrict__ next,
                                                           unsigned long long* __restrict__ n_next) {
    const uint64_t n = *n_ptr, stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t b0 = (uint64_t)blockIdx.x * blockDim.x; b0 < n; b0 += stride) {   // every lane runs every trip
        const uint64_t j = b0 + threadIdx.x;
        bool more = false;
        uint32_t row = 0;
        if (j < n) {
            row = sorted[j].index;
            const FrzOrderKey k = d.keys_row[row];
            const uint32_t s = frz_rank_key_seg(k);
            // the segment's rows start at `parent` in the list and at position s of the order; the rows of the new segment
            // start at `first`
            const uint64_t parent = first_not_ahead(d, sorted, 0, j, k, true);
            const uint64_t first = j > 0 && frz_rank_key_eq(d.keys_row[sorted[j - 1].index], k) ? first_not_ahead(d, sorted, parent, j, k, false) : j;
            const uint32_t seg = s + (uint32_t)(first - parent);
            const bool alone = first == j && (j + 1 == n || !frz_rank_key_eq(d.keys_row[sorted[j + 1].index], k));
            const uint32_t at = d.at_row[row];
            const FrzRankKeyDev& key = d.keys[frz_rank_at_key(at)];
            const uint64_t chunk = ~((k.hi & 0xFFFFu) << 48 | k.lo);
            uint32_t place = 0;
            more = !alone && frz_rank_next(at, frz_rank_chunk_ends(chunk, key.is_text != 0, key.desc != 0), d.n_keys, &place);
            d.seg_of[row] = seg;
            if (first == j) {
                if (more) {
                    d.segs[seg] = make_uint2(row, place);
                    d.skip[seg] = kFrzRankNone;
                } else {
                    atomicOr(&d.heads[seg >> 5], 1u << (seg & 31));
                }
            }
        }
        const uint32_t p = warp_slot(more, n_next);
        if (more) next[p] = FrzMatchDev{row, 0, 0, 0};
    }
}

// One warp per 1024 positions: lane l holds bitmap word l, word_pref its heads before it within the chunk
__global__ void __launch_bounds__(kRankBlock) k_rank_heads(const uint32_t* __restrict__ heads, uint64_t m, uint32_t* __restrict__ word_pref,
                                                           uint32_t* __restrict__ chunk_count) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n_words = (m + 31) / 32, n_chunks = (m + 1023) / 1024;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
    for (uint64_t c = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; c < n_chunks; c += warps) {
        const uint64_t w = c * 32 + lane;
        const uint32_t cnt = w < n_words ? __popc(heads[w]) : 0u;
        uint32_t incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(kFullWarp, incl, o);
            if (lane >= (uint32_t)o) incl += y;
        }
        if (w < n_words) word_pref[w] = incl - cnt;
        if (lane == 31) chunk_count[c] = incl;
    }
}

__global__ void __launch_bounds__(kRankBlock) k_rank_write(const uint32_t* __restrict__ seg_of, uint64_t n, const uint32_t* __restrict__ heads,
                                                           const uint32_t* __restrict__ word_pref, const uint64_t* __restrict__ chunk_base,
                                                           int64_t* __restrict__ values) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint32_t s = seg_of[i];
        values[i] = s == kFrzRankNone ? (int64_t)(1ull << 63)
                                      : (int64_t)(chunk_base[s >> 10] + word_pref[s >> 5] + __popc(heads[s >> 5] & ((1u << (s & 31)) - 1)));
    }
}

}  // namespace

frz_status frz_launch_rank_init(const FrzRankDev& d, FrzMatchDev* list, cudaStream_t stream) {
    if (d.n == 0) return FRZ_OK;
    k_rank_init<<<grid_for(d.n, kRankBlock), kRankBlock, 0, stream>>>(d, list);
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

frz_status frz_launch_rank_round(const FrzRankDev& d, const FrzMatchDev* list, const unsigned long long* n_ptr, uint64_t n_cap,
                                 cudaStream_t stream) {
    const int grid = grid_for(n_cap, kRankBlock);
    if (d.any_text) k_rank_skip<<<grid, kRankBlock, 0, stream>>>(d, list, n_ptr);
    k_rank_chunk<<<grid, kRankBlock, 0, stream>>>(d, list, n_ptr);
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

frz_status frz_launch_rank_split(const FrzRankDev& d, const FrzMatchDev* sorted, const unsigned long long* n_ptr, uint64_t n_cap,
                                 FrzMatchDev* next, unsigned long long* n_next, cudaStream_t stream) {
    k_rank_split<<<grid_for(n_cap, kRankBlock), kRankBlock, 0, stream>>>(d, sorted, n_ptr, next, n_next);
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

frz_status frz_launch_rank_heads(const uint32_t* heads, uint64_t m, uint32_t* word_pref, uint32_t* chunk_count, cudaStream_t stream) {
    const uint64_t n_chunks = (m + 1023) / 1024;
    if (n_chunks == 0) return FRZ_OK;
    k_rank_heads<<<grid_for(n_chunks * 32, kRankBlock), kRankBlock, 0, stream>>>(heads, m, word_pref, chunk_count);
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

frz_status frz_launch_rank_write(const uint32_t* seg_of, uint64_t n, const uint32_t* heads, const uint32_t* word_pref,
                                 const uint64_t* chunk_base, int64_t* values, cudaStream_t stream) {
    if (n == 0) return FRZ_OK;
    k_rank_write<<<grid_for(n, kRankBlock), kRankBlock, 0, stream>>>(seg_of, n, heads, word_pref, chunk_base, values);
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}
