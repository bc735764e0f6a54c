// pack.cu — Arrow-style (bytes, offsets) → tile-bucketed, slot-major corpus (frz_device.cuh).
//
// Replaces the `&[S: AsRef<str>]` argument of Matcher::match_list (src/matcher/mod.rs:212):
// the reference chases one fat pointer per haystack; here the list is packed once and stays
// resident in HBM across queries.
#include "frz_device.cuh"
#include "frz_host.h"

#include <algorithm>

namespace {

// ---- plan: one block per tile: bucket by unit count, emit slot metadata + group descriptors ----
// `offsets` points at the entry of haystack `idx0` (the first haystack of tile `tile0`); n is the global count.
template <typename OffT>
__global__ void __launch_bounds__(256) k_pack_plan(const OffT* __restrict__ offsets, uint64_t n, uint32_t tile0, uint64_t idx0,
                                                   uint32_t* __restrict__ slot_meta, uint16_t* __restrict__ slot_of,
                                                   FrzGroupDesc* __restrict__ groups, uint64_t* __restrict__ tile_units,
                                                   unsigned int* __restrict__ err) {
    __shared__ uint32_t key[FRZ_TILE];
    __shared__ uint32_t len_s[FRZ_TILE];
    __shared__ uint32_t gun[FRZ_GROUPS_PER_TILE];
    const uint32_t tile = tile0 + blockIdx.x;
    const uint64_t base = (uint64_t)tile * FRZ_TILE;
    for (int i = threadIdx.x; i < FRZ_TILE; i += blockDim.x) {
        uint64_t idx = base + i;
        if (idx < n) {
            uint64_t len = (uint64_t)offsets[idx - idx0 + 1] - (uint64_t)offsets[idx - idx0];
            if (len > FRZ_MAX_HAY_LEN) { atomicOr(err, 1u); len = FRZ_MAX_HAY_LEN; }
            uint32_t units = (uint32_t)((len + FRZ_UNIT - 1) / FRZ_UNIT);
            len_s[i] = (uint32_t)len;
            key[i] = (units << FRZ_TILE_SHIFT) | (uint32_t)i;   // units < 2^18, stable via index bits
        } else {
            len_s[i] = 0;
            key[i] = 0xFFFFFFFFu;
        }
    }
    __syncthreads();
    // bitonic sort of 1024 keys (ascending)
    for (int k = 2; k <= FRZ_TILE; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < FRZ_TILE; i += blockDim.x) {
                int ixj = i ^ j;
                if (ixj > i) {
                    uint32_t a = key[i], b = key[ixj];
                    bool up = (i & k) == 0;
                    if ((a > b) == up) { key[i] = b; key[ixj] = a; }
                }
            }
            __syncthreads();
        }
    }
    for (int s = threadIdx.x; s < FRZ_TILE; s += blockDim.x) {
        uint32_t kk = key[s];
        if (kk == 0xFFFFFFFFu) {
            slot_meta[base + s] = FRZ_INVALID_SLOT;
        } else {
            uint32_t li = kk & (FRZ_TILE - 1);
            slot_meta[base + s] = (len_s[li] << FRZ_TILE_SHIFT) | li;
            slot_of[base + li] = (uint16_t)s;
        }
        if (base + s >= n) slot_of[base + s] = 0;  // indices past the end of the list
    }
    if (threadIdx.x < FRZ_GROUPS_PER_TILE) {
        // ascending order ⇒ the last valid lane of the group carries the group's max
        uint32_t g = threadIdx.x, mx = 0;
        for (int l = FRZ_GROUP - 1; l >= 0; l--) {
            uint32_t kk = key[g * FRZ_GROUP + l];
            if (kk != 0xFFFFFFFFu) { mx = kk >> FRZ_TILE_SHIFT; break; }
        }
        gun[g] = mx;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t off = 0, longest = 0;
        for (int g = 0; g < FRZ_GROUPS_PER_TILE; g++) {
            groups[tile * FRZ_GROUPS_PER_TILE + g] = FrzGroupDesc{0ull, off, gun[g]};  // abs_off filled by k_pack_copy
            off += gun[g] * FRZ_GROUP;
            longest = max(longest, gun[g]);   // (the groups ascend, but the trailing groups of a partial last tile are empty)
        }
        atomicMax(err + 1, longest);   // longest haystack of the corpus, in units: kernels stage / specialise on it
        tile_units[tile] = off;
    }
}

// ---- exclusive scan of per-tile unit counts (single block; n_tiles is N/1024) ----
__global__ void __launch_bounds__(1024) k_scan_u64(const uint64_t* __restrict__ in, uint64_t* __restrict__ out,
                                                   uint32_t n, uint64_t carry_in, uint64_t* __restrict__ total) {
    __shared__ uint64_t warp_sum[32];
    __shared__ uint64_t carry_s;
    if (threadIdx.x == 0) carry_s = carry_in;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += blockDim.x) {
        uint32_t i = base + threadIdx.x;
        uint64_t v = i < n ? in[i] : 0;
        uint64_t x = v;
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
            warp_sum[threadIdx.x] = xs - w;  // exclusive
        }
        __syncthreads();
        uint64_t c = carry_s;
        uint64_t incl = c + warp_sum[threadIdx.x >> 5] + x;
        if (i < n) out[i] = incl - v;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry_s = incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry_s;
}

__device__ __forceinline__ uint32_t load_word_safe(const uint8_t* bytes, uint64_t pos, uint64_t total_bytes) {
    // little-endian word at byte position `pos` (pos % 4 == alignment of bytes base assumed by caller)
    if (pos + 4 <= total_bytes) return *reinterpret_cast<const uint32_t*>(bytes + pos);
    uint32_t w = 0;
    for (int b = 0; b < 4; b++)
        if (pos + b < total_bytes) w |= (uint32_t)bytes[pos + b] << (8 * b);
    return w;
}

// ---- copy: one block per tile; thread per output unit so the 16-byte stores are coalesced ----
// `bytes` holds the byte range [off0, off0 + total_bytes) of the caller's value buffer; `offsets` points at the
// entry of haystack `idx0`.  Words past a haystack's end may belong to a chunk that is still in flight on the
// copy engine: they are read (inside the buffer) and masked off, never used.
template <typename OffT>
__global__ void __launch_bounds__(256) k_pack_copy(const uint8_t* __restrict__ bytes, const OffT* __restrict__ offsets,
                                                   uint32_t tile0, uint64_t idx0, uint64_t off0, uint64_t total_bytes,
                                                   const uint32_t* __restrict__ slot_meta,
                                                   FrzGroupDesc* __restrict__ groups, const uint64_t* __restrict__ tile_base,
                                                   uint4* __restrict__ data) {
    __shared__ uint32_t goff[FRZ_GROUPS_PER_TILE + 1];
    const uint32_t tile = tile0 + blockIdx.x;
    if (threadIdx.x < FRZ_GROUPS_PER_TILE) {
        FrzGroupDesc gd = groups[tile * FRZ_GROUPS_PER_TILE + threadIdx.x];
        goff[threadIdx.x] = gd.unit_off;
        if (threadIdx.x == FRZ_GROUPS_PER_TILE - 1) goff[FRZ_GROUPS_PER_TILE] = gd.unit_off + gd.gunits * FRZ_GROUP;
    }
    __syncthreads();
    const uint32_t total_units = goff[FRZ_GROUPS_PER_TILE];
    const uint64_t tb = tile_base[tile];
    if (threadIdx.x < FRZ_GROUPS_PER_TILE) groups[tile * FRZ_GROUPS_PER_TILE + threadIdx.x].abs_off = tb + goff[threadIdx.x];
    const uint64_t misalign = reinterpret_cast<uintptr_t>(bytes) & 3;  // base pointer alignment
    const uint8_t* abase = bytes - misalign;                           // 4-byte aligned
    const uint64_t atotal = total_bytes + misalign;
    for (uint32_t u = threadIdx.x; u < total_units; u += blockDim.x) {
        // group of unit u: largest g with goff[g] <= u (groups with gunits == 0 share an offset)
        int lo = 0, hi = FRZ_GROUPS_PER_TILE - 1;
        while (lo < hi) {
            int mid = (lo + hi + 1) >> 1;
            if (goff[mid] <= u) lo = mid; else hi = mid - 1;
        }
        // skip empty groups that start at the same offset: pick the one whose range contains u
        while (lo < FRZ_GROUPS_PER_TILE - 1 && goff[lo + 1] <= u) lo++;
        // slot-major group: unit `rel` of the group is unit k of slot `lane`, gunits units per slot
        const uint32_t rel = u - goff[lo], gunits = (goff[lo + 1] - goff[lo]) >> 5;
        const uint32_t lane = rel / gunits, k = rel - lane * gunits;
        uint32_t meta = slot_meta[(uint64_t)tile * FRZ_TILE + lo * FRZ_GROUP + lane];
        uint4 v = make_uint4(0, 0, 0, 0);
        if (meta != FRZ_INVALID_SLOT) {
            uint32_t len = meta >> FRZ_TILE_SHIFT;
            uint64_t idx = (uint64_t)tile * FRZ_TILE + (meta & (FRZ_TILE - 1));
            uint32_t b0 = k * FRZ_UNIT;
            if (b0 < len) {
                uint64_t src = (uint64_t)offsets[idx - idx0] - off0 + b0 + misalign;   // position in the aligned view
                uint32_t nvalid = min(len - b0, (uint32_t)FRZ_UNIT);
                uint64_t a = src & ~3ull;
                uint32_t sh = (uint32_t)(src & 3) * 8;
                uint32_t w[5];
#pragma unroll
                for (int j = 0; j < 5; j++) w[j] = load_word_safe(abase, a + 4 * j, atotal);
                uint32_t o[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    o[j] = __funnelshift_r(w[j], w[j + 1], sh);
                    int rem = (int)nvalid - 4 * j;
                    if (rem <= 0) o[j] = 0;
                    else if (rem < 4) o[j] &= (1u << (8 * rem)) - 1;
                }
                v = make_uint4(o[0], o[1], o[2], o[3]);
            }
        }
        data[tb + u] = v;
    }
}

// ---- signature index: one warp per group, lane per slot; classifies the packed bytes of the slot's haystack ----
// .x = byte classes (frz_sig_bucket) that occur, .y = classes that occur at least twice.  The prefilter reads these
// 8 bytes per haystack first and touches the haystack's own bytes only when the needle's classes are all there
// (up to the typo budget) — prefilter.cu, phase A.
__global__ void __launch_bounds__(256) k_pack_sig(const uint4* __restrict__ data, const FrzGroupDesc* __restrict__ groups,
                                                  const uint32_t* __restrict__ slot_meta, uint32_t group0, uint32_t group1,
                                                  uint2* __restrict__ slot_sig) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t g = group0 + ((blockIdx.x * blockDim.x + threadIdx.x) >> 5); g < group1; g += warps) {
        const FrzGroupDesc gd = groups[g];
        const uint32_t meta = slot_meta[(uint64_t)g * FRZ_GROUP + lane];
        const uint32_t len = meta == FRZ_INVALID_SLOT ? 0u : meta >> FRZ_TILE_SHIFT;
        uint32_t p1 = 0, p2 = 0;
        const uint4* gp = data + frz_slot_unit0(gd, lane);
        for (uint32_t k = 0; k < gd.gunits; k++) {   // warp-uniform trip count; the warp walks one contiguous 32 * gunits * 16-byte block
            const uint4 v = __ldg(gp + k);
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int j = 0; j < 16; j++) {
                if (k * FRZ_UNIT + j < len) frz_sig_add(p1, p2, (w[j >> 2] >> ((j & 3) * 8)) & 0xffu);
            }
        }
        slot_sig[(uint64_t)g * FRZ_GROUP + lane] = make_uint2(p1, p2);
    }
}

}  // namespace

// ---- append support: the partial last tile is turned back into raw (bytes, offsets) so that it can be
// re-bucketed together with the appended haystacks.  One block; thread i owns haystack idx0 + i.
__global__ void __launch_bounds__(1024) k_tail_offsets(const uint32_t* __restrict__ slot_meta, const uint16_t* __restrict__ slot_of,
                                                       const uint64_t* __restrict__ tile_base, uint32_t tile, uint32_t cnt,
                                                       uint64_t* __restrict__ out_offsets, uint64_t* __restrict__ out_info) {
    __shared__ uint64_t wsum[32];
    const uint32_t i = threadIdx.x, lane = i & 31, warp = i >> 5;
    uint64_t len = 0;
    if (i < cnt) len = slot_meta[(uint64_t)tile * FRZ_TILE + slot_of[(uint64_t)tile * FRZ_TILE + i]] >> FRZ_TILE_SHIFT;
    uint64_t x = len;
    for (int d = 1; d < 32; d <<= 1) {
        uint64_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= (uint32_t)d) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint64_t w = wsum[lane], xs = w;
        for (int d = 1; d < 32; d <<= 1) {
            uint64_t y = __shfl_up_sync(0xffffffffu, xs, d);
            if (lane >= (uint32_t)d) xs += y;
        }
        wsum[lane] = xs - w;
    }
    __syncthreads();
    const uint64_t incl = wsum[warp] + x;
    if (i < cnt) out_offsets[i] = incl - len;
    if (i == FRZ_TILE - 1) {
        out_offsets[cnt] = incl;       // lanes >= cnt add 0: incl of the last thread is the total
        out_info[0] = incl;            // tail bytes
        out_info[1] = tile_base[tile]; // first unit of the tail tile
    }
}

__global__ void __launch_bounds__(256) k_tail_bytes(const uint4* __restrict__ data, const FrzGroupDesc* __restrict__ groups,
                                                    const uint32_t* __restrict__ slot_meta, const uint16_t* __restrict__ slot_of,
                                                    uint32_t tile, uint32_t cnt, const uint64_t* __restrict__ offsets,
                                                    uint8_t* __restrict__ out_bytes) {
    // one warp per haystack, lanes stride over its bytes
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const uint32_t n_warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = warp; i < cnt; i += n_warps) {
        const uint32_t slot = slot_of[(uint64_t)tile * FRZ_TILE + i];
        const uint32_t len = slot_meta[(uint64_t)tile * FRZ_TILE + slot] >> FRZ_TILE_SHIFT;
        const FrzGroupDesc gd = groups[tile * FRZ_GROUPS_PER_TILE + (slot >> 5)];
        const uint8_t* base = reinterpret_cast<const uint8_t*>(data + frz_slot_unit0(gd, slot & 31));
        uint8_t* dst = out_bytes + offsets[i];
        for (uint32_t b = lane; b < len; b += 32) dst[b] = base[b];
    }
}

template <typename OffT>
__global__ void k_rebase_offsets(const OffT* __restrict__ in, uint64_t n_new, const uint64_t* __restrict__ tail_info,
                                 uint64_t* __restrict__ out) {
    const uint64_t base = tail_info[0], off0 = (uint64_t)in[0];
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j <= n_new; j += (uint64_t)gridDim.x * blockDim.x)
        out[j] = base + ((uint64_t)in[j] - off0);
}

// ------------------------------------------------------------------------------------------------
// Host-side staging.  Three steps so that a streamed ingest can interleave them with H2D chunks:
//   pack_reserve   metadata arrays for tiles [0, n_tiles)
//   pack_plan      bucket tiles [tile0, n_tiles) + running scan of the unit counts → total units (one small
//                  D2H + wait: the packed size is needed to size the data buffer) → grow the data buffer
//   pack_copy      tiles [t0, t1) from the staged bytes into the slot-major layout
namespace {

constexpr const char* kHayTooLong = "haystack longer than %u bytes";

frz_status pack_reserve(FrzCorpusStorage* out, uint32_t n_tiles, uint32_t keep_tiles, cudaStream_t stream) {
    const uint64_t cap = out->tile_base.cap();
    if (cap >= n_tiles) return FRZ_OK;
    const uint32_t want = keep_tiles ? std::max<uint32_t>(n_tiles, (uint32_t)(cap + cap / 2)) : n_tiles;
    const size_t slots = (size_t)want * FRZ_TILE;
    // new arrays next to the old ones, so that an append can carry the existing tiles' metadata over
    FrzDevArray<uint32_t> slot_meta; FrzDevArray<uint16_t> slot_of; FrzDevArray<uint2> slot_sig; FrzDevArray<FrzGroupDesc> groups;
    FrzDevArray<uint64_t> tile_base, scratch;
    FRZ_TRY(slot_meta.reserve(slots));
    FRZ_TRY(slot_of.reserve(slots));
    FRZ_TRY(slot_sig.reserve(slots));
    FRZ_TRY(groups.reserve((size_t)want * FRZ_GROUPS_PER_TILE));
    FRZ_TRY(tile_base.reserve(want));
    FRZ_TRY(scratch.reserve((size_t)want + 2));
    if (keep_tiles) {
        const size_t ks = (size_t)keep_tiles * FRZ_TILE;
        FRZ_CUDA_TRY(cudaMemcpyAsync(slot_meta.get(), out->slot_meta.get(), ks * sizeof(uint32_t), cudaMemcpyDeviceToDevice, stream));
        FRZ_CUDA_TRY(cudaMemcpyAsync(slot_of.get(), out->slot_of.get(), ks * sizeof(uint16_t), cudaMemcpyDeviceToDevice, stream));
        FRZ_CUDA_TRY(cudaMemcpyAsync(slot_sig.get(), out->slot_sig.get(), ks * sizeof(uint2), cudaMemcpyDeviceToDevice, stream));
        FRZ_CUDA_TRY(cudaMemcpyAsync(groups.get(), out->groups.get(), (size_t)keep_tiles * FRZ_GROUPS_PER_TILE * sizeof(FrzGroupDesc), cudaMemcpyDeviceToDevice, stream));
        FRZ_CUDA_TRY(cudaMemcpyAsync(tile_base.get(), out->tile_base.get(), (size_t)keep_tiles * sizeof(uint64_t), cudaMemcpyDeviceToDevice, stream));
        FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    }
    out->slot_meta = std::move(slot_meta); out->slot_of = std::move(slot_of); out->slot_sig = std::move(slot_sig);
    out->groups = std::move(groups); out->tile_base = std::move(tile_base); out->scratch_tile_units = std::move(scratch);
    return FRZ_OK;
}

// carry_in = first free unit (0 for a fresh pack, the first unit of the re-packed tail tile on append)
template <typename OffT>
frz_status pack_plan(FrzCorpusStorage* out, const OffT* d_offsets, uint64_t n, uint32_t tile0, uint64_t idx0, uint64_t carry_in,
                     bool keep_data, cudaStream_t stream) {
    const uint32_t n_tiles = out->n_tiles;
    uint64_t* d_tile_units = out->scratch_tile_units.get();
    uint64_t* d_total = d_tile_units + out->tile_base.cap();
    unsigned int* d_err = reinterpret_cast<unsigned int*>(d_total + 1);
    FRZ_CUDA_TRY(cudaMemsetAsync(d_total, 0, 16, stream));
    k_pack_plan<OffT><<<n_tiles - tile0, 256, 0, stream>>>(d_offsets, n, tile0, idx0, out->slot_meta.get(), out->slot_of.get(),
                                                          out->groups.get(), d_tile_units, d_err);
    k_scan_u64<<<1, 1024, 0, stream>>>(d_tile_units + tile0, out->tile_base.get() + tile0, n_tiles - tile0, carry_in, d_total);
    uint64_t h[2] = {0, 0};
    FRZ_CUDA_TRY(cudaMemcpyAsync(h, d_total, 16, cudaMemcpyDeviceToHost, stream));
    FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    if ((unsigned int)(h[1] & 0xffffffffu)) return frz_fail(FRZ_ERR_UNSUPPORTED, kHayTooLong, FRZ_MAX_HAY_LEN);
    out->total_units = h[0];
    out->max_gunits = std::max<uint32_t>(tile0 ? out->max_gunits : 0u, (uint32_t)(h[1] >> 32));
    if (out->data.cap() < out->total_units + 1) {
        FrzDevArray<uint4> data;
        FRZ_TRY(data.reserve(out->total_units + out->total_units / (keep_data ? 2 : 16) + 1024));
        if (keep_data && carry_in) {
            FRZ_CUDA_TRY(cudaMemcpyAsync(data.get(), out->data.get(), (size_t)carry_in * sizeof(uint4), cudaMemcpyDeviceToDevice, stream));
            FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
        }
        out->data = std::move(data);
    }
    return FRZ_OK;
}

template <typename OffT>
frz_status pack_copy(FrzCorpusStorage* out, const uint8_t* d_bytes, const OffT* d_offsets, uint32_t tile0, uint64_t idx0,
                     uint64_t off0, uint64_t total_bytes, uint32_t t0, uint32_t t1, cudaStream_t stream) {
    if (t1 <= t0) return FRZ_OK;
    (void)tile0;
    k_pack_copy<OffT><<<t1 - t0, 256, 0, stream>>>(d_bytes, d_offsets, t0, idx0, off0, total_bytes, out->slot_meta.get(),
                                                  out->groups.get(), out->tile_base.get(), out->data.get());
    // signature index of the same tiles, from the bytes just interleaved (L2-resident for a streamed chunk)
    const uint32_t g0 = t0 * FRZ_GROUPS_PER_TILE, g1 = t1 * FRZ_GROUPS_PER_TILE;
    const uint32_t sig_blocks = std::min<uint32_t>((g1 - g0 + 7) / 8, frz_sm_count() * 8);
    k_pack_sig<<<sig_blocks, 256, 0, stream>>>(out->data.get(), out->groups.get(), out->slot_meta.get(), g0, g1, out->slot_sig.get());
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

// `d_bytes` is the value buffer the offsets index (haystack i = d_bytes[d_offsets[i], d_offsets[i + 1])), and
// total_bytes = d_offsets[n] - d_offsets[0]; the first and last offsets are read back to check it.
template <typename OffT>
frz_status pack_device_t(const uint8_t* d_bytes, const OffT* d_offsets, uint64_t n, uint64_t total_bytes, cudaStream_t stream,
                         FrzCorpusStorage* out) {
    const uint32_t n_tiles = (uint32_t)((n + FRZ_TILE - 1) / FRZ_TILE);
    if (n_tiles == 0) { out->n = 0; out->n_tiles = 0; out->total_bytes = 0; out->total_units = 0; return FRZ_OK; }
    OffT ends[2] = {0, 0};
    FRZ_CUDA_TRY(cudaMemcpyAsync(&ends[0], d_offsets, sizeof(OffT), cudaMemcpyDeviceToHost, stream));
    FRZ_CUDA_TRY(cudaMemcpyAsync(&ends[1], d_offsets + n, sizeof(OffT), cudaMemcpyDeviceToHost, stream));
    FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    const uint64_t off0 = (uint64_t)ends[0];
    if ((uint64_t)ends[1] < off0 || (uint64_t)ends[1] - off0 != total_bytes)
        return frz_fail(FRZ_ERR_INVALID_ARG, "total_bytes %llu != d_offsets[n] - d_offsets[0] = %llu - %llu", (unsigned long long)total_bytes,
                        (unsigned long long)ends[1], (unsigned long long)off0);
    out->n = n;
    out->n_tiles = n_tiles;
    out->total_bytes = total_bytes;
    FRZ_TRY(pack_reserve(out, n_tiles, 0, stream));
    FRZ_TRY(pack_plan<OffT>(out, d_offsets, n, 0, 0, 0, false, stream));
    return pack_copy<OffT>(out, d_bytes + off0, d_offsets, 0, 0, off0, total_bytes, 0, n_tiles, stream);
}

// Streamed ingest: offsets first, then the value bytes in tile-aligned chunks on a copy stream; the plan runs
// while the first chunks are in flight and every chunk is interleaved as soon as it has landed.
template <typename OffT>
frz_status ingest_host_t(FrzIngest& ing, const uint8_t* h_bytes, const OffT* h_offsets, uint64_t n, cudaStream_t stream,
                         FrzCorpusStorage* out, FrzChunkFn after_chunk, void* ctx) {
    const uint64_t off0 = (uint64_t)h_offsets[0];
    const uint64_t total = (uint64_t)h_offsets[n] - off0;
    const uint32_t n_tiles = (uint32_t)((n + FRZ_TILE - 1) / FRZ_TILE);
    out->n = n;
    out->n_tiles = n_tiles;
    out->total_bytes = total;
    if (n_tiles == 0) { out->total_units = 0; return FRZ_OK; }
    FRZ_TRY(ing.reserve(total, (n + 1) * sizeof(OffT)));
    FRZ_TRY(pack_reserve(out, n_tiles, 0, stream));
    OffT* d_off = reinterpret_cast<OffT*>(ing.d_offsets.get());
    cudaStream_t copy = ing.copy_stream.get();
    cudaEvent_t arena_ev = ing.ev[FrzIngest::kMaxChunks].get();
    // everything already queued on `stream` (a previous call's kernels reading the arena) must finish first
    FRZ_CUDA_TRY(cudaEventRecord(arena_ev, stream));
    FRZ_CUDA_TRY(cudaStreamWaitEvent(copy, arena_ev, 0));
    FRZ_CUDA_TRY(cudaMemcpyAsync(d_off, h_offsets, (n + 1) * sizeof(OffT), cudaMemcpyHostToDevice, copy));
    FRZ_CUDA_TRY(cudaEventRecord(arena_ev, copy));
    // chunk plan: tile-aligned, about equal byte counts, at least kMinChunk bytes each
    int n_chunks = (int)std::min<uint64_t>(FrzIngest::kMaxChunks, std::max<uint64_t>(1, total / FrzIngest::kMinChunkBytes));
    n_chunks = (int)std::min<uint64_t>(n_chunks, n_tiles);
    uint32_t bounds[FrzIngest::kMaxChunks + 1];
    bounds[0] = 0;
    for (int c = 1; c <= n_chunks; c++) {
        uint32_t t = (uint32_t)((uint64_t)n_tiles * c / n_chunks);
        bounds[c] = c == n_chunks ? n_tiles : std::max(t, bounds[c - 1]);
    }
    for (int c = 0; c < n_chunks; c++) {
        const uint64_t i0 = std::min<uint64_t>((uint64_t)bounds[c] * FRZ_TILE, n), i1 = std::min<uint64_t>((uint64_t)bounds[c + 1] * FRZ_TILE, n);
        const uint64_t b0 = (uint64_t)h_offsets[i0] - off0, b1 = (uint64_t)h_offsets[i1] - off0;
        if (b1 > b0) FRZ_CUDA_TRY(cudaMemcpyAsync(ing.d_bytes.get() + b0, h_bytes + off0 + b0, b1 - b0, cudaMemcpyHostToDevice, copy));
        FRZ_CUDA_TRY(cudaEventRecord(ing.ev[c].get(), copy));
    }
    FRZ_CUDA_TRY(cudaStreamWaitEvent(stream, arena_ev, 0));
    FRZ_TRY(pack_plan<OffT>(out, d_off, n, 0, 0, 0, false, stream));   // waits for the plan only; the byte chunks keep flowing
    for (int c = 0; c < n_chunks; c++) {
        FRZ_CUDA_TRY(cudaStreamWaitEvent(stream, ing.ev[c].get(), 0));
        FRZ_TRY(pack_copy<OffT>(out, ing.d_bytes.get(), d_off, 0, 0, off0, total, bounds[c], bounds[c + 1], stream));
        if (after_chunk) FRZ_TRY(after_chunk(ctx, bounds[c], bounds[c + 1], c == n_chunks - 1));
    }
    return FRZ_OK;
}

// Incremental append (SURVEY §8(f) rank 1).  Tiles are independent, so only the partial last tile is
// re-bucketed: it is unpacked to raw bytes, the new haystacks are staged behind it, and tiles
// [n_old / 1024, n_tiles_new) are planned, scanned (carry = first unit of the old tail tile) and copied.
template <typename OffT>
frz_status append_host_t(FrzIngest& ing, const uint8_t* h_bytes, const OffT* h_offsets, uint64_t n_new, cudaStream_t stream,
                         FrzCorpusStorage* st) {
    if (n_new == 0) return FRZ_OK;
    const uint64_t n_old = st->n;
    const uint64_t n = n_old + n_new;
    if (n > 0xFFFFFFFFull) return frz_fail(FRZ_ERR_TOO_MANY_ITEMS, "too many items in haystack: %llu", (unsigned long long)n);
    // a refused append must leave the corpus as it was, so the lengths are checked here, before anything below
    // replaces the metadata of the old tail tile (pack_plan would find them only after that)
    for (uint64_t i = 0; i < n_new; i++)
        if ((uint64_t)h_offsets[i + 1] - (uint64_t)h_offsets[i] > FRZ_MAX_HAY_LEN)
            return frz_fail(FRZ_ERR_UNSUPPORTED, kHayTooLong, FRZ_MAX_HAY_LEN);
    const uint32_t t_last = (uint32_t)(n_old / FRZ_TILE), cnt = (uint32_t)(n_old % FRZ_TILE);
    const uint64_t idx0 = (uint64_t)t_last * FRZ_TILE;
    const uint64_t off0 = (uint64_t)h_offsets[0];
    const uint64_t new_bytes = (uint64_t)h_offsets[n_new] - off0;
    const uint32_t n_tiles = (uint32_t)((n + FRZ_TILE - 1) / FRZ_TILE);
    // staging layout in ing.d_offsets: [tail_info: 2 u64][staged offsets: cnt + n_new + 1 u64][raw new offsets]
    const uint64_t staged_words = 2 + (uint64_t)cnt + n_new + 1;
    FRZ_TRY(ing.reserve(0, staged_words * 8 + (n_new + 1) * sizeof(OffT) + 16));
    uint64_t* d_info = reinterpret_cast<uint64_t*>(ing.d_offsets.get());
    uint64_t* d_staged = d_info + 2;
    OffT* d_raw = reinterpret_cast<OffT*>(d_staged + cnt + n_new + 1);
    uint64_t info[2] = {0, st->total_units};
    if (cnt) {
        k_tail_offsets<<<1, 1024, 0, stream>>>(st->slot_meta.get(), st->slot_of.get(), st->tile_base.get(), t_last, cnt, d_staged, d_info);
        FRZ_CUDA_TRY(cudaMemcpyAsync(info, d_info, 16, cudaMemcpyDeviceToHost, stream));
        FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    } else {
        FRZ_CUDA_TRY(cudaMemcpyAsync(d_info, info, 16, cudaMemcpyHostToDevice, stream));
    }
    const uint64_t tail_bytes = info[0], carry_in = info[1];
    FRZ_TRY(ing.reserve(tail_bytes + new_bytes, 0));
    if (cnt)
        k_tail_bytes<<<32, 256, 0, stream>>>(st->data.get(), st->groups.get(), st->slot_meta.get(), st->slot_of.get(), t_last, cnt, d_staged,
                                             ing.d_bytes.get());
    if (new_bytes) FRZ_CUDA_TRY(cudaMemcpyAsync(ing.d_bytes.get() + tail_bytes, h_bytes + off0, new_bytes, cudaMemcpyHostToDevice, stream));
    FRZ_CUDA_TRY(cudaMemcpyAsync(d_raw, h_offsets, (n_new + 1) * sizeof(OffT), cudaMemcpyHostToDevice, stream));
    k_rebase_offsets<OffT><<<256, 256, 0, stream>>>(d_raw, n_new, d_info, d_staged + cnt);
    FRZ_CUDA_TRY(cudaGetLastError());
    FRZ_TRY(pack_reserve(st, n_tiles, t_last, stream));
    st->n = n;
    st->n_tiles = n_tiles;
    st->total_bytes += new_bytes;
    FRZ_TRY(pack_plan<uint64_t>(st, d_staged, n, t_last, idx0, carry_in, true, stream));
    return pack_copy<uint64_t>(st, ing.d_bytes.get(), d_staged, t_last, idx0, 0, tail_bytes + new_bytes, t_last, n_tiles, stream);
}

}  // namespace

frz_status FrzIngest::reserve(uint64_t bytes, uint64_t offset_bytes) {
    if (!ev[kMaxChunks]) {   // created last: a failed set-up is redone by the next call
        FRZ_TRY(frz_stream_create(copy_stream, cudaStreamNonBlocking));
        for (auto& e : ev) FRZ_TRY(frz_event_create(e, cudaEventDisableTiming));
    }
    FRZ_TRY(d_bytes.reserve(bytes + 16, bytes + bytes / 16 + 4096));
    FRZ_TRY(d_offsets.reserve(offset_bytes, offset_bytes + offset_bytes / 16 + 4096));
    return FRZ_OK;
}

// Builds the packed corpus from device-resident Arrow buffers (64- or 32-bit offsets).  Asynchronous on
// `stream` except for one small D2H copy (the packed size), which it has to wait for to allocate.
frz_status frz_pack_corpus_device(const uint8_t* d_bytes, const void* d_offsets, int offset_width, uint64_t n, uint64_t total_bytes,
                                  cudaStream_t stream, FrzCorpusStorage* out) {
    if (offset_width == 4) return pack_device_t<uint32_t>(d_bytes, static_cast<const uint32_t*>(d_offsets), n, total_bytes, stream, out);
    return pack_device_t<uint64_t>(d_bytes, static_cast<const uint64_t*>(d_offsets), n, total_bytes, stream, out);
}

// Streams host Arrow buffers (ideally pinned) into a packed corpus: H2D chunks overlap the bucketing kernels.
frz_status frz_ingest_host(FrzIngest& ing, const uint8_t* h_bytes, const void* h_offsets, int offset_width, uint64_t n,
                           cudaStream_t stream, FrzCorpusStorage* out, FrzChunkFn after_chunk, void* ctx) {
    if (offset_width == 4) return ingest_host_t<uint32_t>(ing, h_bytes, static_cast<const uint32_t*>(h_offsets), n, stream, out, after_chunk, ctx);
    return ingest_host_t<uint64_t>(ing, h_bytes, static_cast<const uint64_t*>(h_offsets), n, stream, out, after_chunk, ctx);
}

// Appends host Arrow buffers to a packed corpus; indices of the new haystacks continue at the old length.
frz_status frz_append_host(FrzIngest& ing, const uint8_t* h_bytes, const void* h_offsets, int offset_width, uint64_t n_new,
                           cudaStream_t stream, FrzCorpusStorage* st) {
    if (offset_width == 4) return append_host_t<uint32_t>(ing, h_bytes, static_cast<const uint32_t*>(h_offsets), n_new, stream, st);
    return append_host_t<uint64_t>(ing, h_bytes, static_cast<const uint64_t*>(h_offsets), n_new, stream, st);
}
