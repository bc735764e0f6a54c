// pack.cu — Arrow-style (bytes, offsets) → tile-bucketed, slot-major corpus (frz_device.cuh).
//
// Replaces the `&[S: AsRef<str>]` argument of Matcher::match_list (src/matcher/mod.rs:212):
// the reference chases one fat pointer per haystack; here the list is packed once and stays
// resident in HBM across queries.
#include "frz_device.cuh"
#include "frz_host.h"

#include <algorithm>
#include <vector>

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

// ---- unpack: packed tiles turned back into raw (bytes, offsets), so that they can be re-bucketed — the partial last tile
// with the haystacks an append adds behind it, or any list of tiles whose haystacks a replace changes.  Staged haystack
// s = b * 1024 + i is local index i of tiles[b]; the last listed tile holds `last_cnt` haystacks, the others 1024.  A
// replaced haystack (repl[s] = its position in the replacement list) is staged with its new bytes; a removed one that is
// not replaced is staged empty and flagged in `dead`, so that the re-packed tile keeps it removed.
constexpr uint32_t kNoRepl = 0xFFFFFFFFu;
// words of the unpack's info block (device, zeroed by the caller)
enum : int { kInfoOldBytes = 0,   // live bytes the replaced haystacks had
             kInfoRevived = 1,    // replaced haystacks that had been removed
             kInfoOldUnits = 2,   // units the listed tiles occupied
             kInfoTileBase = 3,   // first and one-past-last unit of the (single) listed tile: the append's tail rule
             kInfoTileEnd = 4,
             kInfoStaged = 5,     // staged bytes
             kInfoWords = 8 };

// One block per listed tile: lengths → local exclusive offsets (staged_off[s]) and the tile's byte count (tile_sum[b]).
__global__ void __launch_bounds__(1024) k_unpack_offsets(const uint32_t* __restrict__ slot_meta, const uint16_t* __restrict__ slot_of,
                                                         const FrzGroupDesc* __restrict__ groups, const uint64_t* __restrict__ tile_base,
                                                         const uint32_t* __restrict__ tiles, uint32_t n_list, uint32_t last_cnt,
                                                         const uint32_t* __restrict__ repl, const uint64_t* __restrict__ r_off,
                                                         uint64_t* __restrict__ out_offsets, uint64_t* __restrict__ tile_sum,
                                                         uint8_t* __restrict__ dead, unsigned long long* __restrict__ info) {
    __shared__ uint64_t wsum[32];
    const uint32_t i = threadIdx.x, lane = i & 31, warp = i >> 5, b = blockIdx.x;
    const uint64_t tile = tiles[b];
    const uint32_t cnt = b == n_list - 1 ? last_cnt : FRZ_TILE;
    const uint64_t s = (uint64_t)b * FRZ_TILE + i;
    uint64_t len = 0;
    if (i < cnt) {
        const uint32_t meta = slot_meta[tile * FRZ_TILE + slot_of[tile * FRZ_TILE + i]];
        const uint32_t r = repl ? repl[s] : kNoRepl;
        if (r != kNoRepl) {
            len = r_off[r + 1] - r_off[r];
            if (meta != FRZ_INVALID_SLOT) atomicAdd(info + kInfoOldBytes, (unsigned long long)(meta >> FRZ_TILE_SHIFT));
            else atomicAdd(info + kInfoRevived, 1ull);
        } else if (meta != FRZ_INVALID_SLOT) {
            len = meta >> FRZ_TILE_SHIFT;
        }
        dead[s] = r == kNoRepl && meta == FRZ_INVALID_SLOT;
    }
    if (i == 0) {
        const FrzGroupDesc last = groups[tile * FRZ_GROUPS_PER_TILE + FRZ_GROUPS_PER_TILE - 1];
        const uint64_t units = (uint64_t)last.unit_off + (uint64_t)last.gunits * FRZ_GROUP;
        atomicAdd(info + kInfoOldUnits, (unsigned long long)units);
        if (n_list == 1) {
            info[kInfoTileBase] = tile_base[tile];
            info[kInfoTileEnd] = tile_base[tile] + units;
        }
    }
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
    if (i < cnt) out_offsets[s] = incl - len;
    if (i == FRZ_TILE - 1) tile_sum[b] = incl;   // lanes >= cnt add 0: incl of the last thread is the tile's total
}

// One warp per staged haystack: its offset becomes global (tile_sum holds the tiles' exclusive scan by now) and its bytes
// are copied from the packed tile, or from the uploaded replacement bytes r_bytes[r_off[r], r_off[r + 1]).
__global__ void __launch_bounds__(256) k_unpack_bytes(const uint4* __restrict__ data, const FrzGroupDesc* __restrict__ groups,
                                                      const uint32_t* __restrict__ slot_meta, const uint16_t* __restrict__ slot_of,
                                                      const uint32_t* __restrict__ tiles, uint64_t staged_n,
                                                      const uint32_t* __restrict__ repl, const uint64_t* __restrict__ r_off,
                                                      const uint8_t* __restrict__ r_bytes, const uint8_t* __restrict__ dead,
                                                      const uint64_t* __restrict__ tile_sum, uint64_t* __restrict__ offsets,
                                                      uint8_t* __restrict__ out_bytes) {
    // lanes stride over the haystack's bytes
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t s = warp; s < staged_n; s += n_warps) {
        const uint64_t tile = tiles[s >> FRZ_TILE_SHIFT];
        const uint32_t i = (uint32_t)(s & (FRZ_TILE - 1));
        const uint64_t at = tile_sum[s >> FRZ_TILE_SHIFT] + offsets[s];
        __syncwarp();
        if (lane == 0) offsets[s] = at;
        uint8_t* dst = out_bytes + at;
        const uint32_t r = repl ? repl[s] : kNoRepl;
        if (r != kNoRepl) {
            const uint64_t b0 = r_off[r], len = r_off[r + 1] - b0;
            for (uint64_t b = lane; b < len; b += 32) dst[b] = r_bytes[b0 + b];
        } else if (!dead[s]) {
            const uint32_t slot = slot_of[tile * FRZ_TILE + i];
            const uint32_t len = slot_meta[tile * FRZ_TILE + slot] >> FRZ_TILE_SHIFT;
            const FrzGroupDesc gd = groups[tile * FRZ_GROUPS_PER_TILE + (slot >> 5)];
            const uint8_t* base = reinterpret_cast<const uint8_t*>(data + frz_slot_unit0(gd, slot & 31));
            for (uint32_t b = lane; b < len; b += 32) dst[b] = base[b];
        }
    }
}

// repl[slot_pos[j]] = j: where replacement j lands among the staged haystacks
__global__ void k_mark_repl(const uint32_t* __restrict__ slot_pos, uint64_t n, uint32_t* __restrict__ repl) {
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x)
        repl[slot_pos[j]] = (uint32_t)j;
}

// After the re-pack: a staged haystack flagged dead is removed again (it was packed as an empty haystack).
__global__ void k_mark_dead(const uint8_t* __restrict__ dead, uint64_t staged_n, const uint32_t* __restrict__ tiles,
                            const uint16_t* __restrict__ slot_of, uint32_t* __restrict__ slot_meta) {
    for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < staged_n; s += (uint64_t)gridDim.x * blockDim.x) {
        if (!dead[s]) continue;
        const uint64_t tile = tiles[s >> FRZ_TILE_SHIFT];
        slot_meta[tile * FRZ_TILE + slot_of[tile * FRZ_TILE + (s & (FRZ_TILE - 1))]] = FRZ_INVALID_SLOT;
    }
}

// One block per re-packed tile: its metadata, planned as tile b of a scratch corpus, replaces that of tiles[b].
__global__ void __launch_bounds__(256) k_scatter_tiles(const uint32_t* __restrict__ tiles, const uint64_t* __restrict__ s_tile_base,
                                                       const FrzGroupDesc* __restrict__ s_groups, const uint32_t* __restrict__ s_meta,
                                                       const uint16_t* __restrict__ s_of, const uint2* __restrict__ s_sig,
                                                       uint64_t* __restrict__ tile_base, FrzGroupDesc* __restrict__ groups,
                                                       uint32_t* __restrict__ slot_meta, uint16_t* __restrict__ slot_of,
                                                       uint2* __restrict__ slot_sig) {
    const uint64_t b = blockIdx.x, t = tiles[b];
    if (threadIdx.x == 0) tile_base[t] = s_tile_base[b];
    if (threadIdx.x < FRZ_GROUPS_PER_TILE)
        groups[t * FRZ_GROUPS_PER_TILE + threadIdx.x] = s_groups[b * FRZ_GROUPS_PER_TILE + threadIdx.x];
    for (uint32_t i = threadIdx.x; i < FRZ_TILE; i += blockDim.x) {
        slot_meta[t * FRZ_TILE + i] = s_meta[b * FRZ_TILE + i];
        slot_of[t * FRZ_TILE + i] = s_of[b * FRZ_TILE + i];
        slot_sig[t * FRZ_TILE + i] = s_sig[b * FRZ_TILE + i];
    }
}

// Removal: the slot's metadata becomes FRZ_INVALID_SLOT, which every scan already skips.  info[0] counts the haystacks
// this call removed (a duplicate or an already removed one counts once), info[1] sums their lengths.
__global__ void k_remove(const uint32_t* __restrict__ which, uint64_t n, const uint16_t* __restrict__ slot_of,
                         uint32_t* __restrict__ slot_meta, unsigned long long* __restrict__ info) {
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t idx = which[j], tile = idx >> FRZ_TILE_SHIFT;
        const uint32_t old = atomicExch(slot_meta + tile * FRZ_TILE + slot_of[idx], FRZ_INVALID_SLOT);
        if (old != FRZ_INVALID_SLOT) {
            atomicAdd(info, 1ull);
            atomicAdd(info + 1, (unsigned long long)(old >> FRZ_TILE_SHIFT));
        }
    }
}

// units of every tile, from its last group (the compaction's input)
__global__ void k_tile_units(const FrzGroupDesc* __restrict__ groups, uint32_t n_tiles, uint64_t* __restrict__ out) {
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n_tiles; t += (uint64_t)gridDim.x * blockDim.x) {
        const FrzGroupDesc g = groups[t * FRZ_GROUPS_PER_TILE + FRZ_GROUPS_PER_TILE - 1];
        out[t] = (uint64_t)g.unit_off + (uint64_t)g.gunits * FRZ_GROUP;
    }
}

// Compaction: one block per tile copies its units to new_base[t] of a fresh arena and points tile_base / abs_off there.
__global__ void __launch_bounds__(256) k_compact(const uint4* __restrict__ old_data, uint4* __restrict__ new_data,
                                                 FrzGroupDesc* __restrict__ groups, uint64_t* __restrict__ tile_base,
                                                 const uint64_t* __restrict__ new_base) {
    const uint64_t t = blockIdx.x;
    const uint64_t ob = tile_base[t], nb = new_base[t];
    const FrzGroupDesc last = groups[t * FRZ_GROUPS_PER_TILE + FRZ_GROUPS_PER_TILE - 1];
    const uint64_t units = (uint64_t)last.unit_off + (uint64_t)last.gunits * FRZ_GROUP;
    __syncthreads();   // every thread has read the old tile_base / descriptors before they are rewritten below
    for (uint64_t u = threadIdx.x; u < units; u += blockDim.x) new_data[nb + u] = old_data[ob + u];
    if (threadIdx.x < FRZ_GROUPS_PER_TILE) {
        FrzGroupDesc& g = groups[t * FRZ_GROUPS_PER_TILE + threadIdx.x];
        g.abs_off = nb + g.unit_off;
    }
    if (threadIdx.x == 0) tile_base[t] = nb;
}

// longest group of the corpus, in units per slot (FrzCorpusView::max_gunits)
__global__ void k_max_gunits(const FrzGroupDesc* __restrict__ groups, uint64_t n_groups, unsigned int* __restrict__ out) {
    uint32_t mx = 0;
    for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += (uint64_t)gridDim.x * blockDim.x)
        mx = max(mx, groups[g].gunits);
    for (int d = 16; d > 0; d >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, d));
    if ((threadIdx.x & 31) == 0 && mx) atomicMax(out, mx);
}

template <typename OffT>
__global__ void k_rebase_offsets(const OffT* __restrict__ in, uint64_t n_new, const unsigned long long* __restrict__ base_ptr,
                                 uint64_t* __restrict__ out) {
    const uint64_t base = *base_ptr, off0 = (uint64_t)in[0];
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

// Carves the staging buffer ing.d_offsets into 16-byte aligned pieces.
struct Carve {
    uint8_t* p;
    template <typename T>
    T* take(uint64_t count) {
        T* r = reinterpret_cast<T*>(p);
        p += (count * sizeof(T) + 15) & ~15ull;
        return r;
    }
    static uint64_t size(uint64_t count, uint64_t elem) { return (count * elem + 15) & ~15ull; }
};

// Device buffers of one unpack: staged haystack s = b * 1024 + i is local index i of tiles[b] (see k_unpack_offsets).
struct Unpack {
    unsigned long long* info;   // kInfoWords words
    uint64_t* staged;           // offsets of the staged haystacks (and of an append's new ones behind them)
    uint64_t* tile_sum;         // [n_list] bytes per listed tile → their exclusive scan
    uint32_t* tiles;            // [n_list] ascending; the partial last tile of the corpus can only come last
    uint8_t* dead;              // [n_list * 1024]
    uint32_t* repl = nullptr;   // [n_list * 1024] or nullptr (no replacements)
    uint64_t* r_off = nullptr;  // replacement offsets (from 0)
    uint32_t n_list = 0, last_cnt = 0;
    uint64_t staged_n() const { return (uint64_t)(n_list - 1) * FRZ_TILE + last_cnt; }
};

// Step 1 of an unpack: offsets of the staged haystacks, their total in info[kInfoStaged] and staged[staged_n()], and
// the info block back on the host (the byte count sizes the staging buffer).
frz_status unpack_offsets(const FrzCorpusStorage* st, const Unpack& u, cudaStream_t stream, uint64_t h_info[kInfoWords]) {
    FRZ_CUDA_TRY(cudaMemsetAsync(u.info, 0, kInfoWords * sizeof(uint64_t), stream));
    k_unpack_offsets<<<u.n_list, 1024, 0, stream>>>(st->slot_meta.get(), st->slot_of.get(), st->groups.get(), st->tile_base.get(), u.tiles,
                                                    u.n_list, u.last_cnt, u.repl, u.r_off, u.staged, u.tile_sum, u.dead, u.info);
    k_scan_u64<<<1, 1024, 0, stream>>>(u.tile_sum, u.tile_sum, u.n_list, 0, reinterpret_cast<uint64_t*>(u.info + kInfoStaged));
    FRZ_CUDA_TRY(cudaMemcpyAsync(u.staged + u.staged_n(), u.info + kInfoStaged, sizeof(uint64_t), cudaMemcpyDeviceToDevice, stream));
    FRZ_CUDA_TRY(cudaMemcpyAsync(h_info, u.info, kInfoWords * sizeof(uint64_t), cudaMemcpyDeviceToHost, stream));
    FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    return FRZ_OK;
}

// Step 2: the staged bytes, into out_bytes (r_bytes: the uploaded replacement bytes, if any).
frz_status unpack_bytes(const FrzCorpusStorage* st, const Unpack& u, const uint8_t* r_bytes, uint8_t* out_bytes, cudaStream_t stream) {
    const uint64_t n = u.staged_n();
    const uint32_t blocks = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((n + 7) / 8, (uint64_t)frz_sm_count() * 8));
    k_unpack_bytes<<<blocks, 256, 0, stream>>>(st->data.get(), st->groups.get(), st->slot_meta.get(), st->slot_of.get(), u.tiles, n, u.repl,
                                               u.r_off, r_bytes, u.dead, u.tile_sum, u.staged, out_bytes);
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

// After the re-pack of the listed tiles: their removed, unreplaced haystacks are removed again.
frz_status unpack_mark_dead(FrzCorpusStorage* st, const Unpack& u, cudaStream_t stream) {
    const uint64_t n = u.staged_n();
    const uint32_t blocks = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((n + 255) / 256, (uint64_t)frz_sm_count() * 8));
    k_mark_dead<<<blocks, 256, 0, stream>>>(u.dead, n, u.tiles, st->slot_of.get(), st->slot_meta.get());
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

// Copies every tile's units into a fresh arena, in tile order and without gaps (the layout a fresh pack has).  Peak device
// memory: the old arena plus the new one.
frz_status compact_arena(FrzCorpusStorage* st, cudaStream_t stream) {
    const uint32_t T = st->n_tiles;
    if (T == 0) return FRZ_OK;
    uint64_t* d_units = st->scratch_tile_units.get();
    uint64_t* d_total = d_units + st->tile_base.cap();
    k_tile_units<<<(T + 255) / 256, 256, 0, stream>>>(st->groups.get(), T, d_units);
    k_scan_u64<<<1, 1024, 0, stream>>>(d_units, d_units, T, 0, d_total);
    uint64_t total = 0;
    FRZ_CUDA_TRY(cudaMemcpyAsync(&total, d_total, sizeof total, cudaMemcpyDeviceToHost, stream));
    FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    FrzDevArray<uint4> fresh;
    FRZ_TRY(fresh.reserve(total + total / 16 + 1024));
    k_compact<<<T, 256, 0, stream>>>(st->data.get(), fresh.get(), st->groups.get(), st->tile_base.get(), d_units);
    FRZ_CUDA_TRY(cudaGetLastError());
    FRZ_CUDA_TRY(cudaStreamSynchronize(stream));   // the old arena is freed below
    st->data = std::move(fresh);
    st->total_units = total;
    st->dead_units = 0;
    return FRZ_OK;
}

// An edit that leaves more dead units than live ones compacts the arena.  It runs last, once the edit is complete, and it is
// only an optimisation: when the new arena cannot be allocated, the corpus keeps its dead space (compact_arena changes
// nothing before that allocation has succeeded) and the next edit tries again.
frz_status maybe_compact(FrzCorpusStorage* st, cudaStream_t stream) {
    if (st->dead_units <= st->total_units - st->dead_units) return FRZ_OK;
    const frz_status s = compact_arena(st, stream);
    return s == FRZ_ERR_OOM ? FRZ_OK : s;
}

// Incremental append (SURVEY §8(f) rank 1).  Tiles are independent, so only the partial last tile is
// re-bucketed: it is unpacked to raw bytes, the new haystacks are staged behind it, and tiles
// [n_old / 1024, n_tiles_new) are planned, scanned and copied.  The tail is re-packed in place (carry = first unit of the
// old tail tile) while that tile ends where the arena ends — always so for a corpus that was never edited — and at the
// arena's end otherwise.
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
    // staging layout in ing.d_offsets: [info][staged offsets: cnt + n_new + 1][tile_sum: 1][tiles: 1][dead: 1024][raw new offsets]
    FRZ_TRY(ing.reserve(0, Carve::size(kInfoWords, 8) + Carve::size((uint64_t)cnt + n_new + 1, 8) + 32 + Carve::size(FRZ_TILE, 1) +
                               Carve::size(n_new + 1, sizeof(OffT))));
    Carve cv{ing.d_offsets.get()};
    Unpack u;
    u.info = cv.take<unsigned long long>(kInfoWords);
    u.staged = cv.take<uint64_t>((uint64_t)cnt + n_new + 1);
    u.tile_sum = cv.take<uint64_t>(1);
    u.tiles = cv.take<uint32_t>(1);
    u.dead = cv.take<uint8_t>(FRZ_TILE);
    OffT* d_raw = cv.take<OffT>(n_new + 1);
    u.n_list = 1;
    u.last_cnt = cnt;
    uint64_t info[kInfoWords] = {};
    uint64_t carry_in = st->total_units;
    if (cnt) {
        FRZ_CUDA_TRY(cudaMemcpyAsync(u.tiles, &t_last, sizeof t_last, cudaMemcpyHostToDevice, stream));
        FRZ_TRY(unpack_offsets(st, u, stream, info));
        if (info[kInfoTileEnd] == st->total_units) carry_in = info[kInfoTileBase];   // the tail ends the arena: re-pack it in place
    } else {
        FRZ_CUDA_TRY(cudaMemsetAsync(u.info, 0, kInfoWords * sizeof(uint64_t), stream));
    }
    const uint64_t tail_bytes = info[kInfoStaged];
    FRZ_TRY(ing.reserve(tail_bytes + new_bytes, 0));
    if (cnt) FRZ_TRY(unpack_bytes(st, u, nullptr, ing.d_bytes.get(), stream));
    if (new_bytes) FRZ_CUDA_TRY(cudaMemcpyAsync(ing.d_bytes.get() + tail_bytes, h_bytes + off0, new_bytes, cudaMemcpyHostToDevice, stream));
    FRZ_CUDA_TRY(cudaMemcpyAsync(d_raw, h_offsets, (n_new + 1) * sizeof(OffT), cudaMemcpyHostToDevice, stream));
    k_rebase_offsets<OffT><<<256, 256, 0, stream>>>(d_raw, n_new, u.info + kInfoStaged, u.staged + cnt);
    FRZ_CUDA_TRY(cudaGetLastError());
    FRZ_TRY(pack_reserve(st, n_tiles, t_last, stream));
    st->n = n;
    st->n_tiles = n_tiles;
    st->total_bytes += new_bytes;
    if (cnt && carry_in != info[kInfoTileBase]) st->dead_units += info[kInfoOldUnits];   // the old tail's units are left behind
    FRZ_TRY(pack_plan<uint64_t>(st, u.staged, n, t_last, idx0, carry_in, true, stream));
    FRZ_TRY(pack_copy<uint64_t>(st, ing.d_bytes.get(), u.staged, t_last, idx0, 0, tail_bytes + new_bytes, t_last, n_tiles, stream));
    if (cnt && st->n_removed) FRZ_TRY(unpack_mark_dead(st, u, stream));
    return maybe_compact(st, stream);
}

// Replace: the tiles holding `which` are unpacked in one batch with the new strings substituted, planned as the tiles of
// a scratch corpus whose units go to the end of the arena, and their metadata is scattered over the old tiles'.  Their old
// unit ranges become dead space.  The caller has checked the arguments (indices in range, no duplicates, lengths).
template <typename OffT>
frz_status replace_host_t(FrzIngest& ing, FrzCorpusStorage& scratch, const uint32_t* which, uint64_t n, const uint8_t* h_bytes,
                          const OffT* h_offsets, cudaStream_t stream, FrzCorpusStorage* st) {
    std::vector<uint32_t> tiles(n);
    for (uint64_t j = 0; j < n; j++) tiles[j] = which[j] >> FRZ_TILE_SHIFT;
    std::sort(tiles.begin(), tiles.end());
    tiles.erase(std::unique(tiles.begin(), tiles.end()), tiles.end());
    const uint32_t T = (uint32_t)tiles.size();
    const uint32_t tail_cnt = (uint32_t)(st->n % FRZ_TILE);
    Unpack u;
    u.n_list = T;
    u.last_cnt = (tiles.back() == st->n_tiles - 1 && tail_cnt) ? tail_cnt : FRZ_TILE;
    const uint64_t staged_n = u.staged_n();
    std::vector<uint32_t> slot_pos(n);
    std::vector<uint64_t> r_off(n + 1);
    const uint64_t off0 = (uint64_t)h_offsets[0];
    for (uint64_t j = 0; j < n; j++) {
        const uint32_t b = (uint32_t)(std::lower_bound(tiles.begin(), tiles.end(), which[j] >> FRZ_TILE_SHIFT) - tiles.begin());
        slot_pos[j] = b * FRZ_TILE + (which[j] & (FRZ_TILE - 1));
    }
    for (uint64_t j = 0; j <= n; j++) r_off[j] = (uint64_t)h_offsets[j] - off0;
    const uint64_t r_total = r_off[n];
    const uint64_t slots = (uint64_t)T * FRZ_TILE;
    FRZ_TRY(ing.reserve(0, Carve::size(kInfoWords, 8) + Carve::size(slots + 1, 8) + Carve::size(T, 8) + Carve::size(T, 4) + Carve::size(slots, 4) +
                               Carve::size(slots, 1) + Carve::size(n + 1, 8) + Carve::size(n, 4) + 16));
    Carve cv{ing.d_offsets.get()};
    u.info = cv.take<unsigned long long>(kInfoWords);
    u.staged = cv.take<uint64_t>(slots + 1);
    u.tile_sum = cv.take<uint64_t>(T);
    u.tiles = cv.take<uint32_t>(T);
    u.repl = cv.take<uint32_t>(slots);
    u.dead = cv.take<uint8_t>(slots);
    u.r_off = cv.take<uint64_t>(n + 1);
    uint32_t* d_slot_pos = cv.take<uint32_t>(n);
    // the scratch metadata first: everything that can run out of memory before the corpus changes
    scratch.n = staged_n;
    scratch.n_tiles = T;
    FRZ_TRY(pack_reserve(&scratch, T, 0, stream));
    FRZ_CUDA_TRY(cudaMemcpyAsync(u.tiles, tiles.data(), (size_t)T * 4, cudaMemcpyHostToDevice, stream));
    FRZ_CUDA_TRY(cudaMemcpyAsync(u.r_off, r_off.data(), (n + 1) * 8, cudaMemcpyHostToDevice, stream));
    FRZ_CUDA_TRY(cudaMemcpyAsync(d_slot_pos, slot_pos.data(), n * 4, cudaMemcpyHostToDevice, stream));
    FRZ_CUDA_TRY(cudaMemsetAsync(u.repl, 0xFF, slots * 4, stream));
    k_mark_repl<<<(uint32_t)std::min<uint64_t>((n + 255) / 256, (uint64_t)frz_sm_count() * 8), 256, 0, stream>>>(d_slot_pos, n, u.repl);
    uint64_t info[kInfoWords] = {};
    FRZ_TRY(unpack_offsets(st, u, stream, info));
    const uint64_t staged_bytes = info[kInfoStaged];
    const uint64_t r_at = (staged_bytes + 15) & ~15ull;   // the replacement bytes, behind the staged ones
    FRZ_TRY(ing.reserve(r_at + r_total, 0));
    if (r_total) FRZ_CUDA_TRY(cudaMemcpyAsync(ing.d_bytes.get() + r_at, h_bytes + off0, r_total, cudaMemcpyHostToDevice, stream));
    FRZ_TRY(unpack_bytes(st, u, ing.d_bytes.get() + r_at, ing.d_bytes.get(), stream));
    // plan + copy as a corpus of T tiles whose units start at the arena's end; the arena moves into the scratch for that
    scratch.data = std::move(st->data);
    scratch.total_units = st->total_units;
    frz_status s = pack_plan<uint64_t>(&scratch, u.staged, staged_n, 0, 0, st->total_units, true, stream);
    if (s == FRZ_OK) s = pack_copy<uint64_t>(&scratch, ing.d_bytes.get(), u.staged, 0, 0, 0, staged_bytes, 0, T, stream);
    st->data = std::move(scratch.data);
    FRZ_TRY(s);
    k_scatter_tiles<<<T, 256, 0, stream>>>(u.tiles, scratch.tile_base.get(), scratch.groups.get(), scratch.slot_meta.get(), scratch.slot_of.get(),
                                           scratch.slot_sig.get(), st->tile_base.get(), st->groups.get(), st->slot_meta.get(),
                                           st->slot_of.get(), st->slot_sig.get());
    // from here on the new tiles are in place: the host state follows them at once, and the longest-group bound can only
    // grow with them (the batch's own longest group, from the plan), so that no later failure leaves it below the truth
    const bool had_removed = st->n_removed != 0;
    st->total_units = scratch.total_units;
    st->dead_units += info[kInfoOldUnits];
    st->total_bytes = st->total_bytes + r_total - info[kInfoOldBytes];
    st->n_removed -= info[kInfoRevived];
    st->max_gunits = std::max(st->max_gunits, scratch.max_gunits);
    FRZ_CUDA_TRY(cudaGetLastError());
    if (had_removed) FRZ_TRY(unpack_mark_dead(st, u, stream));
    // the longest group may also have shrunk: recount it over every tile (the kernels specialise on it), before the
    // compaction, which moves units but leaves the groups' sizes as they are
    unsigned int* d_max = reinterpret_cast<unsigned int*>(u.info);
    FRZ_CUDA_TRY(cudaMemsetAsync(d_max, 0, sizeof(unsigned int), stream));
    const uint64_t n_groups = (uint64_t)st->n_tiles * FRZ_GROUPS_PER_TILE;
    k_max_gunits<<<(uint32_t)std::min<uint64_t>((n_groups + 255) / 256, (uint64_t)frz_sm_count() * 8), 256, 0, stream>>>(st->groups.get(),
                                                                                                                        n_groups, d_max);
    unsigned int mx = 0;
    FRZ_CUDA_TRY(cudaMemcpyAsync(&mx, d_max, sizeof mx, cudaMemcpyDeviceToHost, stream));
    FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    st->max_gunits = mx;
    return maybe_compact(st, stream);
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

// Marks haystacks which[0..n) removed (indices checked by the caller).  Their bytes stay where they are.
frz_status frz_remove_host(FrzIngest& ing, const uint32_t* which, uint64_t n, cudaStream_t stream, FrzCorpusStorage* st) {
    FRZ_TRY(ing.reserve(0, 16 + n * sizeof(uint32_t)));
    unsigned long long* d_info = reinterpret_cast<unsigned long long*>(ing.d_offsets.get());
    uint32_t* d_which = reinterpret_cast<uint32_t*>(d_info + 2);
    FRZ_CUDA_TRY(cudaMemsetAsync(d_info, 0, 16, stream));
    FRZ_CUDA_TRY(cudaMemcpyAsync(d_which, which, n * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
    k_remove<<<(uint32_t)std::min<uint64_t>((n + 255) / 256, (uint64_t)frz_sm_count() * 8), 256, 0, stream>>>(d_which, n, st->slot_of.get(),
                                                                                                               st->slot_meta.get(), d_info);
    FRZ_CUDA_TRY(cudaGetLastError());
    uint64_t info[2] = {0, 0};
    FRZ_CUDA_TRY(cudaMemcpyAsync(info, d_info, sizeof info, cudaMemcpyDeviceToHost, stream));
    FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    st->n_removed += info[0];
    st->total_bytes -= info[1];
    return FRZ_OK;
}

// Replaces haystacks which[j] by host Arrow strings (arguments checked by the caller), re-packing only their tiles.
frz_status frz_replace_host(FrzIngest& ing, FrzCorpusStorage& scratch, const uint32_t* which, uint64_t n, const uint8_t* h_bytes,
                            const void* h_offsets, int offset_width, cudaStream_t stream, FrzCorpusStorage* st) {
    if (offset_width == 4)
        return replace_host_t<uint32_t>(ing, scratch, which, n, h_bytes, static_cast<const uint32_t*>(h_offsets), stream, st);
    return replace_host_t<uint64_t>(ing, scratch, which, n, h_bytes, static_cast<const uint64_t*>(h_offsets), stream, st);
}
