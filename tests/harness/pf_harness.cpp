// Host build of frizbee_b200/csrc/prefilter_masks.cuh — the occurrence-mask prefilter windows (0 and 1 typo) the GPU
// kernel runs per warp lane — for tests/test_kernel_logic_cpu.py.  One emulated lane; the haystack is laid out at the
// packed corpus' layout (a haystack's 16-byte units are contiguous).
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../frizbee_b200/csrc/prefilter_masks.cuh"

using namespace frzpf;

extern "C" {
// mode 0: masks_k0, 1: masks_k1, 12: masks_paths<2>, 2: masks_paths<3>, 3: masks_many.  Returns 1/0 = matched, -1 = the pattern has no distinct-class table.
int h_masks_window(const void* pat_bytes, const uint8_t* hay, int len, int mode, int* start, int* end) {
    FrzPatternDev pat;
    memcpy(&pat, pat_bytes, sizeof pat);
    if (pat.n_distinct <= 0) return -1;
    const int units = (len + 15) / 16;
    std::vector<uint4> data((size_t)units + 8, make_uint4(0, 0, 0, 0));
    for (int k = 0; k < units; k++) {
        uint8_t b[16] = {0};
        for (int i = 0; i < 16 && 16 * k + i < len; i++) b[i] = hay[16 * k + i];
        memcpy(&data[(size_t)k], b, 16);
    }
    static uint2 occ[kMaxDistinct][32];
    bool ok;
    if (mode >= 100) {   // single-chunk forms (len <= 64, 64-lane emulation)
        if (!single_chunk_ok(pat, (uint32_t)((len + 15) / 16))) return -2;
        ok = mode == 100 ? masks_k0_single(data.data(), pat, occ, len, true, start, end)
                         : masks_k1_single(data.data(), pat, occ, len, true, start, end);
        return ok ? 1 : 0;
    }
    switch (mode) {
        case 0: ok = masks_k0(data.data(), pat, pat.cid, occ, len, true, start, end); break;
        case 1: ok = masks_k1(data.data(), pat, pat.cid, occ, len, true, start, end); break;
        case 12: ok = masks_paths<2>(data.data(), pat, pat.cid, occ, len, true, start, end); break;
        case 2: ok = masks_paths<3>(data.data(), pat, pat.cid, occ, len, true, start, end); break;
        default: ok = masks_many(data.data(), pat, pat.cid, occ, len, true, start, end); break;
    }
    return ok ? 1 : 0;
}

// the pattern's distinct byte classes (0: more than 16, the kernels take the scanning forms)
int h_n_distinct(const void* pat_bytes) {
    FrzPatternDev pat;
    memcpy(&pat, pat_bytes, sizeof pat);
    return pat.n_distinct;
}

// Phase A of k_prefilter: the signature of the haystack (pack.cu: k_pack_sig uses the same frz_sig_add) against the
// needle's class requirements (host.cu: compile_pattern).  Returns 1 = candidate, 0 = rejected without reading the bytes.
int h_sig_pass(const void* pat_bytes, const uint8_t* hay, int len) {
    FrzPatternDev pat;
    memcpy(&pat, pat_bytes, sizeof pat);
    if (!pat.sig_on) return 1;
    uint32_t p1 = 0, p2 = 0;
    for (int i = 0; i < len; i++) frz_sig_add(p1, p2, hay[i]);
    return frz_sig_pass(pat.sig_need1, pat.sig_need2, pat.sig_k, p1, p2) ? 1 : 0;
}
}
