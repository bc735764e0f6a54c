// CPU build of frizbee_b200/csrc/order_plan.cuh: the order key, the digit schedule and the pick step of the ordered call's
// select, through the header's own functions (tests/test_ordered_host.py).
#include <stdint.h>

#include "../../frizbee_b200/csrc/order_plan.cuh"

// (hi, lo) of each row's key → out[2 * i], out[2 * i + 1]
extern "C" void h_order_keys(uint32_t order, int reversed, const uint32_t* index, const uint16_t* score, const int16_t* boost,
                             const int64_t* value, uint64_t n, uint64_t* out) {
    for (uint64_t i = 0; i < n; i++) {
        const FrzOrderKey k = frz_order_key(order, reversed != 0, score[i], boost[i], index[i], value[i]);
        out[2 * i] = k.hi;
        out[2 * i + 1] = k.lo;
    }
}

extern "C" uint32_t h_order_digit(uint64_t hi, uint64_t lo, uint32_t shift) { return frz_order_digit(FrzOrderKey{hi, lo}, shift); }

extern "C" uint32_t h_order_digits(uint64_t vary_hi, uint64_t vary_lo, uint32_t* shifts) {
    return frz_order_digits(vary_hi, vary_lo, shifts);
}

// out: bucket, take, above
extern "C" void h_order_pick(const uint32_t* hist, uint64_t need, uint64_t n_sel, uint64_t fit, uint64_t* out) {
    const FrzOrderPick p = frz_order_pick(hist, need, n_sel, fit);
    out[0] = p.bucket;
    out[1] = p.take;
    out[2] = p.above;
}
