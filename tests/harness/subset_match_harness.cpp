// CPU build of frizbee_b200/csrc/subset_match_plan.cuh: the steps of a fill, the masked-metadata rule, and the fold as
// subset_match.cu runs it (k_subset_fold's words and chunk counts, step by step), sequentially, through the header's own
// functions (tests/test_subset_match_host.py).
#include <stdint.h>

#include <vector>

#include "../../frizbee_b200/csrc/subset_match_plan.cuh"

// The steps for n patterns with these negation flags → pattern[], op[]; returns their number.
extern "C" uint32_t h_steps(const uint8_t* negated, uint32_t n, int32_t* pattern, uint32_t* op) {
    std::vector<bool> neg(negated, negated + n);
    const std::vector<FrzSubsetMatchStep> steps = frz_subset_match_steps(neg);
    for (size_t k = 0; k < steps.size(); k++) {
        pattern[k] = steps[k].pattern;
        op[k] = steps[k].op;
    }
    return (uint32_t)steps.size();
}

extern "C" int h_masked(uint32_t step, int has_base, uint64_t base_members, uint64_t n) {
    return frz_subset_match_masked(step, has_base != 0, base_members, n) ? 1 : 0;
}

// The fill's fold: step k folds survs[k * surv_words ..] with ops[k] into bits (the first step with base/n_base when
// has_base), and the last step writes chunk_count.  Each word goes through frz_fold_word as one lane of k_subset_fold
// computes it; chunks of kFrzWhereChunkWords words are summed as the warp's reduction does.
extern "C" void h_fold(uint64_t n, const uint32_t* base, uint64_t n_base, uint32_t has_base, const uint32_t* survs, uint64_t surv_words,
                       const uint32_t* ops, uint32_t n_steps, uint32_t* bits, uint32_t* chunk_count) {
    const uint64_t n_words = (n + 31) / 32, n_chunks = (n + kFrzWhereChunk - 1) / kFrzWhereChunk;
    for (uint32_t k = 0; k < n_steps; k++) {
        FrzSubsetFoldDev f = {};
        f.surv = survs + k * surv_words;
        f.bits = bits;
        f.n = n;
        f.op = ops[k];
        f.has_base = k == 0 ? has_base : 0;
        f.base = base;
        f.n_base = n_base;
        f.chunk_count = k + 1 == n_steps ? chunk_count : nullptr;
        for (uint64_t chunk = 0; chunk < n_chunks; chunk++) {
            uint32_t c = 0;
            for (uint32_t lane = 0; lane < kFrzWhereChunkWords; lane++) {
                const uint64_t word = chunk * kFrzWhereChunkWords + lane;
                if (word >= n_words) continue;
                const uint32_t base_word = f.has_base && word * 32 < f.n_base ? f.base[word] : 0u;
                const uint32_t cur = f.op == kFrzFoldFirst ? 0u : f.bits[word];
                const uint32_t x = frz_fold_word(f.op, cur, f.surv[word], frz_fold_base(f.has_base, base_word, word, f.n_base),
                                                 frz_fold_below(word, f.n));
                f.bits[word] = x;
                c += frz_where_popc(x);
            }
            if (f.chunk_count) f.chunk_count[chunk] = c;
        }
    }
}
