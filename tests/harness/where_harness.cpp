// CPU build of frizbee_b200/csrc/where_plan.cuh: the clause test, the set packing, and the fill of frz_subset_where as
// where.cu and host.cu run it (k_where's words and chunk counts, the scan, k_where_members' expansion), sequentially,
// through the header's own functions (tests/test_where_host.py).
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../frizbee_b200/csrc/where_plan.cuh"

// out[i] = the clause holds for values[i]
extern "C" void h_where_holds(const FrzWhereClauseDev* c, const int64_t* sets, const int64_t* values, uint64_t n, uint8_t* out) {
    for (uint64_t i = 0; i < n; i++) out[i] = frz_where_holds(*c, sets, values[i]);
}

// in[0 .. n) packed as the host packs one set clause: out[0 .. return) sorted and distinct
extern "C" uint32_t h_where_pack(const int64_t* in, uint64_t n, int64_t* out) {
    std::vector<int64_t> sets = {42};   // a clause packed before it
    const uint32_t k = frz_where_pack_set(in, n, sets);
    memcpy(out, sets.data() + 1, k * sizeof(int64_t));
    return k;
}

// The fill of w: w->bits, w->chunk_count, members and the member count.  w->bits may be w->base.
extern "C" uint64_t h_where_fill(const FrzWhereDev* w, uint32_t* members) {
    const uint64_t n_words = (w->n + 31) / 32, n_chunks = (w->n + kFrzWhereChunk - 1) / kFrzWhereChunk;
    for (uint64_t word = 0; word < n_words; word++) {   // k_where: the ballot of a word's 32 lanes
        const uint32_t base_word = w->has_base && word * 32 < w->n_base ? w->base[word] : 0u;
        uint32_t b = 0;
        for (uint32_t lane = 0; lane < 32; lane++) {
            const uint64_t i = word * 32 + lane;
            bool keep = frz_where_in_base(*w, base_word, i);
            for (uint32_t c = 0; c < w->n_clauses; c++)
                keep = frz_where_holds(w->clauses[c], w->sets, frz_where_value(w->clauses[c], i)) && keep;
            b |= (uint32_t)keep << lane;
        }
        w->bits[word] = b;
    }
    for (uint64_t c = 0; c < n_chunks; c++) {
        uint32_t t = 0;
        for (uint64_t k = 0; k < kFrzWhereChunkWords && c * kFrzWhereChunkWords + k < n_words; k++)
            t += frz_where_popc(w->bits[c * kFrzWhereChunkWords + k]);
        w->chunk_count[c] = t;
    }
    uint64_t base = 0;   // k_scan_blocks
    for (uint64_t c = 0; c < n_chunks; c++) {
        const uint32_t t = w->chunk_count[c];
        uint32_t excl = 0;   // k_where_members: the word's first slot within its chunk, then each member's rank in it
        for (uint64_t k = 0; k < kFrzWhereChunkWords && c * kFrzWhereChunkWords + k < n_words; k++) {
            const uint64_t word = c * kFrzWhereChunkWords + k;
            const uint32_t x = w->bits[word];
            for (uint32_t lane = 0; lane < 32; lane++)
                if ((x >> lane) & 1u) members[base + excl + frz_where_rank(x, lane)] = (uint32_t)(word * 32 + lane);
            excl += frz_where_popc(x);
        }
        base += t;
    }
    return base;
}
