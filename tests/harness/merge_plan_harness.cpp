// Host build of the k-way merge's position arithmetic (frizbee_b200/csrc/merge_plan.cuh) for tests/test_merge_plan_cpu.py:
// the tables every form reads, the P2P placement (k_place's per-element walk) and the slice exchange (its ranges A[q][p]
// and the scatter of the received pieces), driven through the header's own functions.  Matches are 8-byte frz_match
// records; runs are concatenated, run q at offset sum(counts[0..q)).
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../frizbee_b200/csrc/merge_plan.cuh"

namespace {
struct Match {
    uint32_t index;
    uint16_t score;
    uint8_t exact, pad;
};

struct Runs {
    const Match* m;
    std::vector<uint64_t> start, counts;
    std::vector<uint32_t> gt;   // [q][s], as a run's score table has it (sort.cu / k_merge_bounds)
    int world, bins;

    Runs(const void* matches, const uint64_t* cnt, int world_, int bins_) : m(static_cast<const Match*>(matches)), world(world_), bins(bins_) {
        uint64_t at = 0;
        for (int q = 0; q < world; q++) { start.push_back(at); counts.push_back(cnt[q]); at += cnt[q]; }
        gt.assign((size_t)world * bins, 0);
        for (int q = 0; q < world; q++)
            for (uint64_t i = 0; i < counts[q]; i++) {
                const uint32_t b = frzmerge::bin_of(m[start[q] + i].score, bins);
                for (uint32_t s = 0; s < b; s++) gt[(size_t)q * bins + s]++;
            }
    }
    void plan(bool reversed, int only, uint32_t* rows, const uint64_t* lo, uint64_t* A) const {
        frzmerge::plan_tables(world, bins, reversed, gt.data(), (size_t)bins, counts.data(), only, rows, lo, world, A);
    }
};

uint64_t slices_of(const Runs& R, uint64_t limit, std::vector<uint64_t>& lo) {
    uint64_t total = 0;
    for (uint64_t c : R.counts) total += c;
    const uint64_t kp = total < limit ? total : limit;
    lo.resize(R.world + 1);
    for (int p = 0; p <= R.world; p++) lo[p] = frzmerge::slice_lo(kp, p, R.world);
    return kp;
}
}  // namespace

extern "C" {
// table rows of every run (2 * bins u32 each: pos0 then gt)
void h_tables(const void* matches, const uint64_t* counts, int world, int bins, int reversed, uint32_t* rows) {
    Runs R(matches, counts, world, bins);
    R.plan(reversed != 0, -1, rows, nullptr, nullptr);
}

// P2P placement: every rank plans its own row only and stores its first min(limit, n_q) elements into the slice that holds
// their merged position (k_place).  out: the concatenated slices, K' records.  0, or -1 when an element lands outside the
// slice the lookup chose or outside [0, K').
int h_place(const void* matches, const uint64_t* counts, int world, int bins, int reversed, uint64_t limit, void* out) {
    Runs R(matches, counts, world, bins);
    std::vector<uint64_t> lo;
    const uint64_t kp = slices_of(R, limit, lo);
    std::vector<uint32_t> rows(frzmerge::table_row(world, bins));
    Match* o = static_cast<Match*>(out);
    for (int q = 0; q < world; q++) {
        R.plan(reversed != 0, q, rows.data(), lo.data(), nullptr);
        const uint32_t* pos0 = rows.data() + frzmerge::table_row(q, bins);
        const uint32_t* gt = pos0 + bins;
        const uint64_t n = R.counts[q] < limit ? R.counts[q] : limit;
        for (uint64_t i = 0; i < n; i++) {
            const Match m = R.m[R.start[q] + i];
            const uint32_t s = frzmerge::bin_of(m.score, bins);
            const uint64_t x = pos0[s] + (i - gt[s]);
            if (x >= kp) continue;
            const int p = frzmerge::slice_of(x, kp, world, lo.data());
            if (p < 0 || p >= world || x < lo[p] || x >= lo[p + 1]) return -1;
            o[lo[p] + (x - lo[p])] = m;
        }
    }
    return 0;
}

// Slice exchange: the ranges A[q][p] from the plan, then every rank p scatters the pieces [A[q][p], A[q][p + 1]) of every
// run q into its slice (k_merge_scatter with per-run offsets a = A[q][p] and the output shift lo[p]).  0; -1 when a
// position falls outside the slice; -2 when the piece lengths do not sum to the slice length.
int h_exchange(const void* matches, const uint64_t* counts, int world, int bins, int reversed, uint64_t limit, void* out, uint64_t* A_out) {
    Runs R(matches, counts, world, bins);
    std::vector<uint64_t> lo;
    slices_of(R, limit, lo);
    std::vector<uint32_t> rows(frzmerge::table_row(world, bins));
    std::vector<uint64_t> A((size_t)world * (world + 1));
    R.plan(reversed != 0, -1, rows.data(), lo.data(), A.data());
    memcpy(A_out, A.data(), A.size() * sizeof(uint64_t));
    Match* o = static_cast<Match*>(out);
    for (int p = 0; p < world; p++) {
        const uint64_t len = lo[p + 1] - lo[p];
        uint64_t got = 0;
        for (int q = 0; q < world; q++) {
            const uint64_t a = A[(size_t)q * (world + 1) + p], b = A[(size_t)q * (world + 1) + p + 1];
            const uint32_t* row = rows.data() + frzmerge::table_row(q, bins);
            for (uint64_t i = 0; i < b - a; i++) {
                const Match m = R.m[R.start[q] + a + i];
                const uint32_t s = frzmerge::bin_of(m.score, bins);
                const uint64_t y = (uint32_t)(row[s] + ((uint32_t)(a + i) - row[bins + s]) - (uint32_t)lo[p]);
                if (y >= len) return -1;
                o[lo[p] + y] = m;
            }
            got += b - a;
        }
        if (got != len) return -2;
    }
    return 0;
}
}
