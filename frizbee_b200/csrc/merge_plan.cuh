// merge_plan.cuh — the position arithmetic of the k-way merge of per-GPU runs (src/k_merge.rs:90-131), shared by merge.cu
// and parallel.cu and built for the CPU by tests/test_merge_plan_cpu.py.
//
// Runs are index-range shards in rank order, each ordered by (score desc, index), or by index alone with a one-bin table.
// gt[q][s] counts the elements of run q in score bins above s, so run q's bin-s block is its index range
// [gt[q][s], gt[q][s - 1]).  pos0[q][s] is the merged position of that block's first element: everything in bins above s
// in any run, plus the bin-s blocks of the runs before q in merge order.  Element i of run q, in bin s, lands at
// pos0[q][s] + (i - gt[q][s]).  A merged list of `total` positions is cut into `world` slices [lo[p], lo[p + 1]),
// lo[p] = total * p / world.  The tables are u32 (every form that reads them needs a merged list below 2^32), one row of
// 2 * bins per run: pos0[q][0..bins) then gt[q][0..bins).
#pragma once
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define FRZ_HD __host__ __device__ __forceinline__
#else
#define FRZ_HD inline
#endif

namespace frzmerge {

FRZ_HD size_t table_row(int q, int bins) { return (size_t)q * 2 * (size_t)bins; }

// scores past the last of `bins` >= 1 bins share it (a one-bin table: every score in bin 0)
FRZ_HD uint32_t bin_of(uint32_t score, int bins) { return score < (uint32_t)(bins - 1) ? score : (uint32_t)(bins - 1); }

// the run that comes k-th in merge order: reversed sorts take the runs last to first
FRZ_HD int run_at(int k, int n_runs, bool reversed) { return reversed ? n_runs - 1 - k : k; }

// The bin-s block of every run in merge order, until at(q, pos0, size, gt) returns false.  gt(q, s) as above, count(q) = run
// q's length; T accumulates the positions.
template <class T, class Gt, class Count, class At>
FRZ_HD void block_bases(int s, int n_runs, bool reversed, const Gt& gt, const Count& count, const At& at) {
    T acc = 0;
    for (int q = 0; q < n_runs; q++) acc += (T)gt(q, s);
    for (int k = 0; k < n_runs; k++) {
        const int q = run_at(k, n_runs, reversed);
        const T g = (T)gt(q, s), size = (T)(s == 0 ? count(q) : gt(q, s - 1)) - g;
        if (!at(q, acc, size, g)) return;
        acc += size;
    }
}

FRZ_HD uint64_t slice_lo(uint64_t total, int p, int world) { return total * (uint64_t)p / (uint64_t)world; }

// the slice that holds position x < total: x * world / total is at most one slice off lo[]
FRZ_HD int slice_of(uint64_t x, uint64_t total, int world, const uint64_t* lo) {
    const uint64_t est = x * (uint64_t)world / total;
    int p = est < (uint64_t)(world - 1) ? (int)est : world - 1;
    while (p > 0 && x < lo[p]) p--;
    while (p + 1 < world && x >= lo[p + 1]) p++;
    return p;
}

// Host side of the host-out forms: the table row of run `only` (P2P: the walk stops there), or of every run when only < 0,
// from run q's gt at gt + q * gt_stride (null: one bin, nothing above it) and its length counts[q].  With A ([n_runs][world + 1],
// zeroed) also the slice exchange's ranges: A[q][p] = the elements of run q before lo[p], so run q's elements in slice p
// are [A[q][p], A[q][p + 1]) (a run keeps its order in the merge).
inline void plan_tables(int n_runs, int bins, bool reversed, const volatile uint32_t* gt, size_t gt_stride, const uint64_t* counts, int only,
                        uint32_t* rows, const uint64_t* lo, int world, uint64_t* A) {
    for (int s = bins - 1; s >= 0; s--)
        block_bases<uint64_t>(
            s, n_runs, reversed, [&](int q, int b) { return gt ? gt[q * gt_stride + b] : 0u; }, [&](int q) { return counts[q]; },
            [&](int q, uint64_t pos0, uint64_t size, uint64_t g) {
                if (only >= 0 && q != only) return true;
                rows[table_row(q, bins) + s] = (uint32_t)pos0;
                rows[table_row(q, bins) + bins + s] = (uint32_t)g;
                for (int p = 0; A && size && p <= world; p++)   // the part of the block before lo[p]
                    A[(size_t)q * (world + 1) + p] += lo[p] <= pos0 ? 0 : (lo[p] - pos0 < size ? lo[p] - pos0 : size);
                return only < 0;
            });
}

}  // namespace frzmerge
