"""The specification of the collapsed calls (frz_match_list_collapsed), shared by the tests and tools/bench_collapsed.py.

L is the list the uncollapsed call returns (frz_match_list_ranked with the whole list, frz_match_list_subset or
frz_match_list).  collapse keeps, in L's order, every row in no group and the first per_group rows of each group, and
counts L's rows per group before collapsing.  A row's group is group_of[index], or none (GROUP_NONE) past the array."""
import numpy as np

GROUP_NONE = 0xFFFFFFFF


def groups_of(rows: np.ndarray, group_of) -> np.ndarray:
    """Each row's group id (int64), GROUP_NONE for rows past group_of or with a GROUP_NONE id."""
    group_of = np.asarray(group_of, dtype=np.int64)
    idx = rows["index"].astype(np.int64)
    g = np.full(len(rows), GROUP_NONE, dtype=np.int64)
    inside = idx < len(group_of)
    g[inside] = group_of[idx[inside]]
    return g


def collapse(L: np.ndarray, group_of, per_group, n_groups=None):
    """(C, counts): C is the rows of L kept by the rule above (per_group None: no cap, C = L); counts[j] is the rows of L in
    group j (uint32, n_groups entries; n_groups defaults to one more than the largest id in group_of)."""
    g = groups_of(L, group_of)
    grouped = g != GROUP_NONE
    if n_groups is None:
        ids = np.asarray(group_of, dtype=np.int64)
        ids = ids[ids != GROUP_NONE]
        n_groups = int(ids.max()) + 1 if ids.size else 1
    counts = np.bincount(g[grouped], minlength=n_groups).astype(np.uint32)
    if per_group is None:
        return np.ascontiguousarray(L), counts
    # occurrence of each row within its group, in L's order
    order = np.argsort(g, kind="stable")
    gs = g[order]
    start = np.r_[0, np.flatnonzero(gs[1:] != gs[:-1]) + 1] if len(gs) else np.zeros(0, np.int64)
    run_start = np.zeros(len(gs), dtype=np.int64)
    run_start[start] = start
    run_start = np.maximum.accumulate(run_start) if len(gs) else run_start
    occ = np.empty(len(g), dtype=np.int64)
    occ[order] = np.arange(len(gs)) - run_start
    keep = ~grouped | (occ < per_group)
    return np.ascontiguousarray(L[keep]), counts
