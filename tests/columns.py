"""The specification of the column calls (frz_match_list_columns), shared by the tests and tools/bench_columns.py.

Column c is searched by its own matcher; L_c is that matcher's match_list_into over the column (index order).  Row i
matches when it is live in every column, a member of the subset when one is given, and in every L_c.  Its score is the
saturating sum min(65535, sum_c score_c) and its exact flag the OR of the columns' flags (the multi-pattern rule of
src/matcher/multi.rs:83-152, each pattern reading its own column).  The matching rows in index order, reversed under the
*_DESC strategies, are ranked by boost when one is given (tests/ranking.py), else sorted stably by descending score when
some matcher has a compiled pattern and the strategy sorts by score, else left in that order; groups then collapse the
list (tests/collapsing.py)."""
import numpy as np

from collapsing import collapse
from ranking import MATCH_DTYPE, rank_by_boost


def combine(lists, n: int, live=None, members=None) -> np.ndarray:
    """The matching rows, index-ordered.  lists: one index-ordered L_c per column (indices below n); live (optional): a
    bool per row, False for a row removed in some column; members (optional): the subset's indices (any order, repeats
    and indices >= n allowed)."""
    keep = np.ones(n, dtype=bool)
    if live is not None:
        keep &= np.asarray(live, dtype=bool)
    if members is not None:
        idx = np.asarray(members, dtype=np.int64)
        m = np.zeros(n, dtype=bool)
        m[idx[idx < n]] = True
        keep &= m
    score = np.zeros(n, dtype=np.int64)
    exact = np.zeros(n, dtype=bool)
    for L in lists:
        idx = L["index"].astype(np.int64)
        hit = np.zeros(n, dtype=bool)
        hit[idx] = True
        keep &= hit
        score[idx] += L["score"].astype(np.int64)
        exact[idx] |= L["exact"].astype(bool)
    rows_idx = np.flatnonzero(keep)
    rows = np.zeros(len(rows_idx), dtype=MATCH_DTYPE)
    rows["index"] = rows_idx.astype(np.uint32)
    rows["score"] = np.minimum(score[rows_idx], 65535).astype(np.uint16)
    rows["exact"] = exact[rows_idx]
    return rows


def order(rows: np.ndarray, sort, boost=None, any_compiled: bool = True) -> np.ndarray:
    """L: the index-ordered rows ordered by the strategy (a SortStrategy), the boost, and whether any matcher has a compiled
    pattern (only then does a by-score strategy sort)."""
    if boost is not None:
        return rank_by_boost(rows, boost, sort.is_reversed())
    r = rows[::-1] if sort.is_reversed() else rows
    if sort.is_by_score() and any_compiled:
        r = r[np.argsort(-r["score"].astype(np.int64), kind="stable")]
    return np.ascontiguousarray(r, dtype=MATCH_DTYPE)


def match_list_columns(lists, n: int, sort, live=None, members=None, boost=None, group_of=None, per_group=1, n_groups=None,
                       any_compiled: bool = True):
    """(C, counts) of the call: C is the whole result (a call with k returns C[:k], total len(C)); counts is L's rows per
    group (None without groups).  per_group None is no cap."""
    L = order(combine(lists, n, live, members), sort, boost, any_compiled)
    if group_of is None:
        return L, None
    return collapse(L, group_of, per_group, n_groups)
