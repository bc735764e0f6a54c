"""The specification of the ranked calls (frz_match_list_ranked), shared by the tests and tools/bench_ranked.py.

A row's key is clamp(score + boost[index], 0, 65535) in 32-bit arithmetic, with boost 0 for indices past the boost
array.  rank_by_boost takes the index-ordered rows of match_list_into, reverses them for the *_DESC strategies, and sorts
them stably by descending key: radix_sort_matches (src/sort.rs:6-40) run on the keys instead of the scores."""
import numpy as np

MATCH_DTYPE = np.dtype([("index", "<u4"), ("score", "<u2"), ("exact", "u1"), ("_pad", "u1")])


def keys(matches: np.ndarray, boost) -> np.ndarray:
    """clamp(score + boost[index], 0, 65535) per row (int64); rows whose index lies past `boost` have boost 0."""
    boost = np.asarray(boost if boost is not None else np.zeros(0), dtype=np.int64)
    idx = matches["index"].astype(np.int64)
    b = np.zeros(len(matches), dtype=np.int64)
    inside = idx < len(boost)
    b[inside] = boost[idx[inside]]
    return np.clip(matches["score"].astype(np.int64) + b, 0, 65535)


def rank_by_boost(matches_index_order: np.ndarray, boost, reversed: bool) -> np.ndarray:
    """The whole ranked list; a call with k returns its first min(k, total) rows."""
    m = np.ascontiguousarray(matches_index_order, dtype=MATCH_DTYPE)
    if reversed:
        m = m[::-1]
    return np.ascontiguousarray(m[np.argsort(-keys(m, boost), kind="stable")])
