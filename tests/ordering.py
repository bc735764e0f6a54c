"""The specification of the ordered calls (frz_match_list_ordered), shared by the tests and tools/bench_ordered.py.

L0 is the index-ordered rows of match_list_into, reversed for the *_DESC strategies.  A row's value is attr[index], null
when it equals ATTR_NULL or when the index lies past the attribute's values; its rank value r is clamp(score +
boost[index], 0, 65535) with a boost (ranking.keys), else the raw score.  order_by_attr sorts L0 stably with np.lexsort:
  AttrDesc (0)           non-null first, value descending, r descending
  AttrAsc (1)            non-null first, value ascending, r descending
  ScoreThenAttrDesc (2)  r descending, non-null first, value descending
  ScoreThenAttrAsc (3)   r descending, non-null first, value ascending
Rows still tied keep L0's order."""
import numpy as np

from ranking import MATCH_DTYPE, keys

ATTR_NULL = -(2**63)


def values_of(matches: np.ndarray, attr_values) -> np.ndarray:
    """attr_values[index] per row (int64); rows past the array get ATTR_NULL."""
    attr_values = np.asarray(attr_values, dtype=np.int64)
    idx = matches["index"].astype(np.int64)
    v = np.full(len(matches), ATTR_NULL, dtype=np.int64)
    inside = idx < len(attr_values)
    v[inside] = attr_values[idx[inside]]
    return v


def order_by_attr(matches_index_order: np.ndarray, attr_values, order: int, reversed: bool, boost=None) -> np.ndarray:
    """The whole ordered list; a call with k returns its first min(k, total) rows."""
    m = np.ascontiguousarray(matches_index_order, dtype=MATCH_DTYPE)
    if reversed:
        m = m[::-1]
    v = values_of(m, attr_values)
    null = v == ATTR_NULL
    r = keys(m, boost) if boost is not None else m["score"].astype(np.int64)
    # value keys that sort ascending in the wanted direction: negation is exact for every value but ATTR_NULL, which is
    # ordered by the null key instead
    vkey = np.where(null, 0, -v if order in (0, 2) else v)
    pos = np.arange(len(m))
    # np.lexsort: the last key is the primary one
    if order in (0, 1):
        perm = np.lexsort((pos, -r, vkey, null))
    else:
        perm = np.lexsort((pos, vkey, null, -r))
    return np.ascontiguousarray(m[perm])
