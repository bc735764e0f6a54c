"""Ranked calls without a GPU: the argument checks of frz_boost_create / frz_boost_set / frz_match_list_ranked, which return
before any device access (zero-filled blocks stand in for the handles; the checks below never read them), and the
reference rank_by_boost against a literal restatement of radix_sort_matches' two 8-bit LSD passes on the keys."""
import ctypes

import numpy as np
import pytest

import frizbee_b200 as F
from ranking import keys, rank_by_boost

INVALID_ARG = 1


def test_ranked_argument_checks():
    L = F.lib()
    fake = ctypes.create_string_buffer(4096)
    c = ctypes.addressof(fake)
    vals = np.array([1, -2], dtype=np.int16)
    which = np.array([0, 1], dtype=np.uint32)
    h = ctypes.c_void_p()
    n, total = ctypes.c_uint64(), ctypes.c_uint64()
    out = np.zeros(4, dtype=F.MATCH_DTYPE)
    # frz_boost_create: NULL corpus, NULL out, NULL values with n > 0
    assert L.frz_boost_create(None, vals.ctypes.data, 2, ctypes.byref(h)) == INVALID_ARG
    assert L.frz_boost_create(c, vals.ctypes.data, 2, None) == INVALID_ARG
    assert L.frz_boost_create(c, None, 1, ctypes.byref(h)) == INVALID_ARG
    assert b"null" in L.frz_last_error() and not h.value
    # frz_boost_set: NULL boost, NULL indices or values with n > 0
    assert L.frz_boost_set(None, which.ctypes.data, vals.ctypes.data, 2) == INVALID_ARG
    assert L.frz_boost_set(c, None, vals.ctypes.data, 2) == INVALID_ARG
    assert L.frz_boost_set(c, which.ctypes.data, None, 2) == INVALID_ARG
    assert b"null" in L.frz_last_error()
    # frz_match_list_ranked: a NULL matcher, corpus or boost (the subset may be NULL), and a NULL out with k > 0
    for m_, c_, b_ in ((None, c, c), (c, None, c), (c, c, None)):
        assert L.frz_match_list_ranked(m_, c_, None, b_, 4, out.ctypes.data, ctypes.byref(n), ctypes.byref(total)) == INVALID_ARG
        assert b"null argument" in L.frz_last_error()
    assert L.frz_match_list_ranked(c, c, None, c, 1, None, ctypes.byref(n), ctypes.byref(total)) == INVALID_ARG
    assert b"null out" in L.frz_last_error()
    L.frz_boost_destroy(None)
    assert fake.raw == b"\0" * 4096


def radix_sort_keys(matches: np.ndarray, key: np.ndarray) -> np.ndarray:
    """radix_sort_matches (src/sort.rs:6-40) pass for pass, with the row's key where the reference reads its score."""
    n = len(matches)
    b = np.zeros(n, dtype=matches.dtype)
    kb = np.zeros(n, dtype=np.int64)
    out = np.zeros(n, dtype=matches.dtype)
    # pass 1
    hist = [0] * 256
    for k in key:
        hist[k & 0xFF] += 1
    offsets = [0] * 256
    for idx in range(255, 0, -1):
        offsets[idx - 1] = offsets[idx] + hist[idx]
    for i in range(n):
        r = key[i] & 0xFF
        b[offsets[r]] = matches[i]
        kb[offsets[r]] = key[i]
        offsets[r] += 1
    # pass 2
    hist = [0] * 256
    for k in kb:
        hist[(k >> 8) & 0xFF] += 1
    offsets[255] = 0
    for idx in range(255, 0, -1):
        offsets[idx - 1] = offsets[idx] + hist[idx]
    for i in range(n):
        r = (kb[i] >> 8) & 0xFF
        out[offsets[r]] = b[i]
        offsets[r] += 1
    return out


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("reversed_", [False, True])
def test_rank_by_boost_equals_the_radix_passes(seed, reversed_):
    """Random index-ordered lists with scores over the whole u16 range and boosts that push keys past both clamps."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(0, 3000))
    m = np.zeros(n, dtype=F.MATCH_DTYPE)
    m["index"] = np.sort(rng.choice(4 * n + 1, n, replace=False)).astype(np.uint32)
    hi = [40, 300, 1100, 65535][seed % 4]
    m["score"] = rng.integers(0, hi + 1, n).astype(np.uint16)
    m["exact"] = rng.integers(0, 2, n).astype(np.uint8)
    # boosts of a shorter array than the index range (the rest have 0): small, extreme and a few of each sign
    boost = rng.choice(np.array([-32768, -1000, -300, -1, 0, 0, 1, 5, 300, 1000, 32767]), 3 * n + 1).astype(np.int16)
    small = rng.random(len(boost)) < 0.5
    boost[small] = rng.integers(-40, 41, int(small.sum()))   # many equal keys: ties decide most of the order
    want_in = m[::-1] if reversed_ else m
    k = keys(want_in, boost)
    if n > 100:   # the clamp at 0 is reached, and the one at 65535 where scores reach past 32768
        assert k.min() == 0 and (hi < 65535 or k.max() == 65535)
    got = rank_by_boost(m, boost, reversed_)
    want = radix_sort_keys(want_in, k)
    assert np.array_equal(got, want)


def test_rank_by_boost_clamps_and_ties():
    """Both clamps, ties between a clamped and an unclamped key, ties in both index directions, rows past the boost."""
    m = np.zeros(6, dtype=F.MATCH_DTYPE)
    m["index"] = [0, 1, 2, 3, 4, 9]
    m["score"] = [10, 65000, 5, 65535, 0, 7]
    boost = np.array([-32768, 32767, -5, 0, 0], dtype=np.int16)   # index 9 lies past the array: boost 0
    assert keys(m, boost).tolist() == [0, 65535, 0, 65535, 0, 7]
    assert rank_by_boost(m, boost, False)["index"].tolist() == [1, 3, 9, 0, 2, 4]
    assert rank_by_boost(m, boost, True)["index"].tolist() == [3, 1, 9, 4, 2, 0]
    for rev in (False, True):
        src = m[::-1] if rev else m
        assert np.array_equal(rank_by_boost(m, boost, rev), radix_sort_keys(src, keys(src, boost)))
