"""Collapsed calls without a GPU: the argument checks of frz_groups_create / frz_groups_set / frz_groups_count /
frz_groups_destroy / frz_match_list_collapsed and the missing-device status, the specification tests/collapsing.py
against a literal per-row loop, and frizbee_b200/csrc/collapse_plan.cuh built for the CPU (tests/harness/
collapse_harness.cpp): its order keys reproduce L's order, and its count pass, rounds and keep rule reproduce collapse."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from collapsing import GROUP_NONE, collapse
from cpu_harness import load
from frizbee_b200.types import SortStrategy
from ranking import rank_by_boost

INVALID, UNSUPPORTED, NO_DEVICE = 1, 9, 8
U64_MAX = 2**64 - 1
BY_INDEX, BY_SCORE, BY_KEY = 0, 1, 2
vp, u64, u32, u8 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint8


@pytest.fixture(scope="module")
def H():
    L = load("collapse_harness")
    L.h_collapse_keys.argtypes = [vp, u64, u8, u8, vp, u64, vp]
    L.h_collapse_keys.restype = None
    L.h_collapse.argtypes = [vp, u64, vp, u64, u64, u32, u8, u8, vp, u64, vp, vp]
    L.h_collapse.restype = None
    return L


def test_argument_checks_and_no_device():
    import torch
    L = F.lib()
    fake = C.create_string_buffer(4096)           # a corpus of 0 haystacks; never dereferenced past its length
    c = C.addressof(fake)
    other = C.create_string_buffer(64)            # a handle whose corpus (its first field) is NULL: another corpus
    mine = C.create_string_buffer(c.to_bytes(8, "little"), 64)   # a handle of the fake corpus
    ids = np.array([0, 1], dtype=np.uint32)
    which = np.array([0, 1], dtype=np.uint32)
    h = C.c_void_p()
    n, total = C.c_uint64(), C.c_uint64()
    out = np.zeros(4, dtype=F.MATCH_DTYPE)
    counts = np.zeros(4, dtype=np.uint32)
    o, cn = out.ctypes.data, counts.ctypes.data
    # frz_groups_create: NULL corpus, NULL out, NULL ids with n > 0, n > the corpus's length, n_groups out of range
    assert L.frz_groups_create(None, ids.ctypes.data, 2, 2, C.byref(h)) == INVALID
    assert L.frz_groups_create(c, ids.ctypes.data, 2, 2, None) == INVALID
    assert L.frz_groups_create(c, None, 1, 2, C.byref(h)) == INVALID
    assert b"null" in L.frz_last_error()
    assert L.frz_groups_create(c, ids.ctypes.data, 2, 2, C.byref(h)) == INVALID
    assert b"haystacks" in L.frz_last_error()
    for bad in (0, 2**32, U64_MAX):
        assert L.frz_groups_create(c, None, 0, bad, C.byref(h)) == INVALID
        assert b"n_groups" in L.frz_last_error()
    assert not h.value
    # frz_groups_set: NULL handle, NULL indices or ids with n > 0; n == 0 does nothing
    assert L.frz_groups_set(None, which.ctypes.data, ids.ctypes.data, 2) == INVALID
    assert L.frz_groups_set(C.addressof(mine), None, ids.ctypes.data, 2) == INVALID
    assert L.frz_groups_set(C.addressof(mine), which.ctypes.data, None, 2) == INVALID
    assert b"null" in L.frz_last_error()
    assert L.frz_groups_set(C.addressof(mine), None, None, 0) == 0
    assert L.frz_groups_count(None) == 0
    L.frz_groups_destroy(None)
    # frz_match_list_collapsed: NULL matcher, corpus or groups; per_group 0 and above 32; NULL out with k > 0; a handle
    # of another corpus
    g, oth = C.addressof(mine), C.addressof(other)
    fn = L.frz_match_list_collapsed
    for m_, c_, g_ in ((None, c, g), (c, None, g), (c, c, None)):
        assert fn(m_, c_, None, None, g_, 1, 4, o, C.byref(n), C.byref(total), cn) == INVALID
        assert b"null argument" in L.frz_last_error()
    assert fn(c, c, None, None, g, 0, 4, o, C.byref(n), C.byref(total), cn) == INVALID
    for pg in (33, 1000, 2**63, U64_MAX - 1):
        assert fn(c, c, None, None, g, pg, 4, o, C.byref(n), C.byref(total), cn) == UNSUPPORTED
        assert b"per_group" in L.frz_last_error()
    assert fn(c, c, None, None, g, 1, 1, None, C.byref(n), C.byref(total), cn) == INVALID
    assert b"null out" in L.frz_last_error()
    assert fn(c, c, None, None, oth, 1, 4, o, C.byref(n), C.byref(total), cn) == INVALID
    assert b"groups were made on another corpus" in L.frz_last_error()
    assert fn(c, c, None, oth, g, 1, 4, o, C.byref(n), C.byref(total), cn) == INVALID
    assert b"boost was made on another corpus" in L.frz_last_error()
    assert fn(c, c, oth, None, g, 1, 4, o, C.byref(n), C.byref(total), cn) == INVALID
    assert b"subset was made on another corpus" in L.frz_last_error()
    assert fake.raw == b"\0" * 4096
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    # every argument is valid: the call reaches the device check
    for s_, b_, pg, k in ((None, None, 1, 4), (g, g, 32, 4), (None, g, U64_MAX, 0), (g, None, 3, U64_MAX)):
        assert fn(c, c, s_, b_, g, pg, k, o, C.byref(n), C.byref(total), cn) == NO_DEVICE
    assert fn(c, c, None, None, g, 1, 0, None, None, None, None) == NO_DEVICE


def literal_collapse(L, group_of, per_group, n_groups):
    """collapse restated one row at a time."""
    seen, keep = {}, []
    counts = [0] * n_groups
    for r in L:
        i = int(r["index"])
        g = int(group_of[i]) if i < len(group_of) else GROUP_NONE
        if g == GROUP_NONE:
            keep.append(r)
            continue
        counts[g] += 1
        if per_group is None or seen.get(g, 0) < per_group:
            keep.append(r)
        seen[g] = seen.get(g, 0) + 1
    return np.array(keep, dtype=F.MATCH_DTYPE), np.array(counts, dtype=np.uint32)


def random_rows(rng, n, score_hi, n_index=None):
    rows = np.zeros(n, dtype=F.MATCH_DTYPE)
    rows["index"] = np.sort(rng.choice(n_index or 4 * max(n, 1), n, replace=False)).astype(np.uint32)
    rows["score"] = rng.integers(0, score_hi, n).astype(np.uint16)
    rows["exact"] = rng.integers(0, 2, n)
    return rows


def group_shapes(rng, n_index):
    """(name, group_of, n_groups): the shapes the GPU tests use too."""
    dup = rng.integers(0, max(n_index // 20, 1), n_index).astype(np.uint32)
    short = rng.integers(0, 7, n_index // 2).astype(np.uint32)        # ids past the array: rows in no group
    mixed = rng.integers(0, 50, n_index).astype(np.uint32)
    mixed[rng.random(n_index) < 0.3] = GROUP_NONE
    return [("none", np.full(n_index, GROUP_NONE, np.uint32), 3), ("own", np.arange(n_index, dtype=np.uint32), n_index),
            ("one", np.zeros(n_index, np.uint32), 1), ("dup", dup, max(n_index // 20, 1)), ("short", short, 9),
            ("mixed", mixed, 50)]


@pytest.mark.parametrize("seed", range(4))
def test_collapse_equals_the_literal_loop(seed):
    rng = np.random.default_rng(seed)
    rows = random_rows(rng, int(rng.integers(0, 2000)), 300)
    L = rows[np.argsort(-rows["score"].astype(np.int64), kind="stable")]
    for name, group_of, n_groups in group_shapes(rng, 4 * max(len(rows), 1)):
        for per_group in (1, 2, 3, 32, None):
            got, cnt = collapse(L, group_of, per_group, n_groups)
            want, wcnt = literal_collapse(L, group_of, per_group, n_groups)
            assert np.array_equal(got, want), (name, per_group)
            assert np.array_equal(cnt, wcnt), (name, per_group)


def want_L(base, sort, boost, empty):
    """L of the uncollapsed call from the index-ordered rows: ranked, else by score (non-empty matcher), else index order."""
    if boost is not None:
        return rank_by_boost(base, boost, sort.is_reversed())
    rows = base[::-1] if sort.is_reversed() else base
    if sort.is_by_score() and not empty:
        rows = rows[np.argsort(-rows["score"].astype(np.int64), kind="stable")]
    return np.ascontiguousarray(rows)


def order_of(sort, boost, empty):
    return BY_KEY if boost is not None else BY_SCORE if sort.is_by_score() and not empty else BY_INDEX


def keys_of(H, lst, order, reversed_, boost):
    b = np.ascontiguousarray(boost if boost is not None and len(boost) else np.zeros(1, np.int16))
    keys = np.zeros(max(len(lst), 1), dtype=np.uint64)
    H.h_collapse_keys(lst.ctypes.data, len(lst), order, reversed_, b.ctypes.data, 0 if boost is None else len(boost), keys.ctypes.data)
    return keys[:len(lst)]


@pytest.mark.parametrize("score_hi", [4, 1100, 65536])
def test_order_keys_reproduce_L(H, score_hi):
    """Scores over the whole u16 range and boosts that clamp keys at 0 and at 65535; every strategy, ranked and not, and the
    empty matcher (every score 0)."""
    rng = np.random.default_rng(score_hi)
    for empty in (False, True):
        base = random_rows(rng, 3000, score_hi)
        if empty:
            base["score"] = 0
            base["exact"] = 0
        boosts = [None, rng.integers(-40, 41, 4 * 3000).astype(np.int16),
                  rng.choice(np.array([-32768, -1000, 0, 1000, 32767], np.int16), 2 * 3000)]   # shorter than the indices
        for sort in SortStrategy:
            lst = np.ascontiguousarray(base[::-1] if sort.is_reversed() else base)
            for boost in boosts:
                keys = keys_of(H, lst, order_of(sort, boost, empty), sort.is_reversed(), boost)
                assert len(np.unique(keys)) == len(keys)
                if boost is not None and boost.min() == -32768:   # both clamps are reached
                    assert (keys >> np.uint64(32)).min() == 0 and (empty or score_hi < 65536 or (keys >> np.uint64(32)).max() == 65535)
                got = lst[np.argsort(keys)[::-1]]
                assert np.array_equal(got, want_L(base, sort, boost, empty)), (empty, sort, boost is not None)


@pytest.mark.parametrize("seed", range(3))
def test_rounds_reproduce_collapse(H, seed):
    rng = np.random.default_rng(100 + seed)
    for empty in (False, True):
        base = random_rows(rng, int(rng.integers(1, 2500)), [4, 300, 65536][seed])
        if empty:
            base["score"] = 0
        n_index = 4 * len(base)
        boost = rng.integers(-300, 301, n_index).astype(np.int16)
        for name, group_of, n_groups in group_shapes(rng, n_index):
            for sort in SortStrategy:
                lst = np.ascontiguousarray(base[::-1] if sort.is_reversed() else base)
                for b in (None, boost):
                    order = order_of(sort, b, empty)
                    L = want_L(base, sort, b, empty)
                    bb = np.ascontiguousarray(b if b is not None else np.zeros(1, np.int16))
                    for per_group in (1, 2, 3, 32, None):
                        keep = np.zeros(len(lst), dtype=np.uint8)
                        counts = np.zeros(n_groups, dtype=np.uint32)
                        H.h_collapse(lst.ctypes.data, len(lst), group_of.ctypes.data, len(group_of), n_groups, per_group or 0, order,
                                     sort.is_reversed(), bb.ctypes.data, 0 if b is None else len(b), keep.ctypes.data,
                                     counts.ctypes.data)
                        kept = lst[keep.astype(bool)]
                        got = kept[np.argsort(keys_of(H, kept, order, sort.is_reversed(), b))[::-1]]
                        want, wcounts = collapse(L, group_of, per_group, n_groups)
                        ctx = (name, sort, b is not None, per_group, empty)
                        assert np.array_equal(got, want), ctx
                        assert np.array_equal(counts, wcounts), ctx
