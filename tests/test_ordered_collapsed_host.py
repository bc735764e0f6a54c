"""Ordered collapsed calls without a GPU.  The rounds on the order key (frizbee_b200/csrc/collapse_plan.cuh's two-step max
over order_plan.cuh's keys, built for the CPU by tests/harness/ordered_collapse_harness.cpp) run pass by pass, each pass
over the rows in a random order, and are compared with the specification collapse(order_by_attr(...)) on random and
adversarial lists.  The argument checks of frz_match_list_ordered_collapsed and frz_match_list_columns_ordered run on
zero-filled stand-in handles.  The behaviour on a real corpus is in tests/test_gpu_ordered_collapsed.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import frizbee_b200 as F
from collapsing import GROUP_NONE, collapse
from ordering import ATTR_NULL, order_by_attr
from ranking import MATCH_DTYPE
from test_columns_host import _field_offset

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "frizbee_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "harness", "ordered_collapse_harness.cpp")
LIB = os.path.join(ROOT, "tests", "harness", "libordered_collapse_harness.so")
DEPS = [SRC] + [os.path.join(CSRC, h) for h in ("collapse_plan.cuh", "order_plan.cuh", "batch_plan.cuh")]
INVALID, TOO_MANY_ITEMS, NO_DEVICE, UNSUPPORTED = 1, 4, 8, 9
U64_MAX = 2**64 - 1
I64_MAX = 2**63 - 1
vp, u64, u32, i32 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", LIB, SRC], check=True)
    L = C.CDLL(LIB)
    L.h_ordered_collapse.argtypes = [vp, u64, vp, u64, vp, u32, u32, i32, vp, u64, u64, u32, u64, vp, vp]
    L.h_ordered_collapse.restype = C.c_int
    return L


def rounds(H, rows, values, boost, order, reversed_, group_of, n_groups, per_group, seed):
    """C as the device builds it: the rounds and the keep rule over L0, then the kept rows ordered (order_list).  Returns
    (C, counts, whether both round tables were left zero)."""
    l0 = np.ascontiguousarray(rows[::-1] if reversed_ else rows)
    vals = np.ascontiguousarray(values, dtype=np.int64)
    b = np.ascontiguousarray(boost if boost is not None and len(boost) else np.zeros(1, np.int16), dtype=np.int16)
    ids = np.ascontiguousarray(group_of, dtype=np.uint32)
    keep = np.zeros(max(len(l0), 1), np.uint8)
    counts = np.zeros(n_groups, np.uint32)
    zero = H.h_ordered_collapse(l0.ctypes.data, len(l0), vals.ctypes.data, len(vals), b.ctypes.data,
                                0 if boost is None else len(boost), order, int(reversed_), ids.ctypes.data, len(ids), n_groups,
                                per_group or 0, seed, keep.ctypes.data, counts.ctypes.data)
    kept = l0[keep[: len(l0)].astype(bool)]
    kept = kept[::-1] if reversed_ else kept   # back to index order: order_by_attr reverses it itself
    return order_by_attr(kept, values, order, reversed_, boost), counts, zero == 1


def spec(rows, values, boost, order, reversed_, group_of, n_groups, per_group):
    return collapse(order_by_attr(rows, values, order, reversed_, boost), group_of, per_group, n_groups)


def index_rows(rng, n, n_index, scores=400, first=False):
    idx = np.sort(rng.choice(n_index, n, replace=False)).astype(np.uint32)
    if first and n:
        idx[0] = 0   # x = 0 under the *_DESC strategies
    m = np.zeros(n, MATCH_DTYPE)
    m["index"] = idx
    m["score"] = rng.integers(0, scores, n)
    m["exact"] = rng.integers(0, 2, n)
    return m


def value_shapes(rng, n_index):
    """(name, values): every kind of attribute the rounds must order, adversarial ones included."""
    ts = 1_600_000_000_000 + rng.permutation(n_index).astype(np.int64) * 7
    nulls = rng.integers(-1000, 1000, n_index).astype(np.int64)
    nulls[rng.random(n_index) < 0.3] = ATTR_NULL
    extremes = rng.choice([ATTR_NULL, ATTR_NULL + 1, -1, 0, 1, I64_MAX - 1, I64_MAX], n_index).astype(np.int64)
    return [("timestamps", ts), ("nulls", nulls), ("all_null", np.full(n_index, ATTR_NULL, np.int64)),
            ("max", np.full(n_index, I64_MAX, np.int64)),   # hi = 2^64 - 1 under ATTR_DESC
            ("min", np.full(n_index, ATTR_NULL + 1, np.int64)),   # hi = 1 under ATTR_DESC, 2^64 - 1 under ATTR_ASC
            ("ties", rng.choice([0, 1, 127], n_index).astype(np.int64)), ("extremes", extremes),
            ("short", rng.integers(-5, 5, n_index // 3).astype(np.int64))]


def group_shapes(rng, n_index):
    """(name, group_of, n_groups), the shapes of test_collapsed_host plus a group per attribute value (every row of a
    group tied on hi)."""
    dup = rng.integers(0, max(n_index // 20, 1), n_index).astype(np.uint32)
    short = rng.integers(0, 7, n_index // 2).astype(np.uint32)        # ids past the array: rows in no group
    mixed = rng.integers(0, 50, n_index).astype(np.uint32)
    mixed[rng.random(n_index) < 0.3] = GROUP_NONE
    return [("none", np.full(n_index, GROUP_NONE, np.uint32), 3), ("own", np.arange(n_index, dtype=np.uint32), n_index),
            ("one", np.zeros(n_index, np.uint32), 1), ("dup", dup, max(n_index // 20, 1)), ("short", short, 9),
            ("mixed", mixed, 50)]


PER_GROUP = (1, 2, 3, 32, None)


@pytest.mark.parametrize("seed", range(3))
def test_rounds_equal_the_specification(H, seed):
    """Random lists over every attribute and group shape, all four orders, both index directions, with and without a
    boost, every per_group."""
    rng = np.random.default_rng(500 + seed)
    n_index = int(rng.integers(40, 1200))
    rows = index_rows(rng, int(rng.integers(1, n_index)), n_index, first=seed == 0)
    boost = rng.choice([-32768, -400, -1, 0, 1, 200, 32767], n_index).astype(np.int16)
    for vname, values in value_shapes(rng, n_index):
        for gname, group_of, n_groups in group_shapes(rng, n_index):
            for order in range(4):
                for reversed_ in (False, True):
                    for b in (None, boost):
                        for per_group in PER_GROUP:
                            got, cnt, zero = rounds(H, rows, values, b, order, reversed_, group_of, n_groups, per_group,
                                                    int(rng.integers(0, 2**63)))
                            want, wcnt = spec(rows, values, b, order, reversed_, group_of, n_groups, per_group)
                            ctx = (vname, gname, order, reversed_, b is not None, per_group)
                            assert zero, ctx
                            assert np.array_equal(got, want), ctx
                            assert np.array_equal(cnt, wcnt), ctx


def test_groups_tied_on_hi(H):
    """Every row of a group shares its attribute value (and under SCORE_THEN_* its score), so each round is decided by lo
    alone; and a group whose every row is null (hi = 0) or at the top value (hi = 2^64 - 1)."""
    rng = np.random.default_rng(7)
    n_index = 600
    rows = index_rows(rng, 500, n_index, scores=3, first=True)
    group_of = rng.integers(0, 12, n_index).astype(np.uint32)
    per_value = np.array([ATTR_NULL, I64_MAX, ATTR_NULL + 1, 0, 5, -5, 1 << 40, -(1 << 40), 3, 4, 6, 7], np.int64)
    values = per_value[group_of]
    boost = np.zeros(n_index, np.int16)
    for order in range(4):
        for reversed_ in (False, True):
            for b in (None, boost):
                for per_group in PER_GROUP:
                    for seed in range(3):
                        got, cnt, zero = rounds(H, rows, values, b, order, reversed_, group_of, 12, per_group, seed)
                        want, wcnt = spec(rows, values, b, order, reversed_, group_of, 12, per_group)
                        assert zero and np.array_equal(got, want) and np.array_equal(cnt, wcnt), (order, reversed_, per_group)


def test_the_latest_row_of_each_group(H):
    """The empty matcher's list (every row, score 0) at per_group 1 under ATTR_DESC: each group's newest row, newest first."""
    rng = np.random.default_rng(11)
    n = 3000
    rows = np.zeros(n, MATCH_DTYPE)
    rows["index"] = np.arange(n)
    ts = rng.integers(0, 10**6, n).astype(np.int64)
    group_of = rng.integers(0, 40, n).astype(np.uint32)
    got, cnt, zero = rounds(H, rows, ts, None, 0, False, group_of, 40, 1, 3)
    assert zero
    newest = {}
    for i in range(n):   # the largest timestamp, ties to the lower index
        g = int(group_of[i])
        if g not in newest or ts[i] > ts[newest[g]]:
            newest[g] = i
    want = sorted(newest.values(), key=lambda i: (-ts[i], i))
    assert got["index"].tolist() == want
    assert cnt.tolist() == np.bincount(group_of, minlength=40).tolist()


def test_argument_checks_in_order_and_no_device():
    import torch
    L = F.lib()
    n_at, dev_at = _field_offset(L.frz_corpus_len, 8, 0x1234_5678_9A), _field_offset(L.frz_corpus_device, 4, 5)

    def fake_corpus(n, device=0):
        buf = C.create_string_buffer(4096)
        C.memmove(C.addressof(buf) + n_at, int(n).to_bytes(8, "little"), 8)
        C.memmove(C.addressof(buf) + dev_at, int(device).to_bytes(4, "little"), 4)
        return buf

    c0, c1, longer, elsewhere, stranger = fake_corpus(0), fake_corpus(0), fake_corpus(8), fake_corpus(0, 1), fake_corpus(0)
    huge, huge2 = fake_corpus(2**32), fake_corpus(2**32)
    before = [b.raw for b in (c0, c1, longer, elsewhere, stranger)]
    handle = {name: C.create_string_buffer(C.addressof(c).to_bytes(8, "little"), 256)
              for name, c in (("c0", c0), ("c1", c1), ("stranger", stranger))}
    h = {k: C.addressof(v) for k, v in handle.items()}
    snap = {k: v.raw for k, v in handle.items()}
    mfake = C.create_string_buffer(64)           # a matcher, never dereferenced before the device check
    m, c = C.addressof(mfake), C.addressof(c0)
    out = np.zeros(4, dtype=F.MATCH_DTYPE)
    counts = np.zeros(4, dtype=np.uint32)
    n, total = C.c_uint64(), C.c_uint64()

    def single(m_=m, c_=c, s=None, b=None, a=h["c0"], order=0, g=h["c0"], per_group=1, k=4, o=out.ctypes.data, cnt=None):
        return L.frz_match_list_ordered_collapsed(m_, c_, s, b, a, order, g, per_group, k, o, C.byref(n), C.byref(total), cnt)

    def arr(*xs):
        return (C.c_void_p * len(xs))(*xs)

    def cols_call(ms=None, cols=None, n_cols=2, sort=0, s=None, b=None, a=h["c0"], order=0, g=None, per_group=1, k=4,
                  o=out.ctypes.data, cnt=None):
        ms = arr(m, m) if ms is None else ms
        cols = arr(C.addressof(c0), C.addressof(c1)) if cols is None else cols
        return L.frz_match_list_columns_ordered(ms, cols, n_cols, sort, s, b, a, order, g, per_group, k, o, C.byref(n),
                                                C.byref(total), cnt)

    def refused(fn, status, text, **kw):
        assert fn(**kw) == status, kw
        assert text.encode() in L.frz_last_error(), (kw, L.frz_last_error())

    # frz_match_list_ordered_collapsed: NULL matcher, corpus, attribute or groups; then per_group; then a NULL out with
    # k > 0; then the order; then handles of another corpus in the order subset, boost, groups, attribute
    for kw in ({"m_": None}, {"c_": None}, {"a": None}, {"g": None}, {"g": None, "per_group": 0, "order": 9, "o": None}):
        refused(single, INVALID, "null argument", **kw)
    refused(single, INVALID, "per_group = 0", per_group=0, order=9, o=None, s=h["stranger"])
    for pg in (33, 1000, 2**63, U64_MAX - 1):
        refused(single, UNSUPPORTED, "per_group", per_group=pg, order=9, o=None)
    refused(single, INVALID, "null out", o=None, order=9, s=h["stranger"])
    for order in (4, 2**32 - 1):
        refused(single, INVALID, "order", order=order, s=h["stranger"])
    st = h["stranger"]
    refused(single, INVALID, "subset was made on another corpus", s=st, b=st, g=st, a=st)
    refused(single, INVALID, "boost was made on another corpus", b=st, g=st, a=st)
    refused(single, INVALID, "groups were made on another corpus", g=st, a=st)
    refused(single, INVALID, "attribute was made on another corpus", a=st)
    # frz_match_list_columns_ordered: the column checks first, then a NULL attribute, per_group (only with groups), a NULL
    # out with k > 0, the order, and handles made on none of the columns
    refused(cols_call, INVALID, "n_cols", n_cols=0, a=None, order=9)
    refused(cols_call, INVALID, "null argument", ms=0)
    refused(cols_call, INVALID, "column 1", ms=arr(m, None), a=None)
    refused(cols_call, INVALID, "device", cols=arr(C.addressof(c0), C.addressof(elsewhere)), a=None)
    refused(cols_call, INVALID, "index space", cols=arr(C.addressof(c0), C.addressof(longer)), a=None)
    refused(cols_call, TOO_MANY_ITEMS, "u32 index", cols=arr(C.addressof(huge), C.addressof(huge2)), a=None)
    refused(cols_call, INVALID, "sort", sort=4, a=None)
    refused(cols_call, INVALID, "null argument", a=None, g=h["c0"], per_group=0, order=9, o=None)
    refused(cols_call, INVALID, "per_group = 0", g=h["c0"], per_group=0, order=9, o=None)
    refused(cols_call, UNSUPPORTED, "per_group", g=h["c0"], per_group=33, order=9, o=None)
    refused(cols_call, INVALID, "null out", o=None, order=9, s=st)
    refused(cols_call, INVALID, "order", order=4, s=st)
    refused(cols_call, INVALID, "subset was made on none", s=st, b=st, g=st, a=st)
    refused(cols_call, INVALID, "boost was made on none", b=st, g=st, a=st)
    refused(cols_call, INVALID, "groups were made on none", g=st, a=st)
    refused(cols_call, INVALID, "attribute was made on none", a=st)
    assert [b.raw for b in (c0, c1, longer, elsewhere, stranger)] == before
    assert {k: v.raw for k, v in handle.items()} == snap
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    # every argument is valid: the call reaches the device check
    for kw in ({}, {"order": 3}, {"b": h["c0"], "s": h["c0"]}, {"per_group": 32, "cnt": counts.ctypes.data},
               {"per_group": U64_MAX, "k": 0, "o": None}, {"k": U64_MAX}):
        assert single(**kw) == NO_DEVICE, kw
    # per_group is not read without groups; a handle of any column serves
    for kw in ({}, {"per_group": 0}, {"per_group": 77}, {"a": h["c1"], "s": h["c1"], "b": h["c0"], "g": h["c1"], "per_group": 32,
                                                          "cnt": counts.ctypes.data},
               {"g": h["c0"], "per_group": U64_MAX, "k": 0, "o": None}, {"k": U64_MAX, "sort": 3, "order": 3}, {"n_cols": 1}):
        assert cols_call(**kw) == NO_DEVICE, kw
