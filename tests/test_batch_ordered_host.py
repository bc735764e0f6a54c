"""The batched ordered call without a GPU: the argument checks of frz_match_list_batch_ordered and their order, the
missing-device status, and frizbee_b200/csrc/batch_order_plan.cuh built for the CPU (tests/harness/batch_order_harness.cpp):
the budget arithmetic against a numpy restatement, each query's digit sequence, and one whole sub-batch (keys, shared
tables, the count pass, the rounds on the order key, the member rule, the select's passes and the sort) against the
specifications tests/ordering.py and tests/collapsing.py, query by query."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import frizbee_b200 as F
from collapsing import collapse
from frizbee_b200.types import SortStrategy
from ordering import ATTR_NULL, order_by_attr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "frizbee_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "harness", "batch_order_harness.cpp")
LIB = os.path.join(ROOT, "tests", "harness", "libbatch_order_harness.so")
DEPS = [SRC] + [os.path.join(CSRC, h) for h in ("batch_order_plan.cuh", "batch_collapse_plan.cuh", "collapse_plan.cuh", "order_plan.cuh",
                                                 "batch_plan.cuh")]
INVALID, UNSUPPORTED, NO_DEVICE = 1, 9, 8
U64_MAX = 2**64 - 1
I64_MAX = 2**63 - 1
BUDGET = 512 << 20
PASSES = 15
vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", LIB, SRC], check=True)
    L = C.CDLL(LIB)
    L.h_sizes.argtypes = [u32]
    L.h_sizes.restype = u64
    L.h_order_bytes.argtypes = [u64, u64]
    L.h_order_bytes.restype = u64
    L.h_order_fit.argtypes = [u64, u64, u64, u64]
    L.h_order_fit.restype = u64
    L.h_shifts.argtypes = [u64, u64, vp]
    L.h_shifts.restype = u32
    L.h_key.argtypes = [vp, vp, u64, vp, u32, u32, C.c_int, vp]
    L.h_batch_order.argtypes = [u32, u64] + [vp] * 14 + [u64] + [vp] * 5
    L.h_batch_order.restype = u32
    return L


def ptrs(xs):
    return (C.c_void_p * max(len(xs), 1))(*[x.ctypes.data if x is not None else None for x in xs])


def test_argument_checks_and_no_device():
    import torch
    L = F.lib()
    fake = C.create_string_buffer(4096)           # a corpus of 0 haystacks; never dereferenced past its length
    c = C.addressof(fake)
    other = C.create_string_buffer(64)            # a handle whose corpus (its first field) is NULL: another corpus
    mine = C.create_string_buffer(c.to_bytes(8, "little"), 64)   # a handle of the fake corpus
    g, oth = C.addressof(mine), C.addressof(other)
    fn = L.frz_match_list_batch_ordered
    ms = (C.c_void_p * 2)(c, c)
    out = np.zeros(8, dtype=F.MATCH_DTYPE)
    n_out, n_total = np.zeros(2, np.uint64), np.zeros(2, np.uint64)
    cnt = np.zeros(4, np.uint32)
    o, no, nt = out.ctypes.data, n_out.ctypes.data, n_total.ctypes.data
    hc = (C.c_void_p * 2)(cnt.ctypes.data, None)

    def arr(dtype, *v):
        a = np.array(v, dtype=dtype)
        return a, a.ctypes.data

    def h(*v):
        return (C.c_void_p * 2)(*v)

    ok_pg, ok = arr(np.uint64, 1, U64_MAX)
    ok_od, od = arr(np.uint32, 0, 3)
    mine_a, mine_g = h(g, None), h(None, g)
    # NULL matchers array or corpus, a NULL matcher
    assert fn(None, 2, c, None, None, mine_a, od, mine_g, ok, 4, o, no, nt, hc) == INVALID
    assert fn(ms, 2, None, None, None, mine_a, od, mine_g, ok, 4, o, no, nt, hc) == INVALID
    assert b"null argument" in L.frz_last_error()
    assert fn(h(c, None), 2, c, None, None, mine_a, od, mine_g, ok, 4, o, no, nt, hc) == INVALID
    assert b"null matcher at 1" in L.frz_last_error()
    # per_group first, before the orders and the handles
    for v, want in (((0, 1), INVALID), ((33, 0), UNSUPPORTED), ((1, 0), INVALID)):
        a, p = arr(np.uint64, *v)
        bad_o, bo = arr(np.uint32, 4, 4)
        assert fn(ms, 2, c, h(oth, None), None, h(oth, oth), bo, h(oth, oth), p, 4, o, no, nt, hc) == want, v
        assert b"per_group" in L.frz_last_error()
    # then every order, with or without an attribute, before the handles
    for v, at in (((4, 0), "at 0"), ((0, 4), "at 1"), ((0xFFFFFFFF, 0), "at 0")):
        a, p = arr(np.uint32, *v)
        assert fn(ms, 2, c, h(oth, None), None, None, p, h(oth, oth), ok, 4, o, no, nt, hc) == INVALID, v
        assert b"order" in L.frz_last_error() and at.encode() in L.frz_last_error()
    # q = 0 reads no entry and is a no-op
    assert fn(ms, 0, c, None, None, None, None, None, None, 4, None, None, None, None) == 0
    # handles of another corpus: query order, then subset, boost, groups, attribute within a query
    assert fn(ms, 2, c, None, None, h(g, oth), od, None, ok, 4, o, no, nt, hc) == INVALID
    assert b"attribute of query 1 was made on another corpus" in L.frz_last_error()
    assert fn(ms, 2, c, None, None, h(oth, None), od, h(oth, None), ok, 4, o, no, nt, hc) == INVALID
    assert b"groups of query 0" in L.frz_last_error()
    assert fn(ms, 2, c, None, h(oth, None), h(oth, None), od, h(oth, None), ok, 4, o, no, nt, hc) == INVALID
    assert b"boost of query 0" in L.frz_last_error()
    assert fn(ms, 2, c, h(None, oth), h(oth, None), h(None, oth), od, None, ok, 4, o, no, nt, hc) == INVALID
    assert b"boost of query 0" in L.frz_last_error()
    # then the outputs: NULL n_out, q * k overflow, NULL out
    assert fn(ms, 2, c, None, None, mine_a, od, mine_g, ok, 4, o, None, nt, hc) == INVALID
    assert b"null n_out" in L.frz_last_error()
    assert fn(ms, 2, c, None, None, mine_a, od, mine_g, ok, 2**63, o, no, nt, hc) == INVALID
    assert b"overflows" in L.frz_last_error()
    assert fn(ms, 2, c, None, None, mine_a, od, mine_g, ok, 4, None, no, nt, hc) == INVALID
    assert b"null out" in L.frz_last_error()
    assert fake.raw == b"\0" * 4096 and not cnt.any()
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    # every argument is valid: the call reaches the device check (NULL orders, per_group, attributes and k = 0 included)
    for ats, ods, gs, p, k in ((mine_a, od, mine_g, ok, 4), (None, None, None, None, 4), (h(g, g), None, h(g, g), None, 0),
                               (mine_a, od, None, ok, 0)):
        assert fn(ms, 2, c, h(g, None), h(None, g), ats, ods, gs, p, k, o if k else None, no, None, hc) == NO_DEVICE
    assert not cnt.any()


def test_budget_arithmetic(H):
    rec, key, state, passes = (H.h_sizes(i) for i in range(4))
    assert (rec, key, state, passes) == (40, 16, 88, PASSES)
    rng = np.random.default_rng(2)
    for _ in range(500):
        base = int(rng.integers(1, 64 << 20))
        groups = int(rng.choice([0, 1, 7, 1000, int(rng.integers(1, 2**28))]))
        rows = int(rng.integers(1, 1 << 21))
        order = rec + rows * (key + 8) + 4096 * 4 + state + 256 * 4 + groups * 8
        assert H.h_order_bytes(groups, rows) == order
        collapse_bytes = groups * 12 + rows + 32 if groups else 0
        q = BUDGET // (base + collapse_bytes + order)
        assert H.h_order_fit(BUDGET, base, groups, rows) == (q if q >= 2 else 0)
    # a 1 M-row corpus's ordered queries still fit two to a sub-batch; 14 M groups beside them do not
    assert H.h_order_fit(BUDGET, 40 << 20, 0, 1 << 20) >= 2
    assert H.h_order_fit(BUDGET, 100_000, 14_000_000, 3000) == 0


def key112(L, row, values, boost, order, reversed_):
    hl = np.zeros(2, np.uint64)
    r = np.ascontiguousarray(row)
    L.h_key(r.ctypes.data, values.ctypes.data, len(values), boost.ctypes.data if boost is not None else None,
            0 if boost is None else len(boost), order, int(reversed_), hl.ctypes.data)
    return int(hl[0]) << 48 | int(hl[1])


def test_digit_sequencing(H):
    """frz_batch_order_shift gives exactly the digits in which two of the rows' keys differ, most significant first."""
    rng = np.random.default_rng(3)
    for trial in range(60):
        n = int(rng.integers(1, 200))
        rows = np.zeros(n, dtype=F.MATCH_DTYPE)
        rows["index"] = np.sort(rng.choice(5000, n, replace=False)).astype(np.uint32)
        rows["score"] = rng.integers(0, [2, 300, 65536][trial % 3], n).astype(np.uint16)
        values = rng.choice([ATTR_NULL, -1, 0, 1, 5, I64_MAX], 5000).astype(np.int64) if trial % 2 else \
            rng.integers(-2**40, 2**40, 5000).astype(np.int64)
        order, rev = trial % 4, bool(trial % 3)
        keys = [key112(H, rows[i:i + 1], values, None, order, rev) for i in range(n)]
        want = [s for s in range(104, -1, -8) if len({(k >> s) & 255 for k in keys}) > 1]
        vary = flip = 0
        for k in keys:
            vary |= k
            flip |= ~k & ((1 << 112) - 1)
        v = vary & flip
        shifts = np.zeros(PASSES, np.uint32)
        got = H.h_shifts(v >> 48, v & ((1 << 48) - 1), shifts.ctypes.data)
        assert list(shifts[:got]) == want, (trial, want, shifts[:got])


def random_query(rng, n_index):
    # a third of the queries have more rows than the block sort holds: their rows are selected first
    rows = np.zeros(int(rng.integers(4500, n_index) if rng.random() < 0.3 else rng.integers(0, 1500)), dtype=F.MATCH_DTYPE)
    rows["index"] = np.sort(rng.choice(n_index, len(rows), replace=False)).astype(np.uint32)
    rows["score"] = rng.integers(0, [4, 300, 65536][int(rng.integers(0, 3))], len(rows)).astype(np.uint16)
    rows["exact"] = rng.integers(0, 2, len(rows))
    sort = list(SortStrategy)[int(rng.integers(0, 4))]
    kind = int(rng.integers(0, 5))   # extremes and nulls, ties, uniform, shorter than the corpus, all null
    n_values = n_index // 3 if kind == 3 else n_index
    values = [rng.choice([ATTR_NULL, ATTR_NULL + 1, -1, 0, 1, I64_MAX - 1, I64_MAX], n_values),
              rng.choice([0, 1, 127], n_values), rng.integers(-2**62, 2**62, n_values), rng.integers(-5, 5, n_values),
              np.full(n_values, ATTR_NULL)][kind].astype(np.int64)
    boost = rng.integers(-40000, 40000, int(rng.integers(0, n_index + 1))).astype(np.int16) if rng.random() < 0.4 else None
    members = np.flatnonzero(rng.random(n_index) < rng.choice([0.0, 0.3, 1.0])) if rng.random() < 0.4 else None
    gkind = int(rng.integers(0, 5))   # no groups, own, one, dup, short
    if gkind == 0:
        ids, n_groups = None, 0
    else:
        n_groups = [0, n_index, 1, int(rng.integers(1, 60)), 9][gkind]
        ids = [None, np.arange(n_index, dtype=np.uint32), np.zeros(n_index, np.uint32),
               rng.integers(0, n_groups, n_index).astype(np.uint32), rng.integers(0, 9, n_index // 3).astype(np.uint32)][gkind]
        if gkind == 3:
            ids[rng.random(n_index) < 0.2] = 0xFFFFFFFF
    per_group = [1, 2, 3, 32, None][int(rng.integers(0, 5))]
    return dict(rows=rows, sort=sort, values=values, order=int(rng.integers(0, 4)), boost=boost, members=members, ids=ids,
                n_groups=n_groups, per_group=per_group, wants=bool(rng.random() < 0.6))


@pytest.mark.parametrize("seed", range(8))
def test_sub_batch_reproduces_the_ordered_calls(H, seed):
    """ns queries of every shape share one ordered sub-batch: each query's rows are the first k of collapse(order_by_attr
    (its members)), its total is their number, its counts are the ordered list's, and its passes visit a prefix of its
    varying digits."""
    rng = np.random.default_rng(seed)
    n_index = G = 12000
    ns = int(rng.integers(1, 65))
    k = int(rng.choice([0, 1, 10, 700, 1024]))
    qs = [random_query(rng, n_index) for _ in range(ns)]
    lists, bits = [], []
    for q in qs:
        lists.append(np.ascontiguousarray(q["rows"][::-1] if q["sort"].is_reversed() else q["rows"]))
        if q["members"] is None:
            bits.append(None)
        else:
            b = np.zeros((n_index + 31) // 32, np.uint32)
            np.bitwise_or.at(b, q["members"] >> 5, (np.uint32(1) << (q["members"] & 31).astype(np.uint32)))
            bits.append(b)
    u64s = [np.array(v or [0], np.uint64) for v in (
        [len(x) for x in lists], [len(q["values"]) for q in qs], [0 if q["boost"] is None else len(q["boost"]) for q in qs],
        [n_index] * ns, [0 if q["ids"] is None else len(q["ids"]) for q in qs],
        [U64_MAX if q["per_group"] is None else q["per_group"] for q in qs])]
    n, n_values, n_boost, n_bits, n_ids, per_group = (a.ctypes.data for a in u64s)
    reversed_ = np.array([q["sort"].is_reversed() for q in qs], np.uint8)
    orders = np.array([q["order"] for q in qs], np.uint32)
    wants = np.array([q["wants"] for q in qs], np.uint8)
    pos = np.zeros(max(ns * k, 1), np.uint32)
    totals = np.zeros(ns, np.uint64)
    visited = np.zeros(ns * PASSES, np.uint32)
    n_visited = np.zeros(ns, np.uint32)
    counts_back = np.zeros(ns * G, np.uint32)
    n_back = H.h_batch_order(ns, k, ptrs(lists), n, reversed_.ctypes.data, ptrs([q["values"] for q in qs]), n_values,
                             ptrs([q["boost"] for q in qs]), n_boost, orders.ctypes.data, ptrs(bits), n_bits, ptrs([q["ids"] for q in qs]),
                             n_ids, per_group, wants.ctypes.data, G, pos.ctypes.data, totals.ctypes.data, visited.ctypes.data,
                             n_visited.ctypes.data, counts_back.ctypes.data)
    assert n_back != 0xFFFFFFFF, "a round table is not zero after the rounds, or a selection outgrew the block sort"
    assert n_back == sum(1 for q in qs if q["wants"] and q["ids"] is not None)
    slot = 0
    for j, q in enumerate(qs):
        rows = q["rows"] if q["members"] is None else q["rows"][np.isin(q["rows"]["index"], q["members"])]
        L = order_by_attr(rows, q["values"], q["order"], q["sort"].is_reversed(), q["boost"])
        if q["ids"] is None:
            want, wcounts = L, None
        else:
            want, wcounts = collapse(L, q["ids"], q["per_group"], q["n_groups"])
        assert totals[j] == len(want), (j, totals[j], len(want))
        m = min(k, len(want))
        got = lists[j][pos[j * k: j * k + m]]
        assert np.array_equal(got, want[:m]), (j, q["order"], q["sort"], q["per_group"])
        # the passes visit the query's varying digits in order, and stop when the selection is complete
        if k and len(want) > 4096:
            keys = [key112(H, want[i:i + 1], q["values"], q["boost"], q["order"], q["sort"].is_reversed()) for i in range(len(want))]
            digits = [s for s in range(104, -1, -8) if len({(x >> s) & 255 for x in keys}) > 1]
            v = list(visited[j * PASSES: j * PASSES + n_visited[j]])
            assert v == digits[:len(v)] and v, (j, v, digits)
        else:
            assert n_visited[j] == 0, j   # the rows fit the block sort, or k = 0: nothing to select
        if q["wants"] and q["ids"] is not None:
            assert np.array_equal(counts_back[slot * G: slot * G + q["n_groups"]], wcounts), j
            slot += 1
