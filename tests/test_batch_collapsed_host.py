"""The batched collapsed call without a GPU: the argument checks of frz_match_list_batch_collapsed and their order, the
missing-device status, and frizbee_b200/csrc/batch_collapse_plan.cuh built for the CPU (tests/harness/
batch_collapse_harness.cpp): the budget arithmetic against a numpy restatement, and one sub-batch's slots, shared tables,
count pass, rounds and keep rule against the specification tests/collapsing.py, query by query."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import frizbee_b200 as F
from collapsing import collapse
from frizbee_b200.types import SortStrategy
from ranking import rank_by_boost

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "frizbee_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "harness", "batch_collapse_harness.cpp")
LIB = os.path.join(ROOT, "tests", "harness", "libbatch_collapse_harness.so")
DEPS = [SRC] + [os.path.join(CSRC, h) for h in ("batch_collapse_plan.cuh", "collapse_plan.cuh", "batch_plan.cuh")]
INVALID, UNSUPPORTED, NO_DEVICE = 1, 9, 8
U64_MAX = 2**64 - 1
BY_INDEX, BY_SCORE, BY_KEY = 0, 1, 2
BUDGET = 512 << 20
vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", LIB, SRC], check=True)
    L = C.CDLL(LIB)
    L.h_record_bytes.restype = u64
    L.h_collapse_bytes.argtypes = [u64, u64]
    L.h_collapse_bytes.restype = u64
    L.h_collapse_fit.argtypes = [u64, u64, u64, u64]
    L.h_collapse_fit.restype = u64
    L.h_rounds.argtypes = [u64]
    L.h_rounds.restype = u32
    L.h_batch_collapse.argtypes = [u32] + [vp] * 12 + [u64, vp, vp]
    L.h_batch_collapse.restype = u32
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
    fn = L.frz_match_list_batch_collapsed
    ms = (C.c_void_p * 2)(c, c)
    out = np.zeros(8, dtype=F.MATCH_DTYPE)
    n_out, n_total = np.zeros(2, np.uint64), np.zeros(2, np.uint64)
    cnt = np.zeros(4, np.uint32)
    o, no, nt = out.ctypes.data, n_out.ctypes.data, n_total.ctypes.data
    hc = (C.c_void_p * 2)(cnt.ctypes.data, None)

    def pg(*v):
        a = np.array(v, dtype=np.uint64)
        return a, a.ctypes.data

    def h(*v):
        return (C.c_void_p * 2)(*v)

    ok_pg, ok = pg(1, U64_MAX)
    mine_g = h(g, None)
    # NULL matchers array or corpus, a NULL matcher
    assert fn(None, 2, c, None, None, mine_g, ok, 4, o, no, nt, hc) == INVALID
    assert fn(ms, 2, None, None, None, mine_g, ok, 4, o, no, nt, hc) == INVALID
    assert b"null argument" in L.frz_last_error()
    assert fn(h(c, None), 2, c, None, None, mine_g, ok, 4, o, no, nt, hc) == INVALID
    assert b"null matcher at 1" in L.frz_last_error()
    # per_group: 0 is invalid, above 32 (but not UINT64_MAX) unsupported; the first bad entry decides, before the handles
    for v, want in (((0, 1), INVALID), ((1, 0), INVALID), ((33, 0), UNSUPPORTED), ((0, 33), INVALID), ((U64_MAX - 1, 1), UNSUPPORTED),
                    ((32, 2**63), UNSUPPORTED)):
        a, p = pg(*v)
        assert fn(ms, 2, c, h(oth, None), None, h(oth, oth), p, 4, o, no, nt, hc) == want, v
        assert b"per_group" in L.frz_last_error()
    # q = 0 reads no entry and is a no-op
    a, p = pg(0, 0)
    assert fn(ms, 0, c, None, None, None, p, 4, None, None, None, None) == 0
    # handles of another corpus: query order, then subset, boost, groups within a query
    assert fn(ms, 2, c, None, None, h(g, oth), ok, 4, o, no, nt, hc) == INVALID
    assert b"groups of query 1 were made on another corpus" in L.frz_last_error()
    assert fn(ms, 2, c, h(None, oth), None, h(oth, g), ok, 4, o, no, nt, hc) == INVALID
    assert b"groups of query 0" in L.frz_last_error()
    assert fn(ms, 2, c, h(oth, None), h(oth, None), h(oth, None), ok, 4, o, no, nt, hc) == INVALID
    assert b"subset of query 0" in L.frz_last_error()
    assert fn(ms, 2, c, None, h(oth, None), h(oth, None), ok, 4, o, no, nt, hc) == INVALID
    assert b"boost of query 0" in L.frz_last_error()
    # then frz_match_list_batch's: NULL n_out, q * k overflow, NULL out
    assert fn(ms, 2, c, None, None, mine_g, ok, 4, o, None, nt, hc) == INVALID
    assert b"null n_out" in L.frz_last_error()
    assert fn(ms, 2, c, None, None, mine_g, ok, 2**63, o, no, nt, hc) == INVALID
    assert b"overflows" in L.frz_last_error()
    assert fn(ms, 2, c, None, None, mine_g, ok, 4, None, no, nt, hc) == INVALID
    assert b"null out" in L.frz_last_error()
    assert fake.raw == b"\0" * 4096 and not cnt.any()
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    # every argument is valid: the call reaches the device check (NULL per_group, groups, counts and k = 0 included)
    for gs, p, k, counts in ((mine_g, ok, 4, hc), (None, None, 4, None), (h(g, g), None, 0, None), (mine_g, ok, 0, h(None, None))):
        assert fn(ms, 2, c, h(g, None), h(None, g), gs, p, k, o if k else None, no, None, counts) == NO_DEVICE
    assert not cnt.any()


def test_budget_arithmetic(H):
    rec = H.h_record_bytes()
    assert rec == 32
    rng = np.random.default_rng(1)
    for _ in range(500):
        base = int(rng.integers(1, 64 << 20))
        groups = int(rng.choice([0, 1, 7, 1000, int(rng.integers(1, 2**32))]))
        rows = int(rng.integers(1, 1 << 21))
        extra = groups * 12 + rows + rec if groups else 0
        assert H.h_collapse_bytes(groups, rows) == extra
        q = BUDGET // (base + extra)
        assert H.h_collapse_fit(BUDGET, base, groups, rows) == (q if q >= 2 else 0)
    # at the 512 MiB budget, a small corpus's queries fit two to a sub-batch up to about 22 M groups
    base = 100_000
    assert H.h_collapse_fit(BUDGET, base, 22_000_000, 3000) == 2
    assert H.h_collapse_fit(BUDGET, base, 23_000_000, 3000) == 0
    assert H.h_collapse_fit(BUDGET, base, 24_000_000, 3000) == 0
    assert [H.h_rounds(p) for p in (1, 3, 32, 33, U64_MAX, 0xFFFFFFFF)] == [1, 3, 32, 0, 0, 0]


def random_query(rng, n_index, n_groups_max):
    rows = np.zeros(int(rng.integers(0, 1500)), dtype=F.MATCH_DTYPE)
    rows["index"] = np.sort(rng.choice(n_index, len(rows), replace=False)).astype(np.uint32)
    rows["score"] = rng.integers(0, [4, 300, 65536][int(rng.integers(0, 3))], len(rows)).astype(np.uint16)
    rows["exact"] = rng.integers(0, 2, len(rows))
    sort = list(SortStrategy)[int(rng.integers(0, 4))]
    kind = int(rng.integers(0, 6))   # every row in no group, own, one, dup, short (ids past the array: no group), no groups
    n_groups = [1, n_index, 1, int(rng.integers(1, 60)), 9, 0][kind]
    if kind == 5:
        ids = None
    else:
        ids = [np.full(n_index, 0xFFFFFFFF, np.uint32), np.arange(n_index, dtype=np.uint32), np.zeros(n_index, np.uint32),
               rng.integers(0, n_groups, n_index).astype(np.uint32), rng.integers(0, 9, n_index // 3).astype(np.uint32)][kind]
        if kind == 3:
            ids[rng.random(n_index) < 0.2] = 0xFFFFFFFF
    boost = rng.integers(-300, 301, int(rng.integers(0, n_index + 1))).astype(np.int16) if rng.random() < 0.4 else None
    members = np.flatnonzero(rng.random(n_index) < rng.choice([0.0, 0.3, 1.0])) if rng.random() < 0.4 else None
    per_group = [1, 2, 3, 32, None][int(rng.integers(0, 5))]
    return dict(rows=rows, sort=sort, ids=ids, n_groups=n_groups, boost=boost, members=members, per_group=per_group,
                wants=bool(rng.random() < 0.6))


@pytest.mark.parametrize("seed", range(6))
def test_sub_batch_reproduces_collapse(H, seed):
    """ns queries of every shape share one sub-batch's tables and rounds: each query's kept rows, in L's order, are the
    collapse of its L, and the counts read back are its counts."""
    rng = np.random.default_rng(seed)
    n_index, G = 4000, 4000
    ns = int(rng.integers(1, 65))
    qs = [random_query(rng, n_index, G) for _ in range(ns)]
    lists, bits, keeps = [], [], []
    for q in qs:
        lists.append(np.ascontiguousarray(q["rows"][::-1] if q["sort"].is_reversed() else q["rows"]))
        if q["members"] is None:
            bits.append(None)
        else:
            b = np.zeros((n_index + 31) // 32, np.uint32)
            np.bitwise_or.at(b, q["members"] >> 5, (np.uint32(1) << (q["members"] & 31).astype(np.uint32)))
            bits.append(b)
        keeps.append(np.zeros(max(len(q["rows"]), 1), np.uint8))
    orders = np.array([BY_KEY if q["boost"] is not None else BY_SCORE if q["sort"].is_by_score() else BY_INDEX for q in qs], np.uint8)
    counts_back = np.zeros(ns * G, np.uint32)
    args = [np.array(v or [0], np.uint64) for v in (
        [len(x) for x in lists], [0 if q["ids"] is None else len(q["ids"]) for q in qs],
        [U64_MAX if q["per_group"] is None else q["per_group"] for q in qs], [0 if q["boost"] is None else len(q["boost"]) for q in qs],
        [n_index] * ns)]
    n, n_ids, per_group, n_boost, n_bits = (a.ctypes.data for a in args)
    reversed_ = np.array([q["sort"].is_reversed() for q in qs], np.uint8)
    wants = np.array([q["wants"] for q in qs], np.uint8)
    n_back = H.h_batch_collapse(ns, ptrs(lists), n, ptrs([q["ids"] for q in qs]), n_ids, per_group, orders.ctypes.data,
                                reversed_.ctypes.data, ptrs([q["boost"] for q in qs]), n_boost, ptrs(bits), n_bits, wants.ctypes.data,
                                G, ptrs(keeps), counts_back.ctypes.data)
    assert n_back != 0xFFFFFFFF, "a round table is not zero after the rounds"
    assert n_back == sum(1 for q in qs if q["wants"] and q["ids"] is not None)
    slot = 0
    for j, q in enumerate(qs):
        rows = q["rows"] if q["members"] is None else q["rows"][np.isin(q["rows"]["index"], q["members"])]
        if q["boost"] is not None:
            L = rank_by_boost(rows, q["boost"], q["sort"].is_reversed())
        else:
            L = rows[::-1] if q["sort"].is_reversed() else rows
            if q["sort"].is_by_score():
                L = L[np.argsort(-L["score"].astype(np.int64), kind="stable")]
        kept = set(lists[j][keeps[j][:len(lists[j])].astype(bool)]["index"].tolist())
        got = L[np.isin(L["index"], list(kept))]
        if q["ids"] is None:
            assert np.array_equal(got, L), j   # a query without groups keeps its members
            continue
        want, wcounts = collapse(L, q["ids"], q["per_group"], q["n_groups"])
        assert len(kept) == len(want) and np.array_equal(got, want), (j, q["per_group"], q["sort"])
        if q["wants"]:
            assert np.array_equal(counts_back[slot * G: slot * G + q["n_groups"]], wcounts), j
            slot += 1
