"""The batched top-K call without a GPU: frz_match_list_batch_top's argument checks and missing-device status, and its
per-query position arithmetic (frizbee_b200/csrc/batch_plan.cuh, built for the CPU from tests/harness/batch_plan_harness.cpp)
against a numpy restatement of frz_match_list_top for every query of a batch."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200.types import Config, SortStrategy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "harness", "batch_plan_harness.cpp")
LIB = os.path.join(ROOT, "tests", "harness", "libbatch_plan_harness.so")
DEPS = [SRC, os.path.join(ROOT, "frizbee_b200", "csrc", "batch_plan.cuh")]
INVALID, NO_DEVICE = 1, 8


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", LIB, SRC], check=True)
    L = C.CDLL(LIB)
    L.h_batch_top.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]
    L.h_batch_top.restype = None
    return L


def _fn():
    L = F.lib()
    L.frz_match_list_batch_top.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
    return L.frz_match_list_batch_top


def test_argument_checks_and_no_device():
    import torch
    fn = _fn()
    m = F.Matcher("foo", Config())
    ms = (C.c_void_p * 2)(m._h.value, m._h.value)
    fake_corpus = C.create_string_buffer(64)   # never dereferenced: every check below comes first
    out = np.zeros(8, dtype=F.MATCH_DTYPE)
    n_out, n_total = np.zeros(2, dtype=np.uint64), np.zeros(2, dtype=np.uint64)
    o, no, nt = out.ctypes.data, n_out.ctypes.data, n_total.ctypes.data
    assert fn(None, 2, fake_corpus, 4, o, no, nt) == INVALID                          # NULL ms
    assert fn(None, 0, fake_corpus, 4, o, no, nt) == INVALID
    assert fn((C.c_void_p * 2)(m._h.value, None), 2, fake_corpus, 4, o, no, nt) == INVALID   # a NULL matcher
    assert fn(ms, 2, None, 4, o, no, nt) == INVALID                                  # NULL corpus
    assert fn(ms, 0, None, 4, o, no, nt) == INVALID
    assert fn(ms, 2, fake_corpus, 4, o, None, nt) == INVALID                         # NULL n_out, q > 0
    assert fn(ms, 2, fake_corpus, 4, None, no, nt) == INVALID                        # NULL out, q * k > 0
    assert fn(ms, 2, fake_corpus, 2**63, o, no, nt) == INVALID                       # q * k overflows
    assert fn(ms, 2, fake_corpus, 2**62, o, no, nt) == INVALID                       # q * k * sizeof(match) overflows size_t
    assert fn(ms, 0, fake_corpus, 4, None, None, None) == 0                          # q = 0: no-op
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    assert fn(ms, 2, fake_corpus, 4, o, no, nt) == NO_DEVICE
    assert fn(ms, 2, fake_corpus, 0, None, no, None) == NO_DEVICE                    # k = 0: out and n_total may be NULL
    assert F.batch_last() == {"batched": 0, "overflowed": 0, "sub_batches": 0, "launches": 0}
    m.close()


def _lists(rng, q, n_max, score_hi):
    """Per-query index-ordered lists as the scoring kernels leave them (reversed for the *_DESC strategies)."""
    sorts = rng.integers(0, 4, q)
    lists = []
    for j in range(q):
        n = int(rng.choice([0, 1, 2, rng.integers(0, n_max + 1)]))
        r = np.zeros(n, dtype=F.MATCH_DTYPE)
        r["index"] = np.sort(rng.choice(10 * max(n, 1), size=n, replace=False)).astype(np.uint32)
        r["score"] = rng.integers(0, score_hi, n).astype(np.uint16)
        if rng.random() < 0.3 and n:   # a block of tied scores
            r["score"][rng.random(n) < 0.6] = int(rng.integers(0, score_hi))
        r["exact"] = rng.integers(0, 2, n)
        if SortStrategy(int(sorts[j])).is_reversed():
            r = r[::-1]
        lists.append(np.ascontiguousarray(r))
    return sorts, lists


def _want(r, sort, k):
    if SortStrategy(int(sort)).is_by_score():
        r = r[np.argsort(-r["score"].astype(np.int64), kind="stable")]
    return r[:k]


@pytest.mark.parametrize("score_hi", [4, 300, 65536])
def test_plan_equals_the_truncated_stable_sort(H, score_hi):
    rng = np.random.default_rng(score_hi)
    for q in (1, 2, 33):
        sorts, lists = _lists(rng, q, 3000, score_hi)
        counts = np.array([len(r) for r in lists], dtype=np.uint64)
        cat = np.ascontiguousarray(np.concatenate(lists)) if counts.sum() else np.zeros(1, dtype=F.MATCH_DTYPE)
        by_score = np.array([SortStrategy(int(s)).is_by_score() for s in sorts], dtype=np.uint8)
        for k in (0, 1, 10, 1024, int(counts.max()) + 5):
            out = np.zeros(max(q * k, 1), dtype=F.MATCH_DTYPE)
            n_out = np.zeros(q, dtype=np.uint64)
            H.h_batch_top(cat.ctypes.data, counts.ctypes.data, by_score.ctypes.data, q, k, out.ctypes.data, n_out.ctypes.data)
            for j in range(q):
                want = _want(lists[j], sorts[j], k)
                assert n_out[j] == len(want), (q, k, j)
                assert np.array_equal(out[j * k:j * k + len(want)], want), (q, k, j, SortStrategy(int(sorts[j])))
                assert not out[j * k + len(want):(j + 1) * k].view(np.uint64).any()
