"""The batched call with per-query subsets and boosts without a GPU: frz_match_list_batch's argument checks and
missing-device status, and the per-query member test, ranked value and row choice (frizbee_b200/csrc/batch_plan.cuh, built
for the CPU from tests/harness/batch_scoped_harness.cpp) against a numpy restatement of frz_match_list_subset_top and
frz_match_list_ranked for every query of a batch."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from cpu_harness import load
from frizbee_b200.types import Config, SortStrategy
from ranking import rank_by_boost

INVALID, NO_DEVICE = 1, 8
vp, u64 = C.c_void_p, C.c_uint64


@pytest.fixture(scope="module")
def H():
    L = load("batch_scoped_harness")
    L.h_batch_scoped_top.argtypes = [vp] * 9 + [u64, u64, vp, vp, vp]
    L.h_batch_scoped_top.restype = None
    return L


def _fn():
    L = F.lib()
    L.frz_match_list_batch.argtypes = [vp, u64, vp, vp, vp, u64, vp, vp, vp]
    return L.frz_match_list_batch


def test_argument_checks_and_no_device():
    import torch
    fn = _fn()
    m = F.Matcher("foo", Config())
    ms = (vp * 2)(m._h.value, m._h.value)
    fake_corpus = C.create_string_buffer(64)   # never dereferenced: every check below comes first
    # Without a device no real subset or boost can be made.  Stand-ins whose first field, the handle's corpus, is another
    # corpus (NULL) or fake_corpus: the corpus check reads nothing else.
    other = C.create_string_buffer(64)
    mine = C.create_string_buffer(C.addressof(fake_corpus).to_bytes(8, "little"), 64)
    none2 = (vp * 2)(None, None)
    out = np.zeros(8, dtype=F.MATCH_DTYPE)
    n_out, n_total = np.zeros(2, dtype=np.uint64), np.zeros(2, dtype=np.uint64)
    o, no, nt = out.ctypes.data, n_out.ctypes.data, n_total.ctypes.data
    assert fn(None, 2, fake_corpus, None, None, 4, o, no, nt) == INVALID                        # NULL ms
    assert fn((vp * 2)(m._h.value, None), 2, fake_corpus, none2, none2, 4, o, no, nt) == INVALID   # a NULL matcher
    assert fn(ms, 2, None, None, None, 4, o, no, nt) == INVALID                                 # NULL corpus
    for j in range(2):   # a subset or boost of another corpus, at either position
        h = [None, None]
        h[j] = C.addressof(other)
        assert fn(ms, 2, fake_corpus, (vp * 2)(*h), None, 4, o, no, nt) == INVALID
        assert fn(ms, 2, fake_corpus, None, (vp * 2)(*h), 4, o, no, nt) == INVALID
        assert fn(ms, 2, fake_corpus, none2, (vp * 2)(*h), 4, o, no, nt) == INVALID
    # ... checked before the other arguments' checks and the device check
    bad = (vp * 2)(None, C.addressof(other))
    assert fn(ms, 2, fake_corpus, bad, None, 4, None, None, None) == INVALID
    assert fn(ms, 2, fake_corpus, None, None, 4, o, None, nt) == INVALID                        # NULL n_out, q > 0
    assert fn(ms, 2, fake_corpus, none2, none2, 4, None, no, nt) == INVALID                     # NULL out, q * k > 0
    assert fn(ms, 2, fake_corpus, None, None, 2**63, o, no, nt) == INVALID                      # q * k overflows
    assert fn(ms, 2, fake_corpus, None, None, 2**62, o, no, nt) == INVALID                      # ... size_t
    assert fn(ms, 0, fake_corpus, None, None, 4, None, None, None) == 0                         # q = 0: no-op
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    mine2 = (vp * 2)(C.addressof(mine), C.addressof(mine))
    assert fn(ms, 2, fake_corpus, None, None, 4, o, no, nt) == NO_DEVICE
    assert fn(ms, 2, fake_corpus, none2, none2, 4, o, no, nt) == NO_DEVICE                      # NULL entries
    assert fn(ms, 2, fake_corpus, mine2, mine2, 4, o, no, nt) == NO_DEVICE                      # this corpus's handles
    assert fn(ms, 2, fake_corpus, mine2, None, 0, None, no, None) == NO_DEVICE                  # k = 0
    assert F.batch_last() == {"batched": 0, "overflowed": 0, "sub_batches": 0, "launches": 0}
    m.close()


def test_python_sequence_lengths():
    m = F.Matcher("foo", Config())
    corpus = object.__new__(F.Corpus)   # never reached: the lengths are checked first
    with pytest.raises(ValueError):
        F.match_list_batch([m, m], corpus, 4, subsets=[None])
    with pytest.raises(ValueError):
        F.match_list_batch([m, m], corpus, 4, boosts=[None, None, None])
    m.close()


def _bitmap(members, n_bits):
    """frz_subset's bitmap: the members below n_bits (at least one word, so that it has an address)."""
    words = np.zeros(max((n_bits + 31) // 32, 1), dtype=np.uint32)
    for i in members:
        if i < n_bits:
            words[i >> 5] |= np.uint32(1 << (i & 31))
    return words


def _query(rng, n_max, score_hi):
    """One query: its index-ordered rows, strategy, subset (or None: not scoped) and boost (or None: not ranked)."""
    n = int(rng.choice([0, 1, 2, rng.integers(0, n_max + 1)]))
    base = np.zeros(n, dtype=F.MATCH_DTYPE)
    n_index = 4 * max(n, 1)
    base["index"] = np.sort(rng.choice(n_index, size=n, replace=False)).astype(np.uint32)
    base["score"] = rng.integers(0, score_hi, n).astype(np.uint16)
    if rng.random() < 0.3 and n:   # a block of tied scores
        base["score"][rng.random(n) < 0.6] = int(rng.integers(0, score_hi))
    base["exact"] = rng.integers(0, 2, n)
    sort = SortStrategy(int(rng.integers(0, 4)))
    kind = int(rng.integers(0, 4))   # plain, scoped, ranked, both
    subset = boost = None
    if kind & 1:
        density = rng.choice([0.0, 0.01, 0.1, 0.5, 0.9, 1.0])
        n_bits = int(rng.choice([n_index, n_index // 2, 0]))   # rows past n_bits (appended later) are not members
        members = [i for i in range(n_bits) if rng.random() < density]
        subset = (_bitmap(members, n_bits), n_bits)
    if kind & 2:
        n_boost = int(rng.choice([n_index, n_index // 3, 0]))
        lo, hi = [(0, 256), (-1000, 1000), (-32768, 32768), (0, 1)][int(rng.integers(0, 4))]
        boost = rng.integers(lo, hi, max(n_boost, 1)).astype(np.int16)[:n_boost]
        if n_boost and rng.random() < 0.5:   # boosts that clamp at 0 and at 65535
            boost[rng.random(n_boost) < 0.3] = rng.choice([-32768, 32767])
    return base, sort, subset, boost


def _want(base, sort, subset, boost, k):
    """frz_match_list_ranked / _subset_top / _top restated: the members of the index-ordered list, then the ranked or the
    strategy's order, truncated.  Returns (rows, total)."""
    rows = base
    if subset is not None:
        words, n_bits = subset
        idx = rows["index"].astype(np.int64)
        inside = idx < n_bits
        bit = np.zeros(len(rows), dtype=bool)
        bit[inside] = (words[idx[inside] >> 5] >> (idx[inside] & 31).astype(np.uint32)) & 1 == 1
        rows = rows[bit]
    if boost is not None:
        rows = rank_by_boost(rows, boost, sort.is_reversed())
    else:
        if sort.is_reversed():
            rows = rows[::-1]
        if sort.is_by_score():
            rows = rows[np.argsort(-rows["score"].astype(np.int64), kind="stable")]
    return rows[:k], len(rows)


@pytest.mark.parametrize("score_hi", [4, 300, 65536])
def test_plan_equals_the_filtered_ranked_sort(H, score_hi):
    rng = np.random.default_rng(score_hi)
    for q in (1, 2, 33):
        qs = [_query(rng, 3000, score_hi) for _ in range(q)]
        lists = [np.ascontiguousarray(b[::-1] if s.is_reversed() else b) for b, s, _, _ in qs]
        counts = np.array([len(r) for r in lists], dtype=np.uint64)
        cat = np.ascontiguousarray(np.concatenate(lists)) if counts.sum() else np.zeros(1, dtype=F.MATCH_DTYPE)
        by_score = np.array([s.is_by_score() for _, s, _, _ in qs], dtype=np.uint8)
        scoped = np.array([sub is not None for _, _, sub, _ in qs], dtype=np.uint8)
        ranked = np.array([bo is not None for _, _, _, bo in qs], dtype=np.uint8)
        keep = []   # the arrays the pointers below point into
        bits, n_bits, boosts, n_boost = (vp * q)(), np.zeros(q, np.uint64), (vp * q)(), np.zeros(q, np.uint32)
        for j, (_, _, sub, bo) in enumerate(qs):
            if sub is not None:
                keep.append(sub[0])
                bits[j], n_bits[j] = sub[0].ctypes.data, sub[1]
            if bo is not None:
                b = np.ascontiguousarray(bo if len(bo) else np.zeros(1, np.int16))
                keep.append(b)
                boosts[j], n_boost[j] = b.ctypes.data, len(bo)
        total_max = max(int(counts.max()), 1)
        for k in (0, 1, 10, 1024, total_max + 5):
            out = np.zeros(max(q * k, 1), dtype=F.MATCH_DTYPE)
            n_out, n_total = np.zeros(q, dtype=np.uint64), np.zeros(q, dtype=np.uint64)
            H.h_batch_scoped_top(cat.ctypes.data, counts.ctypes.data, by_score.ctypes.data, scoped.ctypes.data, bits,
                                 n_bits.ctypes.data, ranked.ctypes.data, boosts, n_boost.ctypes.data, q, k, out.ctypes.data,
                                 n_out.ctypes.data, n_total.ctypes.data)
            for j, (base, sort, sub, bo) in enumerate(qs):
                want, total = _want(base, sort, sub, bo, k)
                ctx = (q, k, j, sort, sub is not None, bo is not None)
                assert n_total[j] == total and n_out[j] == len(want), ctx
                assert np.array_equal(out[j * k:j * k + len(want)], want), ctx
                assert not out[j * k + len(want):(j + 1) * k].view(np.uint64).any(), ctx


def test_member_and_ranked_value_edges(H):
    """Member densities 0 % and 100 %, a bitmap shorter than the list, and values that clamp at both ends, on one list."""
    n = 2000
    base = np.zeros(n, dtype=F.MATCH_DTYPE)
    base["index"] = np.arange(n, dtype=np.uint32) * 2
    base["score"] = (np.arange(n) * 37 % 65536).astype(np.uint16)
    cases = [(np.zeros(0, dtype=np.uint32), 0, None),                       # no member
             (_bitmap(range(2 * n), 2 * n), 2 * n, None),                     # every row
             (_bitmap(range(2 * n), n), n, None),                             # n_bits short of the list: the first half
             (None, 0, np.full(2 * n, -32768, np.int16)),                     # every value clamps at 0: index order
             (None, 0, np.full(2 * n, 32767, np.int16)),                      # most clamp at 65535
             (_bitmap(range(0, 2 * n, 6), 2 * n), 2 * n, np.full(n, 32767, np.int16))]   # boost shorter than the list
    for sort in SortStrategy:
        lst = np.ascontiguousarray(base[::-1] if sort.is_reversed() else base)
        for words, nb, bo in cases:
            k = 50
            sub = None if words is None else (words if len(words) else np.zeros(1, np.uint32), nb)
            out = np.zeros(k, dtype=F.MATCH_DTYPE)
            n_out, n_total = np.zeros(1, np.uint64), np.zeros(1, np.uint64)
            bits, boosts = (vp * 1)(sub[0].ctypes.data if sub else None), (vp * 1)(bo.ctypes.data if bo is not None else None)
            # (the argument arrays are named: a temporary's .ctypes.data outlives the array)
            args = [np.array([n], np.uint64), np.array([sort.is_by_score()], np.uint8), np.array([sub is not None], np.uint8),
                    np.array([nb], np.uint64), np.array([bo is not None], np.uint8),
                    np.array([len(bo) if bo is not None else 0], np.uint32)]
            cnt, bysc, scp, nbits, rk, nbo = args
            H.h_batch_scoped_top(lst.ctypes.data, cnt.ctypes.data, bysc.ctypes.data, scp.ctypes.data, bits, nbits.ctypes.data,
                                 rk.ctypes.data, boosts, nbo.ctypes.data, 1, k, out.ctypes.data, n_out.ctypes.data,
                                 n_total.ctypes.data)
            want, total = _want(base, sort, sub, bo, k)
            assert n_total[0] == total and n_out[0] == len(want), (sort, nb)
            assert np.array_equal(out[:len(want)], want), (sort, nb)
