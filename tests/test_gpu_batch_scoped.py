"""The batched call with per-query subsets and boosts on the GPU (frz_match_list_batch): for every query j, its rows, n_out
and n_total must be exactly what its single-query call returns (frz_match_list_ranked with a boost, else
frz_match_list_subset_top with a subset, else frz_match_list_top), across batched-class and fallback queries, batch sizes
around the sub-batch size, subsets and boosts of every shape, corpora edited after the handles were made, repeated handles
and matchers, and survivor lists that overflow.  Needs a CUDA device."""
import ctypes as C
import random

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200.types import CaseMatching, Config, Matching, Pattern, Scoring, SortStrategy
from ranking import rank_by_boost
from scorings import scorings

pytestmark = pytest.mark.gpu

WORDS = ["foo", "fooBar", "foo_bar", "barfoo", "FooBaz", "f-o-o", "xyz", "abcdefghijklmnop", "a/b/c/foo.rs", "fo", "oof",
         "src/matcher/mod.rs", "needle in a haystack", "Hello, World", ""]


def corpus_list(n, seed=1, long_every=0):
    rng = random.Random(seed)
    out = []
    for i in range(n):
        s = rng.choice(WORDS) + ("" if rng.random() < 0.5 else rng.choice(WORDS))
        if long_every and i % long_every == 0:
            s = s + "x" * rng.randrange(60, 300) + rng.choice(WORDS)
        out.append(s)
    return out


def needle_from(rows, rng, lo=1, hi=12):
    s = ""
    while not s:
        s = rng.choice(rows)
    a = rng.randrange(len(s))
    return s[a:a + rng.randrange(lo, hi + 1)]


def batch_matchers(rows, q, seed, with_fallbacks=True):
    """Batched-class queries over the configuration space, with fallback queries interleaved (multi-pattern, negated,
    literal, unicode, long and empty needles).  Returns the matchers and how many of them are of the batched class (on
    corpora of at most 65536 rows, where max_typos=None qualifies too)."""
    rng = random.Random(seed)
    scs = scorings(seed, 8, 64)
    out, n_batchable = [], 0
    for j in range(q):
        kind = j % 7 if with_fallbacks else 0
        cfg = Config(max_typos=rng.choice([0, 1, 2, 3, 15, None]), casing=rng.choice(list(CaseMatching)),
                     sort=rng.choice(list(SortStrategy)), emulate_lanes=rng.choice([16, 32, 64]),
                     scoring=rng.choice(scs))
        if kind == 1:
            out.append(F.Matcher([Pattern(needle_from(rows, rng, 1, 4)), Pattern(needle_from(rows, rng, 1, 3))], cfg))
        elif kind == 2:
            out.append(F.Matcher([Pattern(needle_from(rows, rng, 1, 4)), Pattern("zz", negated=True)], cfg))
        elif kind == 3:
            out.append(F.Matcher(needle_from(rows, rng, 1, 4), cfg.with_(matching=rng.choice(
                [Matching.Exact, Matching.Prefix, Matching.Suffix, Matching.Substring]))))
        elif kind == 4:
            out.append(F.Matcher(needle_from(rows, rng, 1, 3) + "é", cfg))
        elif kind == 5:
            out.append(F.Matcher("f" * rng.randrange(65, 120), cfg.with_(max_typos=None, scoring=Scoring())))
        elif kind == 6 and j % 2:
            out.append(F.Matcher("", cfg))
        else:
            n = rng.choice([1, 2, 3, 5, 8, 12, 20, 40, 64])
            out.append(F.Matcher(needle_from(rows, rng, n, n) if n <= 12 else ("foo_bar" * 10)[:n], cfg))
            n_batchable += 1
    return out, n_batchable


def scopes_for(corpus, q, seed):
    """Per query an independent random subset, boost, both or neither (None).  Returns (subsets, boosts, their members and
    boost values for the spec)."""
    rng = np.random.default_rng(seed)
    n = len(corpus)
    subsets, boosts, members, values = [], [], [], []
    for j in range(q):
        kind = j % 4 if j < 8 else int(rng.integers(0, 4))   # neither, subset, boost, both
        s = b = mem = val = None
        if kind & 1:
            density = rng.choice([0.0, 0.01, 0.2, 0.5, 1.0])
            mem = np.flatnonzero(rng.random(n) < density).astype(np.uint32)
            s = corpus.subset(mem)
        if kind & 2:
            lo, hi = [(0, 256), (-1000, 1000), (-32768, 32768)][int(rng.integers(0, 3))]
            val = rng.integers(lo, hi, int(rng.integers(0, n + 1))).astype(np.int16)   # rows past it have boost 0
            b = corpus.boost(val)
        subsets.append(s)
        boosts.append(b)
        members.append(mem)
        values.append(val)
    return subsets, boosts, members, values


def single(m, corpus, k, s, b):
    """The query's single-query call: (rows, total)."""
    if b is not None:
        return m.match_list_ranked_array(corpus, b, k, subset=s)
    if s is not None:
        return m.match_list_subset_top_array(corpus, s, k)
    return m.match_list_top_array(corpus, k)


@pytest.fixture
def limits():
    """Sets the batched path's limits for one test (F.batch_limits) and restores the defaults afterwards."""
    yield F.batch_limits
    F.batch_limits()


def check(ms, corpus, k, subsets, boosts, batched, overflowed=0):
    """Every query equals its single-query call, and `batched` of them were answered by the batched kernels."""
    rows, n_out, n_total = F.match_list_batch(ms, corpus, k, subsets=subsets, boosts=boosts)
    last = F.batch_last()
    assert last["batched"] == batched and last["overflowed"] == overflowed, (last, batched)
    assert rows.shape == (len(ms), k)
    for j, m in enumerate(ms):
        top, total = single(m, corpus, k, subsets[j] if subsets else None, boosts[j] if boosts else None)
        assert n_total[j] == total and n_out[j] == len(top), (j, k, n_total[j], total)
        assert np.array_equal(rows[j, :len(top)], top), (j, k)
        assert not rows[j, len(top):].view(np.uint64).any(), (j, k)   # unused rows are not written
    return rows, n_out, n_total


@pytest.mark.parametrize("forced", [False, True], ids=["default-limits", "batched-from-2"])
@pytest.mark.parametrize("q", [1, 2, 31, 32, 33, 64, 257])
def test_mixed_scoped_batches_equal_the_single_query_calls(q, forced, limits):
    rows = corpus_list(5000, seed=q, long_every=97)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, q, seed=q)
    subsets, boosts, _, _ = scopes_for(corpus, q, seed=q)
    if forced:
        limits(0, 2)
    want = nb if nb >= (2 if forced else 32) else 0
    for k in (0, 1, 10):
        check(ms, corpus, k, subsets, boosts, want)


def _spec(m, corpus, k, members, boost):
    """rank_by_boost (or the strategy's stable order) of match_list_into filtered by membership, truncated."""
    rows = m.match_list_into_array(corpus)
    if members is not None:
        rows = rows[np.isin(rows["index"], members)]
    sort = m.config.sort
    if boost is not None:
        rows = rank_by_boost(rows, boost, sort.is_reversed())
    else:
        rows = rows[::-1] if sort.is_reversed() else rows
        if sort.is_by_score():
            rows = rows[np.argsort(-rows["score"].astype(np.int64), kind="stable")]
    return rows[:k], len(rows)


def test_against_the_spec(limits):
    rows = corpus_list(6000, seed=21)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, 96, seed=21, with_fallbacks=False)
    subsets, boosts, members, values = scopes_for(corpus, len(ms), seed=21)
    for k in (10, 300):
        out, n_out, n_total = F.match_list_batch(ms, corpus, k, subsets=subsets, boosts=boosts)
        assert F.batch_last()["batched"] == nb
        for j in random.Random(k).sample(range(len(ms)), 32):
            want, total = _spec(ms[j], corpus, k, members[j], values[j])
            assert n_total[j] == total and np.array_equal(out[j, :n_out[j]], want), j


def test_subset_shapes_and_shared_handles(limits):
    """Empty subsets, every row, duplicates in `which`; the same subset, boost and matcher for many queries."""
    rows = corpus_list(3000, seed=4)
    corpus = F.Corpus.from_list(rows)
    base, _ = batch_matchers(rows, 6, seed=4, with_fallbacks=False)
    n = len(rows)
    shapes = [corpus.subset([]), corpus.subset(np.arange(n)), corpus.subset(np.r_[np.arange(0, n, 5), np.arange(0, n, 10)]),
              corpus.subset([n - 1, n - 1, 0])]
    boost = corpus.boost(np.arange(n) % 200)
    ms, subsets, boosts = [], [], []
    for m in base:
        for s in shapes:
            for b in (None, boost):
                ms.append(m)
                subsets.append(s)
                boosts.append(b)
    limits(0, 2)
    for k in (0, 1, 10, 1024):   # 10 and 1024 lie past the totals of the small subsets
        check(ms, corpus, k, subsets, boosts, len(ms))


@pytest.mark.parametrize("n", [0, 700, 5 * 1024 + 300])
def test_corpus_shapes_and_edits(n, limits):
    """The empty corpus, one partial tile, several tiles; then, with the same handles, removed members, replaced rows, and
    appended rows (not members, boost 0 until Boost.set)."""
    rows = corpus_list(n, seed=n, long_every=53)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows or ["foo"], 40, seed=n, with_fallbacks=False)
    more, nb2 = batch_matchers(rows or ["foo"], 14, seed=n + 1)
    ms, nb = ms + more, nb + nb2
    subsets, boosts, _, _ = scopes_for(corpus, len(ms), seed=n)
    limits(0, 2)
    check(ms, corpus, 10, subsets, boosts, nb)
    if n:
        corpus.remove(np.arange(0, n, 3, dtype=np.uint32))
        check(ms, corpus, 10, subsets, boosts, nb)
        corpus.replace_list(np.arange(1, n, 7, dtype=np.uint32), ["foo_bar"] * len(range(1, n, 7)))
        check(ms, corpus, 10, subsets, boosts, nb)
        corpus.append_list(corpus_list(1500, seed=n + 1))
        check(ms, corpus, 10, subsets, boosts, nb)
        new = np.arange(n, n + 1500, dtype=np.uint32)
        for b in boosts:
            if b is not None:
                b.set(new, (new % 300).astype(np.int16))
        check(ms, corpus, 10, subsets, boosts, nb)


def test_k_past_the_totals_and_past_the_batched_limit(limits):
    rows = corpus_list(900, seed=8)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, 40, seed=8, with_fallbacks=False)
    subsets, boosts, _, _ = scopes_for(corpus, len(ms), seed=8)
    limits(0, 2)
    check(ms, corpus, len(rows) + 5, subsets, boosts, nb)
    check(ms, corpus, 1024, subsets, boosts, nb)
    check(ms, corpus, 1025, subsets, boosts, 0)   # k > 1024: every query runs its single-query call


def test_plain_batches_are_unchanged(limits):
    """No subsets and no boosts (None, or lists of None) equal match_list_batch_top, with the same launches per sub-batch;
    a sub-batch with scoped queries launches as many kernels."""
    rows = corpus_list(4000, seed=12)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, 70, seed=12, with_fallbacks=False)
    limits(0, 2)
    top = F.match_list_batch_top(ms, corpus, 10)
    last_top = F.batch_last()
    assert last_top["batched"] == nb
    for subsets, boosts in ((None, None), ([None] * len(ms), [None] * len(ms)), ([None] * len(ms), None)):
        got = F.match_list_batch(ms, corpus, 10, subsets=subsets, boosts=boosts)
        assert F.batch_last() == last_top
        for x, y in zip(top, got):
            assert np.array_equal(x, y)
    subsets, boosts, _, _ = scopes_for(corpus, len(ms), seed=12)
    check(ms, corpus, 10, subsets, boosts, nb)
    assert F.batch_last()["launches"] == last_top["launches"]


def test_handles_of_another_corpus_are_refused():
    rows = corpus_list(500, seed=3)
    a, b = F.Corpus.from_list(rows), F.Corpus.from_list(rows)
    ms, _ = batch_matchers(rows, 4, seed=3, with_fallbacks=False)
    sa, sb, ba, bb = a.subset([1, 2]), b.subset([1, 2]), a.boost([1, 2]), b.boost([1, 2])
    for subsets, boosts in (([sa, sb, None, None], None), (None, [None, None, ba, bb]), ([sa] * 4, [bb, ba, ba, ba])):
        with pytest.raises(F.FrizbeeError) as e:
            F.match_list_batch(ms, a, 10, subsets=subsets, boosts=boosts)
        assert e.value.status == 1
    check(ms, a, 10, [sa] * 4, [ba] * 4, 0)


def test_overflowing_survivor_lists_give_equal_results():
    """Every row survives a one-byte needle with one typo: the per-query lists of the batched path overflow, and the
    sub-batch runs again query by query through the scoped and ranked single-query calls."""
    n = 200_000
    rows = ["ab"] * n
    corpus = F.Corpus.from_list(rows)
    ms = [F.Matcher(c, Config(max_typos=1, sort=s)) for c, s in zip("ab" * 20, list(SortStrategy) * 10)]
    subsets, boosts, _, _ = scopes_for(corpus, len(ms), seed=5)
    assert any(s is not None for s in subsets) and any(b is not None for b in boosts)
    check(ms, corpus, 10, subsets, boosts, 0, overflowed=len(ms))


def _bytes():
    L = F.lib()
    L.frz_debug_device_bytes.restype = C.c_uint64
    L.frz_debug_device_bytes.argtypes = []
    L.frz_debug_device_bytes_peak.restype = C.c_uint64
    L.frz_debug_device_bytes_peak.argtypes = [C.c_int]
    return L


def test_device_memory_returns_and_does_not_grow_with_q():
    rows = corpus_list(20000, seed=9)
    corpus = F.Corpus.from_list(rows)
    ms, _ = batch_matchers(rows, 1024, seed=9, with_fallbacks=False)
    subsets, boosts, _, _ = scopes_for(corpus, 16, seed=9)
    subsets, boosts = (subsets * 64)[:1024], (boosts * 64)[:1024]
    for m, s, b in zip(ms, subsets, boosts):   # the single-query workspaces first, so that they do not count below
        single(m, corpus, 10, s, b)
    start = _bytes().frz_debug_device_bytes()
    _bytes().frz_debug_device_bytes_peak(1)
    F.match_list_batch(ms[:64], corpus, 10, subsets=subsets[:64], boosts=boosts[:64])
    assert F.batch_last()["batched"] == 64
    peak64 = _bytes().frz_debug_device_bytes_peak(1) - start
    assert _bytes().frz_debug_device_bytes() == start
    F.match_list_batch(ms, corpus, 10, subsets=subsets, boosts=boosts)
    assert F.batch_last()["batched"] == 1024
    peak1024 = _bytes().frz_debug_device_bytes_peak(1) - start
    assert _bytes().frz_debug_device_bytes() == start
    assert peak1024 <= peak64 + (1024 - 64) * (10 * 8 + 2048 + 64)
