"""Batched top-K on the GPU (frz_match_list_batch_top): for every query j, its rows, n_out and n_total must be exactly what
frz_match_list_top returns for that matcher on the same corpus, across batched-class queries and the queries that run the
single-query pipeline inside the call, batch sizes around the sub-batch size, corpora with removed, replaced and appended
rows, repeated matchers, and survivor lists that overflow.  Needs a CUDA device."""
import ctypes as C
import random

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200 import synth
from frizbee_b200.types import CaseMatching, Config, Matching, Pattern, Scoring, SortStrategy
from oracle import pyoracle
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
    """Batched-class queries over the configuration space, with fallback queries interleaved.  Returns the matchers and how
    many of them are of the batched class (on corpora of at most 65536 rows, where max_typos=None qualifies too)."""
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


@pytest.fixture
def limits():
    """Sets the batched path's limits for one test (F.batch_limits) and restores the defaults afterwards."""
    yield F.batch_limits
    F.batch_limits()


def check(ms, corpus, k, batched):
    """Every query equals its frz_match_list_top call, and `batched` of them were answered by the batched kernels."""
    rows, n_out, n_total = F.match_list_batch_top(ms, corpus, k)
    last = F.batch_last()
    assert last["batched"] == batched and last["overflowed"] == 0, (last, batched)
    assert rows.shape == (len(ms), k)
    for j, m in enumerate(ms):
        top, total = m.match_list_top_array(corpus, k)
        assert n_total[j] == total and n_out[j] == len(top), (j, k, n_total[j], total)
        assert np.array_equal(rows[j, :len(top)], top), (j, k)
        assert not rows[j, len(top):].view(np.uint64).any(), (j, k)   # unused rows are not written
    return rows, n_out, n_total


@pytest.mark.parametrize("forced", [False, True], ids=["default-limits", "batched-from-2"])
@pytest.mark.parametrize("q", [1, 2, 31, 32, 33, 64, 257])
def test_mixed_batches_equal_the_single_query_calls(q, forced, limits):
    """With the default limits the call batches from 32 batched-class queries on; with the query limit at 2 every batch of
    two or more such queries runs the batched kernels."""
    rows = corpus_list(5000, seed=q, long_every=97)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, q, seed=q)
    if forced:
        limits(0, 2)
    want = nb if nb >= (2 if forced else 32) else 0
    for k in (0, 1, 10):
        check(ms, corpus, k, want)


def test_k_at_and_past_the_totals():
    """A corpus of fewer rows than the batched path's largest k: k = 1, 10, the largest total and more than the corpus all
    run k_batch_top, the largest total through its full sort of every kept row."""
    rows = corpus_list(900, seed=7)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, 40, seed=7, with_fallbacks=False)
    _, _, tot = check(ms, corpus, 10, nb)
    check(ms, corpus, 1, nb)
    check(ms, corpus, int(tot.max()) if tot.max() > 0 else 1, nb)
    check(ms, corpus, len(rows) + 5, nb)


def test_thousand_queries_and_the_oracle():
    rows = corpus_list(2000, seed=11)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, 1000, seed=11, with_fallbacks=False)
    out, n_out, _ = check(ms, corpus, 10, nb)
    assert F.batch_last()["sub_batches"] == 16
    data, offsets = F.pack_host(rows)
    rng = random.Random(3)
    for j in rng.sample(range(len(ms)), 20):
        want = pyoracle.match_list_packed(ms[j]._patterns, ms[j].config, data, offsets)[:10]
        assert np.array_equal(out[j, :n_out[j]], want), j


@pytest.mark.parametrize("n", [0, 700, 5 * 1024 + 300])
def test_corpus_shapes_and_edits(n):
    """The empty corpus, one partial tile, several tiles with a partial last one, and the same after removing, replacing and
    appending rows, on the batched kernels, with fallback queries in the same call."""
    rows = corpus_list(n, seed=n, long_every=53)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows or ["foo"], 40, seed=n, with_fallbacks=False)
    more, nb2 = batch_matchers(rows or ["foo"], 14, seed=n + 1)
    ms, nb = ms + more, nb + nb2
    check(ms, corpus, 10, nb)
    if n:
        corpus.remove(np.arange(0, n, 3, dtype=np.uint32))
        check(ms, corpus, 10, nb)
        corpus.replace_list(np.arange(1, n, 7, dtype=np.uint32), ["foo_bar"] * len(range(1, n, 7)))
        check(ms, corpus, 10, nb)
        corpus.append_list(corpus_list(1500, seed=n + 1))
        check(ms, corpus, 10, nb)


def test_repeated_matchers_and_repeatable_calls():
    """The same matchers several times in one sub-batch; two identical calls agree, and every matcher's own call afterwards
    equals its call before."""
    rows = corpus_list(4000, seed=5)
    corpus = F.Corpus.from_list(rows)
    base, _ = batch_matchers(rows, 8, seed=5, with_fallbacks=False)
    before = [m.match_list_top_array(corpus, 10) for m in base]
    ms = base * 4 + base[::-1] + [base[0]] * 5
    a = check(ms, corpus, 10, len(ms))
    assert F.batch_last()["sub_batches"] == 1
    b = F.match_list_batch_top(ms, corpus, 10)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    for m, (top, total) in zip(base, before):
        t2, tot2 = m.match_list_top_array(corpus, 10)
        assert tot2 == total and np.array_equal(t2, top)


def test_overflowing_survivor_lists_give_equal_results():
    """Every row survives a one-byte needle with one typo: the per-query lists of the batched path (max(n / 4, 65536) records
    per class) overflow, and the sub-batch runs again query by query."""
    n = 200_000
    rows = ["ab"] * n
    corpus = F.Corpus.from_list(rows)
    ms = [F.Matcher(c, Config(max_typos=1, sort=s)) for c, s in zip("ab" * 20, list(SortStrategy) * 10)]
    data, offsets = F.pack_host(rows)
    counts = pyoracle.match_list_packed(ms[0]._patterns, ms[0].config, data, offsets)
    assert len(counts) > max(n // 4, 1 << 16)   # one class list would have to hold more than its capacity
    out, n_out, n_total = F.match_list_batch_top(ms, corpus, 10)
    last = F.batch_last()
    assert last["overflowed"] == len(ms) and last["batched"] == 0, last
    for j, m in enumerate(ms):
        top, total = m.match_list_top_array(corpus, 10)
        assert n_total[j] == total and n_out[j] == len(top) and np.array_equal(out[j, :len(top)], top), j


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
    for m in ms:   # the single-query workspaces first, so that they do not count below
        m.match_list_top_array(corpus, 10)
    start = _bytes().frz_debug_device_bytes()
    _bytes().frz_debug_device_bytes_peak(1)
    F.match_list_batch_top(ms[:64], corpus, 10)
    assert F.batch_last()["batched"] == 64
    peak64 = _bytes().frz_debug_device_bytes_peak(1) - start
    assert _bytes().frz_debug_device_bytes() == start
    F.match_list_batch_top(ms, corpus, 10)
    assert F.batch_last()["batched"] == 1024
    peak1024 = _bytes().frz_debug_device_bytes_peak(1) - start
    assert _bytes().frz_debug_device_bytes() == start
    assert peak1024 <= peak64 + (1024 - 64) * (10 * 8 + 2048 + 64)


def test_corpus_size_limit_by_typo_budget(limits):
    """Past the corpus-size limit only max_typos = 0 queries batch (up to 2^21 rows); the others run the loop in the same
    call.  The limit is lowered below this corpus's size to show both sides on a small corpus."""
    rows = corpus_list(5000, seed=13)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, 80, seed=13, with_fallbacks=False)
    assert nb == len(ms)
    no_typo = sum(1 for m in ms if m.config.max_typos == 0)
    assert 2 <= no_typo < len(ms)
    limits(1000, 2)
    check(ms, corpus, 10, no_typo)
    limits(0, 2)
    check(ms, corpus, 10, len(ms))
