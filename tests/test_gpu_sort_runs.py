"""The fused scatter's block-local sort (sort.cu: k_sort_scatter_seg): each 2048-element segment is sorted in shared memory
and written out as whole score runs.  Lists are built from a scored pool of haystacks so that their scores and counts are
chosen: counts around the segment size, one score everywhere, a different score per element, and only the highest and
lowest scores, in each single-pass bin class.  Every sorted list must equal numpy's stable (-score, index) order of the
same call's index-ordered list, and the oracle's list.  Needs a CUDA device."""
import random

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200.types import Config, Scoring, SortStrategy
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

SEG = 2048   # elements per segment of the fused scatter (kFrzSortSegShift in frz_host.h)
NEEDLE = "ab0/"
BINS = [(12, 256), (60, 512), (150, 1024)]   # match_score -> single-pass bin class of the score bound
FILLER = b"xyz_-"                            # no needle byte: never matches


def config(match_score, sort=SortStrategy.ScoreThenIndexAsc):
    return Config(max_typos=1, scoring=Scoring(match_score=match_score), sort=sort)


def numpy_order(idx_list, sort):
    """numpy's stable (-score, index) order (index descending for ScoreThenIndexDesc) of an index-ordered list."""
    idx = idx_list["index"].astype(np.int64)
    key = idx if sort == SortStrategy.ScoreThenIndexAsc else -idx
    return idx_list[np.lexsort((key, -idx_list["score"].astype(np.int64)))]


def pool_by_score(match_score):
    """Matching haystacks grouped by their score under config(match_score): {score: [haystack, ...]}."""
    rng = random.Random(match_score)
    hs = [bytes(rng.choice(b"abAB0/_-x") for _ in range(rng.randint(3, 40))) for _ in range(20000)]
    got = O.match_list(NEEDLE, hs, config(match_score, SortStrategy.IndexAsc))
    by = {}
    for m in got:
        by.setdefault(m.score, []).append(hs[m.index])
    return by


_POOLS = {}


def pool(match_score):
    if match_score not in _POOLS:
        _POOLS[match_score] = pool_by_score(match_score)
    return _POOLS[match_score]


def corpus_of(matching, n_filler, seed):
    """The matching haystacks spread in order over filler rows."""
    rng = random.Random(seed)
    rows = [bytes(rng.choice(FILLER) for _ in range(rng.randint(0, 12))) for _ in range(len(matching) + n_filler)]
    slots = sorted(rng.sample(range(len(rows)), len(matching)))
    for s, h in zip(slots, matching):
        rows[s] = h
    return rows


def check_sorted(m_asc_cfg, hs, expect_total, limits=()):
    """Full sorted lists (both score strategies) == numpy order of the index-ordered list == the oracle; top-K calls
    == the full list's first K rows."""
    data, off = O.pack(hs)
    corpus = F.Corpus.from_arrow(data, off)
    try:
        m = F.Matcher(NEEDLE, m_asc_cfg.with_(sort=SortStrategy.IndexAsc))
        by_index = m.match_list_array(corpus).copy()
        m.close()
        assert len(by_index) == expect_total
        for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.ScoreThenIndexDesc):
            cfg = m_asc_cfg.with_(sort=sort)
            m = F.Matcher(NEEDLE, cfg)
            try:
                full = m.match_list_array(corpus).copy()
                assert np.array_equal(full, numpy_order(by_index, sort)), (sort, expect_total)
                want = O.match_list_packed([NEEDLE], cfg, data, off)
                for f in ("index", "score", "exact"):
                    assert np.array_equal(full[f], want[f]), (f, sort)
                for k in limits:
                    top, total = m.match_list_top_array(corpus, k)
                    assert total == len(full) and np.array_equal(top, full[:k]), (sort, k)
            finally:
                m.close()
    finally:
        corpus.close()


@pytest.mark.parametrize("match_score,bins", BINS)
def test_bin_class(match_score, bins):
    bound = F.Matcher(NEEDLE, config(match_score)).score_bound()
    assert bins // 2 <= bound < bins or (bins == 256 and bound < 256), bound
    assert len(pool(match_score)) > 4


@pytest.mark.parametrize("match_score", [ms for ms, _ in BINS])
@pytest.mark.parametrize("total", [1, SEG - 1, SEG + 1, 2 * SEG + 1])
def test_counts_around_a_segment(match_score, total):
    """Counts that are not a multiple of the segment, including a last segment holding one element; mixed scores."""
    by = pool(match_score)
    rng = random.Random(total)
    scores = sorted(by)
    matching = [rng.choice(by[rng.choice(scores)]) for _ in range(total)]
    check_sorted(config(match_score), corpus_of(matching, 3000, total), total, limits=(1, total // 2 + 1, total, total + 5))


@pytest.mark.parametrize("match_score", [ms for ms, _ in BINS])
def test_one_score_everywhere(match_score):
    """Every element has the same score: one run per segment, index order throughout; K cuts through that run."""
    by = pool(match_score)
    s = max(by, key=lambda x: len(by[x]))
    total = 3 * SEG + 5
    matching = [by[s][i % len(by[s])] for i in range(total)]
    check_sorted(config(match_score), corpus_of(matching, 500, 1), total, limits=(1, SEG + 7, 3 * SEG, total + 1))


@pytest.mark.parametrize("match_score", [ms for ms, _ in BINS])
def test_every_score_different(match_score):
    """Every element has its own score: runs of one element."""
    by = pool(match_score)
    matching = [by[s][0] for s in sorted(by)]
    random.Random(2).shuffle(matching)
    check_sorted(config(match_score), corpus_of(matching, 4000, 2), len(matching), limits=(1, len(matching) // 2))


@pytest.mark.parametrize("match_score", [ms for ms, _ in BINS])
def test_top_and_bottom_scores_only(match_score):
    """Only the highest and the lowest score of the pool, interleaved over several segments."""
    by = pool(match_score)
    hi, lo = max(by), min(by)
    rng = random.Random(4)
    total = 5 * SEG + 77
    matching = [rng.choice(by[hi]) if rng.random() < 0.3 else rng.choice(by[lo]) for _ in range(total)]
    n_hi = sum(1 for h in matching if h in set(by[hi]))
    check_sorted(config(match_score), corpus_of(matching, 1000, 4), total,
                 limits=(1, n_hi - 1, n_hi, n_hi + 1, total - 1, total, 10 * total))


def test_back_to_back_calls_leave_scratch_clean():
    """One matcher, corpora of different match counts in turn: the histogram re-zeroed by the scan and the counters must
    come back clean for every next call."""
    by = pool(12)
    rng = random.Random(8)
    scores = sorted(by)
    lists = []
    for total in (5 * SEG + 3, 17, 2 * SEG, 1):
        hs = corpus_of([rng.choice(by[rng.choice(scores)]) for _ in range(total)], 2000, total)
        data, off = O.pack(hs)
        lists.append((data, off, F.Corpus.from_arrow(data, off), total))
    for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.ScoreThenIndexDesc):
        cfg = config(12, sort)
        m = F.Matcher(NEEDLE, cfg)
        try:
            for data, off, corpus, total in lists + lists[::-1]:
                got = m.match_list_array(corpus)
                want = O.match_list_packed([NEEDLE], cfg, data, off)
                assert len(got) == total == len(want)
                for f in ("index", "score", "exact"):
                    assert np.array_equal(got[f], want[f]), (f, sort, total)
                top, n = m.match_list_top_array(corpus, 3)
                assert n == total and np.array_equal(top, want[:3])
        finally:
            m.close()
    for _, _, c, _ in lists:
        c.close()
