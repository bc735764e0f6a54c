"""The fused single-pass score sort: for a single pattern whose score bound is below 1024, the scoring kernels build the
sort's per-segment score histogram as they emit, and the sort is a scan plus a block-per-segment scatter (sort.cu).
Every other list (several patterns, two-pass bounds) keeps the histogram kernel.  Bit-exact parity with the oracle, and
the sort's launch count tells which path ran.  Needs a CUDA device."""
import random

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200.types import Config, Pattern, Scoring, SortStrategy
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

SEG = 2048            # elements per segment of the fused scatter (kFrzSortSegShift in frz_host.h)
FUSED_LAUNCHES = 2    # scan + scatter
HIST_LAUNCHES = 3     # histogram + scan + scatter
BY_SCORE = (SortStrategy.ScoreThenIndexAsc, SortStrategy.ScoreThenIndexDesc)


def pack(hs):
    return O.pack(hs)


def sweep_list(rng, per_class):
    """Haystacks in every Smith-Waterman work class: k_sw64's four column classes, k_sw (65-128 bytes), k_sw_generic
    (129-1024) and the greedy scorer (> 1024)."""
    spans = [(0, 40), (41, 48), (49, 56), (57, 64), (65, 128), (129, 1024), (1025, 1600)]
    counts = [per_class] * 5 + [per_class // 3, 12]
    pool = b"abAB_/-ab01"
    return [bytes(rng.choice(pool) for _ in range(rng.randint(lo, hi))) for (lo, hi), c in zip(spans, counts) for _ in range(c)]


def check(patterns, config, data, off, corpus):
    """GPU list == oracle list; returns (list, launches of the call)."""
    if isinstance(patterns, (str, Pattern)):
        patterns = [patterns]
    want = O.match_list_packed(patterns, config, data, off)
    m = F.Matcher(patterns, config)
    try:
        got = m.match_list_array(corpus)
        launches = m.last_timings()["launches"]
    finally:
        m.close()
    assert len(got) == len(want), (len(got), len(want), patterns, config)
    for f in ("index", "score", "exact"):
        bad = np.nonzero(got[f] != want[f])[0]
        assert bad.size == 0, (f, bad[:5], got[bad[:5]], want[bad[:5]], patterns, config)
    return got, launches


def sort_launches(patterns, config, data, off, corpus):
    """Per score sort: parity with the oracle (under every strategy), and the launches the sort added over the call that
    returns the same list in index order (several patterns reverse with a kernel of their own, a single one while it emits)."""
    res = {sort: check(patterns, config.with_(sort=sort), data, off, corpus) for sort in SortStrategy}
    partner = {SortStrategy.ScoreThenIndexAsc: SortStrategy.IndexAsc, SortStrategy.ScoreThenIndexDesc: SortStrategy.IndexDesc}
    return {sort: (res[sort][0], res[sort][1] - res[partner[sort]][1]) for sort in BY_SCORE}


@pytest.mark.parametrize("match_score,bins", [(12, 256), (60, 512), (150, 1024)])
def test_fused_sort_bin_classes(match_score, bins):
    """A score bound in each single-pass bin class, every SW kernel, every sort strategy (reversed ones included)."""
    cfg = Config(max_typos=1, scoring=Scoring(match_score=match_score))
    bound = F.Matcher("ab0/", cfg).score_bound()
    assert bins // 2 <= bound < bins or (bins == 256 and bound < 256), bound
    rng = random.Random(bins)
    data, off = pack(sweep_list(rng, per_class=2000))
    corpus = F.Corpus.from_arrow(data, off)
    try:
        res = sort_launches("ab0/", cfg, data, off, corpus)
    finally:
        corpus.close()
    for sort in BY_SCORE:
        got, extra = res[sort]
        assert extra == FUSED_LAUNCHES, (sort, extra)
        assert len(got) > SEG and len(got) % SEG != 0


def test_fused_sort_small_totals():
    """0 matches, exactly 1 match, and totals just under, at and over one segment."""
    rng = random.Random(5)
    filler = [bytes(rng.choice(b"xyz_-") for _ in range(rng.randint(0, 30))) for _ in range(20000)]
    hs = list(filler)
    hs[1234] = b"xx_needle_xx"
    data, off = pack(hs)
    corpus = F.Corpus.from_arrow(data, off)
    try:
        for sort in BY_SCORE:
            got, _ = check("qqqq", Config(max_typos=0, sort=sort), data, off, corpus)
            assert len(got) == 0
            got, _ = check("needle", Config(max_typos=0, sort=sort), data, off, corpus)
            assert len(got) == 1 and got["index"][0] == 1234
    finally:
        corpus.close()
    for total in (SEG - 1, SEG, SEG + 1, 3 * SEG + 17):
        hs = [b"needle_%d" % i if i % 3 == 0 and i // 3 < total else h for i, h in enumerate(filler)]
        hs = [h.replace(b"needle", b"ne_edle") if i % 7 == 0 else h for i, h in enumerate(hs)]   # two scores
        data, off = pack(hs)
        corpus = F.Corpus.from_arrow(data, off)
        try:
            for sort in BY_SCORE:
                got, _ = check("needle", Config(max_typos=1, sort=sort), data, off, corpus)
                assert len(got) == total and len(np.unique(got["score"])) > 1
        finally:
            corpus.close()


def test_fused_sort_many_segments_and_reuse():
    """More segments than the scatter's persistent grid (> 1 M matches), lists overflowing the first survivor lists
    (the call re-runs), and one matcher over corpora of different sizes in turn: the histogram the scan re-zeroes must
    be clean for every next call."""
    rng = np.random.default_rng(9)
    n = 1_300_000
    lens = rng.integers(1, 14, n)
    pool = np.frombuffer(b"abAB_/-ab01xyz", dtype=np.uint8)
    big = pool[rng.integers(0, len(pool), int(lens.sum()))]
    big_off = np.zeros(n + 1, dtype=np.uint64)
    big_off[1:] = np.cumsum(lens)
    small, small_off = pack(sweep_list(random.Random(3), per_class=300))
    for k in (None, 1):
        cfg = Config(max_typos=k, sort=SortStrategy.ScoreThenIndexAsc)
        m = F.Matcher("ab", cfg)
        corpora = [(big, big_off, F.Corpus.from_arrow(big, big_off)), (small, small_off, F.Corpus.from_arrow(small, small_off))]
        try:
            for data, off, corpus in corpora + corpora:
                want = O.match_list_packed(["ab"], cfg, data, off)
                got = m.match_list_array(corpus)
                assert len(got) == len(want)
                for f in ("index", "score", "exact"):
                    assert np.array_equal(got[f], want[f]), (f, k, len(got))
                if k is None and corpus is corpora[0][2]:
                    assert len(got) == n and n > 528 * SEG   # more segments than a 132-SM H100's 4-blocks-per-SM grid
        finally:
            m.close()
            for _, _, c in corpora:
                c.close()


def test_fused_sort_unicode_path():
    """Unicode needles are scored by unicode.cu and placed by k_emit_literal, which builds the histogram too."""
    rng = random.Random(17)
    alphabet = ["é", "É", "다", "😀", "a", "-", "_", "x"]
    hs = ["".join(rng.choice(alphabet) for _ in range(rng.randint(0, 24))) for _ in range(20000)]
    data, off = pack(hs)
    corpus = F.Corpus.from_arrow(data, off)
    try:
        res = sort_launches("é다😀", Config(max_typos=1), data, off, corpus)
    finally:
        corpus.close()
    for sort in BY_SCORE:
        got, extra = res[sort]
        assert extra == FUSED_LAUNCHES and len(got) > SEG


def test_histogram_kernel_paths_unchanged():
    """Several patterns, and a single pattern whose bound needs two passes, keep the histogram kernel."""
    rng = random.Random(23)
    data, off = pack(sweep_list(rng, per_class=300))
    corpus = F.Corpus.from_arrow(data, off)
    try:
        multi = sort_launches([Pattern("ab"), Pattern("b_", max_typos=1)], Config(max_typos=1), data, off, corpus)
        high = Scoring(match_score=300, mismatch_penalty=10, gap_open_penalty=20, gap_extend_penalty=0)
        two_pass = sort_launches("ab0/", Config(max_typos=1, scoring=high), data, off, corpus)
    finally:
        corpus.close()
    for sort in BY_SCORE:
        assert multi[sort][1] == HIST_LAUNCHES and len(multi[sort][0]) > 100
        assert two_pass[sort][1] == 2 * HIST_LAUNCHES and two_pass[sort][0]["score"].max() > 1023
