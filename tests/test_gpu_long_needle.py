"""Needles of 65..1024 bytes on the GPU (k_scan_window_long / k_prefilter_list_long and k_sw_long), bit-exact against the
oracle's match_list at every emulated lane width, typo budget, case mode, literal mode and sort strategy, through every
entry point that takes a matcher.  The oracle is slow on long needles, so every case keeps its corpus small."""
import random

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200 import parallel, synth
from frizbee_b200.types import CaseMatching, Config, Matching, Pattern, Scoring, SortStrategy
from oracle import pyoracle as O
from scorings import scorings

pytestmark = pytest.mark.gpu

LENGTHS = [65, 96, 128, 129, 255, 256, 257, 511, 512, 513, 1000, 1024]
TYPOS = [0, 1, 2, 3, 15, None]
FILLER = b"abcdefghijklmnopqrstuvwxyz_-/ .0123ABCXYZ"


def needle_of(rng, n, dense=False):
    pool = b"abAB" if dense else b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_-/. "
    return bytes(rng.choice(pool) for _ in range(n))


def plant(rng, needle, W, typos=0, spread=False):
    """A haystack of W bytes holding the needle (case flips, `typos` bytes dropped, optionally spread out)."""
    nb = bytearray(b ^ 0x20 if (chr(b).isalpha() and rng.random() < 0.1) else b for b in needle)
    for _ in range(typos):
        if len(nb) > 1:
            del nb[rng.randrange(len(nb))]
    if len(nb) > W:
        nb = nb[:W]
    out = bytearray(rng.choice(FILLER) for _ in range(W))
    pos = sorted(rng.sample(range(W), len(nb))) if spread else list(range(s := rng.randint(0, W - len(nb)), s + len(nb)))
    for p, b in zip(pos, nb):
        out[p] = b
    return bytes(out)


def haystacks_for(rng, needle, count=24):
    """Shorter than the needle, equal to it, and windows in every span the scorers split on: <= 64 (max_typos None only),
    65-128, 129-256, 257-512, 513-1024 and over 1024 (the greedy scorer)."""
    n = len(needle)
    hs = [needle, needle.swapcase(), needle[: n - 1], needle[: max(1, n // 2)], b"", b"x" * 40]
    spans = [(1, 64), (65, 128), (129, 256), (257, 512), (513, 1024), (1025, 2600)]
    while len(hs) < count:
        lo, hi = rng.choice(spans)
        W = rng.randint(max(lo, 1), hi)
        r = rng.random()
        if W >= n and r < 0.7:
            hs.append(plant(rng, needle, W, typos=rng.choice([0, 0, 1, 2, 4]), spread=rng.random() < 0.4))
        else:
            hs.append(bytes(rng.choice(FILLER) for _ in range(W)))
    rng.shuffle(hs)
    return hs


def check(patterns, cfg, hs):
    """match_list on the GPU == the oracle at the lane width the library emulates; returns the GPU's list."""
    m = F.Matcher(patterns, cfg)
    lanes = m.backend_info()["prefilter_lanes"]
    data, off = O.pack(hs)
    want = O.match_list_packed(patterns if isinstance(patterns, list) else [patterns], cfg.with_(emulate_lanes=lanes), data, off)
    got = m.match_list_array(hs)
    m.close()
    assert len(got) == len(want), (len(got), len(want))
    for f in ("index", "score", "exact"):
        assert np.array_equal(got[f], want[f]), f
    return got


@pytest.mark.parametrize("n", LENGTHS)
def test_lengths_typos_lanes_and_cases(n):
    rng = random.Random(90000 + n)
    for j, k in enumerate(TYPOS):
        needle = needle_of(rng, n, dense=j % 3 == 2)
        em = [16, 32, 64][(j + n) % 3]
        casing = [CaseMatching.Smart, CaseMatching.Ignore, CaseMatching.Respect][(j + n // 7) % 3]
        check(needle, Config(max_typos=k, emulate_lanes=em, casing=casing), haystacks_for(rng, needle, 18))


def test_long_needle_scorings_and_sorts():
    rng = random.Random(91000)
    single_pass = Scoring(match_score=1, mismatch_penalty=0, gap_open_penalty=1, gap_extend_penalty=0, prefix_bonus=0,
                          capitalization_bonus=0, matching_case_bonus=0, exact_match_bonus=0, delimiter_bonus=0)
    m = F.Matcher(b"q" * 300, Config(scoring=single_pass))
    assert m.score_bound() < 1024   # the fused single-pass sort, with the histogram built by k_sw_long
    m.close()
    scs = [single_pass, Scoring(gap_open_penalty=5, gap_extend_penalty=0)] + scorings(9100, 8, 1024)
    run = 0
    for i, sc in enumerate(scs):
        n = [300, 1000, 100][i % 3]
        needle = needle_of(rng, n)
        for sort in SortStrategy:
            cfg = Config(max_typos=[1, None, 2, 0][(i + int(sort)) % 4], emulate_lanes=[16, 32, 64][i % 3], scoring=sc, sort=sort)
            check(needle, cfg, haystacks_for(rng, needle, 14))   # scorings(..., 1024) accepts every needle of up to 1024 bytes
            run += 1
    assert run == 4 * len(scs)
    # a 100-byte needle whose scoring keeps it in the u8 family (every window scored per thread, at 16, 32 or 64 lanes)
    for em in (16, 32, 64):
        needle = needle_of(rng, 100)
        cfg = Config(max_typos=None, emulate_lanes=em, scoring=single_pass)
        m = F.Matcher(needle, cfg)
        assert (m.backend_info()["score_bits"], m.backend_info()["lanes"]) == (8, em)
        m.close()
        check(needle, cfg, haystacks_for(rng, needle, 20))


def test_literal_modes():
    rng = random.Random(92000)
    for n in (65, 300, 1024):
        needle = needle_of(rng, n)
        hs = [needle, b"x" + needle, needle + b"y", b"__" + needle.swapcase() + b"__", needle[:-1], b"a" * 2000 + needle]
        hs += haystacks_for(rng, needle, 12)
        for mode in (Matching.Exact, Matching.Prefix, Matching.Suffix, Matching.Substring):
            for cs in (CaseMatching.Ignore, CaseMatching.Respect):
                check(needle, Config(matching=mode, casing=cs), hs)


def test_multi_pattern_long_and_short_atoms():
    rng = random.Random(93000)
    long1, long2 = needle_of(rng, 150), needle_of(rng, 90)
    hs = []
    for _ in range(40):
        parts = [rng.choice(FILLER) for _ in range(rng.randint(0, 40))]
        s = bytes(parts)
        if rng.random() < 0.6:
            s += plant(rng, long1, rng.randint(150, 400), typos=rng.choice([0, 1]))
        if rng.random() < 0.4:
            s += b"foo" + plant(rng, long2, 120)
        hs.append(s)
    for k in (0, 1, None):
        cfg = Config(max_typos=k)
        check([Pattern(long1), Pattern(b"foo")], cfg, hs)
        check([Pattern(long1), Pattern(long2, negated=True)], cfg, hs)
        check([Pattern(b"foo"), Pattern(long1, negated=True)], cfg, hs)
        check([Pattern(long2), Pattern(b"ab"), Pattern(long1)], cfg, hs)


def test_top_k_and_into_with_offset():
    rng = random.Random(94000)
    needle = needle_of(rng, 200)
    hs = haystacks_for(rng, needle, 60)
    for sort in SortStrategy:
        m = F.Matcher(needle, Config(max_typos=None, sort=sort))
        full = m.match_list_array(hs)
        for k in (1, 5, len(full), len(full) + 3):
            top, total = m.match_list_top_array(hs, k)
            assert total == len(full) and np.array_equal(top, full[:k]), (sort, k)
        m.close()
    m = F.Matcher(needle, Config(max_typos=1))
    data, off = O.pack(hs)
    want = O.match_list_into_packed([needle], Config(max_typos=1, emulate_lanes=m.backend_info()["prefilter_lanes"]), data, off,
                                    index_offset=1000)
    got = m.match_list_into_array(hs, index_offset=1000)
    assert all(np.array_equal(got[f], want[f]) for f in ("index", "score", "exact"))
    m.close()


def long_corpus(n_items, seed):
    """synth corpus of 80..600-byte haystacks with a 100-byte needle planted fully and partially"""
    rng = random.Random(seed)
    needle = needle_of(rng, 100).decode()
    data, off = synth.generate(needle, n_items, 200, 600, seed=seed)
    lens = np.diff(off.astype(np.int64))
    return needle, data, off, lens


def test_streamed_end_to_end_equals_resident():
    needle, data, off, _ = long_corpus(150_000, 95)   # >= 64 tiles: the end-to-end call takes its streamed form
    whole = F.Corpus.from_arrow(data, off)
    for k in (0, 1, None):
        for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexAsc):
            m = F.Matcher(needle, Config(max_typos=k, sort=sort))
            res = m.match_list_array(whole)
            assert len(res) > 0
            for width in (np.uint64, np.uint32):
                e2e = m.match_list_host_array(data, off.astype(width))
                assert np.array_equal(e2e, res), (k, sort, width)
            m.close()
    whole.close()


def test_parallel_world1():
    needle, data, off, _ = long_corpus(60_000, 96)
    comm = parallel.Comm.local(1)
    shards = comm.shard_arrow(data, off)
    whole = F.Corpus.from_arrow(data, off)
    for k in (1, None):
        m = F.Matcher(needle, Config(max_typos=k))
        full = comm.match_list_parallel(m, shards).copy()
        assert np.array_equal(full, m.match_list_array(whole))
        top, total = comm.match_list_parallel_top(m, shards, 50)
        assert total == len(full) and np.array_equal(top, full[:50])
        m.close()
    for s in shards:
        s.close()
    whole.close()
    comm.close()


def test_empty_tiles_and_survivor_retry():
    """Tiles without a single match, and a corpus where more haystacks survive than the first survivor lists hold (the
    call re-runs with worst-case lists).  Eight distinct haystacks repeated: the oracle scores the eight."""
    rng = random.Random(97000)
    needle = needle_of(rng, 120)
    distinct = [plant(rng, needle, 200 + 40 * i, typos=i % 2) for i in range(6)] + [b"no match here", b"z" * 300]
    n_items = 128 * 1024
    idx = np.arange(n_items) % 8
    idx[10 * 1024: 20 * 1024] = 6   # ten tiles of non-matching haystacks
    hs = [distinct[i] for i in idx]
    for k in (1, None):
        cfg = Config(max_typos=k, sort=SortStrategy.IndexAsc, casing=CaseMatching.Ignore)   # planted bytes are case-flipped
        m = F.Matcher(needle, cfg)
        lanes = m.backend_info()["prefilter_lanes"]
        d, o = O.pack(distinct)
        w = O.match_list_packed([needle], cfg.with_(emulate_lanes=lanes), d, o)
        by_hay = {int(r["index"]): (int(r["score"]), int(r["exact"])) for r in w}
        got = m.match_list_array(hs)
        want_idx = [i for i in range(n_items) if int(idx[i]) in by_hay]
        assert got["index"].tolist() == want_idx
        assert all((int(g["score"]), int(g["exact"])) == by_hay[int(idx[int(g["index"])])] for g in got[:5000])
        assert len(got) > 65536   # more survivors of one list (windows over 128 bytes) than the first lists hold
        m.close()


def test_match_indices_refuses_long_needles():
    corpus = F.Corpus.from_list([b"a" * 100, b"b"])
    m = F.Matcher(b"a" * 100, Config())
    with pytest.raises(F.FrizbeeError) as e:
        m.match_indices(corpus, [0, 1])
    assert e.value.status == 9   # FRZ_ERR_UNSUPPORTED
    m.close()
    corpus.close()
