"""Byte needles of 13..64 bytes on the short-needle kernels (k_scan_window / k_prefilter_list, k_sw64 in both score
families, the two-pass sort, k_match_indices, k_unicode), bit-exact against the oracle's match_list: every typo budget the
kernels accept (0..15, >= n, None) and the ones the host refuses, needles with few byte classes (the occurrence-mask
trackers) and with many (the scanning forms), windows in every scorer class, the corpus shapes that change the launch
(staged units, unstaged units, survivor-list retry), all sort strategies, the 64 / 65-byte boundary with the long-needle
kernels, multi-pattern queries, the traceback and unicode needles of up to 64 bytes.  The oracle is the cost: every corpus
is small."""
import random

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200.types import CaseMatching, Config, Pattern, Scoring, SortStrategy
from needles import case_sensitive, n_distinct, plant
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

UNSUPPORTED = 9   # FRZ_ERR_UNSUPPORTED
LENGTHS = [13, 16, 17, 23, 24, 25, 32, 33, 49, 50, 63, 64]
TYPOS = [0, 1, 2, 3, 4, 7, 15, None]
CASINGS = [CaseMatching.Smart, CaseMatching.Ignore, CaseMatching.Respect]
FEW = b"abAB_-"                                          # <= 6 byte classes: the occurrence-mask trackers
MANY = b"abcdefghijklmnopqrstuvwxyz0123456789_-/."      # 40 classes: the scanning forms once n > 16
FILLER = b"abcdefghijklmnopqrstuvwxyz_-/ .0123ABCXYZ\x00\x80\xff"
# windows of every scorer class: CC40, CC48, CC56, COLS64 (k_sw64), COLS128, generic (k_sw_generic) and greedy
SPANS = [(1, 40), (41, 48), (49, 56), (57, 64), (65, 128), (129, 1024), (1025, 1600)]


def needle_of(rng, n, many):
    """a needle of n bytes with few byte classes, or with min(n, 40) distinct ones (> 16 once n > 16)"""
    if not many:
        return bytes(rng.choice(FEW) for _ in range(n))
    head = rng.sample(MANY, min(n, len(MANY)))
    out = bytes(head + [rng.choice(MANY) for _ in range(n - len(head))])
    return bytes(b - 32 if 97 <= b <= 122 and rng.random() < 0.2 else b for b in out)


def haystacks_for(rng, needle, count=22):
    """The needle itself and its case flip, shorter haystacks, and haystacks in every window class, most of them holding
    the needle with case flips, up to 16 bytes deleted, contiguous or spread out."""
    n = len(needle)
    hs = [needle, needle.swapcase(), needle[: n - 1], b"", b"x" * 40, b"-" + needle + b"-"]
    while len(hs) < count:
        lo, hi = SPANS[len(hs) % len(SPANS)]
        W = rng.randint(lo, hi)
        if rng.random() < 0.7:
            drops = rng.choice([0, 0, 1, 2, 3, 4, 7, 8, 15, 16])
            hs.append(plant(rng, needle, W, FILLER, drops=drops, spread=W > n + 8 and rng.random() < 0.4))
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


def form(needle, casing):
    """True: the scanning forms (> 16 byte classes), False: the occurrence-mask trackers"""
    return n_distinct(needle, case_sensitive(needle, casing)) == 0


@pytest.mark.parametrize("n", LENGTHS)
def test_lengths_typos_lanes_and_cases(n):
    rng = random.Random(120000 + n)
    budgets = TYPOS + [n, n + 5]
    for many in (False, True):
        needle = needle_of(rng, n, many)
        hs = haystacks_for(rng, needle)
        for j, k in enumerate(budgets):
            em = [16, 32, 64][(j + n) % 3]
            casing = CASINGS[(j + n // 3 + many) % 3]
            assert form(needle, casing) == (many and n > 16), (needle, casing)
            got = check(needle, Config(max_typos=k, emulate_lanes=em, casing=casing), hs)
            if k is None or k >= n:   # no prefilter, or a budget of the whole needle: everything matches
                assert len(got) == len(hs), (k, len(got))
            else:   # (the empty haystack is below the length gate)
                assert 2 <= len(got) < len(hs), (k, len(got))


def test_column_classes_of_long_needles():
    """Windows of 33..40 bytes ending in a prefix of a 25..64-byte needle, under scorings where a gap costs more than a
    mismatch: the best cell of the needle's last row then lies up to n columns past the window's end, which the column
    class of the window (prefilter.cu: sw_class_of, W + n columns) must keep."""
    rng = random.Random(128500)
    scs = [Scoring(mismatch_penalty=0, gap_open_penalty=9, gap_extend_penalty=6),
           Scoring(match_score=16, mismatch_penalty=1, gap_open_penalty=12, gap_extend_penalty=8)]
    for sc in scs:
        for n in (25, 40, 64):
            needle = needle_of(rng, n, many=n == 40)
            hs = []
            for _ in range(24):
                W = rng.randint(33, 40)
                k = rng.randint(10, min(W, n))
                hs.append(bytes(rng.choice(b"xyz") for _ in range(W - k)) + needle[:k])
            for em in (32, 64):   # (no prefilter: the haystack is the window)
                got = check(needle, Config(max_typos=None, emulate_lanes=em, scoring=sc), hs)
                assert len(got) == len(hs)


def test_budgets_the_host_refuses():
    needle = needle_of(random.Random(121000), 40, many=True)
    for k in (16, 39):
        with pytest.raises(F.FrizbeeError) as e:
            F.Matcher(needle, Config(max_typos=k))
        assert e.value.status == UNSUPPORTED
    hs = [b"", b"x", b"zzzz", needle, b"q" * 70, b"0" * 1100]
    got = check(needle, Config(max_typos=40), hs)
    assert sorted(got["index"].tolist()) == list(range(len(hs)))


def survivor_corpus(rng, needle):
    """eight distinct haystacks of 200..480 bytes (the generic scorer's list), six holding the needle, repeated to 128 Ki
    haystacks: more survivors of one list than the first survivor lists hold"""
    distinct = [plant(rng, needle, 200 + 40 * i, FILLER, drops=i % 3) for i in range(6)] + [b"no match here", b"z" * 300]
    idx = np.arange(128 * 1024) % 8
    return distinct, idx


@pytest.mark.parametrize("many", [False, True])
def test_corpus_shapes(many):
    """k = 7 on a corpus of <= 64-byte haystacks (k_scan_window stages their units in shared memory), the same plus one
    100-byte haystack (units read from the corpus), and a corpus whose survivors overflow the first survivor lists."""
    rng = random.Random(122000 + many)
    needle = needle_of(rng, 40, many)
    assert form(needle, CaseMatching.Ignore) == many
    cfg = Config(max_typos=7, casing=CaseMatching.Ignore)
    short = [needle, needle[:33]]
    while len(short) < 120:
        W = rng.randint(1, 64)
        short.append(plant(rng, needle, W, FILLER, drops=rng.randint(0, 9)) if W >= 30 and rng.random() < 0.6
                     else bytes(rng.choice(FILLER) for _ in range(W)))
    got = check(needle, cfg, short)
    assert 20 <= len(got) <= 100, len(got)
    got = check(needle, cfg, short + [plant(rng, needle, 100, FILLER, drops=3, spread=True)])
    assert len(short) in got["index"].tolist()   # the 100-byte haystack matches
    distinct, idx = survivor_corpus(rng, needle)
    cfg = cfg.with_(sort=SortStrategy.IndexAsc)
    m = F.Matcher(needle, cfg)
    d, o = O.pack(distinct)
    w = O.match_list_packed([needle], cfg.with_(emulate_lanes=m.backend_info()["prefilter_lanes"]), d, o)
    by_hay = {int(r["index"]): (int(r["score"]), int(r["exact"])) for r in w}
    assert len(by_hay) == 6
    got = m.match_list_array([distinct[i] for i in idx])
    m.close()
    assert got["index"].tolist() == [i for i in range(len(idx)) if int(idx[i]) in by_hay]
    assert all((int(g["score"]), int(g["exact"])) == by_hay[int(idx[int(g["index"])])] for g in got[::97])
    assert len(got) > 65536


def test_sort_classes_and_top_k():
    """score_bound() picks the sort: < 512 and < 1024 take the fused single-pass forms, >= 1024 the two-pass sort, which
    needles of 50..64 bytes reach at the default scoring."""
    rng = random.Random(123000)
    bounds = {}
    for n in (23, 24, 50, 64):
        m = F.Matcher(b"a" * n, Config(max_typos=1))
        bounds[n] = m.score_bound()
        m.close()
    assert bounds[23] < 512 <= bounds[24] < 1024 <= bounds[50] <= bounds[64], bounds
    for n in (24, 50, 64):
        needle = needle_of(rng, n, many=n != 50)
        hs = haystacks_for(rng, needle, 30)
        for k in (1, 7):
            for sort in SortStrategy:
                got = check(needle, Config(max_typos=k, sort=sort, emulate_lanes=[16, 32, 64][int(sort) % 3]), hs)
                assert len(got) >= 3
    needle = needle_of(rng, 64, many=False)
    hs = haystacks_for(rng, needle, 80)
    for sort in SortStrategy:
        m = F.Matcher(needle, Config(max_typos=7, sort=sort))
        full = m.match_list_array(hs)
        assert len(full) > 10
        for k in (1, 10, len(full), len(full) + 3):
            top, total = m.match_list_top_array(hs, k)
            assert total == len(full) and np.array_equal(top, full[:k]), (sort, k)
        m.close()


def test_64_65_boundary():
    """the same haystacks against a 64-byte needle (short kernels) and the 65-byte needle that extends it (long kernels)"""
    rng = random.Random(124000)
    for many in (False, True):
        needle = needle_of(rng, 64, many)
        hs = haystacks_for(rng, needle, 16) + haystacks_for(rng, needle + b"x", 12)
        for j, k in enumerate((0, 2, 15, None)):
            cfg = Config(max_typos=k, emulate_lanes=[16, 32, 64][j % 3], casing=CASINGS[(j + many) % 3])
            a = check(needle, cfg, hs)
            b = check(needle + b"x", cfg, hs)
            assert len(a) > 0 and len(b) > 0


def test_multi_pattern_long_atoms():
    """a 40-byte atom with its own max_typos = 7 (k_prefilter_list<FRZ_T_MANY> on the candidates of the first atom), with
    few and with many byte classes, and a negated 64-byte atom"""
    rng = random.Random(125000)
    few40, many40, neg64 = needle_of(rng, 40, False), needle_of(rng, 40, True), needle_of(rng, 64, True)
    hs = []
    for i in range(60):
        s = bytes(rng.choice(FILLER) for _ in range(rng.randint(0, 30)))
        if i % 2 == 0:
            s += b"ab_"
        if rng.random() < 0.5:
            s += plant(rng, rng.choice([few40, many40]), rng.randint(40, 200), FILLER, drops=rng.randint(0, 9), spread=rng.random() < 0.3)
        if rng.random() < 0.3:
            s += plant(rng, neg64, rng.randint(64, 120), FILLER, drops=rng.randint(0, 2))
        hs.append(s)
    for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexAsc):
        cfg = Config(max_typos=1, sort=sort)
        for atom in (few40, many40):
            got = check([Pattern(b"ab_"), Pattern(atom, max_typos=7)], cfg, hs)
            assert 0 < len(got) < len(hs)
        got = check([Pattern(b"ab_"), Pattern(neg64, negated=True)], cfg, hs)
        assert 0 < len(got) < len(hs)
        check([Pattern(few40, max_typos=7), Pattern(neg64, negated=True, max_typos=3)], cfg, hs)


def test_match_indices_traceback():
    """match_indices == the oracle's traceback for needles of 33 and 64 bytes, windows up to and over 1024 bytes"""
    rng = random.Random(126000)
    for n in (33, 64):
        for many in (False, True):
            needle = needle_of(rng, n, many)
            hs = haystacks_for(rng, needle, 18)
            data, off = O.pack(hs)
            corpus = F.Corpus.from_arrow(data, off)
            which = list(range(len(hs)))
            for j, k in enumerate((0, 3, 15, None)):
                cfg = Config(max_typos=k, emulate_lanes=[16, 32, 64][(j + n) % 3], casing=CASINGS[(j + many) % 3])
                m = F.Matcher(needle, cfg)
                got = m.match_indices(corpus, which)
                want = O.match_indices(needle, cfg.with_(emulate_lanes=m.backend_info()["prefilter_lanes"]), data, off, which)
                assert got == want, (n, k, [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w][:2])
                ml = {int(x["index"]): x for x in m.match_list_array(corpus)}
                assert {i for i, g in enumerate(got) if g is not None} == set(ml) and len(ml) > 0
                assert all(got[i][0] == int(ml[i]["score"]) and got[i][1] == bool(ml[i]["exact"]) for i in ml)
                m.close()
            corpus.close()


U_POOLS = ["aéAÉ_다", "abé✓😀", "éÉeE-/x", "нНaя_Я", "fooBar_/-é다😀"]


def unicode_needles(rng):
    four = "".join(rng.choice("😀😁😂🙂🎉") for _ in range(16))
    three = "".join(rng.choice("다✓한€") for _ in range(21)) + "a"
    two = "".join(rng.choice("éÉяЯß") for _ in range(32))
    mixed = list("abcdefgh_-/ABCDEFGHxyzXYZ01" + "q") + [rng.choice("éÉяЯ") for _ in range(8)] + [rng.choice("다✓€") for _ in range(4)]
    rng.shuffle(mixed)
    needles = [four, three, two, "".join(mixed)]
    assert [len(x.encode()) for x in needles] == [64, 64, 64, 56] and [len(x) for x in needles] == [16, 22, 32, 40]
    return needles


def unicode_haystacks(rng, needle, count=26):
    out = ["", "é다😀", "x" * 1100 + "é" + "y" * 50 + "다😀", needle, needle.swapcase()]
    while len(out) < count:
        pool = rng.choice(U_POOLS)
        ln = rng.choice([0, 5, 14, 31, 40, 70, 130, 300])
        hay = [rng.choice(pool) for _ in range(ln)]
        if rng.random() < 0.6:   # the needle's scalars, some dropped or case-flipped, contiguous or spread out
            chars = [c.swapcase() if rng.random() < 0.1 and len(c.swapcase()) == 1 else c for c in needle]
            for _ in range(rng.choice([0, 0, 1, 2, 5, 15])):
                if chars:
                    del chars[rng.randrange(len(chars))]
            at = sorted(rng.choices(range(len(hay) + 1), k=len(chars))) if rng.random() < 0.4 else [rng.randint(0, len(hay))] * len(chars)
            for c, p in reversed(list(zip(chars, at))):
                hay.insert(p, c)
        out.append("".join(hay))
    return out


def test_unicode_needles_up_to_64_bytes():
    rng = random.Random(127000)
    for i, needle in enumerate(unicode_needles(rng)):
        hs = unicode_haystacks(rng, needle)
        data, off = O.pack(hs)
        corpus = F.Corpus.from_arrow(data, off)
        for j, k in enumerate((0, 1, 2, 5, 15, None)):
            cfg = Config(max_typos=k, emulate_lanes=[16, 32, 64][(i + j) % 3])
            m = F.Matcher(needle, cfg)
            want = O.match_list_packed([needle], cfg.with_(emulate_lanes=m.backend_info()["prefilter_lanes"]), data, off)
            got = m.match_list_array(corpus)
            m.close()
            assert len(got) == len(want) and len(got) > 0, (i, k, len(got), len(want))
            for f in ("index", "score", "exact"):
                assert np.array_equal(got[f], want[f]), (i, k, f)
        corpus.close()
    with pytest.raises(F.FrizbeeError) as e:
        F.Matcher("é" * 32 + "a", Config())
    assert e.value.status == UNSUPPORTED
