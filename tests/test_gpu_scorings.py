"""The unicode, literal and traceback paths of the GPU across scoring configurations, against the oracle: k_match_indices
(match_indices), k_unicode and the literal emit (match_list_array / match_list_top_array), multi-pattern queries whose
atoms carry their own scoring, and scores of 32 768-65 535 — which only unicode and literal patterns reach — through the
two-pass score sort, top-K and a multi-pattern bound that clamps at 0xFFFF.  Every matcher is compared with the oracle
at the backend it selected (emulate_lanes = the prefilter lanes of its fuzzy patterns).  Needs a CUDA device."""
import random

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200.types import CaseMatching, Config, Matching, Pattern, Scoring, SortStrategy, UnicodeMatching
from oracle import pyoracle as O
from scorings import TIES, high_match_score, literal_scorings, scorings, unicode_scorings

pytestmark = pytest.mark.gpu

B_POOLS = ["abAB_/-ab01", "ab", "fooBar_x", "aA bB/cC", "abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_-/."]
U_POOLS = ["aéAÉ_다", "abé✓😀", "éÉeE-/x", "нНaя_Я", "fooBar_/-é다😀", "aA_bB-"]
LITERAL_MODES = [Matching.Exact, Matching.Prefix, Matching.Suffix, Matching.Substring]
CASINGS = [CaseMatching.Ignore, CaseMatching.Smart, CaseMatching.Respect]
BYTE_SC = scorings(seed=8300, count=20, max_needle=64)
UNI_SC = unicode_scorings(seed=8400, count=24, max_needle=64)
LIT_SC = literal_scorings(seed=8500, count=16, max_needle=64)
# a 13-byte needle whose u8 cells wrap at the default scoring, and the WRAP8 edge case of tests/scorings.py (cells wrap
# for needles of 3-4 bytes): the traceback kernel must wrap exactly as the reference's u8 backend does
WRAP_NEEDLE = "aB-cD-eF-gH-i"
WRAP_SCORING = Scoring(match_score=16, mismatch_penalty=0, gap_open_penalty=64, gap_extend_penalty=1, prefix_bonus=0,
                       capitalization_bonus=64, matching_case_bonus=0, exact_match_bonus=0, delimiter_bonus=64)


def rand_str(rng, pool, n):
    return "".join(rng.choice(pool) for _ in range(n))


def needle_of_bytes(rng, pool, nbytes):
    s = rng.choice(pool)
    while True:
        c = rng.choice(pool)
        if len((s + c).encode()) > nbytes:
            return s
        s += c


def planted(rng, needle, W, filler):
    """`needle` (letters case-flipped here and there, a scalar dropped now and then) inside about W scalars of filler"""
    chars = [c.swapcase() if rng.random() < 0.15 else c for c in needle]
    if len(chars) > 1 and rng.random() < 0.3:
        del chars[rng.randrange(len(chars))]
    body = "".join(chars)
    pad = max(0, W - len(chars))
    a = rng.randint(0, pad)
    return rand_str(rng, filler, a) + body + rand_str(rng, filler, pad - a)


def corpus_for(rng, needles):
    """Byte and mixed-width unicode haystacks of 0-64, 65-128, 129-1024 and a few over 1024 bytes; every needle alone
    (the exact bonus), case-flipped, planted in short and long haystacks, and twice in one haystack."""
    hs = []
    for _ in range(700):
        pool = rng.choice(B_POOLS + U_POOLS)
        hs.append(rand_str(rng, pool, rng.choice([0, 1, 3, 9, 20, 40, 64, rng.randint(65, 128), rng.randint(129, 400), 1000])))
    for needle in needles:
        filler = rng.choice(B_POOLS + U_POOLS) + "x_"
        hs += [needle, needle.swapcase(), "_" + needle, needle + needle, "a" + needle + "/" + needle]
        hs += [planted(rng, needle, W, filler) for W in (len(needle) + 2, rng.randint(65, 128), rng.randint(129, 1000))]
    hs += [planted(rng, rng.choice(needles), W, "xyz_") for W in (1030, 1100, 1500)]
    hs += [WRAP_NEEDLE, "x" + WRAP_NEEDLE, WRAP_NEEDLE + "J", WRAP_NEEDLE * 3, WRAP_NEEDLE[:-1]]
    rng.shuffle(hs)
    return hs


def indices_cases(rng):
    """(pattern, config) pairs: byte needles of 1-64 bytes and unicode needles of up to 64 bytes, typo budgets 0 / 1 / 2 /
    many / None, lanes 16 / 32 / 64, all case modes and scorings, the four literal modes, and the u8 wrap needles."""
    cases = []
    for i in range(48):
        kind = ["byte", "unicode", "byte-literal", "unicode-literal"][i % 4]
        uni = kind.startswith("unicode")
        pool = rng.choice(U_POOLS if uni else B_POOLS)
        needle = needle_of_bytes(rng, pool, rng.choice([rng.randint(1, 8), rng.randint(9, 64), 64]))
        lanes = [16, 32, 64][i % 3]
        casing = CASINGS[(i // 4) % 3]
        if kind.endswith("literal"):
            cfg = Config(matching=LITERAL_MODES[(i // 4) % 4], casing=casing, scoring=LIT_SC[i % len(LIT_SC)], emulate_lanes=lanes,
                         unicode=UnicodeMatching.Always if uni else UnicodeMatching.Ignore)
        else:
            k = [0, 1, 2, 3, 9, None][(i // 2) % 6]
            sc = (UNI_SC if uni else BYTE_SC)[i % (len(UNI_SC) if uni else len(BYTE_SC))]
            cfg = Config(max_typos=k, casing=casing, scoring=sc, emulate_lanes=lanes,
                         unicode=UnicodeMatching.Always if uni else UnicodeMatching.Ignore)
        cases.append((needle, cfg))
    cases.append((Pattern(needle_of_bytes(rng, B_POOLS[0], 64)), Config(max_typos=None, scoring=TIES)))
    for lanes in (16, 32, 64):
        for k in (0, None):
            cases.append((WRAP_NEEDLE, Config(max_typos=k, emulate_lanes=lanes)))
        cases.append(("aB-c", Config(max_typos=1, scoring=WRAP_SCORING, emulate_lanes=lanes)))
    return cases


@pytest.fixture(scope="module")
def scoring_corpus():
    rng = random.Random(8000)
    cases = indices_cases(rng)
    needles = [c[0].needle if isinstance(c[0], Pattern) else c[0] for c in cases]
    hs = corpus_for(rng, needles)
    data, off = O.pack(hs)
    corpus = F.Corpus.from_arrow(data, off)
    yield cases, hs, data, off, corpus
    corpus.close()


def oracle_lanes(m, cfg):
    """the lanes to emulate in the oracle: the configured ones, else the prefilter lanes the library chose for its first
    fuzzy pattern (a literal pattern reports 64 whatever the fuzzy ones use)"""
    if cfg.emulate_lanes:
        return cfg.emulate_lanes
    infos = [m.backend_info(i) for i in range(m.num_patterns())]
    return next((x for x in infos if not x["literal"]), infos[0])["prefilter_lanes"]


def check_indices(pattern, cfg, data, off, corpus, n):
    """match_indices == the oracle's match_list_indices, and its score / exact flag == match_list_array's for every row"""
    m = F.Matcher(pattern, cfg)
    try:
        lanes = oracle_lanes(m, cfg)
        which = list(range(n))
        got = m.match_indices(corpus, which)
        want = O.match_indices(pattern, cfg.with_(emulate_lanes=lanes), data, off, which)
        bad = [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w]
        assert not bad, (pattern, cfg, len(bad), bad[:3])
        ml = {int(x["index"]): x for x in m.match_list_array(corpus) if int(x["index"]) < n}
        assert {i for i, g in enumerate(got) if g is not None} == set(ml), (pattern, cfg)
        assert all(got[i][0] == int(ml[i]["score"]) and got[i][1] == bool(ml[i]["exact"]) for i in ml), (pattern, cfg)
        return sum(g is not None for g in got), m.backend_info()
    finally:
        m.close()


def test_match_indices_across_scorings(scoring_corpus):
    cases, hs, data, off, corpus = scoring_corpus
    matched = wrapped = 0
    for pattern, cfg in cases:
        cnt, info = check_indices(pattern, cfg, data, off, corpus, len(hs))
        matched += cnt > 0
        wrapped += info["score_bits"] == 8 and isinstance(pattern, str) and pattern in (WRAP_NEEDLE, "aB-c") and cnt > 0
    assert matched > len(cases) * 3 // 4 and wrapped == 9, (matched, wrapped, len(cases))


def multi_queries(rng, hs):
    """multi-pattern queries whose atoms carry their own scoring: byte and unicode atoms cut from one haystack of the
    corpus (so that some haystacks match them all), literal atoms, and negated atoms"""
    qs = []
    long_hs = [h for h in hs if len(h) >= 8]
    for i in range(12):
        h = rng.choice(long_hs)
        atoms = []
        for j in range(rng.randint(2, 3)):
            negated = j > 0 and rng.random() < 0.3
            matching = rng.choice([None, None, Matching.Substring, Matching.Prefix])
            if negated:
                needle = needle_of_bytes(rng, rng.choice(U_POOLS + B_POOLS), rng.randint(2, 6))
            else:
                a = 0 if matching == Matching.Prefix else rng.randrange(len(h) - 1)
                needle = h[a:a + rng.randint(1, 12)]
            uni = not needle.isascii() or rng.random() < 0.3
            sc = rng.choice(LIT_SC) if matching else rng.choice(UNI_SC if uni else BYTE_SC)
            atoms.append(Pattern(needle, negated=negated, matching=matching, scoring=sc, max_typos=rng.choice([None, 0, 1, 2]),
                                 unicode=UnicodeMatching.Always if uni else None))
        qs.append((atoms, Config(max_typos=rng.choice([0, 1, None]), emulate_lanes=rng.choice([16, 32, 64]),
                                 sort=rng.choice(list(SortStrategy)))))
    return qs


def gpu_vs_oracle(patterns, cfg, data, off, corpus):
    if isinstance(patterns, (str, Pattern)):
        patterns = [patterns]
    m = F.Matcher(patterns, cfg)
    try:
        lanes = oracle_lanes(m, cfg)
        got = m.match_list_array(corpus).copy()
    finally:
        m.close()
    want = O.match_list_packed(patterns, cfg.with_(emulate_lanes=lanes), data, off)
    assert len(got) == len(want), (patterns, cfg, len(got), len(want))
    for f in ("index", "score", "exact"):
        bad = np.nonzero(got[f] != want[f])[0]
        assert bad.size == 0, (f, bad[:5], got[bad[:5]], want[bad[:5]], patterns, cfg)
    return got


def test_multi_pattern_atom_scorings(scoring_corpus):
    _, hs, data, off, corpus = scoring_corpus
    rng = random.Random(8100)
    nonempty = 0
    for atoms, cfg in multi_queries(rng, hs):
        nonempty += len(gpu_vs_oracle(atoms, cfg, data, off, corpus)) > 0
        check_indices(atoms, cfg, data, off, corpus, len(hs))
    assert nonempty >= 9, nonempty


@pytest.mark.parametrize("sort", list(SortStrategy))
def test_unicode_match_list_across_scorings(scoring_corpus, sort):
    """k_unicode across scorings for needles of up to 64 bytes, every sort strategy, and top-K == oracle[:K]"""
    _, hs, data, off, corpus = scoring_corpus
    rng = random.Random(8200 + int(sort))
    total = 0
    for i in range(14):
        needle = needle_of_bytes(rng, rng.choice(U_POOLS), rng.choice([rng.randint(1, 12), rng.randint(13, 64)]))
        cfg = Config(max_typos=[0, 1, 2, 3, None][i % 5], casing=CASINGS[i % 3], scoring=UNI_SC[(i + 5 * int(sort)) % len(UNI_SC)],
                     unicode=UnicodeMatching.Always, sort=sort, emulate_lanes=[16, 32, 64][i % 3])
        got = gpu_vs_oracle(needle, cfg, data, off, corpus)
        total += len(got)
        m = F.Matcher(needle, cfg)
        for k in (1, 7, len(got) // 2 + 1):
            top, n = m.match_list_top_array(corpus, k)
            assert n == len(got) and np.array_equal(top, got[:k]), (needle, cfg, k)
        m.close()
    assert total > 500, total


# ---------------------------------------------------------------- scores of 32 768-65 535
HIGH_NEEDLE = "abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMN"   # 40 scalars


@pytest.fixture(scope="module")
def high_corpus():
    """Haystacks around HIGH_NEEDLE: whole, case-flipped, with a scalar dropped or changed, behind a prefix — and a block
    of 400 identical haystacks that tie on one high score."""
    rng = random.Random(8600)
    hs = []
    for _ in range(3000):
        chars = list(HIGH_NEEDLE)
        for _ in range(rng.choice([0, 0, 1, 2, 4])):
            i = rng.randrange(len(chars))
            chars[i] = rng.choice([chars[i].swapcase(), "é", "_", ""])
        hs.append(rng.choice(["", "", "x", "_", "é다", "ab/"]) + "".join(chars) + rng.choice(["", "", "y", "😀"]))
    hs += ["zz_" + HIGH_NEEDLE] * 400
    rng.shuffle(hs)
    data, off = O.pack(hs)
    corpus = F.Corpus.from_arrow(data, off)
    yield hs, data, off, corpus
    corpus.close()


def high_patterns():
    n = len(HIGH_NEEDLE)
    uni = Scoring(match_score=high_match_score(n))
    lit = Scoring(match_score=(0xFFFF - 40) // n - 8)
    return [(Pattern(HIGH_NEEDLE), Config(max_typos=2, unicode=UnicodeMatching.Always, scoring=uni)),
            (Pattern(HIGH_NEEDLE), Config(max_typos=None, unicode=UnicodeMatching.Always, scoring=uni, emulate_lanes=16)),
            (Pattern("é" + HIGH_NEEDLE[:30]), Config(max_typos=3, scoring=Scoring(match_score=high_match_score(31)))),
            (Pattern(HIGH_NEEDLE, matching=Matching.Substring), Config(scoring=lit, casing=CaseMatching.Ignore)),
            (Pattern(HIGH_NEEDLE[-20:], matching=Matching.Suffix), Config(scoring=Scoring(match_score=(0xFFFF - 40) // 20 - 8)))]


@pytest.mark.parametrize("sort", [SortStrategy.ScoreThenIndexAsc, SortStrategy.ScoreThenIndexDesc])
def test_high_scores_sorted(high_corpus, sort):
    """scores of 32 768-65 535 from unicode and literal patterns through the two-pass score sort, and a top-K cut inside
    the block of tied high scores"""
    hs, data, off, corpus = high_corpus
    for pattern, cfg in high_patterns():
        cfg = cfg.with_(sort=sort)
        got = gpu_vs_oracle(pattern, cfg, data, off, corpus)
        sc = got["score"].astype(np.int64)
        assert (sc > 32767).sum() > 1000 and len(np.unique(sc[sc > 32767])) >= 2, (pattern, cfg, np.unique(sc)[-5:])
        m = F.Matcher(pattern, cfg)
        assert m.score_bound() > 32767
        # the block of the 400 tied haystacks ("zz_" + needle) where it is one run of equal scores
        tied = np.nonzero(np.array([hs[i] == "zz_" + HIGH_NEEDLE for i in got["index"]]))[0]
        ks = [1, len(got) // 3]
        if len(tied) and np.all(sc[tied] == sc[tied[0]]):
            block = np.nonzero(sc == sc[tied[0]])[0]
            ks += [int(block[0]) + 1, int(block[0] + block[-1]) // 2, int(block[-1])]
        for k in ks:
            top, n = m.match_list_top_array(corpus, k)
            assert n == len(got) and np.array_equal(top, got[:k]), (pattern, cfg, k)
        m.close()


def test_high_score_two_atom_bound_clamps(high_corpus):
    """two high-scoring atoms: the summed score bound clamps at 0xFFFF and the summed scores sort as the oracle's"""
    hs, data, off, corpus = high_corpus
    half = Scoring(match_score=high_match_score(40) // 2)
    lit = Scoring(match_score=(0xFFFF - 40) // 20 - 8)
    for atoms in ([Pattern(HIGH_NEEDLE, scoring=half, unicode=UnicodeMatching.Always), Pattern(HIGH_NEEDLE[:20], matching=Matching.Substring, scoring=lit)],
                  [Pattern(HIGH_NEEDLE, scoring=half, unicode=UnicodeMatching.Always, max_typos=1),
                   Pattern("é" + HIGH_NEEDLE[:20], scoring=Scoring(match_score=high_match_score(21)), max_typos=3)]):
        for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.ScoreThenIndexDesc, SortStrategy.IndexAsc):
            cfg = Config(max_typos=2, sort=sort)
            m = F.Matcher(atoms, cfg)
            assert m.score_bound() == 0xFFFF
            m.close()
            got = gpu_vs_oracle(atoms, cfg, data, off, corpus)
            assert len(got) > 1000 and int(got["score"].max()) > 32767, (atoms, len(got))
            check_indices(atoms, cfg, data, off, corpus, 600)
