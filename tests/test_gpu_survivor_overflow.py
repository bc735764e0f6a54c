"""Survivor-list overflow and its retry, on every prefilter kernel and scoring class that emits survivor records.

A match call sizes each of its six per-class survivor lists for max(n/4, 65536) records (host.cu: initial_survivor_cap)
unless the pattern can match every haystack.  A prefilter kernel with more survivors in one class drops the rest and sets
FRZ_DEVERR_SURVIVOR_OVERFLOW; the call sees the flag, grows every list to n and runs again.  Each case below puts more
than the cap into the class it targets on the first call of a fresh matcher:

    cols128           k_scan_window -> k_sw<.., 128, ..>        windows of 65-128 bytes               class COLS128
    generic           k_scan_window -> k_sw_generic             windows of 129-1024 and > 1024 bytes  class GENERIC
    long              k_scan_window_long -> k_sw_long           a 70-byte needle, 100-150-byte windows COLS128
    unicode           k_sig_scan -> k_unicode                   a unicode needle                      COLS64
    exact .. substring  literal prefilter -> k_emit_literal     the four literal modes                COLS64
    multi_base        run_pattern of the base atom, then a non-negated and a negated extra atom
    multi_extra       k_prefilter_list: the base's survivors spread over three classes, each under the cap, the extra
                      atom's all in GENERIC
    multi_long_extra  k_prefilter_list_long: the same with a 70-byte extra atom, its windows all in COLS128

The subset list form cannot overflow: it runs only when the members are at most 2 % of the corpus
(FRZ_SUBSET_LIST_PERMILLE), and its lists hold a quarter of the corpus.

Every case asserts that the oracle puts more than the cap into the targeted class, and that the first call overflowed:
the library counts the launches of both attempts of a retried call in frz_matcher_last_timings, so a retried call
reports the launches of the call that follows it twice (a multi-pattern query that stopped at an atom, more).  Results
are bit-exact on (index, score, exact) and order against the CPU oracle.  The large corpora repeat a few thousand
distinct haystacks: the oracle scores those, and each corpus checks that expansion against the oracle's own match_list on
its first rows.  Needs a CUDA device."""

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200.types import Config, Matching, Pattern, SortStrategy
from oracle import pyoracle as O
from ranking import rank_by_boost

pytestmark = pytest.mark.gpu

NOISE = np.frombuffer(b"vwxyzVWXYZ_-. /", dtype=np.uint8)   # none of the needles' bytes, in either case
LONG_ALPHABET = np.frombuffer(b"ijklmnopqrstu", dtype=np.uint8)
GENERIC, COLS128, SHORT = "GENERIC", "COLS128", "<=64"   # SHORT: the four classes of windows of up to 64 bytes
SORTS = [SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexDesc]


def cap_of(n):
    """initial_survivor_cap (host.cu) for a pattern with a typo budget: records per class list before a retry"""
    return min(max(n // 4, 1 << 16), n)


# ---------------------------------------------------------------------------------------------------- haystacks
def noise(rng, lo, hi):
    return bytes(NOISE[rng.integers(0, NOISE.size, size=int(rng.integers(lo, hi + 1)))])


def cased(rng, s):
    """s with each ASCII letter upper-cased with probability 1/3 (the needles are lower case, so they match either)"""
    b = np.frombuffer(s, dtype=np.uint8).copy()
    letter = (b >= ord("a")) & (b <= ord("z"))
    b[letter & (rng.random(b.size) < 1 / 3)] -= 32
    return bytes(b)


def spaced(rng, needle, lo, hi):
    """needle's bytes in order, with lo..hi noise bytes between consecutive ones"""
    out = needle[:1]
    for ch in needle[1:]:
        out += noise(rng, lo, hi) + bytes([ch])
    return cased(rng, out)


def long_needle(seed):
    return bytes(LONG_ALPHABET[np.random.default_rng(seed).integers(0, LONG_ALPHABET.size, size=70)]).decode()


def long_span(rng, needle, lo, hi):
    """needle in three pieces with lo..hi noise bytes between them"""
    b = needle.encode()
    return cased(rng, b[:23] + noise(rng, lo, hi) + b[23:46] + noise(rng, lo, hi) + b[46:])


def expand(rows, ids):
    """the corpus whose haystack i is rows[ids[i]]: (Arrow bytes, offsets)"""
    udata, uoff = O.pack(rows)
    lens = np.diff(uoff).astype(np.int64)[ids]
    off = np.zeros(len(ids) + 1, dtype=np.uint64)
    off[1:] = np.cumsum(lens)
    src = np.repeat(uoff[:-1].astype(np.int64)[ids] - off[:-1].astype(np.int64), lens) + np.arange(int(off[-1]))
    return udata[src], off


# ---------------------------------------------------------------------------------------------------- cases
def case_cols128(rng):
    rows = [noise(rng, 0, 1) + spaced(rng, b"abcd", 21, 40) for _ in range(3000)]
    return ["abcd"], Config(max_typos=1), rows, 140_000, (0, COLS128)


def case_generic(rng):
    rows = [noise(rng, 0, 1) + spaced(rng, b"abcd", 42, 300) for _ in range(1200)]
    rows += [noise(rng, 0, 1) + spaced(rng, b"abcd", 341, 400) for _ in range(300)]   # windows > 1024: the greedy scorer
    return ["abcd"], Config(max_typos=0), rows, 100_000, (0, GENERIC)


def case_long(rng):
    nd = long_needle(11)
    rows = [noise(rng, 0, 1) + long_span(rng, nd, 15, 28) for _ in range(1700)]
    rows += [noise(rng, 0, 1) + long_span(rng, nd, 31, 40) for _ in range(300)]       # 130-150 bytes: GENERIC
    return [nd], Config(max_typos=0), rows, 100_000, (0, COLS128)


def case_unicode(rng):
    e = ["é".encode(), "É".encode()]
    rows = [noise(rng, 0, 6) + e[int(rng.integers(0, 2))] + noise(rng, 0, 10) + "다".encode() + noise(rng, 0, 6)
            for _ in range(3000)]
    return ["é다"], Config(max_typos=1), rows, 140_000, (0, "COLS64")


def literal_case(mode):
    def case(rng):
        body = {Matching.Exact: lambda: b"abcd",
                Matching.Prefix: lambda: b"abcd" + noise(rng, 0, 12),
                Matching.Suffix: lambda: noise(rng, 0, 12) + b"abcd",
                Matching.Substring: lambda: noise(rng, 0, 8) + b"abcd" + noise(rng, 0, 8)}[mode]
        rows = [cased(rng, body()) for _ in range(3000)]
        return [Pattern("abcd", matching=mode)], Config(max_typos=0), rows, 100_000, (0, "COLS64")
    return case


def case_multi_base(rng):
    def gap(extra, p):   # noise with `extra` planted in it with probability p
        return noise(rng, 10, 19) + (cased(rng, extra) if rng.random() < p else b"") + noise(rng, 10, 19)
    rows = [noise(rng, 0, 1) + cased(rng, b"a") + gap(b"ef", 0.7) + cased(rng, b"b") + gap(b"gh", 0.3) + cased(rng, b"c")
            + noise(rng, 21, 39) + cased(rng, b"d") for _ in range(3000)]
    return [Pattern("abcd"), Pattern("ef"), Pattern("gh", negated=True)], Config(max_typos=0), rows, 100_000, (0, COLS128)


def base_ab(rng, t):
    """the base atom "ab" with a window of <= 64 bytes (t = 0), 65-128 (1) or 129-1024 (2)"""
    return spaced(rng, b"ab", *((5, 20), (70, 110), (140, 170))[t])


def case_multi_extra(rng):
    rows = [cased(rng, b"c") + noise(rng, 2, 5) + base_ab(rng, i % 3) + noise(rng, 130, 150) + cased(rng, b"d")
            for i in range(3000)]
    return [Pattern("ab"), Pattern("cd")], Config(max_typos=0), rows, 100_000, (1, GENERIC)


def case_multi_long_extra(rng):
    nd = long_needle(12)
    rows = [noise(rng, 0, 1) + long_span(rng, nd, 15, 28) + noise(rng, 3, 6) + base_ab(rng, 2 * (i % 2))
            for i in range(2000)]
    return [Pattern("ab"), Pattern(nd)], Config(max_typos=0), rows, 100_000, (1, COLS128)


CASES = {"cols128": case_cols128, "generic": case_generic, "long": case_long, "unicode": case_unicode,
         "exact": literal_case(Matching.Exact), "prefix": literal_case(Matching.Prefix),
         "suffix": literal_case(Matching.Suffix), "substring": literal_case(Matching.Substring),
         "multi_base": case_multi_base, "multi_extra": case_multi_extra, "multi_long_extra": case_multi_long_extra}
SUBSET_CASES = ["cols128", "unicode"]   # the two with 140 000 rows: half of them is still more than the cap


# ---------------------------------------------------------------------------------------------------- oracle
def survivor_classes(p, cfg, rows, lanes):
    """per distinct haystack: the survivor list the atom's prefilter puts it in (None: no survivor)"""
    unicode = any(ord(ch) > 127 for ch in p.needle)
    if unicode or (p.matching or cfg.matching) != Matching.Fuzzy:
        hit = O.match_list_into_packed([Pattern(p.needle, matching=p.matching)], cfg, *O.pack(rows))
        out = [None] * len(rows)
        for i in hit["index"]:
            out[i] = "COLS64"   # unicode and literal survivors carry their score: all of them go to one list
        return out
    out = []
    for h in rows:
        ok, start, end = O.prefilter(p.needle, h, cfg.max_typos, lanes)
        w = end - max(start - 1, 0)   # trim_haystack
        out.append(None if not ok else GENERIC if w > 128 else COLS128 if w > 64 else SHORT)
    return out


def ordered(index_order, sort):
    """Matcher::match_list's order from match_list_into's: reversed for the *_DESC strategies, then the stable descending
    score sort for the by-score ones"""
    m = index_order[::-1] if SortStrategy(sort).is_reversed() else index_order
    return O.radix_sort_matches(m) if SortStrategy(sort).is_by_score() else np.ascontiguousarray(m)


class Case:
    """One corpus, resident on the GPU, and its oracle: `into` is the index-ordered match list of the whole corpus."""

    def __init__(self, name, lanes):
        rng = np.random.default_rng(sum(map(ord, name)))
        self.name = name
        pats, cfg, rows, self.n, (self.target_atom, self.target_class) = CASES[name](rng)
        self.cfg = cfg.with_(emulate_lanes=lanes)   # every atom emulates the same reference backend as the oracle
        self.patterns = [p if isinstance(p, Pattern) else Pattern(p) for p in pats]
        ids = rng.integers(0, len(rows), size=self.n)
        self.data, self.off = expand(rows, ids)
        cfg = self.cfg
        per_row = O.match_list_into_packed(self.patterns, cfg, *O.pack(rows))
        hit = np.zeros(len(rows), dtype=bool)
        hit[per_row["index"]] = True
        score = np.zeros(len(rows), dtype=np.uint16)
        exact = np.zeros(len(rows), dtype=np.uint8)
        score[per_row["index"]], exact[per_row["index"]] = per_row["score"], per_row["exact"]
        idx = np.nonzero(hit[ids])[0]
        self.into = np.zeros(len(idx), dtype=F.MATCH_DTYPE)
        self.into["index"], self.into["score"], self.into["exact"] = idx, score[ids[idx]], exact[ids[idx]]
        # the expansion equals the oracle's own match_list on the corpus's first rows
        head = 2500
        for s in SORTS:
            want = O.match_list_packed(self.patterns, cfg.with_(sort=s), self.data[: int(self.off[head])], self.off[: head + 1])
            expect(want, ordered(self.into[self.into["index"] < head], s))
        # survivors per class of the targeted atom and of the atoms before it, over the haystacks each is run on (an
        # extra atom sees the matches of the atoms before it)
        seen = np.ones(len(rows), dtype=bool)
        self.class_counts = []
        for p in self.patterns[: self.target_atom + 1]:
            cls = np.array([str(k) for k in survivor_classes(p, self.cfg, rows, lanes)])
            vals, cnt = np.unique(cls[ids[seen[ids]]], return_counts=True)
            self.class_counts.append(dict(zip(vals.tolist(), cnt.tolist())))
            seen &= (cls != "None") != p.negated
        self.corpus = F.Corpus.from_arrow(self.data, self.off)

    def want(self, sort, members=None):
        into = self.into if members is None else self.into[np.isin(self.into["index"], members)]
        return ordered(into, sort)

    def matcher(self, sort):
        return F.Matcher(self.patterns, self.cfg.with_(sort=sort))


@pytest.fixture(scope="module")
def lanes():
    m = F.Matcher("abcd", Config())
    try:
        return m.backend_info()["prefilter_lanes"]
    finally:
        m.close()


_cases = {}


@pytest.fixture(scope="module")
def cases(lanes):
    yield lambda name: _cases[name] if name in _cases else _cases.setdefault(name, Case(name, lanes))
    for c in _cases.values():
        c.corpus.close()
    _cases.clear()


# ---------------------------------------------------------------------------------------------------- checks
def expect(got, want):
    assert len(got) == len(want), (len(got), len(want))
    for f in ("index", "score", "exact"):
        bad = np.nonzero(got[f] != want[f])[0]
        assert bad.size == 0, (f, bad[:5], got[bad[:5]], want[bad[:5]])


def check_case_overflows(c):
    """the oracle puts more than the cap into the targeted class, and (for an extra atom) no class of the atoms before it
    goes past the cap"""
    cap = cap_of(c.n)
    counts = c.class_counts[c.target_atom]
    assert counts.get(c.target_class, 0) > cap, (c.name, counts, cap)
    for before in c.class_counts[: c.target_atom]:
        assert all(v <= cap for k, v in before.items() if k != "None"), (c.name, before, cap)


def launches(m):
    return m.last_timings()["launches"]


def first_call_overflows(c, m, call):
    """call() on a fresh matcher, twice: the first overflows its lists and runs again, the second (lists grown to n) runs
    once and returns the same rows.  Returns the first call's result."""
    got = call()
    l1 = launches(m)
    again = call()
    l2 = launches(m)
    if len(c.patterns) == 1:
        assert l1 == 2 * l2, (c.name, l1, l2)
    else:
        assert l1 > l2, (c.name, l1, l2)
    for a, b in zip(got if isinstance(got, tuple) else (got,), again if isinstance(again, tuple) else (again,)):
        if isinstance(a, np.ndarray):
            expect(a, b)
        else:
            assert a == b
    return got


# ---------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("sort", SORTS, ids=lambda s: s.name)
@pytest.mark.parametrize("name", list(CASES))
def test_full_list(cases, name, sort):
    c = cases(name)
    check_case_overflows(c)
    m = c.matcher(sort)
    try:
        if name in ("long", "multi_long_extra"):
            assert m.score_bound() >= 1024   # the two-pass sort
        got = first_call_overflows(c, m, lambda: m.match_list_array(c.corpus))
        expect(got, c.want(sort))
    finally:
        m.close()


@pytest.mark.parametrize("name", list(CASES))
def test_top_k(cases, name):
    c = cases(name)
    sort = SORTS[list(CASES).index(name) % 2]
    want = c.want(sort)
    k = len(want) // 3 + 7
    m = c.matcher(sort)
    try:
        got, total = first_call_overflows(c, m, lambda: m.match_list_top_array(c.corpus, k))
        assert total == len(want)
        expect(got, want[:k])
    finally:
        m.close()


@pytest.mark.parametrize("name", SUBSET_CASES)
def test_masked_subset(cases, name):
    """half of the rows as a subset: the masked form (the corpus's slot metadata with the non-members' slots unused)"""
    c = cases(name)
    rng = np.random.default_rng(5)
    members = np.nonzero(rng.random(c.n) < 0.5)[0].astype(np.uint32)
    want = c.want(SortStrategy.ScoreThenIndexAsc, members)
    assert len(want) > cap_of(c.n)
    sub = c.corpus.subset(members)
    m = c.matcher(SortStrategy.ScoreThenIndexAsc)
    try:
        expect(first_call_overflows(c, m, lambda: m.match_list_subset_array(c.corpus, sub)), want)
        got, total = m.match_list_subset_top_array(c.corpus, sub, 1000)
        assert total == len(want)
        expect(got, want[:1000])
    finally:
        m.close()
        sub.close()


@pytest.mark.parametrize("name", SUBSET_CASES)
def test_ranked(cases, name):
    c = cases(name)
    sort = SORTS[SUBSET_CASES.index(name)]
    rng = np.random.default_rng(6)
    values = rng.integers(-40, 41, size=c.n).astype(np.int16)
    want = rank_by_boost(c.into, values, SortStrategy(sort).is_reversed())
    boost = c.corpus.boost(values)
    m = c.matcher(sort)
    try:
        got, total = first_call_overflows(c, m, lambda: m.match_list_ranked_array(c.corpus, boost))
        assert total == len(want)
        expect(got, want)
        got, total = m.match_list_ranked_array(c.corpus, boost, k=500)
        assert total == len(want)
        expect(got, want[:500])
    finally:
        m.close()
        boost.close()


def test_small_corpus_first(cases):
    """the lists are grow-only and sized by the first call: after a call on 3 000 rows they hold 3 000 records, and the
    large corpus still overflows them, grows them and runs again"""
    c = cases("cols128")
    sort = SortStrategy.ScoreThenIndexAsc
    small_n = 3000
    small = F.Corpus.from_arrow(c.data[: int(c.off[small_n])], c.off[: small_n + 1])
    m = c.matcher(sort)
    try:
        expect(m.match_list_array(small), c.want(sort, np.arange(small_n)))
        expect(first_call_overflows(c, m, lambda: m.match_list_array(c.corpus)), c.want(sort))
        expect(m.match_list_array(small), c.want(sort, np.arange(small_n)))
    finally:
        m.close()
        small.close()
