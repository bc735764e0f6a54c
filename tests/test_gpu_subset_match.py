"""Subsets filled from text queries on the GPU (frz_subset_match, Subset.matching / Corpus.matching).  The contract: the
filled subset holds {r.index for r in frz_match_list_into(m, T)} ∩ base and behaves bit for bit like frz_subset_create over
those indices.  Checked for every typo mode, short, long and unicode needles, the four literal modes, negated, multi-atom,
all-negated and empty queries, edited corpora, a text corpus other than the subset's, bases (shorter than the corpus, and
the subset itself), both prefilter forms (full and masked slot metadata), survivor-list overflow, every subset-taking call,
the matcher's later match calls, and device memory on refills.  Needs a CUDA device."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200.types import Config, Matching, Pattern, SortStrategy

pytestmark = pytest.mark.gpu

DIRS = ["src", "lib", "test", "tests", "docs", "node_modules", "Src", "été", "데이터", "matcher", "src/matcher"]
EXTS = ["rs", "py", "toml", "md", "RS", "txt", "é"]
LONG = "abcdefghij" * 7          # a 70-byte needle
LONGER = "klmnopqrst" * 40       # a 400-byte needle


def path_rows(n, seed):
    """n path-like rows: a few directories deep, a name and an extension; some rows carry a long needle's text."""
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(n):
        parts = [DIRS[int(j)] for j in rng.integers(0, len(DIRS), int(rng.integers(0, 4)))]
        name = "".join(chr(int(c)) for c in rng.integers(97, 123, int(rng.integers(1, 9))))
        r = rng.random()
        if r < 0.03:
            name += LONG[: int(rng.integers(60, 71))]
        elif r < 0.05:
            name += LONGER[: int(rng.integers(395, 401))]
        rows.append("/".join(parts + [name + "." + EXTS[int(rng.integers(len(EXTS)))]]))
    return rows


def expected(m, text, base_mask=None):
    mask = np.zeros(len(text), bool)
    mask[m.match_list_into_array(text)["index"]] = True
    if base_mask is not None:
        mask &= base_mask
    return mask


def base_mask_of(sub, n, which):
    mask = np.zeros(n, bool)
    mask[which[which < n]] = True
    return mask


def assert_same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), what


PROBES = [F.Matcher("src", Config(max_typos=1)), F.Matcher.from_query("", Config()), F.Matcher("é", Config(max_typos=0)),
          F.Matcher.from_query("rs !test", Config(max_typos=0, sort=SortStrategy.IndexDesc))]


def check(corpus, filled, mask, what, heavy=False):
    """filled behaves as frz_subset_create over np.flatnonzero(mask)."""
    ref = corpus.subset(np.flatnonzero(mask))
    try:
        assert len(filled) == len(ref) == int(mask.sum()), what
        for m in PROBES if heavy else PROBES[:2]:
            assert_same(m.match_list_subset_array(corpus, filled), m.match_list_subset_array(corpus, ref), (what, "list"))
            a, ta = m.match_list_subset_top_array(corpus, filled, 50)
            b, tb = m.match_list_subset_top_array(corpus, ref, 50)
            assert ta == tb, what
            assert_same(a, b, (what, "top"))
        if not heavy:
            return
        rng = np.random.default_rng(len(corpus))
        m = PROBES[0]
        boost = corpus.boost(rng.integers(-300, 300, len(corpus)).astype(np.int16))
        groups = corpus.groups(rng.integers(0, 17, len(corpus)).astype(np.uint32), 17)
        attr = corpus.attr(rng.integers(0, 50, len(corpus)).astype(np.int64))
        try:
            a, ta = m.match_list_ranked_array(corpus, boost, 20, filled)
            b, tb = m.match_list_ranked_array(corpus, boost, 20, ref)
            assert ta == tb and np.array_equal(a, b), (what, "ranked")
            a = m.match_list_ordered_array(corpus, attr, k=20, subset=filled)
            b = m.match_list_ordered_array(corpus, attr, k=20, subset=ref)
            assert a[1] == b[1] and np.array_equal(a[0], b[0]), (what, "ordered")
            a = m.match_list_collapsed_array(corpus, groups, 20, 2, filled, boost, counts=True)
            b = m.match_list_collapsed_array(corpus, groups, 20, 2, ref, boost, counts=True)
            assert a[1] == b[1] and np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2]), (what, "collapsed")
            ms = [F.Matcher(w, Config(max_typos=0, sort=SortStrategy(j % 4))) for j, w in enumerate(["src", "rs", "ab", "lib"] * 10)]
            a = F.match_list_batch(ms, corpus, 10, subsets=[filled if j % 2 else None for j in range(40)])
            b = F.match_list_batch(ms, corpus, 10, subsets=[ref if j % 2 else None for j in range(40)])
            for x, y in zip(a, b):
                assert np.array_equal(x, y), (what, "batch")
        finally:
            boost.close()
            groups.close()
            attr.close()
    finally:
        ref.close()


QUERIES = ["src", "^src/", ".rs$", "'test", "!test", "src !test", "^src/ .rs$ !test", "!^docs !.md$", "!node_modules",
           "", "été", "!데이터 rs", "^데이터/", "'é", LONG, "src " + LONGER, "!" + LONG, "matcher/mod", "rs toml"]
TYPOS = [0, 1, 2, 3, 7, 15, None]


@pytest.fixture(scope="module")
def corpus():
    rows = path_rows(40_000, 1)
    c = F.Corpus.from_list(rows)
    yield c
    c.close()


@pytest.mark.parametrize("typos", TYPOS)
def test_queries_every_typo_mode(corpus, typos):
    s = corpus.subset([])
    try:
        for q in QUERIES:
            m = F.Matcher.from_query(q, Config(max_typos=typos))
            want = expected(m, corpus)
            for force in ("full", "masked"):
                F.subset_match_debug(force)
                s.matching(m)
                assert len(s) == int(want.sum()), (q, typos, force)
                check(corpus, s, want, (q, typos, force))
    finally:
        F.subset_match_debug("rule")
        s.close()


@pytest.mark.parametrize("mode", [Matching.Exact, Matching.Prefix, Matching.Suffix, Matching.Substring])
def test_literal_modes(corpus, mode):
    for needle in ["src/matcher", "rs", "é", "데이터/", LONG[:66]]:
        for cfg in (Config(matching=mode), Config(matching=mode, max_typos=2)):
            m = F.Matcher(Pattern(needle=needle), cfg)
            s = corpus.matching(m)
            check(corpus, s, expected(m, corpus), (needle, mode))
            s.close()
    rows = ["src/a.rs", "src", "xsrc", "SRC", "src/"]   # Exact: whole rows only
    small = F.Corpus.from_list(rows)
    m = F.Matcher(Pattern(needle="src"), Config(matching=mode))
    s = small.matching(m)
    assert len(s) == int(expected(m, small).sum())
    s.close()
    small.close()


def test_bases_and_in_place(corpus):
    n = len(corpus)
    rng = np.random.default_rng(3)
    s = corpus.subset([])
    try:
        for q in ["^src/", "rs !test", "!docs", ""]:
            m = F.Matcher.from_query(q, Config(max_typos=1))
            for which in (rng.integers(0, n, 300), rng.integers(0, n // 3, n // 2), np.arange(n // 2), np.arange(n)):
                base = corpus.subset(which.astype(np.uint32))
                bm = base_mask_of(base, n, which)
                for force in ("rule", "full", "masked"):
                    F.subset_match_debug(force)
                    s.matching(m, base=base)
                    check(corpus, s, expected(m, corpus, bm), (q, len(which), force))
                base.close()
            # base = s: refines in place
            s.matching(F.Matcher.from_query("src", Config(max_typos=0)))
            before = expected(F.Matcher.from_query("src", Config(max_typos=0)), corpus)
            s.matching(m, base=s)
            check(corpus, s, expected(m, corpus, before), (q, "in place"))
        # a base made before an append is shorter than the corpus: the appended rows are not its members
        c = F.Corpus.from_list(path_rows(5000, 9))
        short = c.subset(np.arange(0, 5000, 2, dtype=np.uint32))
        c.append_list(path_rows(3000, 10))
        m = F.Matcher.from_query("^src/ !test", Config(max_typos=0))
        bm = np.zeros(len(c), bool)
        bm[:5000:2] = True
        for force in ("full", "masked"):
            F.subset_match_debug(force)
            t = c.matching(m, base=short)
            check(c, t, expected(m, c, bm), ("short base", force))
            t.matching(m, base=t)   # a bitmap that grows while it is the base
            check(c, t, expected(m, c, bm), ("short base in place", force))
            t.close()
        short.close()
        c.close()
    finally:
        F.subset_match_debug("rule")
        s.close()


def test_masked_rule(corpus):
    n = len(corpus)
    m = F.Matcher.from_query("^src/ .rs$ !test", Config(max_typos=0))
    small = corpus.subset(np.arange(0, n, 50, dtype=np.uint32))   # 2 % of the rows
    every = corpus.subset(np.arange(n, dtype=np.uint32))
    F.subset_match_debug("rule")
    s = corpus.matching(m)
    assert F.subset_match_debug() == 2   # the patterns after the first
    s.matching(m, base=small)
    assert F.subset_match_debug() == 3   # and the first, inside a base that leaves rows out
    s.matching(m, base=every)
    assert F.subset_match_debug() == 2
    s.matching(F.Matcher.from_query("src", Config()))
    assert F.subset_match_debug() == 0
    for h in (s, small, every):
        h.close()


def test_edited_corpora():
    rows = path_rows(20_000, 5)
    c = F.Corpus.from_list(rows)
    rng = np.random.default_rng(5)
    c.remove(rng.integers(0, len(rows), 2000).astype(np.uint32))
    which = rng.choice(len(rows), 1500, replace=False).astype(np.uint32)
    c.replace_list(which, path_rows(1500, 6))
    c.append_list(path_rows(3000, 7))
    for q in ["^src/ .rs$ !test", "!test", "", "été", LONG, "rs !" + LONG]:
        for typos in (0, 1, None):
            m = F.Matcher.from_query(q, Config(max_typos=typos))
            s = c.matching(m)
            check(c, s, expected(m, c), (q, typos, "edited"))
            s.close()
    c.close()


def test_another_text_corpus():
    n = 30_000
    rng = np.random.default_rng(8)
    dirs = [DIRS[int(j)] + "/" + DIRS[int(k)] for j, k in rng.integers(0, len(DIRS), (n, 2))]
    names = ["".join(chr(int(c)) for c in rng.integers(97, 123, 6)) + "." + EXTS[int(e)] for e in rng.integers(0, len(EXTS), n)]
    dcol, ncol = F.Corpus.from_list(dirs), F.Corpus.from_list(names)
    dcol.remove(np.arange(0, n, 97, dtype=np.uint32))   # removed directory rows never match
    base = ncol.subset(np.arange(0, n, 3, dtype=np.uint32))
    bm = np.zeros(n, bool)
    bm[::3] = True
    for q in ["^src/", "!test", "matcher", "", "été !docs"]:
        m = F.Matcher.from_query(q, Config(max_typos=1))
        s = ncol.matching(m, text=dcol)
        check(ncol, s, expected(m, dcol), (q, "text"))
        s.matching(m, text=dcol, base=base)
        check(ncol, s, expected(m, dcol, bm), (q, "text + base"))
        s.close()
    other = F.Corpus.from_list(names[:-1])
    s = ncol.subset([])
    with pytest.raises(F.FrizbeeError, match="index space"):
        s.matching(F.Matcher("src", Config()), text=other)
    with pytest.raises(F.FrizbeeError, match="base subset was made on another corpus"):
        s.matching(F.Matcher("src", Config()), base=dcol.subset([1]))
    assert len(s) == 0
    for h in (s, base, other, dcol, ncol):
        h.close()


def test_every_subset_call_and_overflow():
    # 300 k rows that all match: more survivors than the first survivor lists hold (a quarter of the rows)
    n = 300_000
    rows = path_rows(n, 11)
    c = F.Corpus.from_list(rows)
    try:
        for q, typos in [("a", 1), ("!zzzzzzzz", 0), ("'.", 0), ("^src/ .rs$ !test", 0), ("src !test", 1)]:
            # a fresh matcher fills: its lists have their first size (a match call that overflows grows them)
            s = c.matching(F.Matcher.from_query(q, Config(max_typos=typos)))
            check(c, s, expected(F.Matcher.from_query(q, Config(max_typos=typos)), c), (q, "every call"), heavy=True)
            s.close()
        m = F.Matcher.from_query("a", Config(max_typos=1))
        assert expected(m, c).sum() > n // 2
    finally:
        c.close()


def test_match_calls_after_a_fill(corpus):
    for q, typos in [("src !test", 1), ("été", 0), (LONG, 2), ("^src/ .rs$", 0)]:
        m = F.Matcher.from_query(q, Config(max_typos=typos))
        before = m.match_list_array(corpus)
        top = m.match_list_top_array(corpus, 20)
        s = corpus.matching(m)
        assert_same(m.match_list_array(corpus), before, q)
        after = m.match_list_top_array(corpus, 20)
        assert after[1] == top[1] and np.array_equal(after[0], top[0]), q
        s.close()


def _bytes():
    L = F.lib()
    L.frz_debug_device_bytes.restype = C.c_uint64
    L.frz_debug_device_bytes.argtypes = []
    return L.frz_debug_device_bytes()


def test_refills_allocate_nothing(corpus):
    m = F.Matcher.from_query("^src/ .rs$ !test", Config(max_typos=1))
    u = F.Matcher.from_query("été !docs", Config(max_typos=0))
    base = corpus.subset(np.arange(0, len(corpus), 40, dtype=np.uint32))
    s = corpus.subset([])
    for force in ("masked", "full"):   # the first fills of each shape size everything
        F.subset_match_debug(force)
        s.matching(m, base=base)
        s.matching(u)
        s.matching(m)
    F.subset_match_debug("rule")
    start = _bytes()
    for _ in range(3):
        s.matching(m)
        s.matching(m, base=base)
        s.matching(u)
        assert _bytes() == start
    s.close()
    base.close()


def test_empty_corpus_and_null_arguments():
    c = F.Corpus.from_list([])
    s = c.matching(F.Matcher("x", Config()))
    assert len(s) == 0
    assert F.lib().frz_subset_match(s._h, None, None, None) == 1
    assert F.lib().frz_subset_match(None, F.Matcher("x", Config())._h, None, None) == 1
    s.close()
    c.close()
