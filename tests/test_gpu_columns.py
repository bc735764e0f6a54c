"""Column calls on the GPU (frz_match_list_columns): a matcher per column, rows must match every column, scores add up.

With one column the call is the existing single-corpus calls bit for bit (top-K, subset, ranked and collapsed, for every
matcher kind and strategy).  A matcher per atom over repeats of one corpus is the multi-pattern matcher over it.  Distinct
columns follow tests/columns.py over the CPU oracle's per-column lists, with and without subset, boost and groups.  Then
corpus edits in some columns only, a survivor-list overflow in the base column and in a later one, a long needle in a
matcher that has never run, a million rows, and the device memory the calls hold."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from collapsing import GROUP_NONE
from columns import match_list_columns as spec
from frizbee_b200 import synth
from frizbee_b200.types import CaseMatching, Config, Matching, Pattern, Scoring, SortStrategy
from oracle import pyoracle as O
from test_gpu_collapsed import LONG300, MATCHERS, assert_same, gen, shapes
from test_gpu_survivor_overflow import Case, cap_of, launches

pytestmark = pytest.mark.gpu

INVALID_ARG = 1
TILE = 1024
LANES = 32
KS = (0, 1, 50, None)


def cfg(sort, max_typos=0, **kw):
    return Config(max_typos=max_typos, sort=sort, emulate_lanes=LANES, **kw)


# every matcher kind of test_gpu_collapsed.py, and the typo budgets, negations and long needles it lacks
KINDS = dict(MATCHERS)
KINDS.update({
    "typos2": lambda s: F.Matcher("deadbeef", cfg(s, 2)),
    "typos3": lambda s: F.Matcher("deadbeef", cfg(s, 3)),
    "typos15": lambda s: F.Matcher("deadbeefdeadbeefdeadbeef", cfg(s, 15)),
    "long80": lambda s: F.Matcher(LONG300[:80], cfg(s, 1)),
    "long1024": lambda s: F.Matcher((LONG300 * 4)[:1024], cfg(s, 3)),
    "negated": lambda s: F.Matcher.from_query("dead !bar", cfg(s, 1)),
    "all-negated": lambda s: F.Matcher.from_query("!foo !bar", cfg(s, 0)),
    "exact": lambda s: F.Matcher("foobar", cfg(s, 0, matching=Matching.Exact)),
    "suffix": lambda s: F.Matcher("😀", cfg(s, 0, matching=Matching.Suffix)),
})


def columns(ms, cs, k=None, sort=SortStrategy.ScoreThenIndexAsc, **kw):
    return F.match_list_columns(ms, cs, k, sort, **kw)


@pytest.fixture(scope="module")
def small():
    hs = gen(3 * TILE + 77, 21)
    data, off = O.pack(hs)
    corpus = F.Corpus.from_arrow(data, off)
    yield corpus, hs
    corpus.close()


# ------------------------------------------------------------------------------------------------ 1. one column
@pytest.mark.parametrize("kind", list(KINDS))
def test_one_column_equals_the_existing_calls(small, kind):
    corpus, _ = small
    n = len(corpus)
    rng = np.random.default_rng(len(kind))
    sub = corpus.subset(np.nonzero(rng.random(n) < 0.4)[0].astype(np.uint32))
    tiny = corpus.subset(rng.choice(n, 40, replace=False).astype(np.uint32))            # the list form
    boost = corpus.boost(rng.integers(-60, 61, n).astype(np.int16))
    _, ids, n_groups = shapes(n, 3)[5]
    groups = corpus.groups(ids, n_groups)
    try:
        for sort in SortStrategy:
            m = KINDS[kind](sort)
            for k in KS:
                kk = 0xFFFFFFFFFFFFFFFF if k is None else k
                got, total = columns([m], [corpus], k, sort)
                want, wtotal = m.match_list_top_array(corpus, kk)
                assert total == wtotal, (kind, sort, k)
                assert_same(got, want, (kind, sort.name, k, "top"))
                for s in (sub, tiny):
                    got, total = columns([m], [corpus], k, sort, subset=s)
                    want, wtotal = m.match_list_subset_top_array(corpus, s, kk)
                    assert total == wtotal
                    assert_same(got, want, (kind, sort.name, k, "subset"))
                got, total = columns([m], [corpus], k, sort, boost=boost, subset=sub)
                want, wtotal = m.match_list_ranked_array(corpus, boost, k, subset=sub)
                assert total == wtotal
                assert_same(got, want, (kind, sort.name, k, "ranked"))
                for pg in (1, 3, None):
                    got, total, cnt = columns([m], [corpus], k, sort, boost=boost if pg == 3 else None, groups=groups,
                                              per_group=pg, counts=True)
                    want, wtotal, wcnt = m.match_list_collapsed_array(corpus, groups, k, per_group=pg,
                                                                      boost=boost if pg == 3 else None, counts=True)
                    assert total == wtotal
                    assert_same(got, want, (kind, sort.name, k, "collapsed", pg))
                    assert np.array_equal(cnt, wcnt)
            m.close()
    finally:
        for h in (sub, tiny, boost, groups):
            h.close()


# ------------------------------------------------------------------------------------------------ 2. atoms over repeats
@pytest.mark.parametrize("sort", list(SortStrategy), ids=lambda s: s.name)
def test_atoms_over_repeats_equal_the_multi_pattern_matcher(small, sort):
    corpus, _ = small
    for atoms in ([Pattern("foo"), Pattern("bar", negated=True, matching=Matching.Prefix), Pattern("dead", matching=Matching.Substring)],
                  [Pattern("bar", negated=True), Pattern("dbf", max_typos=None), Pattern("é다", max_typos=0)],
                  [Pattern("deadbeef", max_typos=2), Pattern(LONG300[:100], negated=True), Pattern("ef", casing=CaseMatching.Respect)],
                  [Pattern("foo", negated=True), Pattern("bar", negated=True)],
                  [Pattern("a", scoring=Scoring(match_score=40)), Pattern("b")]):
        c = cfg(sort, 1)
        whole = F.Matcher.from_patterns(atoms, c)
        per = [F.Matcher.from_patterns([a], c) for a in atoms]
        want = whole.match_list_array(corpus)
        got, total = columns(per, [corpus] * len(per), None, sort)
        assert total == len(want)
        assert_same(got, want, (atoms, sort))
        for j in range(len(per)):   # the order of the columns changes nothing
            order = per[j:] + per[:j]
            assert_same(columns(order, [corpus] * len(per), None, sort)[0], want, (atoms, sort, j))
        whole.close()
        for m in per:
            m.close()
    q = F.Matcher.from_query("foo !^bar 'dead", cfg(sort, 1))
    parts = [F.Matcher.from_query(a, cfg(sort, 1)) for a in ("foo", "!^bar", "'dead")]
    assert_same(columns(parts, [corpus] * 3, None, sort)[0], q.match_list_array(corpus), ("query", sort))
    for m in parts + [q]:
        m.close()


# ------------------------------------------------------------------------------------------------ 3. distinct columns
def oracle_lists(cols, tables):
    return [O.match_list_into_packed(p, c, *O.pack(t)) if p else
            np.array([(i, 0, 0, 0) for i in range(len(t))], dtype=F.MATCH_DTYPE) for (p, c), t in zip(cols, tables)]


HIGH = Scoring(match_score=(0xFFFF - 40) // 3 - 8)
COLUMN_SETS = {
    "two": [(["deadbeef"], Config(max_typos=1)), (["foo"], Config(max_typos=0, casing=CaseMatching.Respect))],
    "three": [([Pattern("bar", negated=True)], Config(max_typos=0)), (["dbf"], Config(max_typos=None)),
              ([Pattern("é다😀")], Config(max_typos=1))],
    "four": [(["ab"], Config(max_typos=0, scoring=Scoring(gap_open_penalty=1, gap_extend_penalty=0))), ([], Config()),
             ([Pattern("ef", matching=Matching.Substring)], Config()), ([LONG300[:90]], Config(max_typos=2))],
    "saturating": [([Pattern("foo", matching=Matching.Substring, scoring=HIGH)], Config()),
                   ([Pattern("bar", matching=Matching.Substring, scoring=HIGH)], Config())],
}


COLUMN_LANES = (32, 64, 16)


@pytest.mark.parametrize("name", list(COLUMN_SETS))
def test_distinct_columns_against_the_oracle(name):
    # each column emulates its own reference backend: patterns compiled for different lane widths run in one call
    spec_cols = [(p, c.with_(emulate_lanes=COLUMN_LANES[j % len(COLUMN_LANES)])) for j, (p, c) in enumerate(COLUMN_SETS[name])]
    n = 2 * TILE + 300
    tables = [gen(n, 100 + j) for j in range(len(spec_cols))]
    lists = oracle_lists(spec_cols, tables)
    if name == "saturating":
        from columns import combine
        assert (combine(lists, n)["score"] == 65535).any()
    corpora = [F.Corpus.from_list(t) for t in tables]
    rng = np.random.default_rng(len(name))
    members = np.nonzero(rng.random(n) < 0.5)[0].astype(np.uint32)
    values = rng.integers(-100, 101, n).astype(np.int16)
    ids = rng.integers(0, 30, n).astype(np.uint32)
    ids[rng.random(n) < 0.2] = GROUP_NONE
    sub, boost, groups = corpora[0].subset(members), corpora[-1].boost(values), corpora[len(corpora) // 2].groups(ids, 30)
    any_compiled = any(p for p, _ in spec_cols)
    try:
        for sort in SortStrategy:
            ms = [F.Matcher.from_patterns([p if isinstance(p, Pattern) else Pattern(p) for p in pats], c.with_(sort=sort))
                  for pats, c in spec_cols]
            for kw, skw in ((dict(), dict()), (dict(subset=sub), dict(members=members)), (dict(boost=boost), dict(boost=values)),
                            (dict(groups=groups, per_group=2, counts=True), dict(group_of=ids, per_group=2, n_groups=30)),
                            (dict(subset=sub, boost=boost, groups=groups, per_group=None, counts=True),
                             dict(members=members, boost=values, group_of=ids, per_group=None, n_groups=30))):
                want, wcnt = spec(lists, n, sort, any_compiled=any_compiled, **skw)
                for k in (0, 7, None):
                    res = columns(ms, corpora, k, sort, **kw)
                    assert res[1] == len(want), (name, sort, sorted(kw), k)
                    assert_same(res[0], want if k is None else want[:k], (name, sort.name, sorted(kw), k))
                    if wcnt is not None:
                        assert np.array_equal(res[2], wcnt)
            for m in ms:
                m.close()
    finally:
        for h in (sub, boost, groups, *corpora):
            h.close()


# ------------------------------------------------------------------------------------------------ 4. edits
def gpu_lists(ms, cs):
    return [m.match_list_into_array(c).copy() for m, c in zip(ms, cs)]


def check_against_own_lists(ms, cs, sort, what):
    lists = gpu_lists(ms, cs)
    want, _ = spec(lists, len(cs[0]), sort, any_compiled=any(m.num_patterns() for m in ms))
    got, total = columns(ms, cs, None, sort)
    assert total == len(want), what
    assert_same(got, want, what)
    return want


def test_edits_in_some_columns():
    n = 3 * TILE + 5
    t0, t1, t2 = gen(n, 31), gen(n, 32), gen(n, 33)
    c0, c1, c2 = (F.Corpus.from_list(t) for t in (t0, t1, t2))
    sort = SortStrategy.ScoreThenIndexAsc
    ms = [F.Matcher("dbf", cfg(sort, 1)), F.Matcher.from_query("", cfg(sort)), F.Matcher.from_query("!zz d", cfg(sort, 1))]
    try:
        base = check_against_own_lists(ms, [c0, c1, c2], sort, "unedited")
        # a row removed in one later column only (and in the empty column, which scans nothing) leaves the result
        gone = base["index"][: 40].astype(np.uint32)
        c2.remove(gone[:20])
        c1.remove(gone[20:])
        after = check_against_own_lists(ms, [c0, c1, c2], sort, "removed in later columns")
        assert not np.isin(after["index"], gone).any() and len(after) == len(base) - 40
        # removed in the scanned column too; replaced rows in every column
        c0.remove(base["index"][40:45].astype(np.uint32))
        which = np.arange(0, n, 97, dtype=np.uint32)
        for c, t in ((c0, t1), (c1, t0), (c2, t0)):
            c.replace_list(which, [t[int(i)] for i in which])
        for sort2 in SortStrategy:
            check_against_own_lists(ms, [c0, c1, c2], sort2, ("edited", sort2))
        # appends: to one column only is refused until the others catch up, and the refusal changes nothing
        extra = gen(2 * TILE, 34)
        c0.append_list(extra)
        with pytest.raises(F.FrizbeeError) as e:
            columns(ms, [c0, c1, c2])
        assert e.value.status == INVALID_ARG and "index space" in str(e.value)
        c1.append_list(extra[::-1])
        with pytest.raises(F.FrizbeeError):
            columns(ms, [c0, c1, c2])
        c2.append_list(extra)
        check_against_own_lists(ms, [c0, c1, c2], sort, "appended")
        check_against_own_lists(ms[::-1], [c2, c1, c0], sort, "appended, reversed")
    finally:
        for x in ms + [c0, c1, c2]:
            x.close()


def test_removed_rows_in_more_columns_than_one_liveness_pass_covers():
    """eleven copies of one table, each with its own removed rows: ten columns besides the scanned one have removed rows,
    more than one k_keep<LiveInColumns> pass takes (8), so the starting list is filtered in two passes"""
    n = 2 * TILE + 40
    hay = gen(n, 61)
    cs = [F.Corpus.from_list(hay) for _ in range(11)]
    rng = np.random.default_rng(61)
    for c in cs[1:]:
        c.remove(rng.choice(n, 25, replace=False).astype(np.uint32))
    sort = SortStrategy.ScoreThenIndexAsc
    ms = [F.Matcher("dbf", cfg(sort, None))] + [F.Matcher.from_query("" if j % 2 else "!zzz", cfg(sort)) for j in range(10)]
    try:
        want = check_against_own_lists(ms, cs, sort, "ten edited columns")
        listed_later = np.ones(n, dtype=bool)   # in every later column's list (a removed row is in none)
        for m, c in zip(ms[1:], cs[1:]):
            listed_later &= np.isin(np.arange(n), m.match_list_into_array(c)["index"])
        assert len(want) and not np.isin(want["index"], np.nonzero(~listed_later)[0]).any()
        full = ms[0].match_list_into_array(cs[0])
        assert len(want) < len(full)   # some of the scanned column's matches were removed in later columns
        for sort2 in (SortStrategy.IndexDesc, SortStrategy.ScoreThenIndexDesc):
            check_against_own_lists(ms, cs, sort2, ("ten edited columns", sort2))
    finally:
        for x in ms + cs:
            x.close()


# ------------------------------------------------------------------------------------------------ 5. overflow
@pytest.fixture(scope="module")
def lanes():
    m = F.Matcher("abcd", Config())
    try:
        return m.backend_info()["prefilter_lanes"]
    finally:
        m.close()


@pytest.mark.parametrize("name", ["multi_base", "multi_extra"])
def test_survivor_overflow_is_retried(lanes, name):
    """multi_base overflows its base atom's lists, multi_extra its later atom's (tests/test_gpu_survivor_overflow.py): as
    one matcher per atom over repeats of the corpus, the base column and a later column overflow"""
    c = Case(name, lanes)
    try:
        assert c.class_counts[c.target_atom].get(c.target_class, 0) > cap_of(c.n)
        for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexDesc):
            ms = [F.Matcher([p], c.cfg.with_(sort=sort)) for p in c.patterns]
            want = c.want(sort)
            got, total = columns(ms, [c.corpus] * len(ms), None, sort)
            l1 = launches(ms[0])
            again, _ = columns(ms, [c.corpus] * len(ms), 100, sort)
            assert l1 > launches(ms[0]), (name, l1, launches(ms[0]))   # the first call ran twice
            assert total == len(want)
            assert_same(got, want, (name, sort))
            assert_same(again, want[:100], (name, sort, 100))
            for m in ms:
                m.close()
    finally:
        c.corpus.close()


# ------------------------------------------------------------------------------------------------ 6. long needle, fresh
def test_long_needle_in_a_fresh_later_matcher():
    n = 2 * TILE + 17
    t0, t1 = gen(n, 41), gen(n, 42)
    c0, c1 = F.Corpus.from_list(t0), F.Corpus.from_list(t1)
    sort = SortStrategy.ScoreThenIndexDesc
    first = F.Matcher("dbf", cfg(sort, None))
    first.match_list_array(c0)                         # ms[0] has run; the long-needle matcher has not
    fresh = F.Matcher.from_patterns([Pattern(LONG300, max_typos=2), Pattern(LONG300[:70], max_typos=1)], cfg(sort, 2))
    try:
        got, total = columns([first, fresh], [c0, c1], None, sort)
        lists = [O.match_list_into_packed(["dbf"], cfg(sort, None), *O.pack(t0)),
                 O.match_list_into_packed([Pattern(LONG300, max_typos=2), Pattern(LONG300[:70], max_typos=1)], cfg(sort, 2), *O.pack(t1))]
        want, _ = spec(lists, n, sort)
        assert len(want) > 10 and total == len(want)
        assert_same(got, want, "fresh long")
        assert_same(fresh.match_list_into_array(c1), lists[1], "the fresh matcher's own call afterwards")
    finally:
        for x in (first, fresh, c0, c1):
            x.close()


# ------------------------------------------------------------------------------------------------ 7. scale
def test_a_million_rows():
    n = 1_000_000
    d0, o0 = synth.generate("deadbeef", n, 24, 48, seed=1)
    d1, o1 = synth.generate("srcmain", n, 40, 96, seed=2, p_partial=0.4, p_full=0.2)
    c0, c1 = F.Corpus.from_arrow(d0, o0), F.Corpus.from_arrow(d1, o1)
    sort = SortStrategy.ScoreThenIndexAsc
    ms = [F.Matcher("deadbeef", cfg(sort, 1)), F.Matcher("src", cfg(sort, 1))]
    rng = np.random.default_rng(9)
    values = rng.integers(-50, 51, n).astype(np.int16)
    ids = rng.integers(0, 1000, n).astype(np.uint32)
    boost, groups = c1.boost(values), c0.groups(ids, 1000)
    try:
        lists = gpu_lists(ms, [c0, c1])
        want, _ = spec(lists, n, sort)
        assert len(want) > 1000
        got, total = columns(ms, [c0, c1], 50, sort)
        assert total == len(want)
        assert_same(got, want[:50], "1M top-50")
        got, total = columns(ms, [c0, c1], 50, sort, boost=boost)
        assert_same(got, spec(lists, n, sort, boost=values)[0][:50], "1M ranked")
        got, total, cnt = columns(ms, [c0, c1], 50, sort, groups=groups, counts=True)
        w, wcnt = spec(lists, n, sort, group_of=ids, n_groups=1000)
        assert total == len(w) and np.array_equal(cnt, wcnt)
        assert_same(got, w[:50], "1M collapsed")
    finally:
        for x in ms + [boost, groups, c0, c1]:
            x.close()


# ------------------------------------------------------------------------------------------------ 8. memory
def device_bytes():
    L = F.lib()
    L.frz_debug_device_bytes.restype = C.c_uint64
    L.frz_debug_device_bytes.argtypes = []
    return L.frz_debug_device_bytes()


def test_memory_is_steady_and_released():
    start = device_bytes()
    n = 4 * TILE
    cs = [F.Corpus.from_list(gen(n, 50 + j)) for j in range(3)]
    sort = SortStrategy.ScoreThenIndexAsc
    ms = [F.Matcher("deadbeef", cfg(sort, 1)), F.Matcher(LONG300, cfg(sort, 2)), F.Matcher.from_query("!foo b", cfg(sort, 1))]
    sub, boost, groups = cs[1].subset(np.arange(0, n, 3, dtype=np.uint32)), cs[2].boost(np.ones(n, np.int16)), cs[0].groups(np.arange(n, dtype=np.uint32) % 17, 17)
    cs[2].remove(np.arange(0, n, 11, dtype=np.uint32))

    def calls():
        columns(ms, cs, 50, sort)
        columns(ms[::-1], cs[::-1], None, SortStrategy.IndexDesc, subset=sub)
        columns(ms, cs, 10, sort, boost=boost, groups=groups, per_group=2, counts=True)

    calls()
    first = device_bytes()
    for _ in range(3):
        calls()
        assert device_bytes() == first
    for x in ms + [sub, boost, groups] + cs:
        x.close()
    assert device_bytes() == start
