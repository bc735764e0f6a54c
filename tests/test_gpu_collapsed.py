"""Collapsed calls on the GPU (frz_groups_create / frz_groups_set / frz_match_list_collapsed).  The contract: of the list L
the uncollapsed call returns (frz_match_list_ranked with the whole list, frz_match_list_subset or frz_match_list), the
rows in no group and the first per_group rows of each group, in L's order, truncated to the first k; the total is the
number of kept rows and the counts are L's rows per group.  Every check compares with tests/collapsing.py's collapse of
the GPU's own uncollapsed call (pinned to the oracle by the parity tests, and here on a few lists too): for every matcher
kind, sort strategy, ranking and subset form, per_group, k and group shape, across corpus and group edits, after a
survivor-list overflow, at a million rows, and for the device memory the calls hold."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from collapsing import GROUP_NONE, collapse
from frizbee_b200 import synth
from frizbee_b200.types import Config, Matching, SortStrategy
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

INVALID_ARG, UNSUPPORTED = 1, 9
TILE = 1024
LANES = 32          # the reference backend the oracle emulates
ALL = None          # k = None: every kept row
PER_GROUP = (1, 2, 3, 32, ALL)
LONG300 = np.random.default_rng(300).choice(np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", np.uint8), 300).tobytes().decode()


def gen(n, seed):
    """Short random rows; some hold `deadbeef`-like text, `foo`/`bar` prefixes, unicode scalars or the long needle with a
    typo or two."""
    rng = np.random.default_rng(seed)
    pool = np.frombuffer(b"abcdef0123_-/ deadbeefoFOBAR", dtype=np.uint8)
    out = []
    for _ in range(n):
        h = bytearray(rng.choice(pool, int(rng.integers(0, 40))).tobytes())
        r = rng.random()
        if r < 0.10:
            t = bytearray(b"deadbeef")
            for _ in range(int(rng.integers(0, 3))):
                t[int(rng.integers(0, len(t)))] = ord("x")
            h[int(rng.integers(0, len(h) + 1)):0] = t
        elif r < 0.16:
            h = bytearray(rng.choice([b"foo", b"bar", b"foobar", b"barfoo"])) + h
        elif r < 0.20:
            h += "é다x😀".encode()
        elif r < 0.23:
            ln = bytearray(LONG300.encode())
            for _ in range(int(rng.integers(0, 3))):
                ln[int(rng.integers(0, len(ln)))] = ord("q")
            h += ln
        out.append(bytes(h))
    return out


def cfg(sort, max_typos=0, **kw):
    return Config(max_typos=max_typos, sort=sort, emulate_lanes=LANES, **kw)


# name -> matcher factory(sort)
MATCHERS = {
    "typos0": lambda s: F.Matcher("deadbeef", cfg(s, 0)),
    "typos1": lambda s: F.Matcher("deadbeef", cfg(s, 1)),
    "typosNone": lambda s: F.Matcher("dbf", cfg(s, None)),
    "long300": lambda s: F.Matcher(LONG300, cfg(s, 2)),
    "unicode": lambda s: F.Matcher("é다😀", cfg(s, 1)),
    "prefix": lambda s: F.Matcher("foo", cfg(s, 0, matching=Matching.Prefix)),
    "substring": lambda s: F.Matcher("bar", cfg(s, 0, matching=Matching.Substring)),
    "multi": lambda s: F.Matcher.from_query("foo !^bar", cfg(s, 1)),
    "empty": lambda s: F.Matcher.from_query("", cfg(s, 0)),
}


def assert_same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for f in ("index", "score", "exact"):
        bad = np.nonzero(got[f] != want[f])[0]
        assert bad.size == 0, (what, f, bad[:5], got[bad[:5]], want[bad[:5]])


def shapes(n, seed):
    """(name, ids, n_groups) group shapes over n rows"""
    rng = np.random.default_rng(seed)
    mixed = rng.integers(0, 40, n).astype(np.uint32)
    mixed[rng.random(n) < 0.3] = GROUP_NONE
    return [("none", np.full(n, GROUP_NONE, np.uint32), 1),
            ("own", np.arange(n, dtype=np.uint32), n),
            ("one", np.zeros(n, np.uint32), 1),
            ("dup", rng.integers(0, max(n // 50, 1), n).astype(np.uint32), max(n // 50, 1)),
            ("short", rng.integers(0, 5, n // 3).astype(np.uint32), 7),    # rows past n // 3 are in no group
            ("mixed", mixed, 40)]


def uncollapsed(m, corpus, subset=None, boost=None):
    """L: the GPU's own uncollapsed call"""
    if boost is not None:
        return m.match_list_ranked_array(corpus, boost, subset=subset)[0].copy()
    if subset is not None:
        return m.match_list_subset_array(corpus, subset).copy()
    return m.match_list_array(corpus).copy()


def check_collapsed(m, corpus, groups, ids, L, what, subset=None, boost=None, per_groups=PER_GROUP,
                    ks=(0, 1, 50, "total", ALL)):
    """collapsed(k, per_group) == collapse(L)[:k], total == |C| and counts == L's rows per group, at every k"""
    for pg in per_groups:
        want, wcounts = collapse(L, ids, pg, len(groups))
        for k in ks:
            k = len(want) if k == "total" else k
            got, total, counts = m.match_list_collapsed_array(corpus, groups, k, per_group=pg, subset=subset, boost=boost,
                                                              counts=True)
            ctx = what + (pg, k)
            assert total == len(want), (ctx, total, len(want))
            assert_same(got, want if k is None else want[:k], ctx)
            assert np.array_equal(counts, wcounts), ctx


@pytest.fixture(scope="module")
def small():
    hs = gen(3 * TILE + 77, 21)
    data, off = O.pack(hs)
    corpus = F.Corpus.from_arrow(data, off)
    yield corpus, data, off
    corpus.close()


@pytest.mark.parametrize("kind", list(MATCHERS))
def test_collapsed_every_matcher_and_strategy(small, kind):
    corpus, _, _ = small
    for name, ids, n_groups in shapes(len(corpus), 7):
        g = corpus.groups(ids, n_groups)
        for sort in SortStrategy:
            m = MATCHERS[kind](sort)
            L = uncollapsed(m, corpus)
            check_collapsed(m, corpus, g, ids, L, (kind, name, sort.name))
            m.close()
        g.close()


def test_collapsed_anchored_on_the_oracle(small):
    """L of the GPU equals the oracle's match_list, so the collapse of the oracle's list is the GPU's collapsed result."""
    corpus, data, off = small
    ids = np.random.default_rng(3).integers(0, 30, len(corpus)).astype(np.uint32)
    g = corpus.groups(ids)
    try:
        for pats, k, extra in ((["deadbeef"], 1, {}), (["foo"], 0, {"matching": Matching.Prefix}),
                               (F.parse_query("foo !^bar"), 1, {})):
            for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexDesc):
                want_L = O.match_list_packed(pats, cfg(sort, k, **extra), data, off)
                m = F.Matcher(pats, cfg(sort, k, **extra))
                assert_same(uncollapsed(m, corpus), want_L, ("oracle", sort.name))
                check_collapsed(m, corpus, g, ids, want_L, ("oracle", sort.name), per_groups=(1, 3), ks=(50, ALL))
                m.close()
    finally:
        g.close()


def test_collapsed_ranked_and_subsets(small):
    """Ranked (both key-sort paths: the key bound below 1024 and at or above it), the list form (at most 2 % of the rows)
    and the masked form of subsets, and both together."""
    corpus, _, _ = small
    n = len(corpus)
    rng = np.random.default_rng(11)
    ids = rng.integers(0, 25, n).astype(np.uint32)
    ids[rng.random(n) < 0.2] = GROUP_NONE
    g = corpus.groups(ids)
    subs = [corpus.subset(rng.choice(n, 40, replace=False)), corpus.subset(rng.choice(n, n // 2, replace=False))]
    short = F.Matcher("deadbeef", cfg(SortStrategy.ScoreThenIndexAsc, 1))
    assert short.score_bound() + 300 < 1024 <= short.score_bound() + 1000
    try:
        for hi in (300, 1000):
            host = rng.integers(-hi, hi + 1, n).astype(np.int16)
            host[0] = hi   # the bound is reached
            b = corpus.boost(host)
            for sort in SortStrategy:
                for m in (F.Matcher("deadbeef", cfg(sort, 1)), F.Matcher(LONG300, cfg(sort, 2)), F.Matcher.from_query("", cfg(sort))):
                    for sub in (None,) + tuple(subs):
                        for boost in (b, None):
                            if sub is None and boost is None:
                                continue
                            L = uncollapsed(m, corpus, sub, boost)
                            check_collapsed(m, corpus, g, ids, L, ("scoped", hi, sort.name, sub is not None, boost is not None),
                                            subset=sub, boost=boost, per_groups=(1, 3, ALL), ks=(0, 50, ALL))
                    m.close()
            b.close()
    finally:
        for s in subs:
            s.close()
        short.close()
        g.close()


def test_all_none_equals_the_existing_calls(small):
    """Every row in no group: the collapsed call is frz_match_list_top, _ranked or _subset_top exactly, counts all zero."""
    corpus, _, _ = small
    n = len(corpus)
    rng = np.random.default_rng(5)
    g = corpus.groups(np.full(n, GROUP_NONE, np.uint32), 4)
    b = corpus.boost(rng.integers(-300, 301, n).astype(np.int16))
    sub = corpus.subset(rng.choice(n, n // 3, replace=False))
    try:
        for kind in ("typos1", "multi", "empty", "long300"):
            for sort in SortStrategy:
                m = MATCHERS[kind](sort)
                for k in (0, 1, 50, n + 5):
                    for pg in (1, 32, ALL):
                        got, total, counts = m.match_list_collapsed_array(corpus, g, k, per_group=pg, counts=True)
                        top, ttotal = m.match_list_top_array(corpus, k)
                        assert total == ttotal and not counts.any()
                        assert_same(got, top, (kind, sort.name, k, pg, "top"))
                        got, total = m.match_list_collapsed_array(corpus, g, k, per_group=pg, boost=b)
                        want, wtotal = m.match_list_ranked_array(corpus, b, k)
                        assert total == wtotal
                        assert_same(got, want, (kind, sort.name, k, pg, "ranked"))
                        got, total = m.match_list_collapsed_array(corpus, g, k, per_group=pg, subset=sub)
                        want, wtotal = m.match_list_subset_top_array(corpus, sub, k)
                        assert total == wtotal
                        assert_same(got, want, (kind, sort.name, k, pg, "subset"))
                m.close()
    finally:
        sub.close()
        b.close()
        g.close()


def test_collapsed_across_edits():
    """Groups are kept by index: appended rows are in no group until set, a removed row stops matching, a replaced row
    keeps its group, and Groups.set between calls moves rows between groups."""
    corpus = F.Corpus.from_list(gen(2 * TILE + 500, 31))
    rng = np.random.default_rng(32)
    n0 = len(corpus)
    ids = rng.integers(0, 20, n0).astype(np.uint32)
    g = corpus.groups(ids, 30)
    b = corpus.boost(rng.integers(-300, 301, n0).astype(np.int16))
    ms = [F.Matcher("deadbeef", cfg(s, 1)) for s in SortStrategy] + [F.Matcher.from_query("", cfg(SortStrategy.IndexDesc))]

    def check(step, ids):
        for m in ms:
            check_collapsed(m, corpus, g, ids, uncollapsed(m, corpus), (step, m.config.sort.name), per_groups=(1, 2, ALL),
                            ks=(0, 5, ALL))
            check_collapsed(m, corpus, g, ids, uncollapsed(m, corpus, boost=b), (step, "ranked"), boost=b, per_groups=(1,),
                            ks=(5, ALL))

    try:
        check("created", ids)
        corpus.append_list([b"deadbeef", b"foo deadbeef", b"xyz"] * 300)
        check("appended", ids)                                    # the new rows are in no group
        new = np.arange(n0, len(corpus), dtype=np.uint32)
        newv = rng.integers(20, 30, len(new)).astype(np.uint32)
        g.set(new, newv)
        ids = np.concatenate([ids, newv])
        check("appended and set", ids)
        top = ms[0].match_list_collapsed_array(corpus, g, 3)[0]["index"]
        corpus.remove(top[:1])
        check("removed", ids)
        assert top[0] not in ms[0].match_list_collapsed_array(corpus, g)[0]["index"]
        corpus.replace_list(top[1:2], [b"deadbeef replaced"])
        check("replaced", ids)
        moved = rng.choice(len(corpus), 500, replace=False).astype(np.uint32)
        to = rng.integers(0, 3, len(moved)).astype(np.uint32)
        to[::7] = GROUP_NONE
        g.set(moved, to)
        ids[moved] = to
        check("set", ids)
    finally:
        for m in ms:
            m.close()
        b.close()
        g.close()
        corpus.close()


def test_collapsed_after_a_survivor_overflow():
    """100 000 rows that all match an exact literal: more survivors than the first call's lists hold (max(n / 4, 65536)),
    so the first collapsed call of a fresh matcher runs again with lists of n and still returns collapse(L)."""
    n = 100_000
    corpus = F.Corpus.from_list([b"abcd"] * n)
    rng = np.random.default_rng(4)
    ids = rng.integers(0, 1000, n).astype(np.uint32)
    g = corpus.groups(ids)
    ref = F.Matcher(F.Pattern("abcd", matching=Matching.Exact), Config(max_typos=0, sort=SortStrategy.ScoreThenIndexAsc))
    m = F.Matcher(F.Pattern("abcd", matching=Matching.Exact), Config(max_typos=0, sort=SortStrategy.ScoreThenIndexAsc))
    try:
        L = uncollapsed(ref, corpus)
        assert len(L) == n
        want, wcounts = collapse(L, ids, 2, len(g))
        got, total, counts = m.match_list_collapsed_array(corpus, g, 50, per_group=2, counts=True)
        first = m.last_timings()["launches"]
        assert total == len(want) and np.array_equal(counts, wcounts)
        assert_same(got, want[:50], "first")
        got, total = m.match_list_collapsed_array(corpus, g, 50, per_group=2)
        assert m.last_timings()["launches"] < first   # the first call ran twice
        assert_same(got, want[:50], "second")
    finally:
        ref.close()
        m.close()
        g.close()
        corpus.close()


def test_collapsed_at_a_million_rows():
    """About 1 M haystacks at max_typos=None (nearly every row matches): random groups, one group holding every row, and
    every row its own group, ranked in one sort pass and in two."""
    n = 1 << 20
    data, off = synth.generate("deadbeef", n, 48, 64, seed=77)
    corpus = F.Corpus.from_arrow(data, off)
    rng = np.random.default_rng(78)
    try:
        for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexDesc):
            m = F.Matcher("xyz", cfg(sort, None))
            for name, ids in (("random", rng.integers(0, 100_000, n).astype(np.uint32)), ("one", np.zeros(n, np.uint32)),
                              ("own", np.arange(n, dtype=np.uint32))):
                g = corpus.groups(ids)
                L = uncollapsed(m, corpus)
                assert len(L) > n // 2
                check_collapsed(m, corpus, g, ids, L, ("1M", sort.name, name), per_groups=(1, 32, ALL), ks=(50, ALL))
                for hi in (300, 1000):
                    b = corpus.boost(rng.integers(-hi, hi + 1, n).astype(np.int16))
                    check_collapsed(m, corpus, g, ids, uncollapsed(m, corpus, boost=b), ("1M", sort.name, name, hi), boost=b,
                                    per_groups=(3,), ks=(50, ALL))
                    b.close()
                g.close()
            m.close()
    finally:
        corpus.close()


def test_collapsed_refusals():
    """Each refused call leaves the groups as they were: the collapsed list afterwards is the same."""
    L = F.lib()
    a = F.Corpus.from_list([b"deadbeef", b"x", b"deadbeefs", b"dead beef"])
    other = F.Corpus.from_list([b"deadbeef", b"x", b"deadbeefs", b"dead beef"])
    m = F.Matcher("deadbeef", Config(max_typos=1, sort=SortStrategy.ScoreThenIndexAsc))
    ga = a.groups(np.array([0, 0, 1, 0], np.uint32))
    go = other.groups()
    bo = other.boost()
    so = other.subset([0, 2])
    out = np.zeros(8, dtype=F.MATCH_DTYPE)
    n, total = C.c_uint64(), C.c_uint64()
    try:
        assert len(ga) == 2 and len(go) == 1
        before = m.match_list_collapsed_array(a, ga)[0].copy()
        assert sorted(before["index"].tolist()) == [0, 2]   # row 3 shares group 0 with row 0 and scores lower
        fn = L.frz_match_list_collapsed
        for s_, b_, g_ in ((None, None, go._h), (so._h, None, ga._h), (None, bo._h, ga._h)):
            assert fn(m._h, a._h, s_, b_, g_, 1, 8, out.ctypes.data, C.byref(n), C.byref(total), None) == INVALID_ARG
            assert b"another corpus" in L.frz_last_error()
        assert fn(m._h, a._h, None, None, ga._h, 33, 8, out.ctypes.data, C.byref(n), C.byref(total), None) == UNSUPPORTED
        assert fn(m._h, a._h, None, None, ga._h, 0, 8, out.ctypes.data, C.byref(n), C.byref(total), None) == INVALID_ARG
        for which, ids in (([1, 4], [1, 1]), ([3, 3], [1, 0]), ([1], [2])):   # index >= len, duplicate, id >= n_groups
            with pytest.raises(F.FrizbeeError) as e:
                ga.set(which, ids)
            assert e.value.status_name == "FRZ_ERR_INVALID_ARG"
        h = C.c_void_p()
        v = np.zeros(5, np.uint32)
        assert L.frz_groups_create(a._h, v.ctypes.data, 5, 1, C.byref(h)) == INVALID_ARG and not h.value   # n > len
        v = np.array([0, 3], np.uint32)
        assert L.frz_groups_create(a._h, v.ctypes.data, 2, 3, C.byref(h)) == INVALID_ARG and not h.value   # id >= n_groups
        assert_same(m.match_list_collapsed_array(a, ga)[0], before, "after refusals")
        ga.set([], [])
        assert_same(m.match_list_collapsed_array(a, ga)[0], before, "after an empty set")
        got, tot = m.match_list_collapsed_array(a, ga, 0)
        assert len(got) == 0 and tot == len(before)
        # a subset without members: no row, and the counts are zero-filled
        sa = a.subset(np.zeros(0, np.uint32))
        got, tot, counts = m.match_list_collapsed_array(a, ga, 8, subset=sa, counts=True)
        assert len(got) == 0 and tot == 0 and not counts.any()
        sa.close()
    finally:
        so.close()
        bo.close()
        go.close()
        ga.close()
        m.close()
        a.close()
        other.close()


def device_bytes():
    L = F.lib()
    L.frz_debug_device_bytes.restype = C.c_uint64
    L.frz_debug_device_bytes.argtypes = []
    return L.frz_debug_device_bytes()


def device_bytes_peak(reset):
    L = F.lib()
    L.frz_debug_device_bytes_peak.restype = C.c_uint64
    L.frz_debug_device_bytes_peak.argtypes = [C.c_int]
    return L.frz_debug_device_bytes_peak(reset)


def test_collapsed_memory():
    """A group handle holds device memory until closed; repeated collapsed calls hold no more than the first."""
    data, off = O.pack(gen(5 * TILE, 41))
    corpus = F.Corpus.from_arrow(data, off)
    base = device_bytes()
    rng = np.random.default_rng(42)
    g1 = corpus.groups(rng.integers(0, 100, len(corpus)).astype(np.uint32))
    g2 = corpus.groups(np.arange(len(corpus), dtype=np.uint32))
    assert device_bytes() >= base + 2 * 4 * len(corpus)
    m = F.Matcher("deadbeef", cfg(SortStrategy.ScoreThenIndexAsc, 1))
    b = corpus.boost(rng.integers(-3000, 3001, len(corpus)).astype(np.int16))
    for g in (g1, g2):
        m.match_list_collapsed_array(corpus, g, 10, counts=True)
        m.match_list_collapsed_array(corpus, g, 10, per_group=32, boost=b)
    held = device_bytes()
    device_bytes_peak(1)
    for _ in range(20):
        for g in (g1, g2):
            m.match_list_collapsed_array(corpus, g, 10, counts=True)
            m.match_list_collapsed_array(corpus, g, per_group=3)
            m.match_list_collapsed_array(corpus, g, 10, per_group=32, boost=b)
    assert device_bytes() == held
    assert device_bytes_peak(0) == held
    m.close()
    b.close()
    g1.close()
    g2.close()
    assert device_bytes() == base
    corpus.close()
