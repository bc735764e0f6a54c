"""Ranked calls on the GPU (frz_boost_create / frz_boost_set / frz_match_list_ranked).  The contract: the rows of
match_list_into (or of a subset's members), reversed for the *_DESC strategies, sorted stably by descending
clamp(score + boost[index], 0, 65535), truncated to the first k; the reported total is the full count.  Every check
compares with tests/ranking.py's rank_by_boost: against the oracle's index-ordered list on small corpora, against the
GPU's own match_list_into (pinned to the oracle by the parity tests) at about a million rows, for subsets, across corpus
edits, against match_list_top under an all-zero boost, after refused calls, and for the device memory the calls hold."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200 import synth
from frizbee_b200.types import Config, Matching, SortStrategy
from oracle import pyoracle as O
from ranking import keys, rank_by_boost

pytestmark = pytest.mark.gpu

INVALID_ARG = 1
TILE = 1024
LANES = 32          # the reference backend the oracle emulates
ALL = None          # k = None: the whole list
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


# name -> (matcher factory(sort), oracle (patterns, max_typos, extra config); None: the GPU's match_list_into)
MATCHERS = {
    "typos0": (lambda s: F.Matcher("deadbeef", cfg(s, 0)), (["deadbeef"], 0, {})),
    "typos1": (lambda s: F.Matcher("deadbeef", cfg(s, 1)), (["deadbeef"], 1, {})),
    "typosNone": (lambda s: F.Matcher("dbf", cfg(s, None)), (["dbf"], None, {})),
    "long300": (lambda s: F.Matcher(LONG300, cfg(s, 2)), ([LONG300], 2, {})),
    "unicode": (lambda s: F.Matcher("é다😀", cfg(s, 1)), None),   # the oracle does not restate the unicode-needle path
    "prefix": (lambda s: F.Matcher("foo", cfg(s, 0, matching=Matching.Prefix)), (["foo"], 0, {"matching": Matching.Prefix})),
    "substring": (lambda s: F.Matcher("bar", cfg(s, 0, matching=Matching.Substring)),
                  (["bar"], 0, {"matching": Matching.Substring})),
    "multi": (lambda s: F.Matcher.from_query("foo !^bar", cfg(s, 1)), (F.parse_query("foo !^bar"), 1, {})),
    "empty": (lambda s: F.Matcher.from_query("", cfg(s, 0)), None),
}


def reversed_(sort):
    return sort in (SortStrategy.IndexDesc, SortStrategy.ScoreThenIndexDesc)


def assert_same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for f in ("index", "score", "exact"):
        bad = np.nonzero(got[f] != want[f])[0]
        assert bad.size == 0, (what, f, bad[:5], got[bad[:5]], want[bad[:5]])


def check_ranked(m, corpus, boost, host_boost, rows, sort, what, subset=None, ks=(0, 1, 7, "total", "total+5", ALL)):
    """ranked(k) == rank_by_boost(rows)[:k] and total == len(rows) at every k."""
    want = rank_by_boost(rows, host_boost, reversed_(sort))
    for k in ks:
        k = len(want) if k == "total" else len(want) + 5 if k == "total+5" else k
        got, total = m.match_list_ranked_array(corpus, boost, k, subset=subset)
        assert total == len(want), (what, k, total, len(want))
        assert_same(got, want if k is None else want[:k], what + (k,))
    return want


def boosts(n, seed):
    """(name, host array, sparse (which, values) applied with Boost.set or None)"""
    rng = np.random.default_rng(seed)
    sparse_w = rng.choice(n, max(1, n // 50), replace=False).astype(np.uint32)
    sparse_v = rng.integers(-300, 301, len(sparse_w)).astype(np.int16)
    sparse = np.zeros(n, np.int16)
    sparse[sparse_w] = sparse_v
    return [("zero", np.zeros(0, np.int16), None),
            ("pm300", rng.integers(-300, 301, n).astype(np.int16), None),
            ("extremes", rng.choice(np.array([-32768, 32767, 0], np.int16), n), None),
            ("sparse_set", sparse, (sparse_w, sparse_v))]


def make_boost(corpus, host, sparse):
    if sparse is None:
        return corpus.boost(host)
    return corpus.boost().set(*sparse)


@pytest.fixture(scope="module")
def small():
    hs = gen(3 * TILE + 77, 21)
    data, off = O.pack(hs)
    corpus = F.Corpus.from_arrow(data, off)
    yield corpus, data, off
    corpus.close()


@pytest.mark.parametrize("kind", list(MATCHERS))
def test_ranked_against_the_oracle(small, kind):
    corpus, data, off = small
    make, orc = MATCHERS[kind]
    n = len(corpus)
    if kind == "empty":
        rows = np.zeros(n, dtype=F.MATCH_DTYPE)
        rows["index"] = np.arange(n)
    elif orc is None:
        m = make(SortStrategy.IndexAsc)
        rows = m.match_list_into_array(corpus).copy()
        m.close()
    else:
        pats, k, extra = orc
        rows = O.match_list_into_packed(pats, cfg(SortStrategy.IndexAsc, k, **extra), data, off)
    assert len(rows) > 0, kind
    for bname, host, sparse in boosts(n, 5):
        b = make_boost(corpus, host, sparse)
        for sort in SortStrategy:
            m = make(sort)
            check_ranked(m, corpus, b, host, rows, sort, (kind, bname, sort.name))
            m.close()
        b.close()


def test_both_sort_paths(small):
    """The key bound (score bound + the largest positive boost) picks one pass below 1024 and two at or above it: deadbeef
    with boosts of up to 300 takes one pass, and so does the empty matcher with boosts below 1024; the 300-byte needle's
    score bound alone is >= 1024, and boosts of up to 1000 lift deadbeef over it."""
    corpus, data, off = small
    n = len(corpus)
    rng = np.random.default_rng(9)
    short = F.Matcher("deadbeef", cfg(SortStrategy.ScoreThenIndexAsc, 1))
    long_ = F.Matcher(LONG300, cfg(SortStrategy.ScoreThenIndexDesc, 2))
    empty = F.Matcher.from_query("", cfg(SortStrategy.IndexAsc))
    assert short.score_bound() + 300 < 1024 <= short.score_bound() + 1000
    assert long_.score_bound() >= 1024
    try:
        for m, pats, k, hi in ((short, ["deadbeef"], 1, 300), (short, ["deadbeef"], 1, 1000), (long_, [LONG300], 2, 0),
                               (empty, None, 0, 1023), (empty, None, 0, 1024)):
            host = rng.integers(-hi, hi + 1, n).astype(np.int16)
            host[0] = hi   # the bound is reached
            if pats is None:
                rows = np.zeros(n, dtype=F.MATCH_DTYPE)
                rows["index"] = np.arange(n)
            else:
                rows = O.match_list_into_packed(pats, cfg(SortStrategy.IndexAsc, k), data, off)
            b = corpus.boost(host)
            check_ranked(m, corpus, b, host, rows, m.config.sort, ("paths", hi), ks=(0, 3, "total", ALL))
            b.close()
    finally:
        for m in (short, long_, empty):
            m.close()


def test_ranked_at_a_million_rows():
    """About 1 M haystacks at max_typos=None: nearly every row matches, so every histogram segment takes many trips, in
    one pass and in two."""
    n = 1 << 20
    data, off = synth.generate("deadbeef", n, 48, 64, seed=77)
    corpus = F.Corpus.from_arrow(data, off)
    rng = np.random.default_rng(78)
    try:
        for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexDesc):
            m = F.Matcher("xyz", cfg(sort, None))
            rows = m.match_list_into_array(corpus).copy()
            assert len(rows) > n // 2
            for hi in (300, 1000):
                host = rng.integers(-hi, hi + 1, n).astype(np.int16)
                b = corpus.boost(host)
                check_ranked(m, corpus, b, host, rows, sort, ("1M", sort.name, hi), ks=(1000, ALL))
                b.close()
            m.close()
    finally:
        corpus.close()


def test_ranked_subsets(small):
    """The list form (at most 2 % of the rows) and the masked form (dense): the reference restricted to the members."""
    corpus, data, off = small
    n = len(corpus)
    rng = np.random.default_rng(13)
    host = rng.integers(-300, 301, n).astype(np.int16)
    b = corpus.boost(host)
    rows = O.match_list_into_packed(["deadbeef"], cfg(SortStrategy.IndexAsc, 1), data, off)
    empty_rows = np.zeros(n, dtype=F.MATCH_DTYPE)
    empty_rows["index"] = np.arange(n)
    try:
        for which in (rng.choice(n, 40, replace=False), rng.choice(n, n // 2, replace=False)):
            which = which.astype(np.uint32)
            sub = corpus.subset(which)
            mask = np.zeros(n, bool)
            mask[which] = True
            for sort in SortStrategy:
                for m, r in ((F.Matcher("deadbeef", cfg(sort, 1)), rows), (F.Matcher.from_query("", cfg(sort)), empty_rows)):
                    mine = r[mask[r["index"].astype(np.int64)]]
                    check_ranked(m, corpus, b, host, mine, sort, ("subset", len(which), sort.name), subset=sub)
                    m.close()
            sub.close()
    finally:
        b.close()


def test_ranked_across_edits():
    """Boosts are kept by index: appended rows rank with boost 0 until set, a removed row disappears, a replaced row keeps
    its boost."""
    corpus = F.Corpus.from_list(gen(2 * TILE + 500, 31))
    rng = np.random.default_rng(32)
    n0 = len(corpus)
    host = rng.integers(-300, 301, n0).astype(np.int16)
    b = corpus.boost(host)
    ms = [F.Matcher("deadbeef", cfg(s, 1)) for s in SortStrategy] + [F.Matcher.from_query("", cfg(SortStrategy.IndexDesc))]

    def check(step, host):
        for m in ms:
            check_ranked(m, corpus, b, host, m.match_list_into_array(corpus).copy(), m.config.sort, (step,),
                         ks=(0, 5, "total", ALL))

    try:
        check("created", host)
        corpus.append_list([b"deadbeef", b"foo deadbeef", b"xyz"] * 300)
        check("appended", host)                                   # the new rows have boost 0
        new = np.arange(n0, len(corpus), dtype=np.uint32)
        newv = rng.integers(-300, 301, len(new)).astype(np.int16)
        b.set(new, newv)
        host = np.concatenate([host, newv])
        check("appended and set", host)
        top = ms[0].match_list_ranked_array(corpus, b, 3)[0]["index"]   # the best boosted rows
        corpus.remove(top[:1])
        check("removed", host)
        assert top[0] not in ms[0].match_list_ranked_array(corpus, b)[0]["index"]
        corpus.replace_list(top[1:2], [b"deadbeef replaced"])
        check("replaced", host)
        assert top[1] in ms[0].match_list_ranked_array(corpus, b)[0]["index"]
    finally:
        for m in ms:
            m.close()
        b.close()
        corpus.close()


def test_zero_boost_equals_top(small):
    """An all-zero boost under the by-score strategies is frz_match_list_top."""
    corpus, _, _ = small
    b = corpus.boost()
    try:
        for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.ScoreThenIndexDesc):
            for make in (lambda s: F.Matcher("deadbeef", cfg(s, 1)), lambda s: F.Matcher(LONG300, cfg(s, 2)),
                         lambda s: F.Matcher.from_query("foo !^bar", cfg(s, 1))):
                m = make(sort)
                full = m.match_list_array(corpus)
                for k in (0, 1, 7, len(full), len(full) + 5):
                    top, total = m.match_list_top_array(corpus, k)
                    got, gtotal = m.match_list_ranked_array(corpus, b, k)
                    assert gtotal == total
                    assert_same(got, top, (sort.name, k))
                m.close()
    finally:
        b.close()


def test_ranked_refusals():
    """Each refused call leaves the boost as it was: the ranked list afterwards is the same."""
    L = F.lib()
    a = F.Corpus.from_list([b"deadbeef", b"x", b"deadbeefs", b"dead beef"])
    other = F.Corpus.from_list([b"deadbeef", b"x", b"deadbeefs", b"dead beef"])
    m = F.Matcher("deadbeef", Config(max_typos=1, sort=SortStrategy.ScoreThenIndexAsc))
    ba = a.boost(np.array([5, 0, 400, -7], np.int16))
    bo = other.boost()
    so = other.subset([0, 2])
    out = np.zeros(8, dtype=F.MATCH_DTYPE)
    n, total = C.c_uint64(), C.c_uint64()
    try:
        before = m.match_list_ranked_array(a, ba)[0].copy()
        assert before["index"].tolist()[0] == 2
        assert L.frz_match_list_ranked(m._h, a._h, None, bo._h, 8, out.ctypes.data, C.byref(n), C.byref(total)) == INVALID_ARG
        assert b"another corpus" in L.frz_last_error()
        assert L.frz_match_list_ranked(m._h, a._h, so._h, ba._h, 8, out.ctypes.data, C.byref(n), C.byref(total)) == INVALID_ARG
        assert b"another corpus" in L.frz_last_error()
        for which, vals in (([1, 4], [100, 100]), ([3, 3], [100, 200])):   # index >= len (the first one is valid), duplicate
            with pytest.raises(F.FrizbeeError) as e:
                ba.set(which, vals)
            assert e.value.status_name == "FRZ_ERR_INVALID_ARG"
        w = np.array([1], np.uint32)
        assert L.frz_boost_set(ba._h, w.ctypes.data, None, 1) == INVALID_ARG
        h = C.c_void_p()
        v = np.zeros(5, np.int16)
        assert L.frz_boost_create(a._h, v.ctypes.data, 5, C.byref(h)) == INVALID_ARG and not h.value   # n > len
        assert L.frz_boost_create(a._h, None, 1, C.byref(h)) == INVALID_ARG and not h.value
        assert_same(m.match_list_ranked_array(a, ba)[0], before, "after refusals")
        ba.set([], [])   # n == 0: nothing happens
        assert_same(m.match_list_ranked_array(a, ba)[0], before, "after an empty set")
        # k = 0 counts; no capacity error with room for k rows
        got, tot = m.match_list_ranked_array(a, ba, 0)
        assert len(got) == 0 and tot == len(before)
    finally:
        so.close()
        bo.close()
        ba.close()
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


def test_ranked_memory():
    """A boost holds device memory until closed; repeated ranked calls (one pass and two) hold no more than the first."""
    data, off = O.pack(gen(5 * TILE, 41))
    corpus = F.Corpus.from_arrow(data, off)
    base = device_bytes()
    rng = np.random.default_rng(42)
    b1 = corpus.boost(rng.integers(-300, 301, len(corpus)).astype(np.int16))
    b2 = corpus.boost(rng.integers(-3000, 3001, len(corpus)).astype(np.int16))
    assert device_bytes() >= base + 2 * 2 * len(corpus)
    m = F.Matcher("deadbeef", cfg(SortStrategy.ScoreThenIndexAsc, 1))
    sub = corpus.subset(np.arange(0, len(corpus), 3))
    for b in (b1, b2):
        m.match_list_ranked_array(corpus, b, 10)
        m.match_list_ranked_array(corpus, b, 10, subset=sub)
    held = device_bytes()
    device_bytes_peak(1)
    for _ in range(20):
        for b in (b1, b2):
            m.match_list_ranked_array(corpus, b, 10)
            m.match_list_ranked_array(corpus, b)
            m.match_list_ranked_array(corpus, b, 10, subset=sub)
    assert device_bytes() == held
    assert device_bytes_peak(0) == held
    sub.close()
    m.close()
    b1.close()
    b2.close()
    assert device_bytes() == base
    corpus.close()
