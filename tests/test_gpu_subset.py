"""Subset match calls on the GPU (frz_subset_create, frz_match_list_subset, frz_match_list_subset_top).  The contract:
match_list_subset(m, c, s) is the full match_list(m, c) with the rows of non-members dropped, in the same order, and the
top-K call returns that list's first min(K, total) rows with total = its length.  Checked against the full call filtered
in numpy for every matcher kind and sort strategy, on subsets from empty to the whole list (random, contiguous, unsorted
with duplicates, in the partial last tile); on small lists also against the oracle over the members' haystacks; after
appends, removals and replacements; for refused calls; and for the device memory the calls hold."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200.types import Config, Matching, SortStrategy
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

INVALID_ARG, CAPACITY = 1, 6
TILE = 1024
LANES = 32          # the reference backend the oracle emulates
N_BIG = 70 * TILE + 333   # >= 64 tiles, with a partial last tile


def needle(n, seed):
    rng = np.random.default_rng(seed)
    return rng.choice(np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", dtype=np.uint8), n).tobytes().decode()


LONGS = {n: needle(n, n) for n in (65, 300, 1024)}
TYPO_NEEDLE = "deadbeefcafe0123"     # 16 bytes: max_typos 5 and 15 stay below the needle length


def gen(n, seed):
    """Short random rows; some hold `deadbeef`-like text, `foo`/`bar` prefixes, unicode scalars or a long needle with
    a typo or two."""
    rng = np.random.default_rng(seed)
    pool = np.frombuffer(b"abcdef0123_-/ deadbeefoFOBAR", dtype=np.uint8)
    out = []
    for _ in range(n):
        h = bytearray(rng.choice(pool, int(rng.integers(0, 40))).tobytes())
        r = rng.random()
        if r < 0.10:
            t = bytearray(TYPO_NEEDLE.encode())
            for _ in range(int(rng.integers(0, 6))):
                t[int(rng.integers(0, len(t)))] = ord("x")
            h[int(rng.integers(0, len(h) + 1)):0] = t
        elif r < 0.16:
            h = bytearray(rng.choice([b"foo", b"bar", b"foobar", b"barfoo"])) + h
        elif r < 0.20:
            h += "é다x😀".encode()
        elif r < 0.23:
            ln = bytearray(LONGS[int(rng.choice([65, 300, 1024]))].encode())
            for _ in range(int(rng.integers(0, 3))):
                ln[int(rng.integers(0, len(ln)))] = ord("q")
            h += ln
        out.append(bytes(h))
    return out


def cfg(sort, max_typos=0, **kw):
    return Config(max_typos=max_typos, sort=sort, emulate_lanes=LANES, **kw)


# name -> (matcher factory(sort), oracle (patterns, max_typos, extra config) or None)
MATCHERS = {
    "typos0": (lambda s: F.Matcher("deadbeef", cfg(s, 0)), lambda: (["deadbeef"], 0, {})),
    "typos1": (lambda s: F.Matcher("deadbeef", cfg(s, 1)), lambda: (["deadbeef"], 1, {})),
    "typos2": (lambda s: F.Matcher("deadbeef", cfg(s, 2)), lambda: (["deadbeef"], 2, {})),
    "typos5": (lambda s: F.Matcher(TYPO_NEEDLE, cfg(s, 5)), lambda: ([TYPO_NEEDLE], 5, {})),
    "typos15": (lambda s: F.Matcher(TYPO_NEEDLE, cfg(s, 15)), lambda: ([TYPO_NEEDLE], 15, {})),
    "typosNone": (lambda s: F.Matcher("dbf", cfg(s, None)), lambda: (["dbf"], None, {})),
    "long65": (lambda s: F.Matcher(LONGS[65], cfg(s, 2)), lambda: ([LONGS[65]], 2, {})),
    "long300": (lambda s: F.Matcher(LONGS[300], cfg(s, 2)), lambda: ([LONGS[300]], 2, {})),
    "long1024": (lambda s: F.Matcher(LONGS[1024], cfg(s, 2)), lambda: ([LONGS[1024]], 2, {})),
    "unicode": (lambda s: F.Matcher("é다😀", cfg(s, 1)), None),   # the oracle does not restate the unicode-needle path
    "exact": (lambda s: F.Matcher("foobar", cfg(s, 0, matching=Matching.Exact)), lambda: (["foobar"], 0, {"matching": Matching.Exact})),
    "prefix": (lambda s: F.Matcher("foo", cfg(s, 0, matching=Matching.Prefix)), lambda: (["foo"], 0, {"matching": Matching.Prefix})),
    "suffix": (lambda s: F.Matcher("foo", cfg(s, 0, matching=Matching.Suffix)), lambda: (["foo"], 0, {"matching": Matching.Suffix})),
    "substring": (lambda s: F.Matcher("bar", cfg(s, 0, matching=Matching.Substring)),
                  lambda: (["bar"], 0, {"matching": Matching.Substring})),
    "multi": (lambda s: F.Matcher.from_query("foo !^bar", cfg(s, 1)), lambda: (F.parse_query("foo !^bar"), 1, {})),
    "all_negated": (lambda s: F.Matcher.from_query("!foo !dead", cfg(s, 0)), lambda: (F.parse_query("!foo !dead"), 0, {})),
    "empty": (lambda s: F.Matcher.from_query("", cfg(s, 0)), None),
}


def subsets(n, seed):
    """(name, index array) pairs: sizes 0, 1, 100, then 1 %, 50 % and 100 % random and contiguous, unsorted with
    duplicates, and the partial last tile.  Both forms of a subset call are taken: the list form up to 2 % of the list
    (FRZ_SUBSET_LIST_PERMILLE), the masked form above."""
    rng = np.random.default_rng(seed)
    last0 = (n // TILE) * TILE
    out = [("empty", np.zeros(0, np.uint32)), ("one", np.array([n // 2], np.uint32)),
           ("hundred", rng.choice(n, 100, replace=False))]
    for pct in (1, 50, 100):
        k = max(1, n * pct // 100)
        out.append((f"random{pct}", rng.choice(n, k, replace=False)))
        start = int(rng.integers(0, n - k + 1))
        out.append((f"contiguous{pct}", np.arange(start, start + k)))
    dup = rng.integers(0, n, 3000)
    out.append(("unsorted_dups", np.concatenate([dup, dup[::-1][:1500]])))
    out.append(("last_tile", np.arange(last0, n)[::-1]))
    return [(name, np.asarray(w, dtype=np.uint32)) for name, w in out]


def member_mask(n, which):
    mask = np.zeros(n, dtype=bool)
    mask[which.astype(np.int64)] = True
    return mask


def assert_same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for f in ("index", "score", "exact"):
        bad = np.nonzero(got[f] != want[f])[0]
        assert bad.size == 0, (what, f, bad[:5], got[bad[:5]], want[bad[:5]])


def check_subset(m, corpus, sub, mask, full, what):
    """match_list_subset == full filtered to the members; top-K at 0, 1, 5, total and total + 3."""
    want = full[mask[full["index"].astype(np.int64)]] if len(full) else full
    got = m.match_list_subset_array(corpus, sub)
    assert_same(got, want, what)
    for k in sorted({0, 1, 5, len(want), len(want) + 3}):
        top, total = m.match_list_subset_top_array(corpus, sub, k)
        assert total == len(want), what + ("top", k, total, len(want))
        assert_same(top, want[:k], what + ("top", k))
    return want


@pytest.fixture(scope="module")
def big():
    data, off = O.pack(gen(N_BIG, 7))
    corpus = F.Corpus.from_arrow(data, off)
    subs = [(name, w, corpus.subset(w)) for name, w in subsets(N_BIG, 8)]
    yield corpus, subs
    for *_, s in subs:
        s.close()
    corpus.close()


@pytest.mark.parametrize("kind", list(MATCHERS))
def test_subset_equals_filtered_full_list(big, kind):
    corpus, subs = big
    make, _ = MATCHERS[kind]
    for sort in SortStrategy:
        m = make(sort)
        full = m.match_list_array(corpus).copy()
        assert len(full) > 0, (kind, sort)
        for name, w, sub in subs:
            mask = member_mask(N_BIG, w)
            assert len(sub) == int(mask.sum())
            want = check_subset(m, corpus, sub, mask, full, (kind, sort.name, name))
            if kind == "empty":   # the live members in index order, reversed for the *_DESC strategies
                idx = np.nonzero(mask)[0]
                if sort in (SortStrategy.IndexDesc, SortStrategy.ScoreThenIndexDesc):
                    idx = idx[::-1]
                assert want["index"].tolist() == idx.tolist()
        m.close()


@pytest.mark.parametrize("kind", [k for k, (_, orc) in MATCHERS.items() if orc is not None])
def test_subset_against_the_oracle(kind):
    """On a small list: the subset call equals the oracle's match_list over the members' haystacks, indices mapped back."""
    hs = gen(3 * TILE + 77, 21)
    data, off = O.pack(hs)
    corpus = F.Corpus.from_arrow(data, off)
    make, orc = MATCHERS[kind]
    pats, k, extra = orc()
    rng = np.random.default_rng(22)
    try:
        # the masked form (900 random rows, the last tiles) and the list form (25 rows: under 2 % of the list)
        for which in (rng.choice(len(hs), 900, replace=False), np.arange(2 * TILE, len(hs)), rng.integers(0, len(hs), 25)):
            which = which.astype(np.uint32)
            members = np.unique(which)
            sub = corpus.subset(which)
            sd, so = O.pack([hs[i] for i in members])
            for sort in SortStrategy:
                m = make(sort)
                want = O.match_list_packed(pats, cfg(sort, k, **extra), sd, so)
                want["index"] = members[want["index"].astype(np.int64)]
                assert_same(m.match_list_subset_array(corpus, sub), want, (kind, sort.name, len(which)))
                m.close()
            sub.close()
    finally:
        corpus.close()


def test_subset_across_edits():
    """Membership is by index: appended rows are not members, a removed member stops matching, a replaced member stays a
    member with its new text."""
    hs = gen(2 * TILE + 500, 31)
    data, off = O.pack(hs)
    corpus = F.Corpus.from_arrow(data, off)
    rng = np.random.default_rng(32)
    which = rng.choice(len(hs), 800, replace=False).astype(np.uint32)
    few = which[90:110]   # under 2 % of the list: the list form; some of these rows are removed, some replaced below
    scopes = [(which, corpus.subset(which)), (few, corpus.subset(few))]
    n0 = len(hs)
    ms = [F.Matcher("deadbeef", cfg(s, 1)) for s in SortStrategy] + [F.Matcher.from_query("!foo", cfg(SortStrategy.IndexDesc)),
                                                                    F.Matcher.from_query("", cfg(SortStrategy.IndexAsc))]

    def check(step):
        for w, sub in scopes:
            mask = member_mask(len(corpus), w)
            for m in ms:
                full = m.match_list_array(corpus).copy()
                got = check_subset(m, corpus, sub, mask, full, (step, len(w)))
                assert np.all(got["index"] < n0)

    try:
        check("created")
        corpus.append_list([b"deadbeef" * 2, b"foo deadbeef", b"xyz"] * 400)   # none of them is a member
        check("appended")
        rem = np.concatenate([which[:100], np.setdiff1d(np.arange(n0), which)[:100]]).astype(np.uint32)
        corpus.remove(rem)
        check("removed")
        rep = np.concatenate([which[50:250], np.setdiff1d(np.arange(n0), which)[200:300], [n0 + 5]]).astype(np.uint32)
        corpus.replace_list(rep, [b"deadbeef new text"] * len(rep))
        check("replaced")
        for w, sub in scopes:   # replaced members (some had been removed) match
            got = ms[2].match_list_subset_array(corpus, sub)   # IndexAsc
            assert set(np.intersect1d(w, which[50:250]).tolist()) <= set(got["index"].tolist())
    finally:
        for m in ms:
            m.close()
        for _, sub in scopes:
            sub.close()
        corpus.close()


def test_subset_refusals():
    L = F.lib()
    a = F.Corpus.from_list([b"deadbeef", b"x", b"deadbeefs"])
    b = F.Corpus.from_list([b"deadbeef", b"x", b"deadbeefs"])
    m = F.Matcher("deadbeef", Config(sort=SortStrategy.IndexAsc))
    sa = a.subset([0, 2])
    out = np.zeros(8, dtype=F.MATCH_DTYPE)
    n, total = C.c_uint64(), C.c_uint64()
    try:
        assert L.frz_match_list_subset(m._h, b._h, sa._h, out.ctypes.data, 8, C.byref(n)) == INVALID_ARG
        assert b"another corpus" in L.frz_last_error()
        assert L.frz_match_list_subset_top(m._h, b._h, sa._h, 2, out.ctypes.data, C.byref(n), C.byref(total)) == INVALID_ARG
        h = C.c_void_p()
        bad = np.array([0, 3], dtype=np.uint32)
        assert L.frz_subset_create(a._h, bad.ctypes.data, 2, C.byref(h)) == INVALID_ARG and not h.value
        assert b"out of range" in L.frz_last_error()
        assert L.frz_subset_create(a._h, None, 1, C.byref(h)) == INVALID_ARG and not h.value
        with pytest.raises(F.FrizbeeError):
            a.subset([1 << 20])
        # the same calls on the right corpus work; a capacity error reports the needed count
        assert m.match_list_subset_array(a, sa)["index"].tolist() == [0, 2]
        assert L.frz_match_list_subset(m._h, a._h, sa._h, out.ctypes.data, 1, C.byref(n)) == CAPACITY and n.value == 2
    finally:
        sa.close()
        m.close()
        a.close()
        b.close()


def device_bytes():
    L = F.lib()
    L.frz_debug_device_bytes.restype = C.c_uint64
    L.frz_debug_device_bytes.argtypes = []
    return L.frz_debug_device_bytes()


def test_subset_memory():
    """The calls' scratch lives in the matcher: flat over repeated calls, and everything is given back by destroy."""
    data, off = O.pack(gen(5 * TILE, 41))
    corpus = F.Corpus.from_arrow(data, off)
    base = device_bytes()
    m = F.Matcher.from_query("deadbeef !foo", cfg(SortStrategy.ScoreThenIndexAsc, 1))
    subs = [corpus.subset(np.arange(0, 5 * TILE, 3)), corpus.subset(np.arange(7, 5 * TILE, 997))]   # masked form, list form
    for _ in range(2):
        for sub in subs:
            m.match_list_subset_array(corpus, sub)
            m.match_list_subset_top_array(corpus, sub, 10)
    held = device_bytes()
    for _ in range(20):
        for sub in subs:
            m.match_list_subset_array(corpus, sub)
            m.match_list_subset_top_array(corpus, sub, 10)
    assert device_bytes() == held
    for sub in subs:
        sub.close()
    m.close()
    assert device_bytes() == base
    corpus.close()
