"""Many subsets filled from attributes in one call on the GPU (frz_subset_where_batch, F.where_batch).  The contract: each
subset is bit for bit what frz_subset_where leaves for its own clauses and base.  Every batched fill is checked against
twin subsets refilled by a loop of Subset.where: equal len() (and equal to a numpy restatement of the clauses), equal
members as the empty matcher lists them, and one match_list_batch over the filled subsets that takes the batched match
kernels.  Covered: corpus lengths around word and chunk boundaries up to 1 M + 7 rows, 1 to 300 queries of 0-8 range,
set and negated clauses, nulls and attributes shorter than the corpus, bases (none, the query's own subset, a shared
subset, one made before an append), bitmaps that must grow, more distinct attributes than are staged, corpus edits,
device memory on refills, and refused calls.  Needs a CUDA device."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200.types import Config, SortStrategy
from test_gpu_where import BATCH_NEEDLES, NULL, attr_values, full, new_corpus, random_clauses, spec

pytestmark = pytest.mark.gpu

EMPTY = F.Matcher.from_query("", Config(sort=SortStrategy.IndexAsc))
STAGED = 4   # kFrzWhereBatchStaged


@pytest.fixture(autouse=True)
def batched_kernels():
    """Every test here runs the batched kernels at every q, unless it restores the rule itself."""
    F.where_batch_debug(True)
    yield
    F.where_batch_debug(False)


def members(corpus, s):
    return EMPTY.match_list_subset_array(corpus, s)["index"].copy()


def check(corpus, got, twins, masks, what):
    """got[j] (batched) and twins[j] (looped) agree, and both hold masks[j]'s rows."""
    assert len(got) == len(twins) == len(masks)
    for j, (g, t, m) in enumerate(zip(got, twins, masks)):
        assert len(g) == len(t) == int(m.sum()), (what, j, len(g), len(t), int(m.sum()))
        assert np.array_equal(members(corpus, g), members(corpus, t)), (what, j)
    n = len(corpus)
    if 31 <= n <= 100_000 and got:
        ms = [F.Matcher(BATCH_NEEDLES[j % len(BATCH_NEEDLES)], Config(max_typos=0, sort=SortStrategy(j % 4))) for j in range(40)]
        a = F.match_list_batch(ms, corpus, 10, subsets=[got[j % len(got)] for j in range(40)])
        assert F.batch_last()["sub_batches"] > 0, what
        b = F.match_list_batch(ms, corpus, 10, subsets=[twins[j % len(twins)] for j in range(40)])
        for x, y in zip(a, b):
            assert np.array_equal(x, y), what


def fill_both(corpus, got, twins, clauses, bases_got, bases_twin):
    F.where_batch(got, clauses, bases_got)
    for t, cl, b in zip(twins, clauses, bases_twin):
        t.where(*cl, base=b)


@pytest.mark.parametrize("q", [1, 2, 7, 64, 300])
@pytest.mark.parametrize("n", [0, 1, 31, 32, 1023, 1024, 1025, 100_000, 1_000_007])
def test_batch_equals_loop(n, q):
    rng = np.random.default_rng(n * 1000 + q)
    corpus = new_corpus(n, n + 1)
    vals = attr_values(n, rng)                    # the second attribute is shorter than the corpus
    attrs = [corpus.attr(v) for v in vals]
    cl0, m0 = random_clauses(attrs, vals, n, rng, 1)
    shared = corpus.where(*cl0)                   # a base several queries share
    got = [corpus.subset([]) for _ in range(q)]   # empty bitmaps: the first fill grows them
    twins = [corpus.subset([]) for _ in range(q)]
    try:
        prev = [np.zeros(n, bool)] * q
        for rnd in range(3):
            clauses, masks, bg, bt = [], [], [], []
            for j in range(q):
                k = None if j % 5 else (0 if j % 10 == 0 else 8)   # 0-8 clauses, both ends pinned
                cl, mask = random_clauses(attrs, vals, n, rng, k, "sparse" if j % 7 == 3 else None)
                kind = (j + rnd) % 3 if rnd else (j % 2) * 2   # round 0: none or shared; then the own subset too
                if kind == 1:
                    bg.append(got[j]), bt.append(twins[j])
                    mask &= prev[j]
                elif kind == 2:
                    bg.append(shared), bt.append(shared)
                    mask &= m0
                else:
                    bg.append(None), bt.append(None)
                clauses.append(cl)
                masks.append(mask)
            fill_both(corpus, got, twins, clauses, bg if any(x is not None for x in bg) else None, bt)
            assert F.where_batch_debug()   # the batched kernels ran
            check(corpus, got, twins, masks, (n, q, rnd))
            prev = masks
    finally:
        for h in got + twins + [shared] + attrs:
            h.close()
        corpus.close()


def test_more_attributes_than_staged():
    for n in (5000, 100_000):
        rng = np.random.default_rng(n)
        corpus = new_corpus(n, 2)
        vals = attr_values(n, rng) + attr_values(n, rng) + attr_values(n, rng)[:1]   # 7 distinct attributes
        attrs = [corpus.attr(v) for v in vals]
        cols = [full(v, n) for v in vals]
        q = 40
        got = [corpus.subset([]) for _ in range(q)]
        twins = [corpus.subset([]) for _ in range(q)]
        clauses, masks = [], []
        for j in range(q):
            cl, mask = [], np.ones(n, bool)
            for c in range(int(rng.integers(0, 9))):
                a = int(rng.integers(0, len(attrs))) if j % 3 else len(attrs) - 1 - c % 3   # unstaged ones first, often
                real = cols[a][cols[a] != NULL]
                x, y = sorted(int(v) for v in rng.choice(real, 2))
                w = attrs[a].between(x, y) if c % 2 else attrs[a].isin(rng.choice(real, 5))
                w = ~w if rng.random() < 0.25 else w
                cl.append(w)
                mask &= spec(cols[a], w.lo, w.hi, w.values, w.negate)
            clauses.append(cl)
            masks.append(mask)
        assert len({id(w.attr) for cl in clauses for w in cl}) > STAGED
        fill_both(corpus, got, twins, clauses, None, [None] * q)
        check(corpus, got, twins, masks, (n, "attrs"))
        for h in got + twins + attrs:
            h.close()
        corpus.close()


def test_edits_short_attributes_and_bases():
    n = 5000
    corpus = new_corpus(n, 3)
    rng = np.random.default_rng(3)
    v = rng.integers(0, 10, n).astype(np.int64)
    a = corpus.attr(v)
    b = corpus.attr(rng.integers(0, 3, n // 2).astype(np.int64))   # shorter than the corpus
    old = corpus.where(a.between(0, 4))                              # a base made before the append
    q = 12
    got = [corpus.subset([]) for _ in range(q)]
    twins = [corpus.subset([]) for _ in range(q)]
    corpus.remove(rng.choice(n, 300, replace=False))
    corpus.replace_list(rng.choice(n, 200, replace=False), [b"deadbeef dbf foo"] * 200)
    corpus.append_list([b"dbf appended"] * 1500)
    m = n + 1500
    va, vb = full(v, m), full(b.values()[: n // 2], m)
    ob = np.zeros(m, bool)
    ob[:n] = spec(full(v, n), 0, 4)

    def round_(bases_kind):
        clauses, masks, bg, bt = [], [], [], []
        for j in range(q):
            lo = int(rng.integers(0, 8))
            cl = [a.between(lo, lo + 2)] + ([b.isin([j % 3])] if j % 2 else []) + ([~a.isin([lo + 1])] if j % 4 == 3 else [])
            mask = spec(va, lo, lo + 2) & (spec(vb, in_=[j % 3]) if j % 2 else True) & (spec(va, in_=[lo + 1], negate=True) if j % 4 == 3 else True)
            kind = bases_kind(j)
            if kind == "old":
                bg.append(old), bt.append(old)
                mask = mask & ob[: len(mask)]
            elif kind == "own":
                bg.append(got[j]), bt.append(twins[j])
                mask = mask & prev[j]
            else:
                bg.append(None), bt.append(None)
            clauses.append(cl)
            masks.append(mask)
        fill_both(corpus, got, twins, clauses, bg, bt)
        check(corpus, got, twins, masks, "edits")
        return masks

    prev = round_(lambda j: "old" if j % 3 == 0 else None)
    prev = round_(lambda j: ["old", "own", None][j % 3])
    corpus.append_list([b"foo"] * 40)            # every bitmap must grow while some are their own base
    m += 40
    va, vb, ob = full(va, m), full(vb, m), np.concatenate([ob, np.zeros(40, bool)])
    prev = [np.concatenate([p, np.zeros(40, bool)]) for p in prev]
    prev = round_(lambda j: "own" if j % 2 else "old")
    for h in got + twins + [old, a, b]:
        h.close()
    corpus.close()


def _lib():
    L = F.lib()
    L.frz_debug_device_bytes_peak.restype = C.c_uint64
    L.frz_debug_device_bytes_peak.argtypes = [C.c_int]
    return L


def test_refill_allocates_nothing():
    n = 300_000
    corpus = new_corpus(n, 4)
    rng = np.random.default_rng(4)
    vals = attr_values(n, rng)
    attrs = [corpus.attr(v) for v in vals]
    q = 64
    subsets = [corpus.subset([]) for _ in range(q)]
    clauses = [random_clauses(attrs, vals, n, rng, int(rng.integers(0, 9)))[0] for _ in range(q)]
    F.where_batch(subsets, clauses, [s if j % 2 else None for j, s in enumerate(subsets)])
    L = _lib()
    L.frz_debug_device_bytes_peak(1)
    F.where_batch(subsets, clauses, None)
    lens = [len(s) for s in subsets]
    peak = L.frz_debug_device_bytes_peak(0)
    F.where_batch(subsets, clauses, None)
    assert L.frz_debug_device_bytes_peak(0) == peak   # a second identical call allocates nothing
    assert [len(s) for s in subsets] == lens
    for h in subsets + attrs:
        h.close()
    corpus.close()


def test_refused_calls_leave_every_subset():
    c1, c2 = new_corpus(3000, 5), new_corpus(100, 6)
    a1, a2 = c1.attr(np.arange(3000)), c2.attr(np.arange(100))
    s = [c1.subset([1, 2, 3]), c1.subset([7]), c1.subset(np.arange(2000))]
    other = c2.subset([4])
    before = [members(c1, x) for x in s]
    refusals = [
        (lambda: F.where_batch(s, [[a1.between(0, 9)], [a2.between(0, 9)], []]), "query 1: the attribute was made on another corpus"),
        (lambda: F.where_batch(s + [other], [[], [], [], []]), "query 3: the subset was made on another corpus"),
        (lambda: F.where_batch(s, [[], [], []], [None, None, other]), "query 2: the base subset was made on another corpus"),
        (lambda: F.where_batch([s[0], s[1], s[0]], [[], [], []]), "query 2: the subset is also query 0's"),
        (lambda: F.where_batch(s, [[], [], []], [s[1], None, None]), "query 0: the base is query 1's subset"),
        (lambda: F.where_batch(s, [[], [a1.between(0, 9)] * 9, []]), "query 1: 9 clauses"),
        (lambda: F.where_batch(s, [[a1.isin(np.arange(4097))], [], []]), "query 0: more than 4096 set values"),
        (lambda: F.where_batch(s, [[], [], [a1.isin([1, NULL])]]), "query 2: set value 1 of clause 0 is FRZ_ATTR_NULL"),
    ]
    for call, msg in refusals:
        with pytest.raises(F.FrizbeeError, match=msg):
            call()
        for x, want in zip(s, before):   # a refused call leaves every subset as it was
            assert np.array_equal(members(c1, x), want), msg
    assert [len(x) for x in s] == [3, 1, 2000]
    with pytest.raises(ValueError):
        F.where_batch(s, [[], []])
    assert F.where_batch([], []) == []
    # the per-query limits hold per query: 8 clauses and 4096 set values each
    F.where_batch(s, [[a1.between(0, 2999)] * 8, [a1.isin(np.arange(4096))], [a1.isin(np.arange(4096) + 10)]], [None, None, s[2]])
    assert [len(x) for x in s] == [3000, 3000, 1990]
    for h in s + [other, a1, a2, c1, c2]:
        h.close()


def test_small_batch_rule():
    """One query, and two over more than 2^22 rows, run the single fill; the others the batched kernels.  Either way each
    subset is what its own Subset.where leaves."""
    F.where_batch_debug(False)
    for n in (1024, (1 << 22) + 5):
        rng = np.random.default_rng(n)
        corpus = new_corpus(n, 8)
        vals = attr_values(n, rng)
        attrs = [corpus.attr(v) for v in vals]
        for q, want in ((1, False), (2, n <= 1 << 22), (3, True)):
            got = [corpus.subset([]) for _ in range(q)]
            twins = [corpus.subset([]) for _ in range(q)]
            clauses, masks = zip(*[random_clauses(attrs, vals, n, rng, 2) for _ in range(q)])
            fill_both(corpus, got, twins, clauses, None, [None] * q)
            assert F.where_batch_debug() == want, (n, q)
            check(corpus, got, twins, masks, (n, q, "rule"))
            for h in got + twins:
                h.close()
        for a in attrs:
            a.close()
        corpus.close()
