"""frz_attr_rank on the GPU.  The contract: a ranked row (live in the attribute's corpus and in every text key's corpus)
gets the dense rank of its key tuple among the ranked rows, every other row FRZ_ATTR_NULL.  Every check compares with a
numpy restatement (each text key mapped to the rank of its bytes under Python's sorted(), then np.lexsort over the key
tuples), and then orders match lists by the rank with frz_match_list_ordered against tests/ordering.py's order_by_attr,
ATTR_ASC and SCORE_THEN_ATTR_ASC under every sort strategy."""
import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200.types import Config, Order, SortStrategy
from ordering import ATTR_NULL, order_by_attr
from test_gpu_memory import check_cycle

pytestmark = pytest.mark.gpu

I64_MAX = 2**63 - 1
FOLD = bytes(range(65)) + bytes(range(97, 123)) + bytes(range(91, 256))   # A-Z as a-z
ALPHABET = np.frombuffer(b"abAB/._zZ\0\x80\xff\xc3\xa9", np.uint8)


def texts_of(rng, n, max_len=24, alphabet=ALPHABET):
    """Random byte strings with NULs, bytes >= 0x80, case pairs, and proper prefixes / extensions of earlier ones."""
    out = []
    for _ in range(n):
        if out and rng.random() < 0.4:
            t = out[int(rng.integers(len(out)))]
            t = t[: int(rng.integers(0, len(t) + 1))] if rng.random() < 0.5 else t + rng.choice(alphabet, int(rng.integers(1, 4))).tobytes()
        else:
            t = rng.choice(alphabet, int(rng.integers(0, max_len + 1))).tobytes()
        out.append(t)
    return out


def int_keys(key):
    """np.lexsort columns of one key, most significant first.  ("text", texts, desc, fold) or ("attr", values, desc)."""
    if key[0] == "text":
        t = [x.translate(FOLD) if key[3] else x for x in key[1]]
        where = {x: i for i, x in enumerate(sorted(set(t)))}
        r = np.array([where[x] for x in t], np.int64)
        return [-r if key[2] else r]
    v = np.asarray(key[1], np.int64)
    null = v == ATTR_NULL
    return [null.astype(np.int64), np.where(null, 0, -v if key[2] else v)]


def spec(n, keys, ranked):
    """The dense rank of each ranked row's tuple; ATTR_NULL elsewhere."""
    cols = [c for k in keys for c in int_keys(k)]
    rows = np.flatnonzero(ranked)
    out = np.full(n, ATTR_NULL, np.int64)
    if rows.size == 0:
        return out
    tup = np.stack([c[rows] for c in cols])
    perm = np.lexsort(tup[::-1])
    s = tup[:, perm]
    new = np.ones(len(rows), bool)
    new[1:] = (s[:, 1:] != s[:, :-1]).any(axis=0)
    out[rows[perm]] = np.cumsum(new) - 1
    return out


def live(n, removed=()):
    m = np.ones(n, bool)
    m[list(removed)] = False
    return m


def check_ordered(corpus, attr, values, needles=("", "ab")):
    """Ordered calls on the rank against order_by_attr: ATTR_ASC and SCORE_THEN_ATTR_ASC, every strategy, whole and k = 50."""
    for needle in needles:
        for sort in SortStrategy:
            m = F.Matcher.from_query(needle, Config(max_typos=0, sort=sort)) if needle == "" else F.Matcher(needle, Config(max_typos=1, sort=sort))
            try:
                into = m.match_list_into_array(corpus).copy()
                for order in (Order.AttrAsc, Order.ScoreThenAttrAsc):
                    want = order_by_attr(into, values, int(order), SortStrategy(sort).is_reversed())
                    for k in (None, 50):
                        got, total = m.match_list_ordered_array(corpus, attr, order, k)
                        assert total == len(want)
                        w = want if k is None else want[:k]
                        assert np.array_equal(got["index"], w["index"]), (needle, sort, order, k)
                        assert np.array_equal(got["score"], w["score"]), (needle, sort, order, k)
            finally:
                m.close()


def device_values(attr, n):
    got = attr.values()
    assert len(got) == n
    return got


def expect_rank(corpus, attr, keys, ranked, ctx=()):
    want = spec(len(corpus), keys, ranked)
    got = device_values(attr, len(corpus))
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, (ctx, bad[:5], got[bad[:5]], want[bad[:5]])
    return want


@pytest.mark.parametrize("fold", [False, True])
@pytest.mark.parametrize("desc", [False, True])
def test_text_key(fold, desc):
    rng = np.random.default_rng(int(fold) * 2 + int(desc))
    texts = texts_of(rng, 5000)
    c = F.Corpus.from_list(texts)
    try:
        a = c.rank(c.text(desc=desc, fold_case=fold))
        want = expect_rank(c, a, [("text", texts, desc, fold)], live(len(texts)), (fold, desc))
        check_ordered(c, a, want)
        a.close()
    finally:
        c.close()


def test_mixed_and_four_keys_and_other_column():
    rng = np.random.default_rng(11)
    n = 3 * 1024 + 77
    names, exts = texts_of(rng, n, 12), texts_of(rng, n, 3, np.frombuffer(b"abcC", np.uint8))
    c, col = F.Corpus.from_list(names), F.Corpus.from_list(exts)
    v1 = rng.choice([ATTR_NULL, ATTR_NULL + 1, -1, 0, 1, I64_MAX], n).astype(np.int64)
    v2 = rng.integers(-3, 3, n // 2).astype(np.int64)   # shorter than the corpus: null past it
    v2f = np.full(n, ATTR_NULL, np.int64)
    v2f[: len(v2)] = v2
    a1, a2 = c.attr(v1), c.attr(v2)
    out = c.attr()
    try:
        cases = [
            ([a1.asc(), c.text()], [("attr", v1, False), ("text", names, False, False)]),
            ([c.text(fold_case=True), a1.desc()], [("text", names, False, True), ("attr", v1, True)]),
            ([a1.desc(), a2.asc()], [("attr", v1, True), ("attr", v2f, False)]),
            ([col.text(desc=True), a2.desc(), c.text(fold_case=True), a1.asc()],
             [("text", exts, True, False), ("attr", v2f, True), ("text", names, False, True), ("attr", v1, False)]),
            ([col.text()], [("text", exts, False, False)]),
        ]
        for j, (keys, spec_keys) in enumerate(cases):
            want = expect_rank(c, out.rank(*keys), spec_keys, live(n), j)
            if j in (0, 3):
                check_ordered(c, out, want)
    finally:
        for h in (out, a1, a2, c, col):
            h.close()


def test_removed_replaced_and_appended_rows():
    rng = np.random.default_rng(12)
    n = 2 * 1024 + 5
    names, other = texts_of(rng, n), texts_of(rng, n)
    c, col = F.Corpus.from_list(names), F.Corpus.from_list(other)
    try:
        gone, gone_col = [0, 5, 1024, n - 1], [7, 2000]
        c.remove(gone)
        col.remove(gone_col)
        a = c.rank(c.text())
        expect_rank(c, a, [("text", names, False, False)], live(n, gone), "removed in C")
        a.rank(col.text(), c.text(desc=True))
        want = expect_rank(c, a, [("text", other, False, False), ("text", names, True, False)], live(n, gone + gone_col), "removed in col")
        check_ordered(c, a, want)
        # replaced rows: the values are a snapshot until the next refill
        which = [3, 9, 1500]
        repl = [b"ZZZ", b"", b"\0"]
        c.replace_list(which, repl)
        before = device_values(a, n)
        assert np.array_equal(before, want)
        for i, t in zip(which, repl):
            names[i] = t
        a.rank(c.text())
        expect_rank(c, a, [("text", names, False, False)], live(n, gone), "replaced")
        # appended rows are null until the refill (and the values grow to the corpus's length)
        extra = texts_of(rng, 1500)
        c.append_list(extra)
        col.append_list(extra)
        names += extra
        other += extra
        got = device_values(a, len(c))
        assert (got[n:] == ATTR_NULL).all()
        a.rank(c.text(fold_case=True))
        want = expect_rank(c, a, [("text", names, False, True)], live(len(c), gone), "appended")
        check_ordered(c, a, want)
        a.close()
    finally:
        c.close()
        col.close()


@pytest.mark.parametrize("case", ["empty", "equal", "prefix200", "long", "identical_1mib"])
def test_shapes(case):
    rng = np.random.default_rng(13)
    if case == "empty":
        texts = []
    elif case == "equal":
        texts = [b"same text"] * 3000
    elif case == "prefix200":
        p = b"/srv/data/" + b"d" * 190
        texts = [p + rng.choice(np.frombuffer(b"ab/", np.uint8), int(rng.integers(0, 12))).tobytes() for _ in range(4000)]
    elif case == "long":
        base = rng.choice(ALPHABET, 1500).tobytes()
        texts = [base[: int(rng.integers(1000, 1500))] + rng.choice(ALPHABET, int(rng.integers(0, 5))).tobytes() for _ in range(800)]
    else:
        big = rng.integers(0, 256, 1 << 20, dtype=np.uint8).tobytes()
        texts = [big] * 4 + [big[:-1], big + b"\0", b"small", big[:100]]
    c = F.Corpus.from_list(texts)
    try:
        for fold, desc in ((False, False), (True, True)):
            a = c.rank(c.text(desc=desc, fold_case=fold))
            want = expect_rank(c, a, [("text", texts, desc, fold)], live(len(texts)), (case, fold))
            if case in ("equal", "prefix200"):
                check_ordered(c, a, want, needles=("",))
            a.close()
    finally:
        c.close()


def test_own_key_and_refill_allocates_nothing():
    rng = np.random.default_rng(14)
    n = 4 * 1024 + 9
    names = texts_of(rng, n)
    c = F.Corpus.from_list(names)
    v = rng.integers(-5, 5, n).astype(np.int64)
    a = c.attr(v)
    try:
        # a as its own key: the values are written only after the order is known
        a.rank(a.desc(), c.text())
        want = expect_rank(c, a, [("attr", v, True), ("text", names, False, False)], live(n), "own key")
        a.rank(a.asc())   # ranks of ranks: the same order, so the same values
        assert np.array_equal(device_values(a, n), want)
        check_cycle(lambda: a.rank(c.text(fold_case=True), a.asc()))
    finally:
        a.close()
        c.close()
