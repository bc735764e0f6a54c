"""frz_attr_rank at the sizes it is built for: a million rows and more, segment ids past 2^16 and 2^24, text keys spread
over thousands of tiles, re-packed tiles, another corpus's texts, and texts at the 4 MiB - 2 haystack bound.  Below 65 536
ranked rows only the low two bytes of a segment id vary, so the sort's passes on segment bytes 2 and 3, the multi-trip
walk of the sort's segments and the scan over more than 1 024 head chunks never run in tests/test_gpu_rank.py.

Every check compares Attr.values() with tests/test_gpu_rank.py's restatement (text keys ranked by Python's sorted() over
bytes, then np.lexsort over the key tuples, null last), bit for bit.  Each case first asserts, from that restatement, the
shape it exists for (tied segments past 2^16 or 2^24 in the second round, the number of head chunks, the texts at the
bounds), so that it cannot pass vacuously when a generator changes.  Every handle is closed before the test ends: the
2^24-row case alone holds gigabytes of device memory."""
import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200 import synth
from frizbee_b200.types import Config, Order, SortStrategy
from ordering import ATTR_NULL, order_by_attr
from test_gpu_memory import check_cycle
from test_gpu_rank import FOLD, I64_MAX, int_keys, spec

pytestmark = pytest.mark.gpu

CHUNK = 7                    # text bytes per refinement chunk (rank_plan.cuh)
HAY_MAX = 4 * 2**20 - 2      # the longest haystack a corpus takes
DIRS = [b"/home/user/src/", b"/home/User/src/", b"/home/user/src/frizbee/", b"/srv/data/", b"/srv/data/2026/",
        b"/usr/lib/python3/site-packages/", b"/usr/lib/python3/Site-Packages/", b"C:\\Users\\me\\", b""]
ALNUM = np.frombuffer(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_.", np.uint8)


# ------------------------------------------------------------------------------------------------ generators
def synth_rows(n, seed):
    return synth.to_list(*synth.generate("deadbeef", n, 24, 64, seed))


def path_rows(rng, n):
    """Path-like rows: a directory from DIRS (shared prefixes, some differing only in case), one to three components and a
    file name; one row in ten repeats an earlier row exactly and one in ten repeats one with its case flipped."""
    comps = [bytes(rng.choice(ALNUM, int(rng.integers(1, 9)))) for _ in range(400)]
    d = rng.integers(0, len(DIRS), n)
    depth = rng.integers(1, 4, n)
    pick = rng.integers(0, len(comps), (n, 3))
    kind = rng.random(n)
    back = rng.integers(0, n, n)
    out = []
    for i in range(n):
        if i and kind[i] < 0.1:
            out.append(out[back[i] % i])
        elif i and kind[i] < 0.2:
            out.append(out[back[i] % i].swapcase())
        else:
            out.append(DIRS[d[i]] + b"/".join(comps[j] for j in pick[i, : depth[i]]))
    return out


def shuffled(rng, rows):
    return [rows[i] for i in rng.permutation(len(rows))]


# ------------------------------------------------------------------------------------------------ the restatement
def as_attr(key):
    """A text key as the attribute key of its ranks, so a reference over several key sets sorts each text only once."""
    return ("attr", int_keys(key)[0], False)


def tied_text_starts(texts, ranked, desc, fold):
    """The first positions, in the final order, of the segments that a single text key leaves tied after the first round
    (equal on the first chunk after the common prefix of all ranked rows, and not ended there): the segments the second
    round sorts."""
    t = sorted((x.translate(FOLD) if fold else x for x, r in zip(texts, ranked) if r), reverse=desc)
    lo, hi = t[0], t[-1]
    p = next((i for i in range(min(len(lo), len(hi))) if lo[i] != hi[i]), min(len(lo), len(hi)))
    keys = [(x[p: p + CHUNK], min(CHUNK, len(x) - p)) for x in t]
    starts, j = [], 0
    while j < len(keys):
        e = j + 1
        while e < len(keys) and keys[e] == keys[j]:
            e += 1
        if e - j > 1 and keys[j][1] == CHUNK:
            starts.append(j)
        j = e
    return np.array(starts, np.int64)


def tied_attr_starts(values, ranked):
    """The first positions of the segments of more than one row that an attribute key leaves (no nulls)."""
    v = np.sort(np.asarray(values)[ranked])
    _, first, count = np.unique(v, return_index=True, return_counts=True)
    return first[count > 1]


def expect(attr, want, ctx):
    got = attr.values()
    assert len(got) == len(want)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, (ctx, bad.size, bad[:5], got[bad[:5]], want[bad[:5]])


def live(n, removed=()):
    m = np.ones(n, bool)
    m[np.asarray(removed, np.int64)] = False
    return m


# ------------------------------------------------------------------------------------------------ cases
def test_text_key_past_a_million_rows():
    """1.1 M synth and path-like rows with shared directories, exact and case-only duplicates, under every (desc,
    fold_case): the second round sorts tied segments on both sides of position 2^16, and the heads span more than 1 024
    chunks of 1 024 positions."""
    rng = np.random.default_rng(31)
    texts = shuffled(rng, synth_rows(700_000, 31) + path_rows(rng, 400_000))
    n = len(texts)
    assert n > 1024 * 1024
    ranked = live(n)
    c = F.Corpus.from_list(texts)
    a = c.attr()
    try:
        for desc in (False, True):
            for fold in (False, True):
                starts = tied_text_starts(texts, ranked, desc, fold)
                assert len(set(starts >> 16)) > 1, (desc, fold)   # segment byte 2 varies in round 2
                a.rank(c.text(desc=desc, fold_case=fold))
                expect(a, spec(n, [("text", texts, desc, fold)], ranked), (desc, fold))
    finally:
        a.close()
        c.close()


def test_segment_ids_past_2_24():
    """2^24 + 4 099 rows of empty or one-byte texts ranked by a1 = perm(i) // 2 (rows tie in pairs), then by a second
    attribute with nulls and int64 extremes, a few hundred rows removed across the tiles: the second round sorts segment
    ids on both sides of 2^24, so the sort's pass on segment byte 3 runs."""
    n = 2**24 + 4099
    rng = np.random.default_rng(32)
    lens = rng.integers(0, 2, n, dtype=np.uint64)
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    data = rng.integers(0, 256, int(off[-1]), dtype=np.uint8)
    a1 = (rng.permutation(n) // 2).astype(np.int64)
    a2 = rng.integers(-2**62, 2**62, n, dtype=np.int64)
    for v in (ATTR_NULL, ATTR_NULL + 1, -I64_MAX, -1, 0, 1, I64_MAX - 1, I64_MAX):
        a2[rng.integers(0, n, 3000)] = v
    pairs = np.argsort(a1, kind="stable")[: n - 1].reshape(-1, 2)   # the rows of each a1 value but the last
    tie = pairs[rng.choice(len(pairs), 1000, replace=False)]
    a2[tie[:, 1]] = a2[tie[:, 0]]   # 1 000 pairs stay tied
    gone = np.unique(rng.integers(0, n, 400))
    ranked = live(n, gone)
    starts = tied_attr_starts(a1, ranked)
    assert (starts < 2**24).any() and (starts >= 2**24).any()   # segment byte 3 varies in round 2
    c = F.Corpus.from_arrow(data, off)
    h1 = h2 = out = None
    try:
        c.remove(gone)
        h1, h2 = c.attr(a1), c.attr(a2)
        out = c.attr()
        out.rank(h1.asc(), h2.desc())
        want = spec(n, [("attr", a1, False), ("attr", a2, True)], ranked)
        assert want.max() >= 2**24
        expect(out, want, "a1 asc, a2 desc")
    finally:
        for h in (out, h2, h1, c):
            if h is not None:
                h.close()


def test_four_keys_over_two_corpora():
    """Four keys at 1 M rows: the text of another corpus (short extensions with ties and some 100-300 byte rows, so its
    tiles bucket differently), an attribute desc, this corpus's text folded, an attribute asc.  Rows removed only in
    the other corpus have no rank; each key splits ties the keys before it leave."""
    rng = np.random.default_rng(33)
    n = 1_000_000
    names = shuffled(rng, synth_rows(600_000, 33) + path_rows(rng, 400_000))
    ext_vocab = [b"", b"py", b"PY", b"rs", b"c", b"h", b"md", b"tar.gz", b"tar.GZ", b"\0", b"py\0"]
    pick = rng.integers(0, len(ext_vocab), n)
    exts = [ext_vocab[j] for j in pick]
    for i in rng.integers(0, n, 5000):
        exts[i] = b"ext/" * 25 + bytes(rng.choice(ALNUM, int(rng.integers(0, 200))))
    v1 = rng.choice(np.array([ATTR_NULL, -5, 0, 3, 9, I64_MAX], np.int64), n)
    v2 = rng.integers(-2**63 + 1, 2**63 - 1, n, dtype=np.int64)
    v2[rng.integers(0, n, 2000)] = ATTR_NULL
    gone_col = np.unique(rng.integers(0, n, 3000))
    ranked = live(n, gone_col)
    keys = [as_attr(("text", exts, False, False)), ("attr", v1, True), as_attr(("text", names, False, True)), ("attr", v2, False)]
    wants = [spec(n, keys[: j + 1], ranked) for j in range(4)]
    assert all(wants[j].max() < wants[j + 1].max() for j in range(3))   # every key splits ties
    c, col = F.Corpus.from_list(names), F.Corpus.from_list(exts)
    h1 = h2 = out = None
    try:
        col.remove(gone_col)
        h1, h2 = c.attr(v1), c.attr(v2)
        out = c.attr()
        out.rank(col.text(), h1.desc(), c.text(fold_case=True), h2.asc())
        expect(out, wants[3], "four keys")
        assert (out.values()[gone_col] == ATTR_NULL).all()
    finally:
        for h in (out, h2, h1, col, c):
            if h is not None:
                h.close()


def test_edited_corpus_at_scale():
    """1 M rows, then 1 % removed across the tiles, 0.5 % replaced by long rows (some past 1 024 bytes, a few past 64
    KiB) so their tiles are re-packed, then 100 000 rows appended so the values grow, then 1 000 more so they grow into the
    swapped scratch: ranked and compared after every step.  A refill at the same size allocates nothing."""
    rng = np.random.default_rng(34)
    texts = shuffled(rng, synth_rows(600_000, 34) + path_rows(rng, 400_000))
    n = len(texts)
    removed = set()
    c = F.Corpus.from_list(texts)
    a = c.attr()
    try:
        a.rank(c.text())
        expect(a, spec(n, [("text", texts, False, False)], live(n)), "initial")
        gone = np.unique(rng.integers(0, n, n // 100))
        c.remove(gone)
        removed |= set(gone.tolist())
        a.rank(c.text(fold_case=True))
        expect(a, spec(n, [("text", texts, False, True)], live(n, sorted(removed))), "removed")
        which = np.unique(rng.integers(0, n, n // 200))
        base = bytes(rng.choice(ALNUM, 300_000))
        repl = []
        for j in range(len(which)):
            ln = int(rng.integers(70_000, 300_000)) if j % 1000 == 0 else int(rng.integers(100, 3000))
            t = base[:ln] if j % 3 else base[: ln // 2] + bytes(rng.choice(ALNUM, ln - ln // 2))
            repl.append(t.swapcase() if j % 5 == 0 else t)
        assert sum(len(t) > 1024 for t in repl) > 100 and sum(len(t) > 65536 for t in repl) >= 3
        c.replace_list(which, repl)
        for i, t in zip(which, repl):
            texts[i] = t
        removed -= set(which.tolist())   # a replaced row comes back
        a.rank(c.text(desc=True))
        expect(a, spec(n, [("text", texts, True, False)], live(n, sorted(removed))), "replaced")
        for extra in (path_rows(rng, 100_000), synth_rows(1000, 35)):
            c.append_list(extra)
            texts += extra
            a.rank(c.text())
            expect(a, spec(len(texts), [("text", texts, False, False)], live(len(texts), sorted(removed))), ("appended", len(texts)))
        check_cycle(lambda: a.rank(c.text(fold_case=True)))
        expect(a, spec(len(texts), [("text", texts, False, True)], live(len(texts), sorted(removed))), "refilled")
    finally:
        a.close()
        c.close()


def boundary_texts(rng):
    """(texts, pairs, case_pairs): rows at the refinement's boundaries, and index pairs that must rank apart (pairs) or
    apart unless folded (case_pairs)."""
    texts, pairs, case_pairs = [], [], []

    def add(*ts):
        texts.extend(ts)
        return list(range(len(texts) - len(ts), len(texts)))

    for k in (1, 2, 3, 5, 9, 37, 147):
        for d in (CHUNK * k - 1, CHUNK * k, 16 * k - 1, 16 * k):
            base = bytes(rng.choice(ALNUM, d + 5))
            flip = base[:d] + bytes([base[d] ^ 0x01]) + base[d + 1:]
            i, j, _ = add(base, flip, base[:d])   # first differ at byte d; and a proper prefix
            pairs.append((i, j))
        base = bytes(rng.choice(ALNUM, CHUNK * k + 3))
        add(base[: CHUNK * k], base[: CHUNK * k] + b"\0", base[: CHUNK * k] + b"a", base[: CHUNK * k - 1])   # end on a chunk
    for p in (5, 17, 33, 100, 1001):   # shared prefixes that end inside a 16-byte unit
        pre = bytes(rng.choice(ALNUM, p))
        add(*[pre + bytes(rng.choice(ALNUM, int(rng.integers(0, 20)))) for _ in range(40)])
    for depth in (9, 500, 1000, 4099):   # case-only differences deep in the text
        base = bytes(rng.choice(np.frombuffer(b"abcxyz", np.uint8), depth))
        i, j = add(base + b"name", base + b"NAME")
        case_pairs.append((i, j))
        i, j = add(base + b"Name.txt", base + b"nAME.txt")
        case_pairs.append((i, j))
    for size in (1, 2, 33, 1025, 4097):   # tie blocks
        add(*[b"tie/" + bytes(rng.choice(ALNUM, 12)) + b"/%d" % size] * size)
    big = bytes(rng.choice(ALNUM, HAY_MAX))
    i, j, _ = add(big, big[:-1] + bytes([big[-1] ^ 0x01]), big[: HAY_MAX - 9])   # at the bound, last byte apart; a prefix
    pairs.append((i, j))
    return texts, pairs, case_pairs


def test_boundary_texts_in_a_large_corpus():
    """Pairs that first differ at bytes 7k - 1, 7k, 16k - 1 and 16k, texts that end on a chunk, shared prefixes that end
    inside a unit, case-only differences deep in the text, tie blocks of 1 to 4 097 rows and two rows of 4 MiB - 2 bytes
    that differ in the last byte, scattered over 200 000 synth rows: every (desc, fold_case)."""
    rng = np.random.default_rng(35)
    special, pairs, case_pairs = boundary_texts(rng)
    filler = synth_rows(200_000, 35)
    n = len(filler) + len(special)
    where = np.sort(rng.choice(n, len(special), replace=False))   # the special rows' places, spread over the corpus
    texts = [None] * n
    for w, t in zip(where, special):
        texts[w] = t
    it = iter(filler)
    texts = [t if t is not None else next(it) for t in texts]
    assert where[-1] - where[0] > n // 2 and sum(len(t) == HAY_MAX for t in texts) == 2
    c = F.Corpus.from_list(texts)
    a = c.attr()
    try:
        for desc in (False, True):
            for fold in (False, True):
                want = spec(n, [("text", texts, desc, fold)], live(n))
                for i, j in pairs:
                    assert want[where[i]] != want[where[j]]
                for i, j in case_pairs:
                    assert (want[where[i]] == want[where[j]]) == fold
                a.rank(c.text(desc=desc, fold_case=fold))
                expect(a, want, (desc, fold))
    finally:
        a.close()
        c.close()


def test_ordered_calls_on_ranks_at_a_million_rows():
    """The ordered calls on a rank of 1 M rows (synth and path-like rows, case-only duplicates tied under fold_case):
    ATTR_ASC and SCORE_THEN_ATTR_ASC, k of 1, 50, 1 024, 4 097 and all, every sort strategy, against order_by_attr over
    match_list_into_array; then one batched ordered call of max_typos = 0 queries, which takes the batched path."""
    rng = np.random.default_rng(36)
    texts = shuffled(rng, synth_rows(700_000, 36) + path_rows(rng, 300_000))
    n = len(texts)
    assert n <= 2**21
    c = F.Corpus.from_list(texts)
    kind = rng.integers(0, 4, n).astype(np.int64)
    ka = c.attr(kind)
    a = c.attr()
    try:
        a.rank(ka.asc(), c.text(fold_case=True))
        values = spec(n, [("attr", kind, False), ("text", texts, False, True)], live(n))
        expect(a, values, "rank")
        assert len(np.unique(values)) < n   # ties the ordered calls break by score and then by index
        for needle in ("", "deadbeef"):
            for sort in SortStrategy:
                cfg = Config(max_typos=0, sort=sort)
                m = F.Matcher.from_query(needle, cfg) if needle == "" else F.Matcher(needle, Config(max_typos=1, sort=sort))
                try:
                    into = m.match_list_into_array(c).copy()
                    assert len(into) > 10_000, (needle, len(into))
                    for order in (Order.AttrAsc, Order.ScoreThenAttrAsc):
                        want = order_by_attr(into, values, int(order), SortStrategy(sort).is_reversed())
                        for k in (1, 50, 1024, 4097, None):
                            got, total = m.match_list_ordered_array(c, a, order, k)
                            w = want if k is None else want[:k]
                            assert total == len(want) and len(got) == len(w), (needle, sort, order, k)
                            assert np.array_equal(got["index"], w["index"]), (needle, sort, order, k)
                            assert np.array_equal(got["score"], w["score"]), (needle, sort, order, k)
                finally:
                    m.close()
        # batched: 32 needles of 5-8 bytes cut from the rows (few enough matches that no survivor list overflows), max_typos
        # = 0, every strategy and both orders
        q, k = 32, 50
        ms, orders = [], []
        while len(ms) < q:
            row = texts[int(rng.integers(0, n))]
            ln = int(rng.integers(5, 9))
            s = int(rng.integers(0, max(1, len(row) - ln)))
            needle = row[s: s + ln]
            if len(needle) == ln and needle.isalnum():
                ms.append(F.Matcher(needle.decode(), Config(max_typos=0, sort=list(SortStrategy)[len(ms) % 4])))
                orders.append((Order.AttrAsc, Order.ScoreThenAttrAsc)[(len(ms) // 4) % 2])
        try:
            rows, n_out, n_total = F.match_list_batch_ordered(ms, c, k, a, orders)[:3]
            last = F.batch_last()
            assert last["batched"] == q and last["overflowed"] == 0, last
            for j, m in enumerate(ms):
                want = order_by_attr(m.match_list_into_array(c), values, int(orders[j]), SortStrategy(m.config.sort).is_reversed())
                assert n_total[j] == len(want) > 0 and n_out[j] == min(k, len(want)), j
                assert np.array_equal(rows[j, : n_out[j]]["index"], want[:k]["index"]), j
                assert np.array_equal(rows[j, : n_out[j]]["score"], want[:k]["score"]), j
        finally:
            for m in ms:
                m.close()
    finally:
        a.close()
        ka.close()
        c.close()
