"""Column calls without a GPU: the argument checks of frz_match_list_columns, their order and the missing-device status,
and the specification tests/columns.py against a literal per-row loop over the CPU oracle's per-column lists."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from columns import combine, match_list_columns
from frizbee_b200.types import Config, CaseMatching, Matching, Pattern, Scoring, SortStrategy
from oracle import pyoracle as O

INVALID, TOO_MANY_ITEMS, UNSUPPORTED, NO_DEVICE = 1, 4, 9, 8
U64_MAX = 2**64 - 1
GROUP_NONE = 0xFFFFFFFF


def _field_offset(fn, width, marker):
    """The byte offset of the corpus field that fn (frz_corpus_len / frz_corpus_device) reads, found by probing."""
    buf = C.create_string_buffer(4096)
    for off in range(0, 1024, width):
        C.memmove(C.addressof(buf) + off, marker.to_bytes(width, "little"), width)
        if fn(C.addressof(buf)) == marker:
            return off
        C.memmove(C.addressof(buf) + off, b"\0" * width, width)
    raise AssertionError("field not found")


def test_argument_checks_in_order_and_no_device():
    import torch
    L = F.lib()
    n_at, dev_at = _field_offset(L.frz_corpus_len, 8, 0x1234_5678_9A), _field_offset(L.frz_corpus_device, 4, 5)

    def fake_corpus(n, device=0):
        buf = C.create_string_buffer(4096)
        C.memmove(C.addressof(buf) + n_at, int(n).to_bytes(8, "little"), 8)
        C.memmove(C.addressof(buf) + dev_at, int(device).to_bytes(4, "little"), 4)
        return buf

    c0, c1, longer, elsewhere, stranger = fake_corpus(7), fake_corpus(7), fake_corpus(8), fake_corpus(7, 1), fake_corpus(7)
    huge, huge2 = fake_corpus(2**32), fake_corpus(2**32)   # one row past the u32 index space
    before = [b.raw for b in (c0, c1, longer, elsewhere, stranger)]
    assert L.frz_corpus_len(C.addressof(c1)) == 7 and L.frz_corpus_device(C.addressof(elsewhere)) == 1
    # a handle's first field is its corpus
    handle = {name: C.create_string_buffer(C.addressof(c).to_bytes(8, "little"), 64)
              for name, c in (("c0", c0), ("c1", c1), ("stranger", stranger))}
    h = {k: C.addressof(v) for k, v in handle.items()}
    mfake = C.create_string_buffer(64)           # a matcher, never dereferenced before the device check
    m = C.addressof(mfake)
    out = np.zeros(4, dtype=F.MATCH_DTYPE)
    counts = np.zeros(4, dtype=np.uint32)
    n, total = C.c_uint64(), C.c_uint64()
    fn = L.frz_match_list_columns

    def arr(*xs):
        return (C.c_void_p * len(xs))(*xs)

    def call(ms=None, cols=None, n_cols=2, sort=0, s=None, b=None, g=None, per_group=1, k=4, o=out.ctypes.data, cnt=None):
        ms = arr(m, m) if ms is None else ms
        cols = arr(C.addressof(c0), C.addressof(c1)) if cols is None else cols
        return fn(ms, cols, n_cols, sort, s, b, g, per_group, k, o, C.byref(n), C.byref(total), cnt)

    def refused(status, text, **kw):
        assert call(**kw) == status, kw
        assert text.encode() in L.frz_last_error(), (kw, L.frz_last_error())

    refused(INVALID, "n_cols", n_cols=0)
    refused(INVALID, "n_cols", n_cols=0, ms=0, sort=9, k=1, o=None)   # the first check wins
    refused(INVALID, "null argument", ms=0)
    refused(INVALID, "null argument", cols=0)
    refused(INVALID, "column 1", ms=arr(m, None))
    refused(INVALID, "column 0", cols=arr(None, C.addressof(c1)))
    refused(INVALID, "device", cols=arr(C.addressof(c0), C.addressof(elsewhere)))
    refused(INVALID, "index space", cols=arr(C.addressof(c0), C.addressof(longer)))
    refused(INVALID, "index space", cols=arr(C.addressof(c0), C.addressof(longer)), sort=9)
    refused(TOO_MANY_ITEMS, "u32 index", cols=arr(C.addressof(huge), C.addressof(huge2)))
    refused(TOO_MANY_ITEMS, "u32 index", cols=arr(C.addressof(huge), C.addressof(huge2)), sort=9, k=1, o=None)
    for bad in (4, 255):
        refused(INVALID, "sort", sort=bad)
    refused(INVALID, "sort", sort=4, g=h["c0"], per_group=0)
    refused(INVALID, "per_group = 0", g=h["c0"], per_group=0)
    for pg in (33, 1000, 2**63, U64_MAX - 1):
        refused(UNSUPPORTED, "per_group", g=h["c0"], per_group=pg)
    refused(INVALID, "null out", k=1, o=None)
    refused(INVALID, "null out", k=1, o=None, s=h["stranger"])
    refused(INVALID, "subset was made on none", s=h["stranger"])
    refused(INVALID, "boost was made on none", b=h["stranger"])
    refused(INVALID, "groups were made on none", g=h["stranger"])
    assert [b.raw for b in (c0, c1, longer, elsewhere, stranger)] == before
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    # every argument is valid: the call reaches the device check.  per_group is not read without groups; handles of any
    # column serve; a column or matcher may repeat
    for kw in (dict(), dict(per_group=0), dict(per_group=77), dict(s=h["c1"], b=h["c0"], g=h["c1"], per_group=32, cnt=counts.ctypes.data),
               dict(g=h["c0"], per_group=U64_MAX, k=0, o=None), dict(k=U64_MAX, sort=3),
               dict(cols=arr(C.addressof(c0), C.addressof(c0)), ms=arr(m, m)), dict(n_cols=1)):
        assert call(**kw) == NO_DEVICE, kw
    assert fn(arr(m), arr(C.addressof(c0)), 1, 0, None, None, None, 0, 0, None, None, None, None) == NO_DEVICE


# ---------------------------------------------------------------------------- the specification against a literal loop

def literal(lists, n, sort, live=None, members=None, boost=None, group_of=None, per_group=1, n_groups=1, any_compiled=True):
    """The contract restated one row at a time."""
    hits = [{int(r["index"]): (int(r["score"]), bool(r["exact"])) for r in L} for L in lists]
    rows = []
    for i in range(n):
        if (live is not None and not live[i]) or (members is not None and i not in set(int(x) for x in members)):
            continue
        if all(i in d for d in hits):
            rows.append((i, min(65535, sum(d[i][0] for d in hits)), any(d[i][1] for d in hits)))
    if sort.is_reversed():
        rows.reverse()
    if boost is not None:
        key = lambda r: min(65535, max(0, r[1] + (int(boost[r[0]]) if r[0] < len(boost) else 0)))
        rows.sort(key=lambda r: -key(r))
    elif sort.is_by_score() and any_compiled:
        rows.sort(key=lambda r: -r[1])
    counts = None
    if group_of is not None:
        counts = [0] * n_groups
        kept, seen = [], {}
        for r in rows:
            g = int(group_of[r[0]]) if r[0] < len(group_of) else GROUP_NONE
            if g == GROUP_NONE:
                kept.append(r)
                continue
            counts[g] += 1
            if per_group is None or seen.get(g, 0) < per_group:
                kept.append(r)
            seen[g] = seen.get(g, 0) + 1
        rows = kept
    return rows, counts


def as_tuples(a):
    return [(int(r["index"]), int(r["score"]), bool(r["exact"])) for r in a]


WORDS = ["foo", "bar", "baz", "foobar", "FooBar", "é다", "😀x", "naïve", "résumé", "quux", "src", "main", "a/b/c", "über"]


def table(rng, n, extra=()):
    rows = []
    for _ in range(n):
        k = int(rng.integers(0, 4))
        rows.append("_".join(WORDS[int(j)] for j in rng.integers(0, len(WORDS), k)) + "".join(extra[int(rng.integers(0, len(extra)))] if extra and rng.random() < 0.3 else ""))
    return rows


HIGH = Scoring(match_score=(0xFFFF - 40) // 3 - 8)   # an exact 3-byte literal scores above 32 767


def column_cases():
    """(name, [(patterns, config)] per column): mixed literal modes, unicode needles, negations, empty matchers, per-column
    configs, and literal columns whose sum saturates at 65535."""
    return [
        ("fuzzy+fuzzy", [(["foo"], Config(max_typos=1)), (["bar"], Config(casing=CaseMatching.Respect))]),
        ("unicode+negated", [(["é다"], Config(max_typos=0)), ([Pattern("baz", negated=True)], Config())]),
        ("empty+fuzzy+literal", [([], Config()), (["ba"], Config(max_typos=None)),
                                  ([Pattern("main", matching=Matching.Substring)], Config())]),
        ("all-negated", [([Pattern("quux", negated=True)], Config()), ([Pattern("src", negated=True)], Config())]),
        ("saturating", [([Pattern("foo", matching=Matching.Substring, scoring=HIGH)], Config()),
                        ([Pattern("bar", matching=Matching.Substring, scoring=HIGH)], Config()),
                        (["a"], Config(max_typos=0))]),
        ("all-empty", [([], Config()), ([], Config())]),
    ]


@pytest.mark.parametrize("seed", range(3))
def test_specification_equals_the_literal_loop(seed):
    rng = np.random.default_rng(seed)
    n = 300
    for name, cols in column_cases():
        lists, tables = [], []
        for j, (pats, cfg) in enumerate(cols):
            hay = table(rng, n, extra=("foo", "bar", "FOO") if j % 2 == 0 else ("bar", "src"))
            data, off = O.pack(hay)
            tables.append(hay)
            lists.append(O.match_list_into_packed(pats, cfg, data, off) if pats else
                         np.array([(i, 0, 0, 0) for i in range(n)], dtype=F.MATCH_DTYPE))
        any_compiled = any(len(p) for p, _ in cols)
        if name == "saturating":
            both = combine(lists[:2], n)
            assert len(both) and (both["score"] == 65535).any(), "no row saturates"
        live = rng.random(n) > 0.1
        members = rng.choice(n + 20, 180, replace=True)
        boost = rng.integers(-300, 301, n - 10).astype(np.int16)
        group_of = rng.integers(0, 9, n).astype(np.uint32)
        group_of[rng.random(n) < 0.2] = GROUP_NONE
        for sort in SortStrategy:
            for kw in (dict(), dict(live=live), dict(members=members), dict(boost=boost), dict(live=live, members=members, boost=boost),
                       dict(group_of=group_of, per_group=1, n_groups=9), dict(group_of=group_of, per_group=None, n_groups=9, boost=boost),
                       dict(group_of=group_of, per_group=3, n_groups=9, members=members)):
                got, counts = match_list_columns(lists, n, sort, any_compiled=any_compiled, **kw)
                want, wcounts = literal(lists, n, sort, any_compiled=any_compiled, **kw)
                ctx = (name, sort, sorted(kw))
                assert as_tuples(got) == want, ctx
                assert (counts is None) == (wcounts is None), ctx
                if counts is not None:
                    assert counts.tolist() == wcounts, ctx


def test_exact_comes_from_any_column():
    """A row's exact flag is the OR over the columns: one exact column makes the row exact, whichever column it is."""
    hay0 = ["foo", "xfoo", "foo", "fo_o"]
    hay1 = ["xbar", "bar", "bar", "bxar"]
    lists = [O.match_list_into_packed(["foo"], Config(max_typos=1), *O.pack(hay0)),
             O.match_list_into_packed(["bar"], Config(max_typos=1), *O.pack(hay1))]
    got = {int(r["index"]): bool(r["exact"]) for r in combine(lists, 4)}
    assert got == {0: True, 1: True, 2: True, 3: False}, got


def test_atoms_over_repeats_of_one_column_equal_the_multi_pattern_matcher():
    """A matcher per atom over [c, c, ...] is the multi-pattern matcher over c (src/matcher/multi.rs:83-152)."""
    rng = np.random.default_rng(7)
    hay = table(rng, 400, extra=("foo", "bar", "baz"))
    data, off = O.pack(hay)
    cfg = Config(max_typos=1)
    for atoms in ([Pattern("foo"), Pattern("bar", negated=True), Pattern("baz", matching=Matching.Substring)],
                  [Pattern("bar", negated=True), Pattern("fo"), Pattern("é다", max_typos=0)],
                  [Pattern("src", negated=True), Pattern("quux", negated=True)]):
        lists = [O.match_list_into_packed([a], cfg, data, off) for a in atoms]
        whole = O.match_list_into_packed(atoms, cfg, data, off)
        for sort in SortStrategy:
            got, _ = match_list_columns(lists, len(hay), sort)
            want = O.match_list_packed(atoms, cfg.with_(sort=sort), data, off)
            assert as_tuples(got) == as_tuples(want), (atoms, sort)
        assert as_tuples(combine(lists, len(hay))) == as_tuples(whole), atoms
