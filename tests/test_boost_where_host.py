"""frz_boost_where without a GPU: frizbee_b200/csrc/boost_plan.cuh built for the CPU (tests/harness/boost_where_harness.cpp).
Its packer (rules grouped by attribute over the batched plan's distinct-attribute table) and k_boost_where's row rule
over staged chunks against a numpy restatement, and the argument checks of frz_boost_where / frz_boost_where_batch in
their documented order on zero-filled stand-in handles.  The behaviour on a real corpus is in tests/test_gpu_boost_where.py."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from cpu_harness import load
from test_where_batch_host import BAttr, BClause
from test_where_host import NULL, random_values, spec_holds

INVALID, UNSUPPORTED, NO_DEVICE = 1, 9, 8
STAGED = 4            # kFrzWhereBatchStaged
CHUNK = 1024          # kFrzWhereChunk
vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32


class BQuery(C.Structure):   # FrzBoostQuery
    _fields_ = [("rule0", u32), ("n_rules", u32), ("set0", u64), ("base", vp), ("n_base", u64), ("out", vp)]


@pytest.fixture(scope="module")
def H():
    L = load("boost_where_harness")
    L.h_boost_pack.argtypes = [vp, vp, u64]
    L.h_boost_pack.restype = u64
    L.h_boost_plan.argtypes = [vp, vp, vp, vp, vp, vp]
    L.h_boost_plan.restype = None
    L.h_boost_fill.argtypes = [vp, vp, u64, u64, vp, vp, vp, vp, vp]
    L.h_boost_fill.restype = None
    return L


class Attrs:
    """Stand-in attributes: each handle is the address of a FrzWhereBatchAttr over a numpy array."""

    def __init__(self, arrays):
        self.arrays = [np.ascontiguousarray(a, dtype=np.int64) for a in arrays]
        self.recs = (BAttr * max(1, len(arrays)))()
        for j, a in enumerate(self.arrays):
            self.recs[j] = BAttr(a.ctypes.data if a.size else None, len(a))
        self.handles = [C.addressof(self.recs) + j * C.sizeof(BAttr) for j in range(len(arrays))]


def abi_rules(attrs, queries):
    """frz_boost_rule records of queries[j] = [(attr index, lo, hi, set values or None, negate, add), ...], and the counts.
    The set arrays are kept alive on the returned record array."""
    flat = [r for q in queries for r in q]
    arr = (F._CBoostRule * max(1, len(flat)))()
    keep = []
    for j, (a, lo, hi, in_, neg, add) in enumerate(flat):
        w = arr[j].when
        w.attr, w.lo, w.hi, w.negate = attrs.handles[a], lo, hi, int(neg)
        if in_ is not None:
            v = np.ascontiguousarray(in_, dtype=np.int64)
            keep.append(v)
            w.in_, w.n_in = (v.ctypes.data if v.size else None), len(v)
        arr[j].add = add
    arr._keep = keep
    return arr, np.array([len(q) for q in queries] or [0], dtype=np.uint64)


def spec_fill(attrs, rules, n, base=None):
    """The fill restated: clamp(base + the adds of the rules that hold) per row, and max(0, the largest value)."""
    acc = np.zeros(n, np.int64)
    if base is not None:
        acc[: min(n, len(base))] += base[:n].astype(np.int64)
    for a, lo, hi, in_, neg, add in rules:
        v = np.full(n, NULL, np.int64)
        src = attrs.arrays[a]
        v[: min(n, len(src))] = src[:n]
        acc += np.where(spec_holds(v, lo, hi, in_, neg), add, 0)
    out = np.clip(acc, -32768, 32767).astype(np.int16)
    return out, max(0, int(out.max())) if n else 0


def run_fill(H, attrs, queries, n, bases=None, in_place=()):
    """h_boost_fill of every query; bases[j]: an int16 array or None; in_place: queries whose output is their base."""
    arr, counts = abi_rules(attrs, queries)
    q = len(queries)
    bases = bases or [None] * q
    base_arrays = [None if b is None else np.ascontiguousarray(b, dtype=np.int16).copy() for b in bases]
    outs = [base_arrays[j] if j in in_place else np.full(max(n, 1), 0x5A5A, np.int16) for j in range(q)]
    hb = (vp * max(1, q))(*[b.ctypes.data if b is not None and b.size else None for b in base_arrays])
    nb = np.array([0 if b is None else len(b) for b in base_arrays] or [0], dtype=np.uint64)
    ho = (vp * max(1, q))(*[o.ctypes.data for o in outs])
    maxima = np.zeros(max(1, q), np.int32)
    loads = np.zeros(max(1, q), np.uint64)
    H.h_boost_fill(arr, counts.ctypes.data, q, n, hb, nb.ctypes.data, ho, maxima.ctypes.data, loads.ctypes.data)
    return [o[:n] for o in outs], maxima[:q], loads[:q]


def random_rule(rng, n_attrs, pool):
    a = int(rng.integers(n_attrs))
    add = int(rng.integers(-65535, 65536))
    neg = bool(rng.random() < 0.3)
    if rng.random() < 0.5:
        lo, hi = sorted(int(x) for x in rng.choice(pool, 2))
        return (a, lo, hi, None, neg, add)
    k = int(rng.integers(0, 6))
    if k == 0:   # an empty set, as Attr.isin([]) passes it: a range that holds for no value
        return (a, 0, -1, None, neg, add)
    in_ = rng.choice(pool, k)
    if k > 1:
        in_[-1] = in_[0]   # a duplicate
    return (a, 0, 0, in_, neg, add)


@pytest.mark.parametrize("n", [0, 1, 31, 1023, 1025, 3 * CHUNK + 17])
@pytest.mark.parametrize("n_attrs", [1, 3, 6])
def test_fill_against_numpy(H, n, n_attrs):
    rng = np.random.default_rng(n * 10 + n_attrs)
    pool = np.array([NULL + 1, -2**62, -7, -1, 0, 1, 2, 5, 9, 2**62, 2**63 - 1], dtype=np.int64)
    # some attributes shorter than the corpus: null past them
    arrays = [random_values(rng, int(rng.integers(0, n + 1)) if k % 2 else n, pool) for k in range(n_attrs)]
    attrs = Attrs(arrays)
    queries = [[random_rule(rng, n_attrs, pool) for _ in range(int(rng.integers(0, 9)))] for _ in range(5)]
    bases = [None, rng.integers(-32768, 32768, n, dtype=np.int16), rng.integers(-32768, 32768, max(0, n // 2), dtype=np.int16),
             rng.integers(-100, 100, n + 5, dtype=np.int16)[:n], None]
    outs, maxima, loads = run_fill(H, attrs, queries, n, bases)
    for j, rules in enumerate(queries):
        want, want_max = spec_fill(attrs, rules, n, bases[j])
        assert np.array_equal(outs[j], want), j
        assert maxima[j] == want_max, j
        # a row reads each distinct attribute of its query once, however many rules test it
        assert loads[j] == n * len({r[0] for r in rules}), j


def test_clamping_at_both_ends(H):
    n = 5
    attrs = Attrs([np.array([0, 1, NULL, 3, 4], np.int64)])
    up = [(0, 0, 10, None, False, 65535)] * 8
    down = [(0, 0, 10, None, False, -65535)] * 8
    base_hi = np.full(n, 32767, np.int16)
    base_lo = np.full(n, -32768, np.int16)
    outs, maxima, _ = run_fill(H, attrs, [up, down, down, up], n, [base_hi, base_lo, base_hi, base_lo])
    assert outs[0].tolist() == [32767, 32767, 32767, 32767, 32767] and maxima[0] == 32767
    assert outs[1].tolist() == [-32768] * 5 and maxima[1] == 0
    # the row without a value keeps its base; the others are clamped at the far end
    assert outs[2].tolist() == [-32768, -32768, 32767, -32768, -32768] and maxima[2] == 32767
    assert outs[3].tolist() == [32767, 32767, -32768, 32767, 32767] and maxima[3] == 32767
    # +65535 - 65535 nets to the base: the sum is taken before the clamp
    both = [(0, 0, 10, None, False, 65535), (0, 0, 10, None, False, -65535), (0, 0, 10, None, False, 3)]
    outs, maxima, _ = run_fill(H, attrs, [both], n, [base_hi])
    assert outs[0].tolist() == [32767, 32767, 32767, 32767, 32767]
    outs, maxima, _ = run_fill(H, attrs, [both], n, [np.full(n, 10, np.int16)])
    assert outs[0].tolist() == [13, 13, 10, 13, 13] and maxima[0] == 13


def test_in_place_base_and_no_rules(H):
    rng = np.random.default_rng(7)
    n = 2 * CHUNK + 3
    attrs = Attrs([random_values(rng, n, np.arange(-5, 6, dtype=np.int64))])
    base = rng.integers(-1000, 1000, n, dtype=np.int16)
    rules = [(0, -2, 2, None, False, 7), (0, 0, 0, np.array([1, 4, 4]), True, -3)]
    want, want_max = spec_fill(attrs, rules, n, base)
    outs, maxima, _ = run_fill(H, attrs, [rules], n, [base], in_place={0})
    assert np.array_equal(outs[0], want) and maxima[0] == want_max
    # no rules: a copy of the base (a shorter base is 0 past its values), or all zero without one
    outs, maxima, _ = run_fill(H, attrs, [[], []], n, [base[:100], None])
    assert np.array_equal(outs[0], np.concatenate([base[:100], np.zeros(n - 100, np.int16)]))
    assert maxima[0] == max(0, int(base[:100].max()))
    assert not outs[1].any() and maxima[1] == 0
    outs, maxima, _ = run_fill(H, attrs, [[]], n, [np.full(n, -5, np.int16)])
    assert maxima[0] == 0   # the key bound never falls below 0


def plan(H, attrs, queries):
    arr, counts = abi_rules(attrs, queries)
    H.h_boost_pack(arr, counts.ctypes.data, len(queries))
    sizes = np.zeros(4, np.uint64)
    H.h_boost_plan(sizes.ctypes.data, None, None, None, None, None)
    na, nr, ns = (int(x) for x in sizes[:3])
    pa, pc, pq = (BAttr * max(1, na))(), (BClause * max(1, nr))(), (BQuery * max(1, len(queries)))()
    adds, sets = np.zeros(max(1, nr), np.int32), np.zeros(max(1, ns), np.int64)
    H.h_boost_plan(sizes.ctypes.data, pa, pc, adds.ctypes.data, pq, sets.ctypes.data)
    return {"attrs": [pa[k].values for k in range(na)], "staged": int(sizes[3]),
            "queries": [[(pa[pc[pq[j].rule0 + r].attr].values, pc[pq[j].rule0 + r].rule.lo, pc[pq[j].rule0 + r].rule.hi,
                          tuple(sets[pq[j].set0 + pc[pq[j].rule0 + r].rule.in_off:][: pc[pq[j].rule0 + r].rule.n_in]),
                          pc[pq[j].rule0 + r].rule.negate, int(adds[pq[j].rule0 + r]), pc[pq[j].rule0 + r].attr)
                         for r in range(pq[j].n_rules)] for j in range(len(queries))]}


def test_plan_groups_rules_by_attribute(H):
    attrs = Attrs([np.arange(10), np.arange(10) * 2, np.arange(10) * 3])
    # a recency ladder over attribute 0 interleaved with rules over 1 and 2
    rules = [(0, 0, 1, None, False, 30), (1, 0, 5, None, False, 15), (0, 0, 3, None, False, 20), (2, 0, 0, [4, 4, 2], True, 1),
             (0, 0, 7, None, False, 10), (1, 0, 0, [], False, 99), (0, 0, 9, None, False, 5)]
    p = plan(H, attrs, [rules])
    got = p["queries"][0]
    # attributes in order of first appearance, the rules of one attribute adjacent and in their order
    assert [r[6] for r in got] == [0, 0, 0, 0, 1, 1, 2]
    assert [r[5] for r in got] == [30, 20, 10, 5, 15, 99, 1]
    assert got[6][3] == (2, 4) and got[5][3] == ()   # set values sorted and de-duplicated; a range clause has none
    assert p["attrs"] == [attrs.recs[k].values for k in range(3)]
    assert p["staged"] == 3


@pytest.mark.parametrize("q", [1, 2, 7, 20])
def test_batched_plan_equals_single_plans(H, q):
    rng = np.random.default_rng(q)
    pool = np.arange(-4, 5, dtype=np.int64)
    attrs = Attrs([rng.choice(pool, 50) for _ in range(7)])
    queries = [[random_rule(rng, 7, pool) for _ in range(int(rng.integers(0, 9)))] for _ in range(q)]
    batched = plan(H, attrs, queries)
    assert batched["staged"] == min(STAGED, len({r[0] for qr in queries for r in qr}))
    for j in range(q):
        single = plan(H, attrs, [queries[j]])["queries"][0]
        # the same rules, attributes (by their values), bounds, set values and adds; only the table places differ
        assert [r[:6] for r in batched["queries"][j]] == [r[:6] for r in single], j


def test_staged_and_unstaged_attributes(H):
    """More distinct attributes than are staged: the rest are read from the attribute, with the same result."""
    rng = np.random.default_rng(3)
    n = 3 * CHUNK + 100
    pool = np.arange(-3, 4, dtype=np.int64)
    attrs = Attrs([random_values(rng, n - 40 * k, pool) for k in range(7)])
    queries = [[(k, -1, 1, None, False, 100 + k) for k in range(7)] + [(6, 0, 0, [2, 3], True, -9)],
               [(6, 0, 2, None, False, 4), (5, 0, 0, [0], False, 8)]]
    outs, maxima, loads = run_fill(H, attrs, queries, n)
    for j, rules in enumerate(queries):
        want, want_max = spec_fill(attrs, rules, n)
        assert np.array_equal(outs[j], want) and maxima[j] == want_max
    assert list(loads) == [7 * n, 2 * n]


def test_argument_checks_and_no_device():
    import torch
    L = F.lib()
    fake = C.create_string_buffer(4096)            # a corpus of 0 haystacks; never written
    c = C.addressof(fake)
    handles = [C.create_string_buffer(c.to_bytes(8, "little"), 256) for _ in range(5)]   # boosts / attributes of it
    other = C.create_string_buffer(256)            # a handle whose corpus (its first field) is NULL: another corpus
    b0, b1, b2, bx, a = (C.addressof(h) for h in handles)
    oth = C.addressof(other)
    snaps = [h.raw for h in handles] + [other.raw]
    big = np.arange(4097, dtype=np.int64)
    bad = np.array([1, NULL, 2], dtype=np.int64)

    def rules(*rs):
        arr = (F._CBoostRule * max(1, len(rs)))()
        for j, (attr, lo, hi, in_, n_in, add) in enumerate(rs):
            w = arr[j].when
            w.attr, w.lo, w.hi, w.in_, w.n_in = attr, lo, hi, in_, n_in
            arr[j].add = add
        return arr

    def hs(*xs):
        return (vp * max(1, len(xs)))(*xs)

    def counts(*k):
        return np.array(k or [0], dtype=np.uint64)

    one = L.frz_boost_where
    r = (a, 0, 5, None, 0, 10)
    # the single call, in its order; the message names the rule
    cases = [
        ((None, rules(r), 1, None), INVALID, b"null argument"),
        ((b0, None, 1, None), INVALID, b"null argument"),
        ((b0, rules(*[r] * 9), 9, None), UNSUPPORTED, b"9 rules (at most 8)"),
        ((b0, rules(r, (None, 0, 5, None, 0, 1)), 2, None), INVALID, b"null argument in rule 1"),
        ((b0, rules(r, (a, 0, 0, None, 3, 1)), 2, None), INVALID, b"null argument in rule 1"),
        ((b0, rules(r, (a, 0, 5, None, 0, 65536)), 2, None), INVALID, b"rule 1 adds 65536"),
        ((b0, rules((a, 0, 5, None, 0, -65536)), 1, None), INVALID, b"rule 0 adds -65536"),
        ((b0, rules((a, 0, 0, big.ctypes.data, 2048, 1), (a, 0, 0, big.ctypes.data, 2049, 1)), 2, None), UNSUPPORTED,
         b"more than 4096 set values"),
        ((b0, rules((a, 0, 0, big.ctypes.data, 2**64 - 1, 1)), 1, None), UNSUPPORTED, b"more than 4096"),
        ((b0, rules(r, (a, 0, 0, bad.ctypes.data, 3, 1)), 2, None), INVALID, b"set value 1 of rule 1 is FRZ_ATTR_NULL"),
        ((b0, rules(r, (oth, 0, 5, None, 0, 1)), 2, None), INVALID, b"the attribute of rule 1 was made on another corpus"),
        ((b0, rules(r), 1, oth), INVALID, b"the base boost was made on another corpus"),
        # earlier checks win: 3 before 4, 4 before 5, 5 before 6, 6 before 7
        ((b0, rules((a, 0, 5, None, 0, 70000), (None, 0, 5, None, 0, 1)), 2, None), INVALID, b"null argument in rule 1"),
        ((b0, rules((a, 0, 0, big.ctypes.data, 4097, 70000)), 1, None), INVALID, b"rule 0 adds 70000"),
        ((b0, rules((a, 0, 0, bad.ctypes.data, 3, 1), (a, 0, 0, big.ctypes.data, 4096, 1)), 2, None), UNSUPPORTED, b"more than 4096"),
        ((b0, rules((oth, 0, 0, bad.ctypes.data, 3, 1)), 1, None), INVALID, b"set value 1 of rule 0"),
    ]
    for args, status, msg in cases:
        assert one(*args) == status, msg
        assert msg in L.frz_last_error(), (msg, L.frz_last_error())
    # the batch: NULL arrays, then query by query the single call's checks, then corpora, then aliasing
    fn = L.frz_boost_where_batch
    assert fn(None, 2, rules(r, r), counts(1, 1).ctypes.data, None) == INVALID
    assert fn(hs(b0, b1), 2, rules(r, r), None, None) == INVALID
    assert b"null argument" in L.frz_last_error()
    bcases = [
        ((hs(b0, None), rules(r, r), counts(1, 1), None), INVALID, b"query 1: null argument"),
        ((hs(b0, b1), rules(r, *[r] * 9), counts(1, 9), None), UNSUPPORTED, b"query 1: 9 rules"),
        ((hs(b0, b1), rules(r, (a, 0, 5, None, 0, -70000)), counts(1, 1), None), INVALID, b"query 1: rule 0 adds -70000"),
        ((hs(b0, b1), rules(r, (a, 0, 0, bad.ctypes.data, 3, 1)), counts(1, 1), None), INVALID,
         b"query 1: set value 1 of rule 0 is FRZ_ATTR_NULL"),
        # the per-query limits hold per query: 2 x 4096 set values pass them (and fail the corpus check)
        ((hs(b0, b1), rules((a, 0, 0, big.ctypes.data, 4096, 1), (oth, 0, 0, big.ctypes.data, 4096, 1)), counts(1, 1), None),
         INVALID, b"query 1: the attribute of rule 0 was made on another corpus"),
        # query 0's later check is not reached before query 1's earlier one
        ((hs(b0, b1), rules((oth, 0, 5, None, 0, 1), (a, 0, 5, None, 0, 70000)), counts(1, 1), None), INVALID,
         b"query 1: rule 0 adds 70000"),
        ((hs(b0, oth), rules(r, r), counts(1, 1), None), INVALID, b"query 1: the boost was made on another corpus"),
        ((hs(b0, b1), rules(r, r), counts(1, 1), hs(None, oth)), INVALID, b"query 1: the base boost was made on another corpus"),
        # corpora before aliasing
        ((hs(b0, b0), rules(r, (oth, 0, 5, None, 0, 1)), counts(1, 1), None), INVALID, b"query 1: the attribute of rule 0"),
        ((hs(b0, b1, b0), rules(r, r, r), counts(1, 1, 1), hs(None, None, b1)), INVALID, b"query 2: the boost is also query 0's"),
        ((hs(b0, b1, b2), rules(r, r, r), counts(1, 1, 1), hs(None, b0, None)), INVALID, b"query 1: the base is query 0's boost"),
    ]
    for (bs, rl, k, bases), status, msg in bcases:
        assert fn(bs, len(k), rl, k.ctypes.data, bases) == status, msg
        assert msg in L.frz_last_error(), (msg, L.frz_last_error())
    assert [h.raw for h in handles] + [other.raw] == snaps and fake.raw == b"\0" * 4096
    # q == 0 makes no CUDA call, whatever the arrays
    assert fn(None, 0, None, None, None) == 0
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    # every argument is valid: the call reaches the device check, the handles untouched.  A base may be the boost itself
    # or a boost no query fills, shared by several queries.
    ok_set = np.array([3, 1, 3], dtype=np.int64)
    assert one(b0, rules(*[(a, 0, 0, big.ctypes.data, 512, 65535)] * 8), 8, b0) == NO_DEVICE
    assert one(b0, None, 0, None) == NO_DEVICE
    for bs, q, rl, k, bases in ((hs(b0), 1, rules(r), counts(1), None),
                                (hs(b0, b1, b2), 3, None, counts(0, 0, 0), hs(b0, bx, bx)),
                                (hs(b0, b1), 2, rules(*[(a, 0, 0, big.ctypes.data, 512, -65535)] * 16), counts(8, 8), hs(None, b1)),
                                (hs(b0, b1), 2, rules((a, 0, 0, ok_set.ctypes.data, 3, 1)), counts(0, 1), hs(b2, b2))):
        assert fn(bs, q, rl, k.ctypes.data, bases) == NO_DEVICE
    assert [h.raw for h in handles] + [other.raw] == snaps
