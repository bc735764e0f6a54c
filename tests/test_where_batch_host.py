"""frz_subset_where_batch without a GPU: frizbee_b200/csrc/where_plan.cuh built for the CPU
(tests/harness/where_batch_harness.cpp).  Its packer (the call's distinct-attribute table, the clauses as references into
it, every query's set values) against a Python restatement, k_where_batch's staged word rule against numpy, and the
argument checks of frz_subset_where_batch in their documented order on zero-filled stand-in handles.  The behaviour on a
real corpus is in tests/test_gpu_where_batch.py."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from cpu_harness import load
from test_where_host import Clause, NULL, random_values, spec_holds

INVALID, UNSUPPORTED, NO_DEVICE = 1, 9, 8
STAGED = 4            # kFrzWhereBatchStaged
CHUNK = 1024          # kFrzWhereChunk
vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32


class BAttr(C.Structure):     # FrzWhereBatchAttr
    _fields_ = [("values", vp), ("n_values", u64)]


class BClause(C.Structure):   # FrzWhereBatchClause
    _fields_ = [("rule", Clause), ("attr", u32), ("pad_", u32)]


class BQuery(C.Structure):    # FrzWhereBatchQuery
    _fields_ = [("clause0", u32), ("n_clauses", u32), ("set0", u64), ("base", vp), ("n_base", u64), ("has_base", u32),
                ("pad_", u32), ("bits", vp), ("chunk_count", vp), ("chunk_base", vp), ("members", vp)]


class BDev(C.Structure):      # FrzWhereBatchDev
    _fields_ = [("attrs", vp), ("clauses", vp), ("queries", vp), ("sets", vp), ("n", u64), ("q", u32), ("n_staged", u32)]


@pytest.fixture(scope="module")
def H():
    L = load("where_batch_harness")
    L.h_where_batch_pack.argtypes = [vp, vp, u64]
    L.h_where_batch_pack.restype = u64
    L.h_where_batch_plan.argtypes = [vp, vp, vp, vp, vp]
    L.h_where_batch_plan.restype = None
    L.h_where_batch_word.argtypes = [vp, u32, u64]
    L.h_where_batch_word.restype = u32
    return L


class Attrs:
    """Stand-in attributes: each handle is the address of a FrzWhereBatchAttr over a numpy array."""

    def __init__(self, arrays):
        self.arrays = [np.ascontiguousarray(a, dtype=np.int64) for a in arrays]
        self.recs = (BAttr * len(arrays))()
        for j, a in enumerate(self.arrays):
            self.recs[j] = BAttr(a.ctypes.data if a.size else None, len(a))
        self.handles = [C.addressof(self.recs) + j * C.sizeof(BAttr) for j in range(len(arrays))]


def abi_clauses(flat, attrs):
    """frz_where_clause records for (attr index, lo, hi, set values or None, negate); the arrays are kept alive."""
    arr = (F._CWhereClause * max(1, len(flat)))()
    keep = []
    for j, (a, lo, hi, in_, neg) in enumerate(flat):
        arr[j].attr, arr[j].lo, arr[j].hi, arr[j].negate = attrs.handles[a], lo, hi, int(neg)
        if in_ is not None:
            v = np.ascontiguousarray(in_, dtype=np.int64)
            keep.append(v)
            arr[j].in_, arr[j].n_in = v.ctypes.data, len(v)
    return arr, keep


def pack(H, queries, attrs):
    """The harness's plan of `queries` (lists of clause tuples): (attrs, clauses, queries, sets, n_staged)."""
    flat = [c for qc in queries for c in qc]
    arr, keep = abi_clauses(flat, attrs)
    n_cl = np.array([len(qc) for qc in queries] or [0], dtype=np.uint64)
    H.h_where_batch_pack(arr, n_cl.ctypes.data, len(queries))
    sizes = np.zeros(4, np.uint64)
    H.h_where_batch_plan(sizes.ctypes.data, None, None, None, None)
    na, nc, ns, staged = (int(x) for x in sizes)
    pa, pc, pq = (BAttr * max(1, na))(), (BClause * max(1, nc))(), (BQuery * max(1, len(queries)))()
    ps = np.zeros(max(1, ns), np.int64)
    H.h_where_batch_plan(sizes.ctypes.data, pa, pc, pq, ps.ctypes.data)
    return pa, pc, pq, ps, na, nc, ns, staged


def spec_plan(queries):
    """The plan restated: the distinct attributes in order of first appearance, each clause's (place, lo, hi, in_off,
    n_in, negate) with in_off relative to its query's first set value, each query's (clause0, n_clauses, set0), and the
    set values, sorted and de-duplicated per clause."""
    place, table, clauses, qs, sets = {}, [], [], [], []
    for qc in queries:
        qs.append((len(clauses), len(qc), len(sets)))
        set0 = len(sets)
        for a, lo, hi, in_, neg in qc:
            if a not in place:
                place[a] = len(table)
                table.append(a)
            u = np.unique(np.asarray(in_, np.int64)).tolist() if in_ is not None and len(in_) else []
            clauses.append((place[a], lo, hi, len(sets) - set0, len(u), int(neg)))
            sets += u
    return table, clauses, qs, sets


def random_queries(rng, q, n_attrs, max_clauses=8):
    out = []
    for _ in range(q):
        qc = []
        for _ in range(int(rng.integers(0, max_clauses + 1))):
            a = int(rng.integers(0, n_attrs))
            neg = bool(rng.random() < 0.3)
            if rng.random() < 0.5:
                lo, hi = (int(x) for x in rng.integers(-4, 12, 2))
                qc.append((a, lo, hi, None, neg))
            else:
                qc.append((a, 0, -1, rng.integers(-4, 12, int(rng.integers(1, 9))).tolist(), neg))
        out.append(qc)
    return out


@pytest.mark.parametrize("q,n_attrs", [(1, 1), (3, 2), (7, 4), (40, 9), (300, 3)])
def test_packer_against_restatement(H, q, n_attrs):
    rng = np.random.default_rng(q * 100 + n_attrs)
    attrs = Attrs([np.arange(5 + j, dtype=np.int64) for j in range(n_attrs)])
    queries = random_queries(rng, q, n_attrs)
    queries[0] = [(n_attrs - 1, 0, 5, None, False)] + queries[0][:7]   # first appearance is not index order
    pa, pc, pq, ps, na, nc, ns, staged = pack(H, queries, attrs)
    table, clauses, qs, sets = spec_plan(queries)
    assert na == len(table) and staged == min(len(table), STAGED)
    for t, a in enumerate(table):   # each distinct attribute once, with its handle's values
        assert pa[t].values == attrs.recs[a].values and pa[t].n_values == len(attrs.arrays[a])
    assert nc == len(clauses)
    for j, (place, lo, hi, off, nin, neg) in enumerate(clauses):
        c = pc[j]
        assert (c.attr, c.rule.lo, c.rule.hi, c.rule.in_off, c.rule.n_in, c.rule.negate) == (place, lo, hi, off, nin, neg), j
        assert c.rule.values == pa[place].values and c.rule.n_values == pa[place].n_values
    for j, (c0, k, s0) in enumerate(qs):
        assert (pq[j].clause0, pq[j].n_clauses, pq[j].set0) == (c0, k, s0), j
        assert pq[j].base is None and pq[j].has_base == 0 and pq[j].bits is None
    assert ns == len(sets) and ps[:ns].tolist() == sets


def test_packer_shares_attributes_across_queries(H):
    attrs = Attrs([np.zeros(3, np.int64) for _ in range(6)])
    queries = [[(2, 0, 1, None, False), (5, 0, 0, [3, 1, 3], True)], [], [(5, 1, 1, None, False), (2, 0, 0, [7], False)],
               [(0, 0, 0, None, False), (1, 0, 0, None, False), (3, 0, 0, None, False), (4, 0, 0, None, False)]]
    pa, pc, pq, ps, na, nc, ns, staged = pack(H, queries, attrs)
    assert na == 6 and staged == STAGED   # more distinct attributes than are staged
    assert [pc[j].attr for j in range(nc)] == [0, 1, 1, 0, 2, 3, 4, 5]
    assert [(pq[j].clause0, pq[j].n_clauses, pq[j].set0) for j in range(4)] == [(0, 2, 0), (2, 0, 2), (2, 2, 2), (4, 4, 3)]
    assert ps[:ns].tolist() == [1, 3, 7] and pc[3].rule.in_off == 0 and pc[1].rule.in_off == 0


def run_words(H, attrs, queries, n, bases):
    """Every query's bitmap from h_where_batch_word over the packed plan; bases[j]: None or (bitmap words, n_base)."""
    pa, pc, pq, ps, na, nc, ns, staged = pack(H, queries, attrs)
    keep = []
    for j, b in enumerate(bases):
        if b is not None:
            words, n_base = b
            keep.append(words)
            pq[j].base, pq[j].n_base, pq[j].has_base = words.ctypes.data, n_base, 1
    d = BDev(C.addressof(pa), C.addressof(pc), C.addressof(pq), ps.ctypes.data, n, len(queries), staged)
    n_words = (n + 31) // 32
    out = np.zeros((len(queries), n_words), np.uint32)
    for j in range(len(queries)):
        for w in range(n_words):
            out[j, w] = H.h_where_batch_word(C.byref(d), j, w)
    return out


def bits_of(mask):
    n = len(mask)
    padded = np.zeros(((n + 31) // 32) * 32, bool)
    padded[:n] = mask
    return np.packbits(padded.reshape(-1, 32)[:, ::-1], axis=1, bitorder="big").view(">u4").ravel().astype(np.uint32)


@pytest.mark.parametrize("n", [1, 31, 33, 1024, 1025, 3 * 1024 + 7])
def test_staged_words_against_numpy(H, n):
    rng = np.random.default_rng(n)
    n_attrs = 6   # two past the staged limit
    arrays = []
    for a in range(n_attrs):
        m = int(rng.integers(0, n + 1)) if a % 2 else n   # rows past a short attribute are null
        arrays.append(random_values(rng, m, np.arange(-4, 12)) if m else np.zeros(0, np.int64))
    attrs = Attrs(arrays)
    full = []
    for v in arrays:
        f = np.full(n, NULL, np.int64)
        f[: len(v)] = v
        full.append(f)
    q = 9
    queries = random_queries(rng, q, n_attrs)
    bases, masks = [], []
    for j, qc in enumerate(queries):
        mask = np.ones(n, bool)
        for a, lo, hi, in_, neg in qc:
            mask &= spec_holds(full[a], lo, hi, in_, neg)
        base = None
        if j % 3:
            n_base = int(rng.integers(0, n + 1)) if j % 3 == 1 else n   # a base shorter than the corpus
            bm = rng.random(n_base) < 0.6
            base = (bits_of(bm) if n_base else np.zeros(1, np.uint32), n_base)
            full_b = np.zeros(n, bool)
            full_b[:n_base] = bm
            mask &= full_b
        bases.append(base)
        masks.append(mask)
    got = run_words(H, attrs, queries, n, bases)
    for j in range(q):
        assert np.array_equal(got[j], bits_of(masks[j])), j   # the tail of the last word is zero


def test_argument_checks_and_no_device():
    import torch
    L = F.lib()
    L.frz_subset_where_batch.argtypes = [vp, u64, vp, vp, vp]
    fake = C.create_string_buffer(4096)            # a corpus of 0 haystacks; never written
    c = C.addressof(fake)
    handles = [C.create_string_buffer(c.to_bytes(8, "little"), 256) for _ in range(4)]   # subsets / attributes of it
    other = C.create_string_buffer(256)            # a handle whose corpus (its first field) is NULL: another corpus
    s0, s1, s2, a = (C.addressof(h) for h in handles)
    oth = C.addressof(other)
    snaps = [h.raw for h in handles] + [other.raw]

    def subs(*xs):
        return (vp * max(1, len(xs)))(*xs)

    def clauses(*cl):
        arr = (F._CWhereClause * max(1, len(cl)))()
        for j, (attr, lo, hi, in_, n_in, neg) in enumerate(cl):
            arr[j].attr, arr[j].lo, arr[j].hi, arr[j].in_, arr[j].n_in, arr[j].negate = attr, lo, hi, in_, n_in, neg
        return arr

    def counts(*k):
        return np.array(k or [0], dtype=np.uint64)

    fn = L.frz_subset_where_batch
    rng = (a, 0, 5, None, 0, 0)
    one = counts(1, 1)
    big = np.arange(4097, dtype=np.int64)
    bad = np.array([1, NULL, 2], dtype=np.int64)
    # 1. NULL arrays with q > 0
    assert fn(None, 2, clauses(rng, rng), one.ctypes.data, None) == INVALID
    assert fn(subs(s0, s1), 2, clauses(rng, rng), None, None) == INVALID
    assert b"null argument" in L.frz_last_error()
    # 2. query by query, frz_subset_where's checks in its order: the first failing query's first failing check wins
    cases = [
        ((subs(s0, None), clauses(rng, rng), one), INVALID, b"query 1: null argument"),
        ((subs(s0, s1), None, one), INVALID, b"query 0: null argument"),
        ((subs(s0, s1), clauses(*[rng] * 10), counts(1, 9)), UNSUPPORTED, b"query 1: 9 clauses"),
        ((subs(s0, s1), clauses(rng, (None, 0, 5, None, 0, 0)), one), INVALID, b"query 1: null argument in clause 0"),
        ((subs(s0, s1), clauses(rng, (a, 0, 0, None, 3, 0)), one), INVALID, b"query 1: null argument in clause 0"),
        ((subs(s0, s1), clauses(rng, (a, 0, 0, big.ctypes.data, 2048, 0), (a, 0, 0, big.ctypes.data, 2049, 0)), counts(1, 2)),
         UNSUPPORTED, b"query 1: more than 4096 set values"),
        ((subs(s0, s1), clauses((a, 0, 0, big.ctypes.data, 2**64 - 1, 0), rng), one), UNSUPPORTED, b"query 0: more than 4096"),
        ((subs(s0, s1), clauses(rng, (a, 0, 0, bad.ctypes.data, 3, 0)), one), INVALID, b"query 1: set value 1 of clause 0 is FRZ_ATTR_NULL"),
        # the per-query limits hold per query: 2 x 4096 set values and 2 x 8 clauses pass them (and fail the corpus check)
        ((subs(s0, s1), clauses((a, 0, 0, big.ctypes.data, 4096, 0), (oth, 0, 0, big.ctypes.data, 4096, 0)), one), INVALID,
         b"query 1: the attribute was made on another corpus"),
        # query 0's later check is not reached before query 1's earlier one
        ((subs(s0, s1), clauses((a, 0, 0, bad.ctypes.data, 3, 0), *[rng] * 9), counts(1, 9)), UNSUPPORTED, b"query 1: 9 clauses"),
    ]
    for (ss, cl, k), status, msg in cases[:9]:
        assert fn(ss, 2, cl, k.ctypes.data, None) == status, msg
        assert msg in L.frz_last_error(), (msg, L.frz_last_error())
    ss, cl, k = cases[9][0]
    assert fn(ss, 2, cl, k.ctypes.data, None) == INVALID   # query 0's NULL set value comes first: queries go in order
    assert b"query 0: set value 1" in L.frz_last_error()
    # 3. a subset, attribute or base of another corpus, query by query
    assert fn(subs(s0, oth), 2, clauses(rng, rng), one.ctypes.data, None) == INVALID
    assert b"query 1: the subset was made on another corpus" in L.frz_last_error()
    assert fn(subs(s0, s1), 2, clauses(rng, (oth, 0, 5, None, 0, 0)), one.ctypes.data, None) == INVALID
    assert b"query 1: the attribute was made on another corpus" in L.frz_last_error()
    assert fn(subs(s0, s1), 2, clauses(rng, rng), one.ctypes.data, subs(None, oth)) == INVALID
    assert b"query 1: the base subset was made on another corpus" in L.frz_last_error()
    assert fn(subs(s0, s0), 2, clauses(rng, (oth, 0, 5, None, 0, 0)), one.ctypes.data, None) == INVALID   # 3 before 4
    assert b"another corpus" in L.frz_last_error()
    # 4. a duplicate subset
    assert fn(subs(s0, s1, s0), 3, clauses(rng, rng, rng), counts(1, 1, 1).ctypes.data, subs(None, None, s1)) == INVALID
    assert b"query 2: the subset is also query 0's" in L.frz_last_error()   # 4 before 5
    # 5. a base that is another query's subset
    assert fn(subs(s0, s1, s2), 3, clauses(rng, rng, rng), counts(1, 1, 1).ctypes.data, subs(None, s0, None)) == INVALID
    assert b"query 1: the base is query 0's subset" in L.frz_last_error()
    assert [h.raw for h in handles] + [other.raw] == snaps and fake.raw == b"\0" * 4096
    # q == 0 makes no CUDA call, whatever the arrays
    assert fn(None, 0, None, None, None) == 0
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    # every argument is valid: the call reaches the device check, the handles untouched.  Bases may be the query's own
    # subset or a subset no query fills, shared by several queries.
    ok_set = np.array([3, 1, 3], dtype=np.int64)
    for ss, q, cl, k, bs in ((subs(s0), 1, clauses(rng), counts(1), None),
                             (subs(s0, s1, s2), 3, None, counts(0, 0, 0), subs(s0, a, a)),
                             (subs(s0, s1), 2, clauses(*[rng] * 8, (a, 0, 0, big.ctypes.data, 4096, 1), *[rng] * 7),
                              counts(8, 8), subs(None, s1)),
                             (subs(s0, s1), 2, clauses((a, 0, 0, ok_set.ctypes.data, 3, 0)), counts(0, 1), subs(s2, s2))):
        assert fn(ss, q, cl, k.ctypes.data, bs) == NO_DEVICE
    assert [h.raw for h in handles] + [other.raw] == snaps
