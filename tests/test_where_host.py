"""frz_subset_where without a GPU: frizbee_b200/csrc/where_plan.cuh built for the CPU (tests/harness/where_harness.cpp)
against a numpy restatement of the clauses, the set packing and the whole fill (words, chunk counts, scan and member
expansion), and the argument checks of frz_attr_* / frz_subset_where on zero-filled stand-in handles.  The behaviour on a
real corpus is in tests/test_gpu_where.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import frizbee_b200 as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "harness", "where_harness.cpp")
LIB = os.path.join(ROOT, "tests", "harness", "libwhere_harness.so")
DEPS = [SRC, os.path.join(ROOT, "frizbee_b200", "csrc", "where_plan.cuh")]
INVALID, UNSUPPORTED, NO_DEVICE = 1, 9, 8
NULL = -(2**63)
I64_MAX = 2**63 - 1
MAX_CLAUSES = 8
vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32


class Clause(C.Structure):   # FrzWhereClauseDev
    _fields_ = [("values", vp), ("n_values", u64), ("lo", C.c_int64), ("hi", C.c_int64), ("in_off", u32), ("n_in", u32),
                ("negate", u32), ("pad_", u32)]


class Fill(C.Structure):     # FrzWhereDev
    _fields_ = [("clauses", Clause * MAX_CLAUSES), ("sets", vp), ("base", vp), ("bits", vp), ("chunk_count", vp),
                ("n", u64), ("n_base", u64), ("n_clauses", u32), ("n_sets", u32), ("has_base", u32), ("pad_", u32)]


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", LIB, SRC], check=True)
    L = C.CDLL(LIB)
    L.h_where_holds.argtypes = [vp, vp, vp, u64, vp]
    L.h_where_holds.restype = None
    L.h_where_pack.argtypes = [vp, u64, vp]
    L.h_where_pack.restype = u32
    L.h_where_fill.argtypes = [vp, vp]
    L.h_where_fill.restype = u64
    return L


def spec_holds(values, lo=0, hi=-1, in_=None, negate=False):
    """The clause over int64 values, restated: null fails, negated or not."""
    values = np.asarray(values, dtype=np.int64)
    t = np.isin(values, np.asarray(in_, dtype=np.int64)) if in_ is not None else (lo <= values) & (values <= hi)
    return (t != negate) & (values != NULL)


def random_values(rng, n, pool=None):
    v = rng.integers(-2**63 + 1, 2**63 - 1, size=n, dtype=np.int64, endpoint=True) if pool is None else rng.choice(pool, size=n)
    v = np.asarray(v, dtype=np.int64)
    v[rng.random(n) < 0.1] = NULL
    extremes = np.array([NULL + 1, I64_MAX, -1, 0, 1, NULL], dtype=np.int64)
    v[: len(extremes)] = extremes[: n]
    return v


def holds(H, values, lo=0, hi=-1, in_=None, negate=False):
    values = np.ascontiguousarray(values, dtype=np.int64)
    c = Clause(0, 0, lo, hi, 0, 0, int(negate), 0)
    sets = np.zeros(1, np.int64)
    if in_ is not None:
        sets = np.unique(np.asarray(in_, dtype=np.int64))
        c.n_in = len(sets)
    out = np.zeros(len(values), np.uint8)
    H.h_where_holds(C.byref(c), sets.ctypes.data, values.ctypes.data, len(values), out.ctypes.data)
    return out.astype(bool)


def test_range_clauses(H):
    rng = np.random.default_rng(1)
    v = random_values(rng, 4000)
    ranges = [(NULL + 1, I64_MAX), (0, 0), (-5, 5), (5, -5), (I64_MAX, I64_MAX), (NULL + 1, NULL + 1), (NULL, I64_MAX),
              (-2**62, 2**62), (1, 0)]
    for lo, hi in ranges + [tuple(sorted(rng.integers(-2**63 + 1, 2**63 - 1, 2))) for _ in range(20)]:
        for neg in (False, True):
            assert np.array_equal(holds(H, v, lo, hi, negate=neg), spec_holds(v, lo, hi, negate=neg)), (lo, hi, neg)
    # a null value fails every clause, negated or not, even a full-range one
    assert not holds(H, [NULL], NULL, I64_MAX).any() and not holds(H, [NULL], 1, 0, negate=True).any()


def test_set_clauses(H):
    rng = np.random.default_rng(2)
    pool = np.array([NULL + 1, I64_MAX, -7, 0, 3, 1000, 2**40], dtype=np.int64)
    v = random_values(rng, 3000, pool)
    sets = [[3], [I64_MAX, NULL + 1], [3, 3, -7, 3, 0, -7], list(rng.permutation(pool[:5])),
            list(rng.integers(-10**6, 10**6, 4096)), list(np.concatenate([pool, pool]))]
    for s in sets:
        for neg in (False, True):
            assert np.array_equal(holds(H, v, in_=s, negate=neg), spec_holds(v, in_=s, negate=neg))
    big = rng.integers(-2**63 + 1, 2**63 - 1, 4096, dtype=np.int64)
    w = np.concatenate([big, big + 1, random_values(rng, 500)])
    assert np.array_equal(holds(H, w, in_=big), spec_holds(w, in_=big))


def test_set_packing(H):
    rng = np.random.default_rng(3)
    for s in ([5], [3, 1, 2, 3, 1], [I64_MAX, NULL + 1, 0, I64_MAX], rng.integers(-50, 50, 4096)):
        s = np.ascontiguousarray(s, dtype=np.int64)
        out = np.zeros(len(s), np.int64)
        k = H.h_where_pack(s.ctypes.data, len(s), out.ctypes.data)
        assert np.array_equal(out[:k], np.unique(s))


def fill(H, n, clauses, sets, base=None, n_base=0, in_place=False):
    """The harness's fill over n indices; clauses: (values array, lo, hi, in_off, n_in, negate)."""
    f = Fill()
    keep = []
    for j, (vals, lo, hi, off, nin, neg) in enumerate(clauses):
        vals = np.ascontiguousarray(vals, dtype=np.int64)
        keep.append(vals)
        f.clauses[j] = Clause(vals.ctypes.data if vals.size else None, len(vals), lo, hi, off, nin, int(neg), 0)
    sets = np.ascontiguousarray(sets if len(sets) else [0], dtype=np.int64)
    n_words = (n + 31) // 32
    bits = base if in_place else np.full(max(1, n_words), 0xDEADBEEF, np.uint32)
    counts = np.full(max(1, (n + 1023) // 1024), 0xDEADBEEF, np.uint32)
    members = np.zeros(max(1, n), np.uint32)
    f.sets, f.bits, f.chunk_count, f.n, f.n_clauses, f.n_sets = sets.ctypes.data, bits.ctypes.data, counts.ctypes.data, n, len(clauses), len(sets)
    if base is not None:
        f.base, f.n_base, f.has_base = base.ctypes.data, n_base, 1
    total = H.h_where_fill(C.byref(f), members.ctypes.data)
    return bits[:n_words], counts[: (n + 1023) // 1024], members[:total]


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 1023, 1024, 1025, 3 * 1024 + 7, 40000])
def test_fill_against_numpy(H, n):
    rng = np.random.default_rng(n)
    for trial in range(6):
        n_clauses = int(rng.integers(0, MAX_CLAUSES + 1))
        clauses, sets, mask = [], [], np.ones(n, bool)
        for _ in range(n_clauses):
            n_values = int(rng.integers(0, n + 1))   # rows past the attribute's array are null
            vals = random_values(rng, n_values, np.arange(-4, 12)) if n_values else np.zeros(0, np.int64)
            full = np.full(n, NULL, np.int64)
            full[:n_values] = vals
            neg = bool(rng.random() < 0.3)
            if rng.random() < 0.5:
                lo, hi = sorted(rng.integers(-4, 12, 2))
                clauses.append((vals, int(lo), int(hi), 0, 0, neg))
                mask &= spec_holds(full, lo, hi, negate=neg)
            else:
                s = rng.integers(-4, 12, int(rng.integers(1, 6)))
                u = np.unique(s)
                clauses.append((vals, 0, -1, len(sets), len(u), neg))
                sets.extend(u.tolist())
                mask &= spec_holds(full, in_=s, negate=neg)
        base = None
        n_base = 0
        if trial % 2:
            n_base = int(rng.integers(0, n + 1))   # a base made before rows were appended
            bmask = rng.random(n_base) < 0.7
            base = np.zeros(max(1, (n_base + 31) // 32), np.uint32)
            for i in np.flatnonzero(bmask):
                base[i >> 5] |= np.uint32(1 << (i & 31))
            full_b = np.zeros(n, bool)
            full_b[:n_base] = bmask
            mask &= full_b
        in_place = base is not None and trial == 3 and len(base) >= (n + 31) // 32
        bits, counts, members = fill(H, n, clauses, sets, base, n_base, in_place)
        want = np.flatnonzero(mask).astype(np.uint32)
        assert np.array_equal(members, want)
        want_bits = np.zeros((n + 31) // 32, np.uint32)
        for i in want:
            want_bits[i >> 5] |= np.uint32(1 << (i & 31))
        assert np.array_equal(bits, want_bits)   # the tail of the last word is zero
        per_chunk = np.bincount(want // 1024, minlength=(n + 1023) // 1024) if n else np.zeros(0)
        assert np.array_equal(counts, per_chunk)


def test_member_expansion_across_words_and_chunks(H):
    n = 5 * 1024 + 13
    idx = np.array([0, 31, 32, 63, 1023, 1024, 1025, 2047, 2048, 4095, 4096, n - 1], dtype=np.int64)
    vals = np.full(n, 0, np.int64)
    vals[idx] = 7
    _, counts, members = fill(H, n, [(vals, 7, 7, 0, 0, False)], [])
    assert np.array_equal(members, idx.astype(np.uint32))
    _, _, all_ = fill(H, n, [], [])
    assert np.array_equal(all_, np.arange(n, dtype=np.uint32))
    _, _, rest = fill(H, n, [(vals, 7, 7, 0, 0, True)], [])
    assert np.array_equal(rest, np.setdiff1d(np.arange(n), idx).astype(np.uint32))


def test_argument_checks_and_no_device():
    import torch
    L = F.lib()
    fake = C.create_string_buffer(4096)            # a corpus of 0 haystacks; never written
    c = C.addressof(fake)
    mine = C.create_string_buffer(c.to_bytes(8, "little"), 256)    # a subset / attribute of the fake corpus
    other = C.create_string_buffer(256)            # a handle whose corpus (its first field) is NULL: another corpus
    s, a, oth = C.addressof(mine), C.addressof(mine), C.addressof(other)
    snap_mine, snap_other = mine.raw, other.raw
    vals = np.array([1, 2], dtype=np.int64)
    which = np.array([0, 1], dtype=np.uint32)
    h = C.c_void_p()
    # frz_attr_create: NULL corpus, NULL out, NULL values with n > 0, n > the corpus's length
    assert L.frz_attr_create(None, vals.ctypes.data, 2, C.byref(h)) == INVALID
    assert L.frz_attr_create(c, vals.ctypes.data, 2, None) == INVALID
    assert L.frz_attr_create(c, None, 1, C.byref(h)) == INVALID
    assert b"null" in L.frz_last_error()
    assert L.frz_attr_create(c, vals.ctypes.data, 2, C.byref(h)) == INVALID
    assert b"haystacks" in L.frz_last_error() and not h.value
    # frz_attr_set: NULL handle, NULL arrays with n > 0, an index past the corpus; n == 0 does nothing
    assert L.frz_attr_set(None, which.ctypes.data, vals.ctypes.data, 2) == INVALID
    assert L.frz_attr_set(a, None, vals.ctypes.data, 2) == INVALID
    assert L.frz_attr_set(a, which.ctypes.data, None, 2) == INVALID
    assert L.frz_attr_set(a, which.ctypes.data, vals.ctypes.data, 2) == INVALID
    assert b"out of range" in L.frz_last_error()
    assert L.frz_attr_set(a, None, None, 0) == 0
    L.frz_attr_destroy(None)

    def clauses(*cl):
        arr = (F._CWhereClause * max(1, len(cl)))()
        for j, (attr, lo, hi, in_, n_in, neg) in enumerate(cl):
            arr[j].attr, arr[j].lo, arr[j].hi, arr[j].in_, arr[j].n_in, arr[j].negate = attr, lo, hi, in_, n_in, neg
        return arr

    fn = L.frz_subset_where
    rng = clauses((a, 0, 5, None, 0, 0))
    ok_set = np.array([3, 1, 3], dtype=np.int64)
    # NULL subset, NULL clauses with n > 0
    assert fn(None, rng, 1, None) == INVALID
    assert fn(s, None, 1, None) == INVALID
    assert b"null" in L.frz_last_error()
    # more than 8 clauses
    nine = clauses(*[(a, 0, 5, None, 0, 0)] * 9)
    assert fn(s, nine, 9, None) == UNSUPPORTED
    assert b"clauses" in L.frz_last_error()
    # a NULL attribute, NULL set values with n_in > 0
    assert fn(s, clauses((a, 0, 5, None, 0, 0), (None, 0, 5, None, 0, 0)), 2, None) == INVALID
    assert fn(s, clauses((a, 0, 0, None, 3, 0)), 1, None) == INVALID
    assert b"null" in L.frz_last_error()
    # more than 4096 set values over all clauses, including in one clause, and a huge n_in
    big = np.arange(4097, dtype=np.int64)
    assert fn(s, clauses((a, 0, 0, big.ctypes.data, 4097, 0)), 1, None) == UNSUPPORTED
    assert fn(s, clauses((a, 0, 0, big.ctypes.data, 2048, 0), (a, 0, 0, big.ctypes.data, 2049, 1)), 2, None) == UNSUPPORTED
    assert fn(s, clauses((a, 0, 0, big.ctypes.data, 2**64 - 1, 0)), 1, None) == UNSUPPORTED
    assert b"set values" in L.frz_last_error()
    # FRZ_ATTR_NULL as a set value
    bad = np.array([1, NULL, 2], dtype=np.int64)
    assert fn(s, clauses((a, 0, 0, bad.ctypes.data, 3, 0)), 1, None) == INVALID
    assert b"FRZ_ATTR_NULL" in L.frz_last_error()
    # an attribute or base of another corpus
    assert fn(s, clauses((a, 0, 5, None, 0, 0), (oth, 0, 5, None, 0, 0)), 2, None) == INVALID
    assert b"attribute was made on another corpus" in L.frz_last_error()
    assert fn(s, rng, 1, oth) == INVALID
    assert b"base subset was made on another corpus" in L.frz_last_error()
    assert fake.raw == b"\0" * 4096 and mine.raw == snap_mine and other.raw == snap_other
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    # every argument is valid: the call reaches the device check, the handle untouched
    for cl, n_cl, base in ((rng, 1, None), (None, 0, None), (clauses((a, 0, 0, ok_set.ctypes.data, 3, 1)), 1, s),
                           (clauses(*[(a, 1, 0, None, 0, 0)] * 8), 8, s),
                           (clauses((a, 0, 0, big.ctypes.data, 4096, 0)), 1, None)):
        assert fn(s, cl, n_cl, base) == NO_DEVICE
    assert mine.raw == snap_mine
