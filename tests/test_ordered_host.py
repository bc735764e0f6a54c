"""frz_match_list_ordered without a GPU: frizbee_b200/csrc/order_plan.cuh built for the CPU (tests/harness/order_harness.cpp).
The key's descending order is checked against tests/ordering.py's np.lexsort specification on random and adversarial
rows, the keys' uniqueness, and the select's pick rule run pass by pass over random key sets.  The argument checks of the
call run on zero-filled stand-in handles.  The behaviour on a real corpus is in tests/test_gpu_ordered.py."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from cpu_harness import load
from ordering import ATTR_NULL, order_by_attr
from ranking import MATCH_DTYPE

INVALID, NO_DEVICE = 1, 8
I64_MAX = 2**63 - 1
BLOCK_ROWS = 4096   # kFrzOrderBlockRows
vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32


@pytest.fixture(scope="module")
def H():
    L = load("order_harness")
    L.h_order_keys.argtypes = [u32, C.c_int, vp, vp, vp, vp, u64, vp]
    L.h_order_keys.restype = None
    L.h_order_digit.argtypes = [u64, u64, u32]
    L.h_order_digit.restype = u32
    L.h_order_digits.argtypes = [u64, u64, vp]
    L.h_order_digits.restype = u32
    L.h_order_pick.argtypes = [vp, u64, u64, u64, vp]
    L.h_order_pick.restype = None
    return L


def order_keys(H, m, values, order, reversed, boost):
    """The (hi, lo) key of each row of m (int64 values per row, boost per row or None)."""
    n = len(m)
    idx = np.ascontiguousarray(m["index"], dtype=np.uint32)
    sc = np.ascontiguousarray(m["score"], dtype=np.uint16)
    b = np.ascontiguousarray(np.zeros(n, np.int16) if boost is None else boost, dtype=np.int16)
    v = np.ascontiguousarray(values, dtype=np.int64)
    out = np.zeros(2 * max(n, 1), np.uint64)
    H.h_order_keys(order, int(reversed), idx.ctypes.data, sc.ctypes.data, b.ctypes.data, v.ctypes.data, n, out.ctypes.data)
    return out[0: 2 * n: 2], out[1: 2 * n: 2]


def rows(rng, n, kind):
    """Index-ordered rows, attribute values over [0, n_idx), a boost over them."""
    n_idx = n + 5
    idx = np.sort(rng.choice(n_idx, n, replace=False)).astype(np.uint32)
    m = np.zeros(n, MATCH_DTYPE)
    m["index"] = idx
    if kind == "equal_scores":
        m["score"] = 100
    elif kind == "clamp":
        m["score"] = rng.choice([0, 1, 65534, 65535, 300], n)
    else:
        m["score"] = rng.integers(0, 400, n)
    m["exact"] = rng.integers(0, 2, n)
    n_vals = n_idx if kind != "short" else n_idx // 2
    if kind in ("all_equal", "equal_scores"):
        vals = np.full(n_vals, 7, np.int64)
    elif kind == "ties":
        vals = rng.choice([0, 1, 127], n_vals).astype(np.int64)
    elif kind == "extremes":
        vals = rng.choice([ATTR_NULL, ATTR_NULL + 1, ATTR_NULL + 2, -1, 0, 1, I64_MAX - 1, I64_MAX], n_vals).astype(np.int64)
    else:
        vals = rng.integers(-2**63 + 1, 2**63 - 1, n_vals, dtype=np.int64, endpoint=True)
    vals[rng.random(n_vals) < 0.15] = ATTR_NULL
    boost = rng.choice([-32768, -400, -1, 0, 1, 200, 32767], n_idx).astype(np.int16)
    return m, vals, boost


KINDS = ["random", "ties", "extremes", "all_equal", "equal_scores", "clamp", "short"]


@pytest.mark.parametrize("kind", KINDS)
def test_key_order_is_the_specification(H, kind):
    rng = np.random.default_rng(KINDS.index(kind))
    for n in (1, 2, 33, 700):
        m, vals, boost = rows(rng, n, kind)
        for order in range(4):
            for reversed in (False, True):
                for b in (None, boost):
                    want = order_by_attr(m, vals, order, reversed, b)
                    l0 = m[::-1] if reversed else m
                    idx = l0["index"].astype(np.int64)
                    v = np.where(idx < len(vals), vals[np.minimum(idx, len(vals) - 1)], ATTR_NULL)
                    hi, lo = order_keys(H, l0, v, order, reversed, None if b is None else b[idx])
                    got = l0[np.lexsort((~lo, ~hi))]
                    assert np.array_equal(got, want), (kind, n, order, reversed, b is not None)
                    assert len(set(zip(hi.tolist(), lo.tolist()))) == n   # unique keys
                    assert (lo >> np.uint64(48)).max(initial=0) == 0   # 112 bits


def test_attribute_extremes_and_nulls(H):
    """Null is below every value in both directions; INT64_MIN + 1 under DESC and INT64_MAX under ASC are just above it."""
    m = np.zeros(5, MATCH_DTYPE)
    m["index"] = np.arange(5)
    v = np.array([ATTR_NULL, ATTR_NULL + 1, 0, I64_MAX, -1], np.int64)
    for order, want in ((0, [3, 2, 4, 1, 0]), (1, [1, 4, 2, 3, 0]), (2, [3, 2, 4, 1, 0]), (3, [1, 4, 2, 3, 0])):
        hi, lo = order_keys(H, m, v, order, False, None)
        assert np.lexsort((~lo, ~hi)).tolist() == want, order


def select(H, hi, lo, k, fit):
    """The select over keys (hi, lo), pass by pass as order.cu runs it: positions selected.  As in host.cu, a k that
    takes every row (or a list of one row) skips the select."""
    if k >= len(hi) or len(hi) <= 1:
        return np.arange(min(k, len(hi)))
    vary_hi = np.bitwise_or.reduce(hi) & np.bitwise_or.reduce(~hi)
    vary_lo = np.bitwise_or.reduce(lo) & np.bitwise_or.reduce(~lo & np.uint64((1 << 48) - 1))
    shifts = np.zeros(14, np.uint32)
    n_shifts = H.h_order_digits(int(vary_hi), int(vary_lo), shifts.ctypes.data)
    dig = lambda pos, s: np.array([H.h_order_digit(int(hi[p]), int(lo[p]), int(s)) for p in pos], np.int64)
    cand = np.arange(len(hi))
    sel = []
    need = k
    out = np.zeros(3, np.uint64)
    for p in range(n_shifts + 1):
        assert p < n_shifts, "the last digit must complete the selection"
        d = dig(cand, shifts[p])
        hist = np.ascontiguousarray(np.bincount(d, minlength=256).astype(np.uint32))
        H.h_order_pick(hist.ctypes.data, need, len(sel), fit, out.ctypes.data)
        bucket, take, above = (int(x) for x in out)
        sel += cand[d > bucket].tolist()
        if take:
            sel += cand[d == bucket].tolist()
            return np.array(sel, np.int64)
        cand = cand[d == bucket]
        need -= above


@pytest.mark.parametrize("kind", ["random", "ties", "all_equal"])
def test_pick_selects_the_top_k(H, kind):
    rng = np.random.default_rng(40 + ["random", "ties", "all_equal"].index(kind))
    for n in (1, 2, 9, 300, 5000):
        m, vals, boost = rows(rng, n, kind)
        idx = m["index"].astype(np.int64)
        v = np.where(idx < len(vals), vals[np.minimum(idx, len(vals) - 1)], ATTR_NULL)
        hi, lo = order_keys(H, m, v, int(rng.integers(0, 4)), bool(rng.integers(0, 2)), boost[idx])
        ranked = np.lexsort((~lo, ~hi))
        for k in sorted({0, 1, 7, n - 1, n, BLOCK_ROWS + 1} & set(range(0, n + 1))):
            exact = select(H, hi, lo, k, 0)
            assert sorted(exact.tolist()) == sorted(ranked[:k].tolist()), (n, k)
            fitted = select(H, hi, lo, k, BLOCK_ROWS if k <= BLOCK_ROWS else 0)
            assert set(ranked[:k].tolist()) <= set(fitted.tolist())
            assert len(fitted) == len(set(fitted.tolist())) and (len(fitted) == k or len(fitted) <= BLOCK_ROWS)
            # what the selection holds besides the top k lies right behind it
            assert set(fitted.tolist()) == set(ranked[: len(fitted)].tolist())


def test_digit_schedule_skips_constant_digits(H):
    shifts = np.zeros(14, np.uint32)
    assert H.h_order_digits(0, 0, shifts.ctypes.data) == 0
    assert H.h_order_digits(1, 1 << 40, shifts.ctypes.data) == 2 and shifts[:2].tolist() == [48, 40]
    assert H.h_order_digits(2**64 - 1, 2**48 - 1, shifts.ctypes.data) == 14
    assert shifts.tolist() == list(range(104, -1, -8))


def test_ordered_argument_checks():
    import torch
    L = F.lib()
    fake = C.create_string_buffer(4096)            # a corpus of 0 haystacks; never written
    c = C.addressof(fake)
    mine = C.create_string_buffer(c.to_bytes(8, "little"), 256)    # a subset / boost / attribute of the fake corpus
    other = C.create_string_buffer(256)            # a handle whose corpus (its first field) is NULL: another corpus
    h, oth = C.addressof(mine), C.addressof(other)
    snap_mine, snap_other = mine.raw, other.raw
    n, total = C.c_uint64(), C.c_uint64()
    out = np.zeros(4, dtype=F.MATCH_DTYPE)
    fn = L.frz_match_list_ordered

    def call(m_=c, c_=c, s=None, b=None, a=h, order=0, k=4, o=out.ctypes.data):
        return fn(m_, c_, s, b, a, order, k, o, C.byref(n), C.byref(total))

    # a NULL matcher, corpus or attribute (the subset and boost may be NULL), and a NULL out with k > 0
    for kw in ({"m_": None}, {"c_": None}, {"a": None}):
        assert call(**kw) == INVALID
        assert b"null argument" in L.frz_last_error()
    assert call(o=None) == INVALID
    assert b"null out" in L.frz_last_error()
    # an order above FRZ_ORDER_SCORE_THEN_ATTR_ASC
    for order in (4, 2**32 - 1):
        assert call(order=order) == INVALID
        assert b"order" in L.frz_last_error()
    # an attribute, boost or subset of another corpus
    assert call(a=oth) == INVALID
    assert b"attribute was made on another corpus" in L.frz_last_error()
    assert call(b=oth) == INVALID
    assert b"boost was made on another corpus" in L.frz_last_error()
    assert call(s=oth) == INVALID
    assert b"subset was made on another corpus" in L.frz_last_error()
    assert fake.raw == b"\0" * 4096 and mine.raw == snap_mine and other.raw == snap_other
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    # every argument is valid: the call reaches the device check (k = 0 with a NULL out only counts)
    for kw in ({}, {"order": 3}, {"b": h}, {"s": h}, {"k": 0, "o": None}, {"k": 2**64 - 1}):
        assert call(**kw) == NO_DEVICE
    assert mine.raw == snap_mine
