"""The batched column call without a GPU: the argument checks of frz_match_list_batch_columns, their order and the
missing-device status, and frizbee_b200/csrc/batch_columns_plan.cuh built for the CPU (tests/harness/
batch_columns_harness.cpp): random per-column lists folded and compacted as the device does it, against the specification
tests/columns.py (combine), sums that saturate at 65535 included."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from columns import combine
from cpu_harness import load

INVALID, TOO_MANY_ITEMS, UNSUPPORTED, NO_DEVICE = 1, 4, 9, 8
U64_MAX = 2**64 - 1
vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32


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
    huge, huge2 = fake_corpus(2**32), fake_corpus(2**32)
    before = [b.raw for b in (c0, c1, longer, elsewhere, stranger)]
    a0, a1 = C.addressof(c0), C.addressof(c1)
    handle = {name: C.create_string_buffer(C.addressof(c).to_bytes(8, "little"), 64)
              for name, c in (("c0", c0), ("c1", c1), ("stranger", stranger))}
    h = {k: C.addressof(v) for k, v in handle.items()}
    mfake = C.create_string_buffer(64)           # a matcher, never dereferenced before the device check
    m = C.addressof(mfake)
    out = np.zeros(8, dtype=F.MATCH_DTYPE)
    n_out, n_total = np.zeros(2, np.uint64), np.zeros(2, np.uint64)
    cnt = np.zeros(4, dtype=np.uint32)
    fn = L.frz_match_list_batch_columns

    def arr(*xs):
        return (C.c_void_p * max(len(xs), 1))(*xs)

    def pg(*v):
        a = np.array(v, dtype=np.uint64)
        keep.append(a)
        return a.ctypes.data

    keep = []

    def call(ms=None, q=2, cols=None, n_cols=2, sort=0, s=None, b=None, g=None, per_group=None, k=4, o=out.ctypes.data,
             no=n_out.ctypes.data, counts=None):
        ms = arr(m, m, m, m) if ms is None else ms
        cols = arr(a0, a1) if cols is None else cols
        return fn(ms, q, cols, n_cols, sort, s, b, g, per_group, k, o, no, n_total.ctypes.data, counts)

    def refused(status, text, **kw):
        assert call(**kw) == status, kw
        assert text.encode() in L.frz_last_error(), (kw, L.frz_last_error())

    refused(INVALID, "n_cols", n_cols=0)
    refused(INVALID, "n_cols", n_cols=0, ms=0, sort=9, k=1, o=None)   # the first check wins
    refused(INVALID, "null argument", ms=0)
    refused(INVALID, "null argument", cols=0)
    refused(INVALID, "null corpus of column 1", cols=arr(a0, None), ms=arr(m, None, m, m))
    refused(INVALID, "q * n_cols overflows", q=2**63)
    refused(INVALID, "null matcher of query 1, column 0", ms=arr(m, m, None, m), cols=arr(a0, C.addressof(elsewhere)))
    refused(INVALID, "device", cols=arr(a0, C.addressof(elsewhere)))
    refused(INVALID, "index space", cols=arr(a0, C.addressof(longer)))
    refused(INVALID, "index space", cols=arr(a0, C.addressof(longer)), sort=9)
    refused(TOO_MANY_ITEMS, "u32 index", cols=arr(C.addressof(huge), C.addressof(huge2)))
    refused(TOO_MANY_ITEMS, "u32 index", cols=arr(C.addressof(huge), C.addressof(huge2)), sort=9, k=1, o=None)
    for bad in (4, 255):
        refused(INVALID, "sort", sort=bad)
    refused(INVALID, "sort", sort=4, per_group=pg(0, 0))
    # per_group: every entry is checked, with or without groups; the first bad entry decides, before the handles
    for v, want in (((0, 1), INVALID), ((1, 0), INVALID), ((33, 0), UNSUPPORTED), ((0, 33), INVALID), ((U64_MAX - 1, 1), UNSUPPORTED),
                    ((32, 2**63), UNSUPPORTED)):
        assert call(per_group=pg(*v), s=arr(h["stranger"], None), g=arr(None, h["stranger"])) == want, v
        assert b"per_group" in L.frz_last_error()
    # handles made on none of the columns: query order, then subset, boost, groups within a query
    refused(INVALID, "groups of query 1 were made on none", g=arr(h["c1"], h["stranger"]))
    refused(INVALID, "subset of query 0 was made on none", s=arr(h["stranger"], None), b=arr(h["stranger"], None), g=arr(h["stranger"], None))
    refused(INVALID, "boost of query 0 was made on none", b=arr(h["stranger"], None), g=arr(h["stranger"], None))
    refused(INVALID, "groups of query 0 were made on none", s=arr(None, h["stranger"]), g=arr(h["stranger"], None))
    # then NULL n_out, q * k overflow, NULL out
    refused(INVALID, "null n_out", no=None)
    refused(INVALID, "overflows", k=2**63)
    refused(INVALID, "null out", o=None)
    # q = 0 reads no matcher, handle or per_group entry, and is a no-op
    assert fn(arr(), 0, arr(a0, a1), 2, 0, None, None, None, None, 4, None, None, None, None) == 0
    assert [b.raw for b in (c0, c1, longer, elsewhere, stranger)] == before and not cnt.any()
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    # every argument is valid: the call reaches the device check.  Handles of any column serve, NULL arrays stand for NULL
    # entries, a column or matcher may repeat
    for kw in (dict(), dict(per_group=pg(1, U64_MAX)), dict(s=arr(h["c1"], None), b=arr(None, h["c0"]), g=arr(h["c1"], h["c0"]),
                                                          per_group=pg(32, 3), counts=arr(cnt.ctypes.data, None)),
               dict(g=arr(h["c0"], None), per_group=pg(U64_MAX, 1), k=0, o=None), dict(sort=3, k=1025),
               dict(cols=arr(a0, a0)), dict(n_cols=1, ms=arr(m, m)), dict(q=1)):
        assert call(**kw) == NO_DEVICE, kw
    assert not cnt.any()


# ---------------------------------------------------------------------------- the plan header against the specification

@pytest.fixture(scope="module")
def H():
    L = load("batch_columns_harness")
    L.h_columns_bytes.argtypes = [u64, u64, u64]
    L.h_columns_bytes.restype = u64
    L.h_fold.argtypes = [u32, u32, u32, u32]
    L.h_fold.restype = u32
    L.h_join.argtypes = [u64, u32, vp, vp, vp, vp, C.c_int, vp]
    L.h_join.restype = u64
    return L


def ptrs(xs):
    return (C.c_void_p * max(len(xs), 1))(*[x.ctypes.data if x is not None else None for x in xs])


def test_fold_rule(H):
    assert H.h_fold(0, 0, 7, 1) == (1 << 24) | 0x10000 | 7
    assert H.h_fold((1 << 24) | 0xFFF0, 1, 0x20, 0) == (2 << 24) | 0xFFFF   # saturates
    assert H.h_fold((1 << 24) | 0x10000 | 5, 1, 3, 0) == (2 << 24) | 0x10000 | 8   # the exact flag stays
    assert H.h_fold((1 << 24) | 5, 2, 3, 1) == (1 << 24) | 5   # missed the second column: stays out
    assert H.h_fold(0, 1, 3, 1) == 0
    for n_cols, rows, pat in ((1, 1, 1500), (4, 1 << 18, 1536), (255, 1 << 21, 1536)):
        assert H.h_columns_bytes(n_cols, rows, pat) == rows * 4 + 4 + (n_cols - 1) * pat + n_cols * 2 + 1


@pytest.mark.parametrize("seed", range(8))
def test_join_reproduces_combine(H, seed):
    """Columns with and without patterns, rows removed in some columns, scores up to 65535: the device's fold and
    compaction give combine()'s rows, in index order or reversed."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 3000))
    n_cols = int(rng.integers(1, 6))
    live = [rng.random(n) > rng.choice([0.0, 0.1, 0.5]) if rng.random() < 0.5 else None for _ in range(n_cols)]
    has = np.array([rng.random() < 0.75 for _ in range(n_cols)], np.uint8)
    has[int(rng.integers(0, n_cols))] = 1
    lists = []
    for c in range(n_cols):
        if not has[c]:
            lists.append(None)
            continue
        pick = rng.random(n) < rng.choice([0.05, 0.5, 0.97])
        if live[c] is not None:
            pick &= live[c]   # a column's scan never lists a row removed in it
        idx = np.flatnonzero(pick)
        L = np.zeros(len(idx), dtype=F.MATCH_DTYPE)
        L["index"] = idx.astype(np.uint32)
        top = int(rng.choice([40, 300, 65536]))
        L["score"] = rng.integers(0, top, len(idx)).astype(np.uint16)
        if top == 65536:
            L["score"][rng.random(len(idx)) < 0.3] = 65535
        L["exact"] = rng.integers(0, 2, len(idx))
        lists.append(L)
    all_live = np.ones(n, dtype=bool)
    for lv in live:
        if lv is not None:
            all_live &= lv
    want = combine([L for L in lists if L is not None], n, live=all_live)
    live_u8 = [None if lv is None else lv.astype(np.uint8) for lv in live]
    n_list = np.array([0 if L is None else len(L) for L in lists], np.uint64)
    for reversed_ in (0, 1):
        out = np.zeros(max(n, 1), dtype=F.MATCH_DTYPE)
        total = H.h_join(n, n_cols, ptrs(lists), n_list.ctypes.data, ptrs(live_u8), has.ctypes.data, reversed_, out.ctypes.data)
        got = out[:total]
        assert np.array_equal(got, want[::-1] if reversed_ else want), (seed, reversed_)
