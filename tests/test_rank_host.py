"""frz_attr_rank without a GPU: frizbee_b200/csrc/rank_plan.cuh built for the CPU (tests/harness/rank_harness.cpp) against
Python's sorted() on random byte strings and int64 values, the whole refinement with the kernels' per-row steps, and the
argument checks of frz_attr_rank and their order on zero-filled stand-in handles.  The behaviour on a real corpus is in
tests/test_gpu_rank.py."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np
import pytest

import frizbee_b200 as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "harness", "rank_harness.cpp")
LIB = os.path.join(ROOT, "tests", "harness", "librank_harness.so")
DEPS = [SRC] + [os.path.join(ROOT, "frizbee_b200", "csrc", h) for h in ("rank_plan.cuh", "order_plan.cuh", "batch_plan.cuh")]
INVALID, UNSUPPORTED, NO_DEVICE = 1, 9, 8
NULL = -(2**63)
I64_MAX = 2**63 - 1
vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32
FOLD = bytes(range(65)) + bytes(range(97, 123)) + bytes(range(91, 256))   # A-Z as a-z


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", LIB, SRC], check=True)
    L = C.CDLL(LIB)
    L.h_rank_text_chunk.argtypes = [C.c_char_p, u32, u32, u32, u32]
    L.h_rank_text_chunk.restype = u64
    L.h_rank_attr_chunk.argtypes = [C.c_int64, u32]
    L.h_rank_attr_chunk.restype = u64
    L.h_rank_chunk_ends.argtypes = [u64, u32, u32]
    L.h_rank_chunk_ends.restype = u32
    L.h_rank_fold4.argtypes = [u32]
    L.h_rank_fold4.restype = u32
    L.h_rank_common.argtypes = [C.c_char_p, u32, C.c_char_p, u32, u32, u32]
    L.h_rank_common.restype = u32
    L.h_rank.argtypes = [u32, u32, vp, vp, vp, vp, vp, vp, vp, vp]
    L.h_rank.restype = u32
    return L


def padded(b: bytes) -> bytes:
    return b + b"\0" * ((len(b) + 15) // 16 * 16 + 16 - len(b))


# ------------------------------------------------------------------------------------------------ the specification
def spec_ranks(n, keys, ranked):
    """The dense rank of each ranked row's key tuple (None elsewhere).  keys: ("attr", values, desc) or ("text", texts,
    desc, fold)."""
    def cmp_key(k, i, j):
        if k[0] == "attr":
            a, b = int(k[1][i]), int(k[1][j])
            if a == NULL or b == NULL:
                return (a == NULL) - (b == NULL)
            c = (a > b) - (a < b)
        else:
            a, b = k[1][i], k[1][j]
            if k[3]:
                a, b = a.translate(FOLD), b.translate(FOLD)
            c = (a > b) - (a < b)
        return -c if k[2] else c

    def cmp(i, j):
        for k in keys:
            c = cmp_key(k, i, j)
            if c:
                return c
        return 0

    rows = sorted([i for i in range(n) if ranked[i]], key=functools.cmp_to_key(cmp))
    out = [None] * n
    r = -1
    for p, i in enumerate(rows):
        if p == 0 or cmp(rows[p - 1], i) != 0:
            r += 1
        out[i] = r
    return out


def harness_ranks(H, n, keys, ranked):
    nk = len(keys)
    is_text = np.array([k[0] == "text" for k in keys], np.uint32)
    desc = np.array([k[2] for k in keys], np.uint32)
    fold = np.array([k[3] if k[0] == "text" else 0 for k in keys], np.uint32)
    keep, vals, texts, offs = [], (C.c_void_p * nk)(), (C.c_void_p * nk)(), (C.c_void_p * nk)()
    for j, k in enumerate(keys):
        if k[0] == "attr":
            v = np.ascontiguousarray(k[1], np.int64)
            keep.append(v)
            vals[j] = v.ctypes.data
        else:
            data = np.frombuffer(b"".join(k[1]) + b"\0", np.uint8).copy()
            o = np.zeros(n + 1, np.uint64)
            o[1:] = np.cumsum([len(t) for t in k[1]])
            keep += [data, o]
            texts[j], offs[j] = data.ctypes.data, o.ctypes.data
    rk = np.ascontiguousarray(ranked, np.uint8)
    out = np.zeros(max(1, n), np.int64)
    rounds = H.h_rank(n, nk, is_text.ctypes.data, desc.ctypes.data, fold.ctypes.data, C.cast(vals, vp), C.cast(texts, vp),
                      C.cast(offs, vp), rk.ctypes.data, out.ctypes.data)
    return [None if x == NULL else int(x) for x in out[:n]], rounds


def rbytes(rng, alphabet, k):
    return rng.choice(np.frombuffer(alphabet, np.uint8), k).tobytes()


def random_texts(rng, n, alphabet=b"aAbBzZ\0\x80\xff/.", max_len=20, pool=None):
    out = []
    for _ in range(n):
        if pool and rng.random() < 0.4:   # proper prefixes and extensions of earlier texts
            t = pool[int(rng.integers(len(pool)))]
            t = t[: int(rng.integers(0, len(t) + 1))] if rng.random() < 0.5 else t + rbytes(rng, alphabet, int(rng.integers(0, 4)))
        else:
            t = rbytes(rng, alphabet, int(rng.integers(0, max_len + 1)))
        out.append(t)
        pool = (pool or []) + [t]
    return out


def random_values(rng, n):
    v = rng.choice(np.array([NULL, NULL + 1, -1, 0, 1, 7, I64_MAX, 2**40, -2**40], np.int64), n)
    return np.ascontiguousarray(v, np.int64)


# ------------------------------------------------------------------------------------------------ chunk rules
def test_fold4_is_bytewise_fold(H):
    for b in range(256):
        x = b * 0x01010101
        want = int.from_bytes(bytes([b]).translate(FOLD) * 4, "little")
        assert H.h_rank_fold4(x) == want, b
    rng = np.random.default_rng(0)
    for x in rng.integers(0, 2**32, 5000, dtype=np.uint64):
        x = int(x)
        assert H.h_rank_fold4(x) == int.from_bytes(x.to_bytes(4, "little").translate(FOLD), "little")


def test_attr_chunks_order_values_null_last(H):
    vals = [NULL, NULL + 1, NULL + 2, -2**40, -1, 0, 1, 2**40, I64_MAX - 1, I64_MAX]
    for desc in (0, 1):
        chunks = [H.h_rank_attr_chunk(v, desc) for v in vals]
        want = sorted([v for v in vals if v != NULL], reverse=bool(desc)) + [NULL]
        assert [v for _, v in sorted(zip(chunks, vals))] == want
        assert all(H.h_rank_chunk_ends(c, 0, desc) for c in chunks)


def test_text_chunks_order_short_texts(H):
    """Texts of at most 6 bytes fit one chunk: its order is the texts' order, proper prefixes first, NUL an ordinary byte."""
    rng = np.random.default_rng(1)
    texts = sorted({t for t in random_texts(rng, 600, max_len=6) if len(t) <= 6} | {b"", b"\0", b"\0\0", b"a", b"a\0", b"A", b"\xff", b"\x80a"})
    for fold in (0, 1):
        for desc in (0, 1):
            chunks = {t: H.h_rank_text_chunk(padded(t), len(t), 0, fold, desc) for t in texts}
            key = (lambda t: t.translate(FOLD)) if fold else (lambda t: t)
            for a in texts:
                for b in texts[::7]:
                    want = (key(a) > key(b)) - (key(a) < key(b))
                    got = (chunks[a] > chunks[b]) - (chunks[a] < chunks[b])
                    assert got == (-want if desc else want), (a, b, fold, desc)
            assert all(H.h_rank_chunk_ends(c, 1, desc) for c in chunks.values())


def test_text_chunks_step_through_long_texts(H):
    t = bytes(range(1, 30))
    for off in range(0, len(t) + 1):
        c = H.h_rank_text_chunk(padded(t), len(t), off, 0, 0)
        left = min(7, len(t) - off)
        assert c & 0xFF == left
        assert (c >> 8).to_bytes(7, "big") == t[off: off + 7].ljust(7, b"\0")
        assert H.h_rank_chunk_ends(c, 1, 0) == (left < 7)
        assert H.h_rank_chunk_ends(~c & (2**64 - 1), 1, 1) == (left < 7)


def test_common_prefix(H):
    rng = np.random.default_rng(2)
    for _ in range(3000):
        base = rbytes(rng, b"aAbB\0\xff", int(rng.integers(0, 70)))
        a = base + rbytes(rng, b"aAbB\0\xff", int(rng.integers(0, 20)))
        b = base[: int(rng.integers(0, len(base) + 1))] + rbytes(rng, b"aAbB\0\xff", int(rng.integers(0, 20)))
        lim = min(len(a), len(b))
        off = int(rng.integers(0, lim + 1))
        for fold in (0, 1):
            fa, fb = (a.translate(FOLD), b.translate(FOLD)) if fold else (a, b)
            want = next((i for i in range(off, lim) if fa[i] != fb[i]), lim) - off
            assert H.h_rank_common(padded(a), len(a), padded(b), len(b), off, fold) == want, (a, b, off, fold)


# ------------------------------------------------------------------------------------------------ whole refinement
@pytest.mark.parametrize("seed", range(12))
def test_refinement_against_sorted(H, seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(0, 300))
    keys = []
    for _ in range(int(rng.integers(1, 5))):
        if rng.random() < 0.5:
            keys.append(("text", random_texts(rng, n, max_len=int(rng.choice([3, 12, 40]))), int(rng.integers(2)), int(rng.integers(2))))
        else:
            keys.append(("attr", random_values(rng, n), int(rng.integers(2)), 0))
    ranked = rng.random(n) < 0.85
    got, _ = harness_ranks(H, n, keys, ranked)
    assert got == spec_ranks(n, keys, ranked)


def test_shared_prefixes_take_few_rounds(H):
    rng = np.random.default_rng(7)
    prefix = b"/home/user/projects/" + b"x" * 180   # 200 bytes every path shares
    texts = [prefix + rbytes(rng, b"abc/", int(rng.integers(0, 6))) for _ in range(200)]
    got, rounds = harness_ranks(H, len(texts), [("text", texts, 0, 0)], np.ones(len(texts), bool))
    assert got == spec_ranks(len(texts), [("text", texts, 0, 0)], [True] * len(texts))
    assert rounds <= 4
    big = [bytes(rng.integers(0, 256, 20000, dtype=np.uint8))] * 5 + [b"tail"]   # identical long texts
    got, rounds = harness_ranks(H, len(big), [("text", big, 1, 1)], np.ones(len(big), bool))
    assert got == spec_ranks(len(big), [("text", big, 1, 1)], [True] * len(big))
    assert rounds <= 3


def test_all_equal_and_empty(H):
    for n in (0, 1, 5):
        texts = [b"same"] * n
        assert harness_ranks(H, n, [("text", texts, 0, 0)], np.ones(n, bool))[0] == [0] * n
    got, _ = harness_ranks(H, 3, [("attr", np.array([NULL] * 3), 0, 0)], np.array([1, 0, 1], bool))
    assert got == [0, None, 0]


# ------------------------------------------------------------------------------------------------ argument checks
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

    c0, c1, longer, elsewhere = fake_corpus(7), fake_corpus(7), fake_corpus(8), fake_corpus(7, 1)
    corp = {k: C.addressof(v) for k, v in (("c0", c0), ("c1", c1), ("longer", longer), ("elsewhere", elsewhere))}
    # an attribute's first field is its corpus
    handle = {k: C.create_string_buffer(corp[k].to_bytes(8, "little"), 128) for k in corp}
    a = {k: C.addressof(v) for k, v in handle.items()}
    before = [b.raw for b in (c0, c1, longer, elsewhere)] + [h.raw for h in handle.values()]

    def keys(*ks):
        arr = (F._CRankKey * max(1, len(ks)))()
        for j, (attr, text, desc, fold) in enumerate(ks):
            arr[j].attr, arr[j].text, arr[j].desc, arr[j].fold_case = attr, text, desc, fold
        return arr

    fn = L.frz_attr_rank
    ok = keys((None, corp["c1"], 1, 1))
    # 1. NULL attribute, NULL keys with n_keys > 0
    assert fn(None, ok, 1) == INVALID and b"null" in L.frz_last_error()
    assert fn(a["c0"], None, 1) == INVALID and b"null" in L.frz_last_error()
    assert fn(None, None, 0) == INVALID and b"null" in L.frz_last_error()
    # 2. no key
    assert fn(a["c0"], None, 0) == INVALID and b"n_keys = 0" in L.frz_last_error()
    assert fn(a["c0"], ok, 0) == INVALID
    # 3. more than four keys, ahead of any bad key
    five = keys(*[(None, None, 0, 0)] * 5)
    assert fn(a["c0"], five, 5) == UNSUPPORTED and b"keys" in L.frz_last_error()
    # 4. both or neither of attr and text, ahead of fold_case and the corpus rules
    assert fn(a["c0"], keys((a["c1"], None, 0, 1), (None, None, 0, 0)), 2) == INVALID and b"neither" in L.frz_last_error()
    assert fn(a["c0"], keys((a["longer"], corp["c1"], 0, 0)), 1) == INVALID and b"both" in L.frz_last_error()
    # 5. fold_case on an attribute key, ahead of the corpus rules
    assert fn(a["c0"], keys((None, corp["longer"], 0, 0), (a["c1"], None, 0, 1)), 2) == INVALID
    assert b"fold_case" in L.frz_last_error()
    # 6. a key of another device or another length: text or attribute
    assert fn(a["c0"], keys((None, corp["longer"], 0, 0)), 1) == INVALID and b"rows" in L.frz_last_error()
    assert fn(a["c0"], keys((a["longer"], None, 0, 0)), 1) == INVALID and b"rows" in L.frz_last_error()
    assert fn(a["c0"], keys((None, corp["c1"], 0, 0), (None, corp["elsewhere"], 0, 0)), 2) == INVALID
    assert b"device" in L.frz_last_error()
    assert fn(a["c0"], keys((a["elsewhere"], None, 0, 0)), 1) == INVALID and b"device" in L.frz_last_error()
    assert [b.raw for b in (c0, c1, longer, elsewhere)] + [h.raw for h in handle.values()] == before
    # frz_attr_get: NULL handle, NULL out with n > 0, more values than the corpus has rows; an attribute without device
    # values reads as all null
    got = np.zeros(8, np.int64)
    assert L.frz_attr_get(None, got.ctypes.data, 1) == INVALID
    assert L.frz_attr_get(a["c0"], None, 1) == INVALID
    assert L.frz_attr_get(a["c0"], got.ctypes.data, 8) == INVALID and b"haystacks" in L.frz_last_error()
    assert L.frz_attr_get(a["c0"], got.ctypes.data, 7) == 0 and (got[:7] == NULL).all() and got[7] == 0
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    # every argument is valid: the call reaches the device check, the handles untouched; a may be its own key, and an
    # attribute of another corpus of the same length serves
    for ks, nk in ((ok, 1), (keys((a["c0"], None, 1, 0)), 1), (keys((a["c1"], None, 0, 0), (None, corp["c0"], 0, 1),
                                                                    (None, corp["c1"], 1, 0), (a["c0"], None, 0, 0)), 4)):
        assert fn(a["c0"], ks, nk) == NO_DEVICE
    assert [b.raw for b in (c0, c1, longer, elsewhere)] + [h.raw for h in handle.values()] == before


# ------------------------------------------------------------------------------------------------ the digits of a round
def _digits(H, keys):
    """The digit shifts the LSD sort visits for a round's sort keys, from their OR and the OR of their complements as
    k_rank_chunk accumulates them (the low key word holds 48 bits) and rank_fill combines them."""
    m48 = (1 << 48) - 1
    or_hi = or_lo = nor_hi = nor_lo = 0
    for hi, lo in keys:
        or_hi, or_lo = or_hi | hi, or_lo | lo
        nor_hi, nor_lo = nor_hi | (~hi & (2**64 - 1)), nor_lo | (~lo & m48)
    shifts = np.zeros(14, np.uint32)
    n = H.h_order_digits(or_hi & nor_hi, or_lo & nor_lo, shifts.ctypes.data)
    return [int(s) for s in shifts[:n]]


@pytest.mark.parametrize("seg_hi", [2**8 - 1, 2**16 - 1, 2**24, 2**32 - 2], ids=["seg8", "seg16", "seg24", "seg32"])
def test_round_digits_are_the_varying_segment_and_chunk_bytes(H, seg_hi):
    """Sort keys of rows whose segment ids span [0, seg_hi] and whose chunks vary in chosen bytes: the sort visits exactly
    the segment bytes (key bits 64-95) and chunk bytes (key bits 0-63) in which the keys differ, most significant first,
    and never the top 16 bits; the descending key order is the ascending (segment, chunk) order; the segment comes back."""
    rng = np.random.default_rng(seg_hi % 1000)
    H.h_rank_sort_key.argtypes = [u32, u64, vp]
    H.h_rank_key_seg.argtypes = [u64, u64]
    H.h_rank_key_seg.restype = u32
    H.h_order_digits.argtypes = [u64, u64, vp]
    H.h_order_digits.restype = u32
    out = np.zeros(2, np.uint64)
    for chunk_bytes in ([], [0], [7], [0, 3, 6], list(range(8))):
        segs = [0, seg_hi] + [int(x) for x in rng.integers(0, seg_hi + 1, 200, dtype=np.uint64)]
        base = int(rng.integers(0, 2**64, dtype=np.uint64))
        chunks = []
        for _ in segs:
            c = base
            for b in chunk_bytes:
                c = (c & ~(0xFF << 8 * b)) | int(rng.integers(0, 256)) << 8 * b
            chunks.append(c)
        if chunk_bytes:   # the first row keeps the base chunk, the second differs in every chosen byte
            chunks[0] = base
            chunks[1] = base ^ sum(0x5A << 8 * b for b in chunk_bytes)
        keys = []
        for s, c in zip(segs, chunks):
            H.h_rank_sort_key(s, c, out.ctypes.data)
            hi, lo = int(out[0]), int(out[1])
            assert hi >> 48 == 0 and lo >> 48 == 0
            assert H.h_rank_key_seg(hi, lo) == s
            keys.append((hi, lo))
        want = [64 + 8 * b for b in range(3, -1, -1) if len({s >> 8 * b & 0xFF for s in segs}) > 1]
        want += [8 * b for b in range(7, -1, -1) if len({c >> 8 * b & 0xFF for c in chunks}) > 1]
        assert _digits(H, keys) == want, (seg_hi, chunk_bytes)
        assert want[0] == {2**8 - 1: 64, 2**16 - 1: 72, 2**24: 88, 2**32 - 2: 88}[seg_hi]
        # the key, read as one 112-bit number, descends as (segment, chunk) ascends
        as_int = [hi << 48 | lo for hi, lo in keys]
        by_key = sorted(range(len(segs)), key=lambda i: -as_int[i])
        by_tuple = sorted(range(len(segs)), key=lambda i: (segs[i], chunks[i]))
        assert [(segs[i], chunks[i]) for i in by_key] == [(segs[i], chunks[i]) for i in by_tuple]
