"""The unicode, literal and traceback scorers (frizbee_b200/csrc/unicode_path.cuh, indices_path.cuh and the byte literal
matcher of prefilter_scan.cuh) across scoring configurations, run on the CPU with the needle and scoring constants the
library hands to the GPU kernels (frz_matcher_debug_unicode / frz_matcher_debug_pattern) and the backend it selects.

tests/test_unicode_device_code.py checks the same headers with constants the harness builds itself, mostly at the
default scoring, where the capitalization, matching-case and delimiter bonuses are all 4.  Here the library's own
constants are first compared field by field with that construction, then every scorer runs with them against the
oracle: the traceback (byte and scalar rows, needles of 1-64 bytes, every typo budget, windows of 1-1024 bytes and the
greedy form past them), the unicode Smith-Waterman score for needles of 6-64 bytes, and the unicode and byte literal
matchers in all four modes, including which occurrence a substring match picks."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200.types import CaseMatching, Config, Matching, Pattern, Scoring, UnicodeMatching
from needles import case_pairs
from oracle import pyoracle as O
from scorings import TIES, literal_scorings, scorings, unicode_scorings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "frizbee_b200", "csrc")
U_SRC = os.path.join(ROOT, "tests", "harness", "unicode_harness.cpp")
U_LIB = os.path.join(ROOT, "tests", "harness", "libunicode_harness.so")
U_DEPS = [U_SRC] + [os.path.join(CSRC, f) for f in ("unicode_path.cuh", "indices_path.cuh", "unicode_needle.h", "unicode_case.inc")]
PS_SRC = os.path.join(ROOT, "tests", "harness", "pf_scan_harness.cpp")
PS_LIB = os.path.join(ROOT, "tests", "harness", "libpf_scan_harness.so")
PS_DEPS = [PS_SRC] + [os.path.join(CSRC, f) for f in ("prefilter_scan.cuh", "prefilter_masks.cuh", "frz_device.cuh")]
CUDA_INC = "/usr/local/cuda/include"

U_FIELDS = ("gex", "gopx", "match_x", "mismatch", "case_bonus", "cap_bonus", "delim_bonus", "prefix_bonus")
RAW_FIELDS = ("raw_match", "raw_gap_open", "raw_gap_extend", "raw_prefix", "raw_cap", "raw_case", "raw_delim", "exact_bonus")


class UNeedle(C.Structure):   # unicode_path.cuh: FrzUNeedle
    _fields_ = [("c", C.c_uint8 * 64), ("f", C.c_uint8 * 64), ("bflip", C.c_uint8 * 64), ("off", C.c_uint8 * 64),
                ("len", C.c_uint8 * 64), ("n", C.c_int32), ("nbytes", C.c_int32)]


class UScoring(C.Structure):   # unicode_path.cuh: FrzUScoring
    _fields_ = [(f, C.c_int32) for f in U_FIELDS + RAW_FIELDS]


def _stale(lib, deps):
    return not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in deps)


@pytest.fixture(scope="module")
def H():
    if _stale(U_LIB, U_DEPS):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", U_LIB, U_SRC], check=True)
    L = C.CDLL(U_LIB)
    L.h_uneedle_size.restype = L.h_uscoring_size.restype = C.c_size_t
    assert (L.h_uneedle_size(), L.h_uscoring_size()) == (C.sizeof(UNeedle), C.sizeof(UScoring))
    L.h_build_needle.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.POINTER(UNeedle)]
    L.h_needle_has_uppercase.argtypes = [C.c_char_p, C.c_size_t]
    L.h_scoring_of.argtypes = [C.c_void_p, C.c_int, C.POINTER(UScoring)]
    L.h_scoring_of.restype = None
    L.h_sw_score_c.argtypes = [C.POINTER(UNeedle), C.POINTER(UScoring), C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int]
    L.h_sw_indices_c.argtypes = [C.POINTER(UNeedle), C.c_int, C.POINTER(UScoring), C.c_char_p, C.c_int, C.c_int, C.c_int,
                                 C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
    L.h_lit_find_c.argtypes = [C.POINTER(UNeedle), C.POINTER(UScoring), C.c_char_p, C.c_int, C.c_int, C.POINTER(C.c_int),
                               C.POINTER(C.c_uint32)]
    F.lib().frz_matcher_debug_unicode.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    return L


@pytest.fixture(scope="module")
def PS():
    if not os.path.isdir(CUDA_INC):
        pytest.skip("CUDA headers not found")
    if _stale(PS_LIB, PS_DEPS):
        subprocess.run(["g++", "-O2", "-std=c++17", "-I" + CUDA_INC, "-fPIC", "-shared", "-o", PS_LIB, PS_SRC], check=True)
    L = C.CDLL(PS_LIB)
    L.h_pattern_size.restype = C.c_size_t
    L.h_lit_find.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_uint32)]
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    return L


def scoring9(s: Scoring):
    return np.array([s.match_score, s.mismatch_penalty, s.gap_open_penalty, s.gap_extend_penalty, s.prefix_bonus,
                     s.capitalization_bonus, s.matching_case_bonus, s.exact_match_bonus, s.delimiter_bonus], dtype=np.uint16)


def library_constants(needle, cfg):
    """The FrzUNeedle / FrzUScoring of a one-pattern matcher, and its backend_info."""
    m = F.Matcher(needle, cfg)
    try:
        un, usc = UNeedle(), UScoring()
        F._check(F.lib().frz_matcher_debug_unicode(m._h, 0, C.byref(un), C.sizeof(un), C.byref(usc), C.sizeof(usc)))
        return un, usc, m.backend_info()
    finally:
        m.close()


def harness_scoring(H, sc: Scoring, bits: int) -> UScoring:
    out = UScoring()
    s9 = scoring9(sc)
    H.h_scoring_of(s9.ctypes.data, bits, C.byref(out))
    return out


def fields(s):
    return {f: getattr(s, f) for f, _ in s._fields_}


def is_case_sensitive(H, nb: bytes, casing) -> bool:
    if casing == CaseMatching.Smart:
        return bool(H.h_needle_has_uppercase(nb, len(nb)))
    return casing == CaseMatching.Respect


U_POOLS = ["aéAÉ_다", "abé✓😀", "éÉeE-/x", "нНaя_Я", "ab", "fooBar_/-é다😀", "aA_bB-"]
B_POOLS = ["abAB_/-ab01", "ab", "fooBar_x", "aA bB/cC", "abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_-/."]
BYTE_SC = scorings(seed=7300, count=24, max_needle=64)
UNI_SC = unicode_scorings(seed=7400, count=30, max_needle=64)
LIT_SC_U = literal_scorings(seed=7500, count=24, max_needle=64)
LIT_SC_B = literal_scorings(seed=7600, count=20, max_needle=1024)


def needle_of_bytes(rng, pool, nbytes):
    """A string of scalars from `pool` of at most `nbytes` UTF-8 bytes (at least one scalar)."""
    s = rng.choice(pool)
    while True:
        c = rng.choice(pool)
        if len((s + c).encode()) > nbytes:
            return s
        s += c


# ---------------------------------------------------------------- the library's constants
def test_library_constants_equal_the_harness_construction(H):
    """host.cu's FrzUScoring / FrzUNeedle (what k_unicode and k_match_indices receive) equal the construction the CPU
    harness restates (scoring_of, frz_build_uneedle): every field, for ASCII needles on the byte path and unicode needles,
    all three case modes, the u8 and the u16 family; literal patterns carry only the raw fields (lane constants 0)."""
    rng = random.Random(7100)
    checked = {"byte": 0, "unicode": 0, "literal": 0, "u8": 0, "u16": 0}
    pool_sc = [(sc, "fuzzy") for sc in BYTE_SC + UNI_SC] + [(sc, "literal") for sc in LIT_SC_U]
    for sc, kind in pool_sc:
        for trial in range(16):
            uni = trial % 2 == 1
            pool = rng.choice(U_POOLS if uni else B_POOLS)
            needle = needle_of_bytes(rng, pool, rng.choice([rng.randint(1, 13), rng.randint(1, 64)]))
            casing = [CaseMatching.Ignore, CaseMatching.Smart, CaseMatching.Respect][trial % 3]
            matching = rng.choice([Matching.Exact, Matching.Prefix, Matching.Suffix, Matching.Substring]) if kind == "literal" else Matching.Fuzzy
            cfg = Config(max_typos=rng.choice([None, 0, 1, 3]), casing=casing, matching=matching, scoring=sc,
                         unicode=UnicodeMatching.Always if uni else UnicodeMatching.Ignore, emulate_lanes=rng.choice([16, 32, 64]))
            try:
                un, usc, info = library_constants(needle, cfg)
            except F.FrizbeeError:   # the byte path's signed 16-bit cell bound refuses some unicode-accepted scorings
                assert not uni and kind == "fuzzy"
                continue
            nb = needle.encode()
            want = fields(harness_scoring(H, sc, info["score_bits"]))
            got = fields(usc)
            if kind == "literal":
                assert all(got[f] == 0 for f in U_FIELDS), (needle, sc, got)
                assert {f: got[f] for f in RAW_FIELDS} == {f: want[f] for f in RAW_FIELDS}, (needle, sc, got, want)
                checked["literal"] += 1
            else:
                assert got == want, (needle, sc, cfg, got, want)
                checked["u8" if info["score_bits"] == 8 else "u16"] += 1
            cs = is_case_sensitive(H, nb, casing)
            ref = UNeedle()
            assert H.h_build_needle(nb, len(nb), int(cs), C.byref(ref)) == 1
            if uni:
                assert bytes(un) == bytes(ref), (needle, cs)
                checked["unicode"] += 1
            else:
                # byte path: the case_needle pairs only (f holds the needle itself, no scalar table)
                n = len(nb)
                assert (un.nbytes, un.n) == (n, 0)
                assert bytes(un.c)[:n] == nb and bytes(un.f)[:n] == nb, needle
                assert bytes(un.bflip)[:n] == bytes(ref.bflip)[:n] == case_pairs(nb, cs)[1], (needle, cs)
                checked["byte"] += 1
    assert min(checked.values()) > 200, checked


# ---------------------------------------------------------------- traceback (indices_path.cuh)
FORCED = [(8, 16), (16, 16), (32, 16), (16, 8), (32, 8), (64, 8)]
WINDOWS = [1, 2, 3, 7, 15, 16, 17, 31, 33, 63, 64, 65, 100, 127, 128, 129, 200, 255, 256, 300, 511, 700, 1023, 1024]


def traceback_window(rng, nb, pool_b, W):
    """W bytes of filler from `pool_b` with the needle (case-flipped here and there) planted whole or scattered."""
    hay = bytearray(rng.choice(pool_b) for _ in range(W))
    r = rng.random()
    if r < 0.7 and len(nb) <= W:
        if r < 0.35:
            s = rng.randint(0, W - len(nb))
            pos = range(s, s + len(nb))
        else:
            pos = sorted(rng.sample(range(W), len(nb)))
        for p, b in zip(pos, nb):
            hay[p] = b ^ 0x20 if (chr(b).isalpha() and b < 0x80 and rng.random() < 0.15) else b
    return bytes(hay)


def run_traceback(H, rng, trials, unicode_rows, counts):
    out = (C.c_uint32 * 2048)()
    cnt = C.c_int()
    scs = UNI_SC if unicode_rows else BYTE_SC
    for trial in range(trials):
        sc = TIES if trial % 7 == 0 else scs[trial % len(scs)]
        pool = rng.choice(U_POOLS if unicode_rows else B_POOLS)
        nbytes = rng.choice([rng.randint(1, 5), rng.randint(6, 16), rng.randint(1, 64)])
        needle = needle_of_bytes(rng, pool, nbytes)
        nb = needle.encode()
        k = rng.choice([None, 0, 1, 2, 3, 15])
        casing = rng.choice([CaseMatching.Ignore, CaseMatching.Smart, CaseMatching.Respect])
        cfg = Config(max_typos=k, casing=casing, scoring=sc, emulate_lanes=rng.choice([16, 32, 64]),
                     unicode=UnicodeMatching.Always if unicode_rows else UnicodeMatching.Ignore)
        try:
            un, usc, info = library_constants(needle, cfg)
        except F.FrizbeeError:
            continue   # the byte path refuses this needle length at this scoring
        cs = is_case_sensitive(H, nb, casing)
        W = rng.choice(WINDOWS) if rng.random() < 0.93 else rng.randint(1025, 1500)
        pool_b = (pool + "x_").encode()
        hay = traceback_window(rng, nb, pool_b, W)
        sp = rng.choice([0, 0, 1, 5, 300])
        # the backend the library selected, then the forced ones (the u8 family only where the scoring fits in u8: there
        # the library's u16 constants equal the truncated ones)
        backends = [(info["lanes"], info["score_bits"])] + [rng.choice(FORCED)]
        for lanes, bits in backends:
            if bits == 8 and not O.score_fits_in_u8(len(nb), sc):
                continue
            got = H.h_sw_indices_c(C.byref(un), int(unicode_rows), C.byref(usc), hay, len(hay), sp, -1 if k is None else k,
                                   lanes, bits, out, 2048, C.byref(cnt))
            want = O.sw_indices(nb, hay, sp, k, unicode_rows, sc, cs, lanes, bits)
            assert (got, list(out[: cnt.value])) == want, (needle, hay, sp, k, cs, lanes, bits, sc, got, list(out[: cnt.value]), want)
            counts["cases"] += 1
            counts["greedy"] += len(hay) > 1024
            counts["matched"] += got > 0
            counts["ties"] += sc == TIES


@pytest.mark.parametrize("rows", ["bytes", "scalars"])
def test_traceback_across_scorings(H, rows):
    """frzi::sw_indices (score with full matrices + AlignmentPathIter, or the greedy form past 1024 bytes) with the
    library's constants at its own backend and a forced one, vs the oracle's score_haystack_indices: needles of 1-64
    bytes, max_typos None/0/1/2/3/15, start_pos 0 and > 0, windows of 1-1500 bytes; every seventh case scores with zero
    gap and mismatch penalties, where diagonal, left and up cells tie."""
    rng = random.Random(7200 + (rows == "scalars"))
    counts = dict(cases=0, greedy=0, matched=0, ties=0)
    run_traceback(H, rng, 5000, rows == "scalars", counts)
    assert counts["cases"] > 7500 and counts["greedy"] > 400 and counts["ties"] > 1000, counts
    assert counts["matched"] > counts["cases"] // 3, counts


# ---------------------------------------------------------------- unicode Smith-Waterman score
def test_unicode_sw_score_long_needles(H):
    """frzu::sw_score with the library's constants for needles of 6-64 bytes (up to 64 scalars), at the backend the
    library selects and at a forced one, vs the oracle's score_haystack_unicode; scorings include those whose scores
    pass 32 767."""
    rng = random.Random(7250)
    checked = high = 0
    for trial in range(4000):
        sc = UNI_SC[trial % len(UNI_SC)]
        pool = rng.choice(U_POOLS)
        needle = needle_of_bytes(rng, pool, rng.choice([rng.randint(6, 20), rng.randint(6, 64), 64]))
        nb = needle.encode()
        if len(nb) < 6:
            continue
        casing = rng.choice([CaseMatching.Ignore, CaseMatching.Smart, CaseMatching.Respect])
        un, usc, info = library_constants(needle, Config(max_typos=None, casing=casing, scoring=sc, unicode=UnicodeMatching.Always,
                                                         emulate_lanes=rng.choice([16, 32, 64])))
        cs = is_case_sensitive(H, nb, casing)
        W = rng.choice([len(nb), len(nb) + 3, 40, 64, 65, 130, 300, 1024, 1100])
        w = traceback_window(rng, nb, (pool + "x_").encode(), max(W, 1))
        if rng.random() < 0.15 or (sc.match_score > 500 and rng.random() < 0.5):
            w = nb
        pref = rng.random() < 0.5
        for lanes, bits in [(info["lanes"], info["score_bits"]), rng.choice(FORCED)]:
            if bits == 8 and not O.score_fits_in_u8(len(nb), sc):
                continue
            got = H.h_sw_score_c(C.byref(un), C.byref(usc), w, len(w), int(pref), lanes, bits)
            want = O.sw_score_unicode(nb, w, sc, cs, pref, lanes, bits)
            assert got == want, (needle, w, cs, pref, lanes, bits, sc, got, want)
            checked += 1
            high += want > 32767
    assert checked > 5500 and high > 50, (checked, high)


# ---------------------------------------------------------------- literal matchers
MODES = [Matching.Exact, Matching.Prefix, Matching.Suffix, Matching.Substring]


def literal_haystacks(rng, needle: str, filler: str):
    """Haystacks for a literal needle: the needle alone (exact bonus), and the needle twice or three times in contexts
    that earn different bonuses — at position 0 (prefix), after a delimiter, after a lowercase letter (capitalization when
    the needle starts uppercase), after an uppercase letter — or the same context twice (a tie: the earliest wins)."""
    ctx = ["", "_", "a", "Z", "/", rng.choice(filler) if filler else "x"]
    mid = lambda: "".join(rng.choice(filler) for _ in range(rng.choice([0, 1, 3, 9])))
    out = [needle, needle + needle]
    for _ in range(4):
        a, b, c = rng.choice(ctx), rng.choice(ctx), rng.choice(ctx)
        out.append(a + needle + mid() + b + needle + mid())
        out.append(mid() + a + needle + b + needle + c + needle)
    flip = needle.swapcase()
    out.append("a" + flip + "_" + needle)     # the same needle in either case
    out.append(needle + "x" + needle[:-1])    # a cut-off second occurrence
    return out


def check_literal(got, pos, score, want, n, ctx):
    """want: the oracle's match_indices entry (score, exact, reversed contiguous run of the match) or None"""
    assert got == (want is not None), ctx
    if want is not None:
        assert (score, pos) == (want[0], min(want[2])), (ctx, score, pos, want)
        assert want[2] == list(range(pos + n - 1, pos - 1, -1)), (ctx, want)


def test_unicode_literal_across_scorings(H):
    """frzu::lit_find (all four modes) with the library's constants vs the oracle's match_list_indices: score, exact flag
    and the chosen position, for needles of 1-64 bytes, scorings with distinct bonuses and exact_match_bonus up to its
    guard."""
    rng = random.Random(7350)
    pos, score = C.c_int(), C.c_uint32()
    checked = found = subst = exact = 0
    for trial in range(600):
        sc = LIT_SC_U[trial % len(LIT_SC_U)]
        pool = rng.choice(U_POOLS)
        needle = needle_of_bytes(rng, pool, rng.choice([rng.randint(1, 6), rng.randint(1, 64), 64]))
        nb = needle.encode()
        mode = MODES[trial % 4]
        casing = rng.choice([CaseMatching.Ignore, CaseMatching.Respect, CaseMatching.Smart])
        cfg = Config(matching=mode, casing=casing, unicode=UnicodeMatching.Always, scoring=sc)
        un, usc, info = library_constants(needle, cfg)
        assert info["literal"]
        hs = literal_haystacks(rng, needle, pool)
        data, off = O.pack(hs)
        want = O.match_indices(Pattern(needle), cfg, data, off, list(range(len(hs))), stride=256)
        for j, h in enumerate(hs):
            hb = h.encode()
            got = H.h_lit_find_c(C.byref(un), C.byref(usc), hb, len(hb), int(mode), C.byref(pos), C.byref(score))
            check_literal(got, pos.value, score.value, want[j], len(nb), (needle, h, mode, casing, sc))
            if got:
                assert (pos.value == 0 and len(nb) == len(hb)) == want[j][1]
                found += 1
                exact += want[j][1]
                subst += mode == Matching.Substring
            checked += 1
    assert checked == 7200 and found > 3000 and subst == 1800 and exact > 400, (checked, found, subst, exact)


def test_byte_literal_across_scorings(H, PS):
    """lit_find of prefilter_scan.cuh (the byte path's literal matcher, FrzPatternDev and LongPat forms) with the library's
    pattern vs the oracle: score, exact flag and the chosen position, for needles of 1-1024 bytes in all four modes."""
    rng = random.Random(7450)
    pos, score = C.c_int(), C.c_uint32()
    checked = found = longs = subst = 0
    for trial in range(400):
        sc = LIT_SC_B[trial % len(LIT_SC_B)]
        pool = rng.choice(B_POOLS)
        n = rng.choice([rng.randint(1, 8), rng.randint(1, 64), rng.randint(65, 1024), 1024])
        needle = "".join(rng.choice(pool) for _ in range(n))
        nb = needle.encode()
        mode = MODES[trial % 4]
        casing = rng.choice([CaseMatching.Ignore, CaseMatching.Respect])
        cs = casing == CaseMatching.Respect
        cfg = Config(matching=mode, casing=casing, unicode=UnicodeMatching.Ignore, scoring=sc)
        m = F.Matcher(needle, cfg)
        pat = (C.c_uint8 * PS.h_pattern_size())()
        F._check(F.lib().frz_matcher_debug_pattern(m._h, 0, pat, len(pat)))
        m.close()
        c, flip = case_pairs(nb, cs)
        hs = literal_haystacks(rng, needle, pool)
        data, off = O.pack(hs)
        want = O.match_indices(Pattern(needle), cfg, data, off, list(range(len(hs))), stride=1100)
        longs += n > 64
        for j, h in enumerate(hs):
            hb = h.encode()
            got = PS.h_lit_find(pat, c if n > 64 else None, flip if n > 64 else None, hb, len(hb), C.byref(pos), C.byref(score))
            check_literal(got, pos.value, score.value, want[j], n, (needle, h, mode, cs, sc))
            if got:
                found += 1
                subst += mode == Matching.Substring
            checked += 1
    assert checked == 4800 and found > 2000 and subst == 1200 and longs > 150, (checked, found, subst, longs)
