"""The register Smith-Waterman core of the GPU kernels (frizbee_b200/csrc/sw_core.cuh: SwCore, window assembly, exact
check) is compiled here for the CPU — same source, scalar stand-ins for the CUDA SIMD-in-register intrinsics — and run
against the oracle with the pattern constants of the real library (frz_matcher_debug_pattern).  Covers what a GPU is
otherwise needed for: every emulated lane width, the column-limited classes (CC 40/48/56/64), the 128-column variant,
the u8 wrap emulation and the shift-placement variants, across the scorings of tests/scorings.py.  k_sw_generic's scorers
(sw_generic.cuh) are built the same way from tests/harness/sw_generic_harness.cpp."""
import ctypes as C
import random

import numpy as np
import pytest

import frizbee_b200 as F
from cpu_harness import load
from frizbee_b200.types import CaseMatching, Config, Matching, Scoring, UnicodeMatching
from needles import case_pairs, case_sensitive, n_distinct, plant
from oracle import pyoracle as O
from scorings import scorings


@pytest.fixture(scope="module")
def H():
    L = load("sw_harness", opt="-O1", cuda_include=True)
    L.h_pattern_size.restype = C.c_size_t
    L.h_swcore.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                           C.POINTER(C.c_int)]
    L.h_pattern_flags.argtypes = [C.c_void_p] + [C.POINTER(C.c_int)] * 3
    return L


def device_pattern(H, needle, cfg):
    m = F.Matcher(needle, cfg)
    buf = (C.c_uint8 * H.h_pattern_size())()
    F._check(F.lib().frz_matcher_debug_pattern(m._h, 0, buf, len(buf)))
    info = m.backend_info()
    m.close()
    return buf, info


def rand_bytes(rng, pool, n):
    return bytes(rng.choice(pool) for _ in range(n))


POOLS = [b"abAB_/-ab01", b"ab", b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_-/.", b"aAbB_zZ9"]
HAY_EXTRA = b"\xc3\xa9\x00"   # haystacks may hold any bytes (multi-byte scalars, NUL)


# a scoring whose whole score range fits in u8 for needles of up to 64 bytes (and far longer): keeps them in the u8 family
SINGLE_PASS = Scoring(match_score=1, mismatch_penalty=0, gap_open_penalty=1, gap_extend_penalty=0, prefix_bonus=0,
                      capitalization_bonus=0, matching_case_bonus=0, exact_match_bonus=0, delimiter_bonus=0)


@pytest.mark.parametrize("lanes", [16, 32, 64])
def test_swcore_column_classes_equal_oracle(H, lanes):
    """SwCore<LANES, 64, no-wrap, VAR, CC>: the class the prefilter would choose and every wider one give the oracle's score."""
    column_classes_vs_oracle(H, lanes, long_u8=False)


@pytest.mark.parametrize("lanes", [16, 32, 64])
def test_swcore_column_classes_long_u8_needles(H, lanes):
    """The same for needles of up to 64 bytes: at the default scoring a u8 needle has at most 13 bytes, SINGLE_PASS keeps
    longer ones in u8, where the needle is longer than the window and W + n passes every class boundary."""
    column_classes_vs_oracle(H, lanes, long_u8=True)


def column_classes_vs_oracle(H, lanes, long_u8):
    rng = random.Random(5000 + lanes + 100 * long_u8)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    sc = SINGLE_PASS if long_u8 else Scoring()
    checked = 0
    for trial in range(400 if long_u8 else 700):
        pool = rng.choice(POOLS)
        n = rng.choice([rng.randint(1, 64), rng.randint(30, 64)]) if long_u8 else rng.randint(1, 11)
        needle = rand_bytes(rng, pool, n)
        if 0 in needle:
            continue
        cs = rng.random() < 0.3
        cfg = Config(max_typos=None, emulate_lanes=lanes, casing=CaseMatching.Respect if cs else CaseMatching.Ignore, scoring=sc)
        pat, info = device_pattern(H, needle, cfg)
        assert info["score_bits"] == 8 and info["lanes"] == lanes
        wrap8, col_classes, lane_pen = pattern_flags(H, pat)
        assert (wrap8, col_classes, lane_pen) == (False, True, long_u8)   # SINGLE_PASS: gap_extend 0 < gap_open
        for _ in range(6):
            W = rng.randint(1, 64)
            win = rand_bytes(rng, pool + (HAY_EXTRA if rng.random() < 0.3 else b""), W)
            pre = rng.random() < 0.5
            want = O.sw_score(needle, win, sc, cs, pre, lanes, 8)
            chunk_cols = (W + lanes - 1) // lanes * lanes
            need = min(W + n, chunk_cols)
            for cc in (40, 48, 56, 64):
                if cc < need or cc < W:
                    continue
                eq = C.c_int()
                var = rng.choice([0, 8]) | (16 if lane_pen else 0)   # the per-lane gap penalty form, as sw.cu launches it
                got = H.h_swcore(pat, win, W, rng.randint(0, 15), int(pre), lanes, 64, cc, 0, var, C.byref(eq))
                assert got == want, (needle, win, cs, pre, lanes, cc, var, got, want)
                assert bool(eq.value) == (win == needle)
                checked += 1
    assert checked > 3000


@pytest.mark.parametrize("lanes,bits", [(8, 16), (16, 16), (32, 16), (16, 8), (64, 8)])
def test_swcore_128_columns_and_u16_family(H, lanes, bits):
    rng = random.Random(6000 + lanes + bits)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    emulate = {(8, 16): 16, (16, 16): 32, (32, 16): 64, (16, 8): 16, (64, 8): 64}[(lanes, bits)]
    for trial in range(150):
        pool = rng.choice(POOLS)
        n = rng.choice([rng.randint(14, 64), rng.randint(40, 64)]) if bits == 16 else rng.randint(1, 10)
        needle = rand_bytes(rng, pool, n)
        cfg = Config(max_typos=None, emulate_lanes=emulate, casing=CaseMatching.Ignore)
        pat, info = device_pattern(H, needle, cfg)
        assert (info["lanes"], info["score_bits"]) == (lanes, bits)
        for _ in range(3):
            W = rng.choice([rng.randint(1, n), rng.randint(n, 128), rng.randint(1, 64)])
            win = rand_bytes(rng, pool + (HAY_EXTRA if rng.random() < 0.3 else b""), W)
            pre = rng.random() < 0.5
            want = O.sw_score(needle, win, Scoring(), False, pre, lanes, bits)
            eq = C.c_int()
            got = H.h_swcore(pat, win, W, rng.randint(0, 15), int(pre), lanes, 128, 128, 0, 0, C.byref(eq))
            assert got == want, (needle, win, pre, lanes, bits, got, want)
            if W <= 64:
                got64 = H.h_swcore(pat, win, W, rng.randint(0, 15), int(pre), lanes, 64, 64, 0, 0, C.byref(eq))
                assert got64 == want


def test_swcore_u8_wrap_emulation(H):
    """12-13-byte needles at the default scoring can wrap the reference's u8 lanes (DESIGN.md §2 finding 3): the host
    selects WRAP8 and the kernel core must reproduce the wrapped arithmetic."""
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    rng = random.Random(7)
    needle = b"aB-cD-eF-gH-i"
    pat, info = device_pattern(H, needle, Config(max_typos=None, emulate_lanes=64))
    assert info["score_bits"] == 8
    hays = [needle, b"x" + needle, needle + b"yy", b"aB-cD-eF-gH-i_aB-cD-eF-gH-i"]
    hays += [rand_bytes(rng, b"aBcDeFgHi-_", rng.randint(5, 64)) for _ in range(400)]
    for win in hays:
        for pre in (True, False):
            want = O.sw_score(needle, win, Scoring(), True, pre, 64, 8)   # smart case: the needle has uppercase
            eq = C.c_int()
            got = H.h_swcore(pat, win, len(win), 3, int(pre), 64, 64, 64, 1, 0, C.byref(eq))
            assert got == want, (win, pre, got, want)


# ---------------------------------------------------------------- the scorers across the scoring space (tests/scorings.py)
MAX_NEEDLE = 24
SCORINGS = scorings(seed=424242, count=44, max_needle=MAX_NEEDLE)
SWEEP_POOLS = POOLS + [b"aBcD-_Xy", b"fooBAR/._", b"aA\x00b"]
HAY_HIGH = b"\x80\xc3\xa9\xff\x00"


def needle_for(rng, sc, lanes):
    """A needle whose reference backend runs `lanes` wide for scoring `sc`, with the emulate_lanes and score family
    that select it, or None when no such needle is drawn (LANES 8 is u16 only, LANES 64 u8 only)."""
    for _ in range(8):
        pool = rng.choice(SWEEP_POOLS)
        needle = rand_bytes(rng, pool, rng.choice([rng.randint(1, 6), rng.randint(1, MAX_NEEDLE), MAX_NEEDLE]))
        bits = 8 if O.score_fits_in_u8(len(needle), sc) else 16
        em = lanes if bits == 8 else 2 * lanes
        if em in (16, 32, 64):
            return needle, pool, bits, em
    return None


def case_for(rng, needle):
    casing = rng.choice([CaseMatching.Ignore, CaseMatching.Respect, CaseMatching.Smart])
    cs = casing == CaseMatching.Respect or (casing == CaseMatching.Smart and any(65 <= b <= 90 for b in needle))
    return casing, cs


def sweep_window(rng, needle, pool, W):
    r = rng.random()
    if r < 0.08 and len(needle) == W:
        return needle
    if r < 0.12 and len(needle) == W:
        return needle.swapcase()
    extra = rng.choice([b"", b"x", HAY_HIGH])
    return rand_bytes(rng, pool + extra, W)


def pattern_flags(H, pat):
    wrap8, col_classes, lane_pen = C.c_int(), C.c_int(), C.c_int()
    H.h_pattern_flags(pat, C.byref(wrap8), C.byref(col_classes), C.byref(lane_pen))
    return bool(wrap8.value), bool(col_classes.value), bool(lane_pen.value)


@pytest.mark.parametrize("lanes", [8, 16, 32, 64])
def test_swcore_scoring_sweep(H, lanes):
    """SwCore with the constants of generated scorings (tests/scorings.py: zeros, gap_extend = 0 < gap_open,
    gap_open < gap_extend, constants >= 256, both sides of score_fits_in_u8, WRAP8 through the scoring, the signed 16-bit
    bounds) vs the oracle at the same LANES and score family.  Each window is scored by the instantiation the kernels
    launch for it (column class as prefilter.cu: sw_class_of, WRAP8, the per-lane penalty variant) and by every wider
    column class, with both bonus forms (VAR 0 / 8); all three case modes, needles with NUL and uppercase letters,
    haystack bytes >= 0x80 and NUL, every startlo, prefix bonus on and off, and the exact-window check."""
    rng = random.Random(31000 + lanes)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    checked, seen = 0, set()
    for trial in range(400):
        sc = SCORINGS[trial % len(SCORINGS)]
        drawn = needle_for(rng, sc, lanes)
        if drawn is None:
            continue
        needle, pool, bits, em = drawn
        casing, cs = case_for(rng, needle)
        pat, info = device_pattern(H, needle, Config(max_typos=None, emulate_lanes=em, casing=casing, scoring=sc))
        assert (info["lanes"], info["score_bits"]) == (lanes, bits)
        wrap8, col_classes, lane_pen = pattern_flags(H, pat)
        assert col_classes == (not wrap8 and 0 not in needle)
        seen.add((bits, wrap8, lane_pen, cs))
        for _ in range(5):
            W = rng.choice([len(needle), rng.randint(1, 64), rng.randint(1, 64), rng.randint(65, 128)])
            W = max(1, min(W, 128))
            win = sweep_window(rng, needle, pool, W)
            pre = rng.random() < 0.5
            want = O.sw_score(needle, win, sc, cs, pre, lanes, bits)
            if W <= 64:
                cols = 64
                if col_classes:
                    need = min(W + len(needle), (W + lanes - 1) // lanes * lanes)
                    cls_cc = next(cc for cc in (40, 48, 56, 64) if need <= cc)
                    ccs = [cc for cc in (40, 48, 56, 64) if cc >= cls_cc]
                else:
                    ccs = [64]
            else:
                cols = 128
                need = min(W + len(needle), (W + lanes - 1) // lanes * lanes)
                ccs = [128] + ([cc for cc in (80, 96, 112) if cc >= need and cc >= W] if col_classes else [])
            for cc in ccs:
                for var in ((0,) if wrap8 else (0, 8)):
                    v = var | (16 if lane_pen else 0)
                    eq = C.c_int()
                    startlo = rng.randint(0, 15)
                    got = H.h_swcore(pat, win, W, startlo, int(pre), lanes, cols, cc, int(wrap8), v, C.byref(eq))
                    assert got == want, (needle, win, sc, cs, pre, lanes, bits, cols, cc, v, startlo, got, want)
                    assert bool(eq.value) == (win == needle)
                    checked += 1
    assert checked > 2500, checked
    # the sweep reached the variants that matter at this width
    assert any(lp for _, _, lp, _ in seen) and any(cs for *_, cs in seen)
    if lanes != 8:
        assert any(w for _, w, _, _ in seen)
    assert {b for b, *_ in seen} == ({16} if lanes == 8 else {8} if lanes == 64 else {8, 16})


# ---------------------------------------------------------------- k_sw_generic's scorers (sw_generic.cuh)

@pytest.fixture(scope="module")
def G():
    L = load("sw_generic_harness", cuda_include=True)
    L.h_pattern_size.restype = C.c_size_t
    L.h_sw_generic.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int]
    L.h_greedy.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int]
    return L


@pytest.mark.parametrize("lanes", [8, 16, 32, 64])
def test_generic_scorer_across_scorings(H, G, lanes):
    """generic_score (k_sw_generic, windows of 129..1024 bytes: true u8 / u16 element arithmetic) vs the oracle's
    score_haystack at the same LANES and family, over the scoring sweep."""
    assert G.h_pattern_size() == H.h_pattern_size()
    rng = random.Random(33000 + lanes)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    checked, families = 0, set()
    for trial in range(3 * len(SCORINGS)):
        sc = SCORINGS[trial % len(SCORINGS)]
        drawn = needle_for(rng, sc, lanes)
        if drawn is None:
            continue
        needle, pool, bits, em = drawn
        casing, cs = case_for(rng, needle)
        pat, info = device_pattern(H, needle, Config(max_typos=None, emulate_lanes=em, casing=casing, scoring=sc))
        assert (info["lanes"], info["score_bits"]) == (lanes, bits)
        families.add(bits)
        for W in (rng.choice([129, 130, 1023, 1024]), rng.randint(129, 1024)):
            win = rand_bytes(rng, pool + rng.choice([b"", b"x-", HAY_HIGH]), W)
            pre = rng.random() < 0.5
            want = O.sw_score(needle, win, sc, cs, pre, lanes, bits)
            got = G.h_sw_generic(pat, win, W, int(pre))
            assert got == want, (needle, win, sc, cs, pre, lanes, bits, got, want)
            checked += 1
    assert checked > 60, checked
    assert families == ({16} if lanes == 8 else {8} if lanes == 64 else {8, 16})


def test_greedy_scorer_across_scorings(H, G):
    """greedy_score (k_sw_generic, windows over 1024 bytes) vs the oracle's match_greedy, over the scoring sweep: windows
    that hold the needle's bytes spread out (gaps of every length, either case) and windows that miss one of them."""
    rng = random.Random(34000)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    matched = missed = 0
    for trial in range(4 * len(SCORINGS)):
        sc = SCORINGS[trial % len(SCORINGS)]
        pool = rng.choice(SWEEP_POOLS)
        needle = rand_bytes(rng, pool, rng.randint(1, MAX_NEEDLE))
        casing, cs = case_for(rng, needle)
        pat, _ = device_pattern(H, needle, Config(max_typos=None, casing=casing, scoring=sc))
        W = rng.randint(1025, 3000)
        filler = rand_bytes(rng, b"xyz_-/ 019QW" + HAY_HIGH, W)
        if rng.random() < 0.8:   # plant the needle at sorted random positions, some bytes case-flipped
            pos = sorted(rng.sample(range(W), len(needle)))
            win = bytearray(filler)
            for p, b in zip(pos, needle):
                win[p] = b ^ 0x20 if (chr(b).isalpha() and rng.random() < 0.3) else b
            win = bytes(win)
        else:
            win = filler
        pre = rng.random() < 0.5
        want = O.match_greedy(needle, win, sc, cs, pre)
        got = G.h_greedy(pat, win, W, int(pre))
        assert got == (-1 if want is None else want), (needle, sc, cs, pre, got, want)
        matched += want is not None
        missed += want is None
    assert matched > 40 and missed > 10, (matched, missed)


# ---------------------------------------------------------------- occurrence-mask prefilter windows (prefilter_masks.cuh)

@pytest.fixture(scope="module")
def PF():
    L = load("pf_harness", opt="-O1", cuda_include=True)
    L.h_masks_window.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.h_n_distinct.argtypes = [C.c_void_p]
    return L


# needles with few byte classes (the occurrence-mask forms take needles of up to 64 bytes with <= 16 classes)
MASK_POOLS = [b"ab", b"aAbBcC", b"abAB_/-01", b"aAbB_zZ9"]


def mask_needle(rng, pool, n_max=64):
    return rand_bytes(rng, pool, rng.choice([rng.randint(1, 12), rng.randint(1, n_max), rng.randint(13, n_max)]))


def mask_haystack(rng, needle, pool, ln, k):
    """`ln` bytes of the pool, about half of them holding the needle with 0..k+1 of its bytes deleted"""
    filler = pool + (HAY_EXTRA if rng.random() < 0.2 else b"x")
    if ln and rng.random() < 0.5:
        return plant(rng, needle, ln, filler, drops=rng.randint(0, k + 1), spread=rng.random() < 0.4)
    return rand_bytes(rng, filler, ln)


def test_n_distinct_helper_equals_compile_pattern(H, PF):
    """tests/needles.py: n_distinct (used by the GPU tests to tell which prefilter form a needle takes) equals the
    FrzPatternDev.n_distinct host.cu: compile_pattern writes, on both sides of 16 classes and of 64 bytes."""
    rng = random.Random(8800)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    seen = set()
    for trial in range(600):
        pool = rng.choice(MASK_POOLS + POOLS + [b"abcdefghijklmnopq", b"aA\x00zZ"])
        needle = rand_bytes(rng, pool, rng.choice([rng.randint(1, 20), rng.randint(1, 64), rng.randint(60, 70)]))
        casing = rng.choice([CaseMatching.Ignore, CaseMatching.Respect, CaseMatching.Smart])
        pat, _ = device_pattern(H, needle, Config(max_typos=1, casing=casing, unicode=UnicodeMatching.Ignore))
        want = PF.h_n_distinct(pat)
        assert n_distinct(needle, case_sensitive(needle, casing)) == want, (needle, casing, want)
        seen.add((want == 0, len(needle) > 64))
    assert seen == {(False, False), (True, False), (True, True)}


@pytest.mark.parametrize("lanes", [16, 32, 64])
@pytest.mark.parametrize("k", [0, 1])
def test_mask_prefilter_windows_equal_oracle(H, PF, lanes, k):
    """masks_k0 / masks_k1 (DP4A-packed occurrence masks + the reference's mask state machine at chunk width LANES) vs
    Prefilter::match_haystack / match_haystack_1_typo, on haystacks of up to 200 bytes (several 64-byte blocks)."""
    rng = random.Random(8000 + lanes + k)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    checked = matched = long_needles = 0
    for trial in range(500):
        pool = rng.choice(MASK_POOLS)
        needle = mask_needle(rng, pool)
        long_needles += len(needle) > 24
        cs = rng.random() < 0.3
        cfg = Config(max_typos=k, emulate_lanes=lanes, casing=CaseMatching.Respect if cs else CaseMatching.Ignore)
        pat, info = device_pattern(H, needle, cfg)
        assert info["prefilter_lanes"] == lanes
        assert PF.h_n_distinct(pat) == n_distinct(needle, cs) > 0
        for _ in range(12):
            ln = rng.choice([0, 1, 2, 7, 15, 16, 17, 31, 33, 50, 63, 64, 65, 100, 128, 129, 200])
            hay = mask_haystack(rng, needle, pool, ln, k)
            s, e = C.c_int(), C.c_int()
            got = PF.h_masks_window(pat, hay, len(hay), k, C.byref(s), C.byref(e))
            assert got >= 0
            want = O.prefilter(needle, hay, k, lanes, cs)
            assert bool(got) == want[0], (needle, hay, k, lanes, cs, want)
            if want[0]:
                assert (s.value, e.value) == (want[1], want[2]), (needle, hay, k, lanes, cs, want, s.value, e.value)
                matched += 1
            checked += 1
    assert checked > 5000 and matched > 1000 and long_needles > 150


@pytest.mark.parametrize("k", [0, 1])
def test_single_chunk_mask_forms_equal_oracle(H, PF, k):
    """masks_k0_single / masks_k1_single (corpora of <= 64-byte haystacks at the 64-lane width: one block, one chunk,
    per-position masks) vs the oracle's Prefilter::match_haystack / match_haystack_1_typo.  Needles of up to 64 bytes: the
    single-chunk forms take those with n_distinct + n <= 16, the others are refused (the kernel runs masks_k0 / masks_k1,
    checked here too)."""
    rng = random.Random(9100 + k)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    checked = matched = refused = 0
    for trial in range(900):
        pool = rng.choice(POOLS if rng.random() < 0.5 else MASK_POOLS)
        needle = rand_bytes(rng, pool, rng.randint(1, 11) if rng.random() < 0.6 else rng.randint(1, 64))
        cs = rng.random() < 0.3
        cfg = Config(max_typos=k, emulate_lanes=64, casing=CaseMatching.Respect if cs else CaseMatching.Ignore)
        pat, info = device_pattern(H, needle, cfg)
        nd = n_distinct(needle, cs)
        if nd == 0:
            continue
        for _ in range(12):
            ln = rng.choice([0, 1, 2, 3, 7, 15, 16, 17, 31, 32, 33, 47, 48, 50, 63, 64])
            hay = mask_haystack(rng, needle, pool, ln, k)
            s, e = C.c_int(), C.c_int()
            got = PF.h_masks_window(pat, hay, len(hay), 100 + k, C.byref(s), C.byref(e))
            if got == -2:   # n_distinct + n > 16: the kernel takes the general form
                assert nd + len(needle) > 16
                refused += 1
                got = PF.h_masks_window(pat, hay, len(hay), k, C.byref(s), C.byref(e))
            else:
                assert nd + len(needle) <= 16
            want = O.prefilter(needle, hay, k, 64, cs)
            assert bool(got) == want[0], (needle, hay, k, cs, want)
            if want[0]:
                assert (s.value, e.value) == (want[1], want[2]), (needle, hay, k, cs, want, s.value, e.value)
                matched += 1
            checked += 1
    assert checked > 6000 and matched > 1500 and 1000 < refused < checked - 1000


@pytest.mark.parametrize("lanes", [16, 32, 64])
def test_signature_test_is_a_necessary_condition(H, PF, lanes):
    """Phase A of k_prefilter rejects a haystack from its 8-byte class signature alone.  That is only sound if the test is
    a NECESSARY condition of the reference's prefilters (all typo budgets, both case modes) and of the literal modes:
    whenever the oracle accepts, the signature test must pass — checked on dense alphabets (letters in both cases,
    digits, punctuation, non-ASCII bytes, NUL) where class collisions and multiplicities are common."""
    from frizbee_b200.types import Matching, Pattern
    rng = random.Random(4200 + lanes)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    PF.h_sig_pass.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
    pools = POOLS + [b"0123456789", b"a1b2c3_-./ ", b"eeeddd", b"aAzZ@[`{|~!"]
    accepted = rejected_by_sig = 0
    for trial in range(900):
        pool = rng.choice(pools)
        needle = rand_bytes(rng, pool, rng.randint(1, 12))
        k = rng.choice([0, 0, 1, 1, 2, 3, 5])
        cs = rng.random() < 0.3
        cfg = Config(max_typos=k, emulate_lanes=lanes, casing=CaseMatching.Respect if cs else CaseMatching.Ignore)
        pat, info = device_pattern(H, needle, cfg)
        for _ in range(16):
            ln = rng.choice([0, 1, 2, 5, 9, 16, 17, 31, 40, 64, 65, 100, 130])
            hay = rand_bytes(rng, pool + rng.choice([b"", b"x", b"XY9", HAY_EXTRA]), ln)
            ok = O.prefilter(needle, hay, k, lanes, cs)[0]
            sig = PF.h_sig_pass(pat, hay, len(hay))
            if ok:
                assert sig == 1, (needle, hay, k, lanes, cs)
                accepted += 1
            elif not sig:
                rejected_by_sig += 1
    assert accepted > 1500 and rejected_by_sig > 1500
    # literal modes: a literal match contains every needle byte (either case when case-insensitive)
    lit_ok = 0
    for trial in range(400):
        pool = rng.choice(pools)
        needle = rand_bytes(rng, pool, rng.randint(1, 6))
        if 0 in needle or any(b >= 0x80 for b in needle):
            continue
        cs = rng.random() < 0.3
        mode = rng.choice([Matching.Exact, Matching.Prefix, Matching.Suffix, Matching.Substring])
        cfg = Config(matching=mode, casing=CaseMatching.Respect if cs else CaseMatching.Ignore)
        pat, _ = device_pattern(H, needle, cfg)
        for _ in range(10):
            pre, post = rand_bytes(rng, pool, rng.randint(0, 5)), rand_bytes(rng, pool, rng.randint(0, 5))
            mid = bytes((b ^ 0x20) if (not cs and chr(b).isalpha() and rng.random() < 0.5) else b for b in needle)
            hay = {Matching.Exact: mid, Matching.Prefix: mid + post, Matching.Suffix: pre + mid, Matching.Substring: pre + mid + post}[mode]
            got = O.match_list([Pattern(needle.decode("latin-1"), matching=mode)], [hay.decode("latin-1")], cfg)
            if got:
                assert PF.h_sig_pass(pat, hay, len(hay)) == 1, (needle, hay, mode, cs)
                lit_ok += 1
    assert lit_ok > 500


@pytest.mark.parametrize("lanes", [16, 32, 64])
def test_signature_test_is_a_necessary_condition_for_unicode_needles(H, PF, lanes):
    """The unicode-needle path runs the same signature scan before k_unicode, with only the needle's ASCII scalars counted
    (host.cu: compile_pattern).  Necessary-condition check against the oracle's unicode prefilters (all typo budgets,
    both case modes) and unicode literal modes, on alphabets that mix ASCII letters in both cases with multi-byte scalars
    whose case flips differ in every byte."""
    from frizbee_b200.types import Matching, Pattern, UnicodeMatching
    rng = random.Random(9100 + lanes)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    PF.h_sig_pass.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
    pools = ["aéAÉ_다", "abé✓😀", "éÉeE-/x", "нНaя_Я", "ab", "aAbBkK", "sSßxX09"]
    accepted = rejected_by_sig = 0
    for trial in range(700):
        pool = rng.choice(pools)
        needle = "".join(rng.choice(pool) for _ in range(rng.randint(1, 7)))
        k = rng.choice([0, 0, 1, 1, 2, 3, 5])
        cs = rng.random() < 0.3
        cfg = Config(max_typos=k, emulate_lanes=lanes, unicode=UnicodeMatching.Always,
                     casing=CaseMatching.Respect if cs else CaseMatching.Ignore)
        pat, info = device_pattern(H, needle, cfg)
        for _ in range(16):
            hay = "".join(rng.choice(pool + rng.choice(["", "xyz", "XY9", "ÉЯ"])) for _ in range(rng.choice([0, 1, 2, 5, 9, 17, 31, 40, 70])))
            hb = hay.encode()
            ok = O.prefilter_unicode(needle, hay, k, lanes, cs)[0]
            sig = PF.h_sig_pass(pat, hb, len(hb))
            if ok:
                assert sig == 1, (needle, hay, k, lanes, cs)
                accepted += 1
            elif not sig:
                rejected_by_sig += 1
    assert accepted > 1200 and rejected_by_sig > 800, (accepted, rejected_by_sig)
    lit_ok = 0
    for trial in range(300):
        pool = rng.choice(pools)
        needle = "".join(rng.choice(pool) for _ in range(rng.randint(1, 5)))
        cs = rng.random() < 0.3
        mode = rng.choice([Matching.Exact, Matching.Prefix, Matching.Suffix, Matching.Substring])
        cfg = Config(matching=mode, unicode=UnicodeMatching.Always, casing=CaseMatching.Respect if cs else CaseMatching.Ignore)
        pat, _ = device_pattern(H, needle, cfg)
        for _ in range(10):
            pre = "".join(rng.choice(pool) for _ in range(rng.randint(0, 4)))
            post = "".join(rng.choice(pool) for _ in range(rng.randint(0, 4)))
            mid = "".join((ch.swapcase() if (not cs and rng.random() < 0.5 and len(ch.swapcase().encode()) == len(ch.encode())) else ch) for ch in needle)
            hay = {Matching.Exact: mid, Matching.Prefix: mid + post, Matching.Suffix: pre + mid, Matching.Substring: pre + mid + post}[mode]
            if O.match_list([Pattern(needle, matching=mode)], [hay], cfg):
                hb = hay.encode()
                assert PF.h_sig_pass(pat, hb, len(hb)) == 1, (needle, hay, mode, cs)
                lit_ok += 1
    assert lit_ok > 400, lit_ok


@pytest.mark.parametrize("lanes", [16, 32, 64])
@pytest.mark.parametrize("k", [1, 2, 3, 4, 5, 7, 10, 15])
def test_mask_prefilter_groundwork_2_and_n_typos(H, PF, lanes, k):
    """masks_paths<NP> / masks_many (prefilter_masks.cuh; k_scan_window and k_prefilter_list run them at k = 2 and k >= 3
    for needles with <= 16 byte classes, prefilter.cu: process_candidate) vs match_haystack_1_typo / _2_typos /
    _many_typos of the reference (src/prefilter/algo/ascii_typos.rs).  Needles of up to 64 bytes, n = k + 1 and n <= k
    among them; haystacks that hold the needle with 0..k+1 bytes deleted."""
    rng = random.Random(9000 + lanes + k)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    mode = {1: 12, 2: 2}.get(k, 3)
    checked = matched = 0
    lengths = set()
    for trial in range(200):
        pool = rng.choice(MASK_POOLS[:3])
        r = trial % 8
        needle = rand_bytes(rng, pool, k + 1 if r == 0 else rng.randint(1, k) if r == 1 else
                            rng.randint(1, 64) if r < 5 else rng.randint(33, 64))
        lengths.add(len(needle) - k)
        cs = rng.random() < 0.3
        cfg = Config(max_typos=k, emulate_lanes=lanes, casing=CaseMatching.Respect if cs else CaseMatching.Ignore)
        pat, info = device_pattern(H, needle, cfg)
        assert PF.h_n_distinct(pat) == n_distinct(needle, cs) > 0
        for _ in range(12):
            ln = rng.choice([0, 1, 2, 7, 15, 16, 17, 31, 33, 50, 63, 64, 65, 100, 128, 129, 200])
            hay = mask_haystack(rng, needle, pool, ln, k)
            s, e = C.c_int(), C.c_int()
            got = PF.h_masks_window(pat, hay, len(hay), mode, C.byref(s), C.byref(e))
            want = O.prefilter(needle, hay, k, lanes, cs)
            assert bool(got) == want[0], (needle, hay, k, lanes, cs, want)
            if want[0]:
                assert (s.value, e.value) == (want[1], want[2]), (needle, hay, k, lanes, cs, want, s.value, e.value)
                matched += 1
            checked += 1
    assert checked == 2400 and matched > checked // 3, (checked, matched)
    assert 1 in lengths and min(lengths) <= 0 and max(lengths) >= 64 - k - 8


@pytest.mark.parametrize("lanes", [16, 32, 64])
def test_swcore_128_column_classes_groundwork(H, lanes):
    """SwCore<LANES, 128, ., ., CC> with CC in {80, 96, 112}: the column-limited form of the 65..128-byte window class
    (not yet used by the kernels) gives the oracle's score whenever CC >= min(W + n, ceil(W / LANES) * LANES)."""
    rng = random.Random(12000 + lanes)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    checked = 0
    for trial in range(120):
        pool = rng.choice(POOLS)
        n = rng.randint(1, 11)
        needle = rand_bytes(rng, pool, n)
        pat, info = device_pattern(H, needle, Config(max_typos=None, emulate_lanes=lanes, casing=CaseMatching.Ignore))
        for _ in range(4):
            W = rng.randint(40, 120)
            win = rand_bytes(rng, pool + (HAY_EXTRA if rng.random() < 0.3 else b""), W)
            pre = rng.random() < 0.5
            want = O.sw_score(needle, win, Scoring(), False, pre, lanes, 8)
            need = min(W + n, (W + lanes - 1) // lanes * lanes)
            for cc in (80, 96, 112, 128):
                if cc < need or cc < W:
                    continue
                eq = C.c_int()
                got = H.h_swcore(pat, win, W, rng.randint(0, 15), int(pre), lanes, 128, cc, 0, 0, C.byref(eq))
                assert got == want, (needle, win, pre, lanes, cc, got, want)
                checked += 1
    assert checked > 500


# ---------------------------------------------------------------- scanning prefilter forms and the literal matcher (prefilter_scan.cuh)

@pytest.fixture(scope="module")
def PS():
    L = load("pf_scan_harness", cuda_include=True)
    ip = C.POINTER(C.c_int)
    L.h_scan_window.argtypes = [C.c_void_p, C.c_char_p, C.c_int, ip, ip]
    L.h_scan_window_long.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int, ip, ip]
    L.h_lit_find.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int, ip, C.POINTER(C.c_uint32)]
    L.h_pattern_probes.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    return L


SCAN_POOLS = [b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_-/. ", b"abcdefghijklmnopqrs",
              b"aAbBcC", b"abAB_/-01", b"ab\x00-Zz"]
SCAN_LENS = [0, 1, 2, 3, 4, 5, 7, 15, 16, 17, 31, 32, 33, 63, 64, 65, 100, 128, 129, 255, 256, 511, 1024, 1025, 2600]


def scan_case(rng, n):
    """a needle of n bytes (few or many byte classes, NUL among them), its case mode and typo budget"""
    pool = rng.choice(SCAN_POOLS)
    needle = rand_bytes(rng, pool, n)
    casing = rng.choice([CaseMatching.Ignore, CaseMatching.Respect, CaseMatching.Smart])
    k = rng.choice(list(range(16)) + [n, n + rng.randint(1, 5)])
    return needle, pool, casing, case_sensitive(needle, casing), k


def scan_haystack(rng, needle, pool, k):
    ln = rng.choice(SCAN_LENS)
    filler = pool + rng.choice([b"", b"xyz", HAY_EXTRA, b"\x80\xff\x00"])
    if ln >= 1 and rng.random() < 0.55:
        return plant(rng, needle, ln, filler, drops=rng.randint(0, k + 1), spread=rng.random() < 0.4, flip_p=0.15)
    return rand_bytes(rng, filler, ln)


def check_window(got, s, e, want, ctx):
    assert got >= 0, ctx
    assert bool(got) == want[0], (ctx, want)
    if want[0]:
        assert (s.value, e.value) == (want[1], want[2]), (ctx, want, s.value, e.value)


@pytest.mark.parametrize("lanes", [16, 32, 64])
def test_scan_forms_equal_oracle(H, PS, lanes):
    """window_k0 / _k1 / _k2 / _many on FrzPatternDev (the form the pattern's typo mode selects, as k_match_indices and,
    for needles of more than 16 byte classes, k_scan_window / k_prefilter_list run it) vs Prefilter::match_haystack* of
    the reference, window bounds included: needles of 1..64 bytes on both sides of 16 classes, k in 0..15 and >= n, all
    three case modes, haystacks of 0..2600 bytes with NUL and bytes >= 0x80."""
    rng = random.Random(15000 + lanes)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    checked = matched = 0
    forms, budgets = set(), set()
    for trial in range(1500):
        n = rng.choice([rng.randint(1, 16), rng.randint(1, 64), rng.randint(40, 64)])
        needle, pool, casing, cs, k = scan_case(rng, n)
        pat, info = device_pattern(H, needle, Config(max_typos=k, emulate_lanes=lanes, casing=casing,
                                                     unicode=UnicodeMatching.Ignore))
        assert info["prefilter_lanes"] == lanes
        forms.add(n_distinct(needle, cs) > 0)
        budgets.add(min(k, 16) if k < n else "all")
        for _ in range(8):
            hay = scan_haystack(rng, needle, pool, k)
            s, e = C.c_int(), C.c_int()
            got = PS.h_scan_window(pat, hay, len(hay), C.byref(s), C.byref(e))
            want = O.prefilter(needle, hay, k, lanes, cs)
            check_window(got, s, e, want, (needle, hay, k, lanes, cs))
            matched += want[0]
            checked += 1
    assert forms == {True, False} and budgets >= set(range(16)) | {"all"}, (forms, budgets)
    assert checked == 12000 and checked // 4 < matched < checked - checked // 4, matched


@pytest.mark.parametrize("lanes", [16, 32, 64])
def test_scan_forms_long_needles_equal_oracle(H, PS, lanes):
    """The same forms on LongPat (k_scan_window_long / k_prefilter_list_long: needles of 65..1024 bytes, per-position data
    from the needle table) vs the oracle.  The needle table is built from the case_needle pairs with host.cu's probes,
    checked against the pattern's own probes over its first 64 positions."""
    rng = random.Random(16000 + lanes)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    checked = matched = 0
    om, tg = C.create_string_buffer(64), C.create_string_buffer(64)
    for trial in range(300):
        n = rng.choice([65, rng.randint(65, 200), rng.randint(65, 1024), 1024])
        needle, pool, casing, cs, k = scan_case(rng, n)
        pat, info = device_pattern(H, needle, Config(max_typos=k, emulate_lanes=lanes, casing=casing,
                                                     unicode=UnicodeMatching.Ignore))
        c, flip = case_pairs(needle, cs)
        PS.h_pattern_probes(pat, om, tg)
        assert [(om.raw[i], tg.raw[i]) for i in range(64)] == [
            (0x20, x | 0x20) if f != x else (0, x) for x, f in zip(c[:64], flip[:64])]
        for _ in range(6):
            hay = scan_haystack(rng, needle, pool, k)
            s, e = C.c_int(), C.c_int()
            got = PS.h_scan_window_long(pat, c, flip, hay, len(hay), C.byref(s), C.byref(e))
            want = O.prefilter(needle, hay, k, lanes, cs)
            check_window(got, s, e, want, (n, hay, k, lanes, cs))
            matched += want[0]
            checked += 1
    assert checked == 1800 and matched > 200 and checked - matched > 500, matched


def test_literal_matcher_equals_oracle(H, PS):
    """lit_find (the literal modes of the byte path, on FrzPatternDev and on LongPat) vs the oracle's match_list in the
    same mode: match, score and exact flag, for needles of 1..1024 bytes and both case modes."""
    rng = random.Random(17000)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    found = missed = longs = 0
    for trial in range(1000):
        n = rng.choice([rng.randint(1, 8), rng.randint(1, 64), rng.randint(60, 70), rng.randint(65, 1024)])
        pool = rng.choice(SCAN_POOLS)
        needle = rand_bytes(rng, pool, n)
        mode = [Matching.Exact, Matching.Prefix, Matching.Suffix, Matching.Substring][trial % 4]
        casing = rng.choice([CaseMatching.Ignore, CaseMatching.Respect])
        cs = casing == CaseMatching.Respect
        cfg = Config(matching=mode, casing=casing, unicode=UnicodeMatching.Ignore)
        pat, _ = device_pattern(H, needle, cfg)
        c, flip = case_pairs(needle, cs)
        longs += n > 64
        for _ in range(4):
            mid = bytes((b ^ 0x20) if (not cs and chr(b).isalpha() and b < 0x80 and rng.random() < 0.3) else b for b in needle)
            if rng.random() < 0.2 and n > 1:
                i = rng.randrange(n)
                mid = mid[:i] + b"#" + mid[i + 1:]
            pre = rand_bytes(rng, pool + b"_ ", rng.choice([0, 0, 1, 3, 40]))
            post = rand_bytes(rng, pool + b"_ ", rng.choice([0, 0, 1, 3, 40]))
            hay = rng.choice([mid, pre + mid, mid + post, pre + mid + post, pre + mid + post + mid])
            data, off = O.pack([hay])
            want = O.match_list_packed([needle], cfg, data, off)
            pos, score = C.c_int(), C.c_uint32()
            got = PS.h_lit_find(pat, c if n > 64 else None, flip if n > 64 else None, hay, len(hay), C.byref(pos), C.byref(score))
            assert got == len(want), (needle, hay, mode, cs)
            if got:
                exact = pos.value == 0 and n == len(hay)
                assert (score.value, exact) == (int(want["score"][0]), bool(want["exact"][0])), (needle, hay, mode, cs)
                found += 1
            else:
                missed += 1
    assert found > 1400 and missed > 400 and longs > 200, (found, missed, longs)
