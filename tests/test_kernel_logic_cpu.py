"""The register Smith-Waterman core of the GPU kernels (frizbee_b200/csrc/sw_core.cuh: SwCore, window assembly, exact
check) is compiled here for the CPU — same source, scalar stand-ins for the CUDA SIMD-in-register intrinsics — and run
against the oracle with the pattern constants of the real library (frz_matcher_debug_pattern).  Covers what a GPU is
otherwise needed for: every emulated lane width, the column-limited classes (CC 40/48/56/64), the 128-column variant,
the u8 wrap emulation and the shift-placement variants, across the scorings of tests/scorings.py.  k_sw_generic's scorers
(sw_generic.cuh) are built the same way from tests/harness/sw_generic_harness.cpp."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200.types import CaseMatching, Config, Scoring
from oracle import pyoracle as O
from scorings import scorings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "harness", "sw_harness.cpp")
LIB = os.path.join(ROOT, "tests", "harness", "libsw_harness.so")
DEPS = [SRC] + [os.path.join(ROOT, "frizbee_b200", "csrc", f) for f in ("sw_core.cuh", "frz_device.cuh")]
CUDA_INC = "/usr/local/cuda/include"


@pytest.fixture(scope="module")
def H():
    if not os.path.isdir(CUDA_INC):
        pytest.skip("CUDA headers not found")
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
        subprocess.run(["g++", "-O1", "-std=c++17", "-I" + CUDA_INC, "-fPIC", "-shared", "-o", LIB, SRC], check=True)
    L = C.CDLL(LIB)
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


@pytest.mark.parametrize("lanes", [16, 32, 64])
def test_swcore_column_classes_equal_oracle(H, lanes):
    """SwCore<LANES, 64, no-wrap, VAR, CC>: the class the prefilter would choose and every wider one give the oracle's score."""
    rng = random.Random(5000 + lanes)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    checked = 0
    for trial in range(700):
        pool = rng.choice(POOLS)
        n = rng.randint(1, 11)
        needle = rand_bytes(rng, pool, n)
        if 0 in needle:
            continue
        cs = rng.random() < 0.3
        cfg = Config(max_typos=None, emulate_lanes=lanes, casing=CaseMatching.Respect if cs else CaseMatching.Ignore)
        pat, info = device_pattern(H, needle, cfg)
        assert info["score_bits"] == 8 and info["lanes"] == lanes
        for _ in range(6):
            W = rng.randint(1, 64)
            win = rand_bytes(rng, pool + (HAY_EXTRA if rng.random() < 0.3 else b""), W)
            pre = rng.random() < 0.5
            want = O.sw_score(needle, win, Scoring(), cs, pre, lanes, 8)
            chunk_cols = (W + lanes - 1) // lanes * lanes
            need = min(W + n, chunk_cols)
            for cc in (40, 48, 56, 64):
                if cc < need or cc < W:
                    continue
                eq = C.c_int()
                var = rng.choice([0, 8])
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
        n = rng.randint(14, 24) if bits == 16 else rng.randint(1, 10)
        needle = rand_bytes(rng, pool, n)
        cfg = Config(max_typos=None, emulate_lanes=emulate, casing=CaseMatching.Ignore)
        pat, info = device_pattern(H, needle, cfg)
        assert (info["lanes"], info["score_bits"]) == (lanes, bits)
        for _ in range(3):
            W = rng.randint(1, 128)
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
G_SRC = os.path.join(ROOT, "tests", "harness", "sw_generic_harness.cpp")
G_LIB = os.path.join(ROOT, "tests", "harness", "libsw_generic_harness.so")
G_DEPS = [G_SRC] + [os.path.join(ROOT, "frizbee_b200", "csrc", f) for f in ("sw_generic.cuh", "sw_core.cuh", "frz_device.cuh")]


@pytest.fixture(scope="module")
def G():
    if not os.path.isdir(CUDA_INC):
        pytest.skip("CUDA headers not found")
    if not os.path.exists(G_LIB) or any(os.path.getmtime(d) > os.path.getmtime(G_LIB) for d in G_DEPS):
        subprocess.run(["g++", "-O2", "-std=c++17", "-I" + CUDA_INC, "-fPIC", "-shared", "-o", G_LIB, G_SRC], check=True)
    L = C.CDLL(G_LIB)
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
PF_SRC = os.path.join(ROOT, "tests", "harness", "pf_harness.cpp")
PF_LIB = os.path.join(ROOT, "tests", "harness", "libpf_harness.so")
PF_DEPS = [PF_SRC] + [os.path.join(ROOT, "frizbee_b200", "csrc", f) for f in ("prefilter_masks.cuh", "frz_device.cuh")]


@pytest.fixture(scope="module")
def PF():
    if not os.path.isdir(CUDA_INC):
        pytest.skip("CUDA headers not found")
    if not os.path.exists(PF_LIB) or any(os.path.getmtime(d) > os.path.getmtime(PF_LIB) for d in PF_DEPS):
        subprocess.run(["g++", "-O1", "-std=c++17", "-I" + CUDA_INC, "-fPIC", "-shared", "-o", PF_LIB, PF_SRC], check=True)
    L = C.CDLL(PF_LIB)
    L.h_masks_window.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    return L


@pytest.mark.parametrize("lanes", [16, 32, 64])
@pytest.mark.parametrize("k", [0, 1])
def test_mask_prefilter_windows_equal_oracle(H, PF, lanes, k):
    """masks_k0 / masks_k1 (DP4A-packed occurrence masks + the reference's mask state machine at chunk width LANES) vs
    Prefilter::match_haystack / match_haystack_1_typo, on haystacks of up to 200 bytes (several 64-byte blocks)."""
    rng = random.Random(8000 + lanes + k)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    checked = matched = 0
    for trial in range(500):
        pool = rng.choice(POOLS)
        needle = rand_bytes(rng, pool, rng.randint(1, 12))
        cs = rng.random() < 0.3
        cfg = Config(max_typos=k, emulate_lanes=lanes, casing=CaseMatching.Respect if cs else CaseMatching.Ignore)
        pat, info = device_pattern(H, needle, cfg)
        assert info["prefilter_lanes"] == lanes
        for _ in range(12):
            ln = rng.choice([0, 1, 2, 7, 15, 16, 17, 31, 33, 50, 63, 64, 65, 100, 128, 129, 200])
            hay = rand_bytes(rng, pool + (HAY_EXTRA if rng.random() < 0.2 else b"x"), ln)
            s, e = C.c_int(), C.c_int()
            got = PF.h_masks_window(pat, hay, len(hay), k, C.byref(s), C.byref(e))
            assert got >= 0
            want = O.prefilter(needle, hay, k, lanes, cs)
            assert bool(got) == want[0], (needle, hay, k, lanes, cs, want)
            if want[0]:
                assert (s.value, e.value) == (want[1], want[2]), (needle, hay, k, lanes, cs, want, s.value, e.value)
                matched += 1
            checked += 1
    assert checked > 5000 and matched > 500


@pytest.mark.parametrize("k", [0, 1])
def test_single_chunk_mask_forms_equal_oracle(H, PF, k):
    """masks_k0_single / masks_k1_single (corpora of <= 64-byte haystacks at the 64-lane width: one block, one chunk,
    per-position masks) vs the oracle's Prefilter::match_haystack / match_haystack_1_typo."""
    rng = random.Random(9100 + k)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    checked = matched = 0
    for trial in range(900):
        pool = rng.choice(POOLS)
        needle = rand_bytes(rng, pool, rng.randint(1, 11))
        cs = rng.random() < 0.3
        cfg = Config(max_typos=k, emulate_lanes=64, casing=CaseMatching.Respect if cs else CaseMatching.Ignore)
        pat, info = device_pattern(H, needle, cfg)
        for _ in range(12):
            ln = rng.choice([0, 1, 2, 3, 7, 15, 16, 17, 31, 32, 33, 47, 48, 50, 63, 64])
            hay = rand_bytes(rng, pool + (HAY_EXTRA if rng.random() < 0.2 else b"x"), ln)
            s, e = C.c_int(), C.c_int()
            got = PF.h_masks_window(pat, hay, len(hay), 100 + k, C.byref(s), C.byref(e))
            if got == -2:
                continue   # needle too long for the position table: the kernel takes the general form
            want = O.prefilter(needle, hay, k, 64, cs)
            assert bool(got) == want[0], (needle, hay, k, cs, want)
            if want[0]:
                assert (s.value, e.value) == (want[1], want[2]), (needle, hay, k, cs, want, s.value, e.value)
                matched += 1
            checked += 1
    assert checked > 6000 and matched > 800


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
@pytest.mark.parametrize("k", [1, 2, 3, 5])
def test_mask_prefilter_groundwork_2_and_n_typos(H, PF, lanes, k):
    """masks_paths<NP> / masks_many (prefilter_masks.cuh, not yet wired into the kernels) vs match_haystack_1_typo /
    _2_typos / _many_typos of the reference (src/prefilter/algo/ascii_typos.rs)."""
    rng = random.Random(9000 + lanes + k)
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    mode = {1: 12, 2: 2}.get(k, 3)
    checked = matched = 0
    for trial in range(300):
        pool = rng.choice(POOLS)
        needle = rand_bytes(rng, pool, rng.randint(1, 12))
        cs = rng.random() < 0.3
        cfg = Config(max_typos=k, emulate_lanes=lanes, casing=CaseMatching.Respect if cs else CaseMatching.Ignore)
        pat, info = device_pattern(H, needle, cfg)
        for _ in range(12):
            ln = rng.choice([0, 1, 2, 7, 15, 16, 17, 31, 33, 50, 63, 64, 65, 100, 128, 129, 200])
            hay = rand_bytes(rng, pool + (HAY_EXTRA if rng.random() < 0.2 else b"x"), ln)
            s, e = C.c_int(), C.c_int()
            got = PF.h_masks_window(pat, hay, len(hay), mode, C.byref(s), C.byref(e))
            want = O.prefilter(needle, hay, k, lanes, cs)
            assert bool(got) == want[0], (needle, hay, k, lanes, cs, want)
            if want[0]:
                assert (s.value, e.value) == (want[1], want[2]), (needle, hay, k, lanes, cs, want, s.value, e.value)
                matched += 1
            checked += 1
    assert checked > 3000 and matched > 300


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
