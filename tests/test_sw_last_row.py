"""SwCore's last needle row has no gap propagation (frizbee_b200/csrc/sw_core.cuh, run()), and the scoring kernels compare
a window with the needle only when the window record says it can be exact (sw.cu, score_window).  The CPU half runs the
header's g++ build (tests/harness/sw_harness.cpp) against the oracle, at the needle lengths and gap scorings where the
last row's gap step matters most; the GPU half puts exact windows through frz_match_list."""
import ctypes as C
import random

import numpy as np
import pytest

import frizbee_b200 as F
from cpu_harness import load
from frizbee_b200.types import CaseMatching, Config, Scoring
from oracle import pyoracle as O


NEEDLES = [b"a", b"Q", b"ab", b"aB", b"deadbeef", b"dEad-bEf"]


def gap_scorings(lanes):
    """gap_open 0, gap_extend 0, both 0, and both at the largest values a `lanes`-wide backend accepts
    (lanes * gap_extend + gap_open <= 32767)."""
    ge_max = 256
    return [
        Scoring(gap_open_penalty=0),
        Scoring(gap_extend_penalty=0),
        Scoring(gap_open_penalty=0, gap_extend_penalty=0),
        Scoring(gap_open_penalty=32767 - lanes * ge_max, gap_extend_penalty=ge_max),
        Scoring(),
    ]


@pytest.fixture(scope="module")
def H():
    L = load("sw_harness", opt="-O1", cuda_include=True)
    L.h_pattern_size.restype = C.c_size_t
    L.h_swcore.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                           C.POINTER(C.c_int)]
    L.h_pattern_flags.argtypes = [C.c_void_p] + [C.POINTER(C.c_int)] * 3
    return L


def device_pattern(H, needle, cfg):
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    m = F.Matcher(needle, cfg)
    buf = (C.c_uint8 * H.h_pattern_size())()
    F._check(F.lib().frz_matcher_debug_pattern(m._h, 0, buf, len(buf)))
    info = m.backend_info()
    m.close()
    return buf, info


def flags(H, pat):
    wrap8, col_classes, lane_pen = C.c_int(), C.c_int(), C.c_int()
    H.h_pattern_flags(pat, C.byref(wrap8), C.byref(col_classes), C.byref(lane_pen))
    return bool(wrap8.value), bool(col_classes.value), bool(lane_pen.value)


def windows(rng, needle):
    """Random windows, plus windows whose best cell sits left of a long run that only the last row's gap step
    reaches: the needle (or its last byte) followed by filler, at every chunk offset."""
    low = needle.lower()
    out = [needle, needle.swapcase(), low[-1:] + b"." * 40, b"_" + needle + b"x" * 30]
    for lead in (0, 7, 15, 16, 31, 32, 47, 63):
        out.append((b"z" * lead + low[-1:] + b"q" * 64)[:64])
        out.append((b"z" * lead + needle + b"-" * 64)[:64])
        out.append((b"z" * lead + low[:1] + b"yy" + low[1:] + b"w" * 64)[:64])
    for _ in range(40):
        W = rng.randint(1, 64)
        out.append(bytes(rng.choice(low + b"Ab_-/x0" + bytes([0x80, 0])) for _ in range(W)))
    return [w for w in out if w]


def kernel_calls(W, n, lanes, wrap8, col_classes):
    """(cols, cc) of every k_sw64 / k_sw form the host could run this window through."""
    if W > 64:
        return [(128, 128)]
    if not col_classes:
        return [(64, 64)]
    need = min(W + n, (W + lanes - 1) // lanes * lanes)
    return [(64, cc) for cc in (40, 48, 56, 64) if cc >= need and cc >= W]


@pytest.mark.parametrize("em", [16, 32, 64])
def test_last_row_without_gap_step_equals_oracle(H, em):
    """Needles of 1, 2 and 8 bytes (for one byte, row 0 is also the last row) at gap_open 0, gap_extend 0, both 0 and
    both at their largest accepted values: every instantiation the kernels would run gives the oracle's score, whose
    last row does run the gap step, and the exact-window check agrees with a byte compare."""
    rng = random.Random(1700 + em)
    checked, seen = 0, set()
    for sc in gap_scorings(em):
        for needle in NEEDLES:
            for casing in (CaseMatching.Ignore, CaseMatching.Respect):
                cs = casing == CaseMatching.Respect
                pat, info = device_pattern(H, needle, Config(max_typos=None, emulate_lanes=em, casing=casing, scoring=sc))
                lanes, bits = info["lanes"], info["score_bits"]
                wrap8, col_classes, lane_pen = flags(H, pat)
                seen.add((len(needle), bits, wrap8, lane_pen))
                for win in windows(rng, needle):
                    for pre in (False, True):
                        want = O.sw_score(needle, win, sc, cs, pre, lanes, bits)
                        for cols, cc in kernel_calls(len(win), len(needle), lanes, wrap8, col_classes):
                            for var in ((0,) if wrap8 else (0, 8)):
                                v = (var if cols == 64 else 0) | (16 if lane_pen else 0)
                                eq = C.c_int()
                                got = H.h_swcore(pat, win, len(win), rng.randint(0, 15), int(pre), lanes, cols, cc,
                                                 int(wrap8), v, C.byref(eq))
                                assert got == want, (needle, win, sc, cs, pre, lanes, bits, cols, cc, v, got, want)
                                assert bool(eq.value) == (win == needle)
                                checked += 1
    assert checked > 5000, checked
    assert {n for n, *_ in seen} == {1, 2, 8}
    assert any(lp for *_, lp in seen)   # gap_extend 0 < gap_open takes the per-lane penalty form


@pytest.mark.gpu
@pytest.mark.parametrize("em", [16, 32, 64])
def test_exact_windows_through_match_list(em):
    """A list where some haystacks equal the needle (the exact bonus applies), some equal it up to case, and some
    contain it: the gated compare marks exactly the equal ones, and every score, index and exact flag is the oracle's."""
    rng = random.Random(90 + em)
    for needle in ("deadbeef", "ab", "a", "dEad-bEf"):
        hs = [needle, needle.swapcase(), needle + "x", "x" + needle, needle[:-1], needle + needle]
        hs += ["".join(rng.choice(needle + "xyz_-AB") for _ in range(rng.randint(1, 70))) for _ in range(3000)]
        hs += [needle] * 50
        rng.shuffle(hs)
        data, offsets = O.pack(hs)
        for casing in (CaseMatching.Ignore, CaseMatching.Respect):
            for typos in (None, 0, 1):
                cfg = Config(max_typos=typos, emulate_lanes=em, casing=casing)
                want = O.match_list_packed([needle], cfg, data, offsets)
                corpus = F.Corpus.from_arrow(data, offsets)
                try:
                    m = F.Matcher([needle], cfg)
                    got = m.match_list_array(corpus)
                    m.close()
                finally:
                    corpus.close()
                assert len(got) == len(want)
                for f in ("index", "score", "exact"):
                    assert np.array_equal(got[f], want[f]), (f, needle, casing, typos, em)
                exact_idx = {i for i, h in enumerate(hs) if h == needle}
                assert {int(i) for i in got["index"][got["exact"] != 0]} == exact_idx
