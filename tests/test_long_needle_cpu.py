"""Needles of 65..1024 bytes without a GPU: the two long-needle scorers built for the CPU from
tests/harness/sw_wave_harness.cpp (the wavefront arithmetic of k_sw_long, sw_wave.cuh, and generic_score over the needle
view of k_sw_long_thread) against the oracle's score_haystack, and the host-side limits of the byte path (which needles
compile, and the FRZ_ERR_UNSUPPORTED cases that remain)."""
import ctypes as C
import os
import random
import subprocess

import pytest

import frizbee_b200 as F
from frizbee_b200.types import CaseMatching, Config, Matching, Pattern, Scoring, UnicodeMatching
from oracle import pyoracle as O
from scorings import scorings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "harness", "sw_wave_harness.cpp")
LIB = os.path.join(ROOT, "tests", "harness", "libsw_wave_harness.so")
DEPS = [SRC] + [os.path.join(ROOT, "frizbee_b200", "csrc", f) for f in ("sw_wave.cuh", "sw_generic.cuh", "sw_core.cuh", "frz_device.cuh")]
CUDA_INC = "/usr/local/cuda/include"
UNSUPPORTED = 9   # FRZ_ERR_UNSUPPORTED


@pytest.fixture(scope="module")
def W():
    if not os.path.isdir(CUDA_INC):
        pytest.skip("CUDA headers not found")
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
        subprocess.run(["g++", "-O2", "-std=c++17", "-I" + CUDA_INC, "-fPIC", "-shared", "-o", LIB, SRC], check=True)
    L = C.CDLL(LIB)
    L.h_pattern_size.restype = C.c_size_t
    L.h_sw_wave.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_int, C.c_char_p, C.c_int, C.c_int]
    L.h_sw_generic_long.argtypes = L.h_sw_wave.argtypes
    return L


def device_pattern(W, needle, cfg):
    F.lib().frz_matcher_debug_pattern.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    m = F.Matcher(needle, cfg)
    buf = (C.c_uint8 * W.h_pattern_size())()
    F._check(F.lib().frz_matcher_debug_pattern(m._h, 0, buf, len(buf)))
    info = m.backend_info()
    m.close()
    return buf, info


def flip(needle: bytes, cs: bool) -> bytes:
    return needle if cs else needle.swapcase()


POOLS = [b"ab", b"abAB_/-01", b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789 _-/.", b"aAbB_zZ9\x00"]
HAY_EXTRA = b"\xc3\xa9\x80\xff\x00"


def draw_len(rng, lanes):
    """Lengths that cluster around the boundaries of the wavefront's passes of 32 chunks (256 columns at 8 lanes, 512 at
    16), of the chunks themselves and of the split between the two scorers (512 bytes); the rest mostly short, which keeps
    about 3 400 cases per width within a minute."""
    r = rng.random()
    if r < 0.5:
        b = rng.choice([32 * lanes, 64 * lanes, 96 * lanes, 1024, 512, lanes, 65, 128, 129])
        return max(1, min(1024, b + rng.randint(-lanes - 1, lanes + 1)))
    return rng.randint(1, 300) if r < 0.9 else rng.randint(1, 1024)


@pytest.mark.parametrize("em", [16, 32, 64])
def test_wavefront_equals_oracle(W, em):
    """wave_score (k_sw_long's arithmetic) == the oracle's score_haystack at LANES = em / 2 (u16 family): needles of
    65..1024 bytes, windows of 1..1024 bytes, every case mode, needles with NUL, haystack bytes >= 0x80, and the scorings of
    tests/scorings.py for long needles (gap_extend 0 among them: the reference's per-lane penalty form)."""
    lanes = em // 2
    rng = random.Random(71000 + em)
    scs = scorings(7100 + em, 14, 1024)
    checked = 0
    while checked < 3400:   # about 10 000 cases over the three widths
        sc = rng.choice(scs) if rng.random() < 0.5 else Scoring()
        pool = rng.choice(POOLS)
        n = rng.randint(65, 300) if rng.random() < 0.5 else max(65, draw_len(rng, lanes))
        needle = bytes(rng.choice(pool) for _ in range(n))
        casing = rng.choice([CaseMatching.Ignore, CaseMatching.Respect, CaseMatching.Smart])
        cs = casing == CaseMatching.Respect or (casing == CaseMatching.Smart and any(65 <= b <= 90 for b in needle))
        try:
            pat, info = device_pattern(W, needle, Config(max_typos=None, emulate_lanes=em, casing=casing, scoring=sc))
        except F.FrizbeeError as e:
            assert e.status == 2   # FRZ_ERR_NEEDLE_TOO_LONG: this scoring overflows the u16 score at this length
            continue
        if info["score_bits"] == 8:
            continue   # (the u8 family is scored per thread: test_generic_long_needle_u8_family)
        w = draw_len(rng, lanes)
        hp = pool + (HAY_EXTRA if rng.random() < 0.3 else b"")
        if rng.random() < 0.3 and w >= n:   # the needle inside the window, some bytes flipped
            at = rng.randint(0, w - n)
            win = bytearray(rng.choice(hp) for _ in range(w))
            win[at:at + n] = bytes(b ^ 0x20 if (chr(b).isalpha() and rng.random() < 0.2) else b for b in needle)
            win = bytes(win)
        else:
            win = bytes(rng.choice(hp) for _ in range(w))
        pre = rng.random() < 0.5
        want = O.sw_score(needle, win, sc, cs, pre, lanes, 16)
        got = W.h_sw_wave(pat, needle, flip(needle, cs), n, win, w, int(pre))
        assert got == want, (n, w, lanes, sc, casing, pre, got, want)
        assert W.h_sw_generic_long(pat, needle, flip(needle, cs), n, win, w, int(pre)) == want
        checked += 1


@pytest.mark.parametrize("em", [16, 32, 64])
def test_generic_long_needle_u8_family(W, em):
    """Scorings whose whole score range fits in 255 keep a long needle in the u8 family (lanes = emulate_lanes, 8-bit
    elements): k_sw_long_thread scores every window of such a needle with generic_score, equal to the oracle's."""
    rng = random.Random(72000 + em)
    checked = 0
    for trial in range(300):
        sc = Scoring(match_score=rng.choice([0, 1, 2]), mismatch_penalty=rng.choice([0, 1]), gap_open_penalty=rng.randint(0, 5),
                     gap_extend_penalty=rng.randint(0, 2), prefix_bonus=0, capitalization_bonus=rng.choice([0, 0, 1]),
                     matching_case_bonus=0, exact_match_bonus=rng.randint(0, 9), delimiter_bonus=rng.choice([0, 0, 1]))
        n = rng.randint(65, 400)
        pool = rng.choice(POOLS)
        needle = bytes(rng.choice(pool) for _ in range(n))
        casing = rng.choice([CaseMatching.Ignore, CaseMatching.Respect])
        cs = casing == CaseMatching.Respect
        pat, info = device_pattern(W, needle, Config(max_typos=None, emulate_lanes=em, casing=casing, scoring=sc))
        if info["score_bits"] != 8:
            continue
        assert info["lanes"] == em
        w = rng.randint(1, 1024)
        win = bytes(rng.choice(pool + HAY_EXTRA) for _ in range(w))
        pre = rng.random() < 0.5
        want = O.sw_score(needle, win, sc, cs, pre, em, 8)
        assert W.h_sw_generic_long(pat, needle, flip(needle, cs), n, win, w, int(pre)) == want, (n, w, sc, casing, pre)
        checked += 1
    assert checked >= 100, checked


def err(fn):
    with pytest.raises(F.FrizbeeError) as e:
        fn()
    return e.value.status


@pytest.mark.parametrize("n", [65, 100, 1000, 1024])
def test_long_byte_needles_compile(n):
    for em in (16, 32, 64):
        m = F.Matcher(b"ab_C" * (n // 4) + b"x" * (n % 4), Config(emulate_lanes=em))
        info = m.backend_info()
        m.close()
        assert info["score_bits"] == 16 and info["lanes"] == em // 2, info
    for cfg in (Config(max_typos=None), Config(max_typos=15), Config(matching=Matching.Substring),
                Config(unicode=UnicodeMatching.Ignore)):
        F.Matcher(b"\xc3\xa9" * (n // 2) + b"a" * (n % 2), cfg).close() if cfg.unicode == UnicodeMatching.Ignore \
            else F.Matcher(b"q" * n, cfg).close()


def test_long_needle_limits():
    # over 1024 bytes: unsupported, on either path
    assert err(lambda: F.Matcher(b"a" * 1025, Config())) == UNSUPPORTED
    assert err(lambda: F.Matcher("é".encode() * 600, Config())) == UNSUPPORTED
    # over 64 bytes on the unicode path (a non-ASCII needle under Smart, any needle under Always)
    assert err(lambda: F.Matcher("é".encode() * 40, Config())) == UNSUPPORTED
    assert err(lambda: F.Matcher(b"a" * 65, Config(unicode=UnicodeMatching.Always))) == UNSUPPORTED
    F.Matcher("é".encode() * 32, Config()).close()          # 64 bytes: the unicode kernels take it
    # max_typos of 16 or more below the needle length
    assert err(lambda: F.Matcher(b"a" * 100, Config(max_typos=16))) == UNSUPPORTED
    F.Matcher(b"a" * 100, Config(max_typos=100)).close()   # a budget of the whole needle matches everything
    # scorings whose cells would leave the signed 16-bit range
    assert err(lambda: F.Matcher(b"a" * 1024, Config(scoring=Scoring(match_score=40)))) == UNSUPPORTED
    # the earlier guards keep their statuses: the u16 score overflow guard and the gap-penalty guard
    assert err(lambda: F.Matcher(b"a" * 1000, Config(scoring=Scoring(match_score=100)))) == 2   # FRZ_ERR_NEEDLE_TOO_LONG
    assert err(lambda: F.Matcher(b"a" * 100, Config(scoring=Scoring(gap_extend_penalty=3000)))) == 3   # FRZ_ERR_GAP_OVERFLOW
    # a scoring whose score range fits in 255 keeps a long needle in the u8 family, which compiles
    m = F.Matcher(b"q" * 100, Config(scoring=Scoring(match_score=1, mismatch_penalty=0, gap_open_penalty=1, gap_extend_penalty=0,
                                                     prefix_bonus=0, capitalization_bonus=0, matching_case_bonus=0,
                                                     exact_match_bonus=0, delimiter_bonus=0)))
    assert m.backend_info()["score_bits"] == 8
    m.close()
    # long atoms in a query, negated ones included
    F.Matcher([Pattern(b"z" * 300), Pattern(b"y" * 70, negated=True), Pattern(b"ab")], Config()).close()
