"""Scorings for the kernel tests: the edge cases where the Smith-Waterman kernels' arithmetic changes form, followed by
random draws of all nine `Scoring` fields.  Every scoring `scorings` returns is one the library compiles for a fuzzy
needle of up to `max_needle` bytes at every lane width: the library's bounds (score overflow guard, signed 16-bit cell range,
gap-penalty range) all grow with the needle length and the lane width, so checking the longest needle at the widest
lanes checks every shorter one."""
import random
from typing import List

import frizbee_b200 as F
from frizbee_b200.types import Config, Matching, Scoring, UnicodeMatching

FIELDS = ("match_score", "mismatch_penalty", "gap_open_penalty", "gap_extend_penalty", "prefix_bonus",
          "capitalization_bonus", "matching_case_bonus", "exact_match_bonus", "delimiter_bonus")
ZERO = Scoring(**{f: 0 for f in FIELDS})


def accepted(sc: Scoring, max_needle: int) -> bool:
    try:
        F.Matcher(b"a" * max_needle, Config(max_typos=None, scoring=sc, emulate_lanes=64)).close()
    except F.FrizbeeError:
        return False
    return True


def edge_cases(max_needle: int) -> List[Scoring]:
    n = max_needle
    # match_score that puts the signed 16-bit cell bound of host.cu (n * (match + max bonus + case bonus) + prefix +
    # mismatch + match <= 32767) just inside its limit for an n-byte needle
    m_cell = (32767 - 6 - 12 - n * (4 + 4)) // (n + 1)
    wrap_by_scoring = dict(match_score=16, mismatch_penalty=0, gap_open_penalty=64, prefix_bonus=0, capitalization_bonus=64,
                           matching_case_bonus=0, exact_match_bonus=0, delimiter_bonus=64)
    return [
        ZERO,
        Scoring(),
        # gap_extend = 0 < gap_open: the gap penalty is a constant, the per-lane penalty variant of the kernels
        Scoring(gap_open_penalty=1, gap_extend_penalty=0),
        Scoring(gap_open_penalty=5, gap_extend_penalty=0),
        Scoring(match_score=30, gap_open_penalty=60, gap_extend_penalty=0, delimiter_bonus=9),
        Scoring(gap_open_penalty=32767, gap_extend_penalty=0),
        Scoring(**{**{f: 0 for f in FIELDS}, "match_score": 7, "gap_open_penalty": 3}),
        # gap_open < gap_extend: gap_open_x saturates to 0
        Scoring(gap_open_penalty=1, gap_extend_penalty=3),
        Scoring(gap_open_penalty=0, gap_extend_penalty=2, match_score=20),
        # constants of 256 and more (u16 family; the u8 family would truncate them)
        Scoring(mismatch_penalty=260),
        Scoring(match_score=256, capitalization_bonus=300, delimiter_bonus=257, matching_case_bonus=256, prefix_bonus=511,
                gap_open_penalty=256, gap_extend_penalty=0, exact_match_bonus=1000),
        # score_fits_in_u8 switches between needle lengths 4 and 5 (default scoring: between 13 and 14)
        Scoring(match_score=50),
        # u8 family that wraps for needles of 3-4 bytes (cell bound > 255 although score_fits_in_u8 holds): WRAP8
        # selected through the scoring, with and without a gap_extend of 0
        Scoring(gap_extend_penalty=1, **wrap_by_scoring),
        Scoring(gap_extend_penalty=0, **wrap_by_scoring),
        # just inside the kernels' signed 16-bit bounds: the cell bound, and the gap-penalty bound 32 * 1023 + 31
        Scoring(match_score=m_cell),
        Scoring(match_score=m_cell, gap_open_penalty=9, gap_extend_penalty=0),
        Scoring(gap_open_penalty=31, gap_extend_penalty=1023),
    ]


def _draw(rng: random.Random) -> Scoring:
    def one():
        r = rng.random()
        if r < 0.2:
            return 0
        if r < 0.6:
            return rng.randint(1, 8)
        if r < 0.9:
            return rng.randint(0, 64)
        return rng.randint(0, 600)
    return Scoring(**{f: one() for f in FIELDS})


def _sweep(edges: List[Scoring], ok, seed: int, count: int, max_needle: int) -> List[Scoring]:
    out = [sc for sc in edges if ok(sc, max_needle)]
    rng = random.Random(seed)
    while len(out) < count:
        sc = _draw(rng)
        if ok(sc, max_needle):
            out.append(sc)
    return out


def scorings(seed: int, count: int, max_needle: int) -> List[Scoring]:
    """The accepted edge cases, then random accepted scorings up to `count` in all."""
    return _sweep(edge_cases(max_needle), accepted, seed, count, max_needle)


# The unicode kernels keep true u8 / u16 lanes and the literal matcher adds in u32: neither has the byte path's signed
# 16-bit cell bound, only the u16 score guard.  So they accept scorings whose scores reach 32 768-65 535, which
# `accepted` refuses.  A needle of `max_needle` ASCII scalars is the longest the unicode guard (which counts scalars)
# sees for `max_needle` bytes.
def accepted_unicode(sc: Scoring, max_needle: int) -> bool:
    try:
        F.Matcher(b"a" * max_needle, Config(max_typos=None, unicode=UnicodeMatching.Always, scoring=sc, emulate_lanes=64)).close()
    except F.FrizbeeError:
        return False
    return True


def accepted_literal(sc: Scoring, max_needle: int) -> bool:
    try:
        F.Matcher(b"a" * max_needle, Config(matching=Matching.Substring, scoring=sc)).close()
    except F.FrizbeeError:
        return False
    return True


# the bonuses of the default scoring are all 4: these make capitalization, matching case and delimiter distinguishable
DISTINCT_BONUSES = Scoring(capitalization_bonus=3, matching_case_bonus=11, delimiter_bonus=29, prefix_bonus=7)
# zero gap and mismatch penalties: traceback cells tie between diagonal, left and up
TIES = Scoring(mismatch_penalty=0, gap_open_penalty=0, gap_extend_penalty=0)


def high_match_score(max_needle: int, sc: Scoring = Scoring()) -> int:
    """The largest match_score that the unicode guard accepts for `max_needle` scalars with the other fields of `sc`:
    a needle of that many scalars matched in full scores just under 65 536."""
    lo, hi = 0, 0xFFFF
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if accepted_unicode(Scoring(**{**sc.__dict__, "match_score": mid}), max_needle):
            lo = mid
        else:
            hi = mid - 1
    return lo


def unicode_edge_cases(max_needle: int) -> List[Scoring]:
    m_hi = high_match_score(max_needle)
    return [DISTINCT_BONUSES, TIES, Scoring(**{**TIES.__dict__, "prefix_bonus": 0, "matching_case_bonus": 0}),
            Scoring(match_score=m_hi), Scoring(match_score=m_hi // 2 + 1, gap_extend_penalty=0, delimiter_bonus=300),
            Scoring(match_score=m_hi, mismatch_penalty=0, gap_open_penalty=0, gap_extend_penalty=0)] + edge_cases(max_needle)


def literal_edge_cases(max_needle: int) -> List[Scoring]:
    d = Scoring()
    per_char = d.match_score + d.matching_case_bonus + max(d.capitalization_bonus, d.delimiter_bonus)
    # the largest exact_match_bonus the literal guard accepts for a needle of max_needle bytes
    exact_max = 0xFFFF - d.prefix_bonus - d.mismatch_penalty - max_needle * per_char
    return [DISTINCT_BONUSES, Scoring(exact_match_bonus=exact_max), Scoring(exact_match_bonus=exact_max // 2, prefix_bonus=0),
            Scoring(match_score=(0xFFFF - 40) // max_needle - 8), Scoring(**{f: 0 for f in FIELDS}),
            Scoring(capitalization_bonus=500, delimiter_bonus=0, matching_case_bonus=0),
            Scoring(capitalization_bonus=0, delimiter_bonus=500, prefix_bonus=0)]


def unicode_scorings(seed: int, count: int, max_needle: int) -> List[Scoring]:
    """`scorings` for the unicode kernels: accepted for a unicode needle of `max_needle` bytes, high scores included."""
    return _sweep(unicode_edge_cases(max_needle), accepted_unicode, seed, count, max_needle)


def literal_scorings(seed: int, count: int, max_needle: int) -> List[Scoring]:
    """`scorings` for the literal matcher: accepted for a literal needle of `max_needle` bytes, exact_match_bonus up to
    its guard included."""
    return _sweep(literal_edge_cases(max_needle), accepted_literal, seed, count, max_needle)
