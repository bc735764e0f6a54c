"""Scorings for the kernel tests: the edge cases where the Smith-Waterman kernels' arithmetic changes form, followed by
random draws of all nine `Scoring` fields.  Every scoring returned is one the library compiles for a fuzzy needle of up
to `max_needle` bytes at every lane width: the library's bounds (score overflow guard, signed 16-bit cell range,
gap-penalty range) all grow with the needle length and the lane width, so checking the longest needle at the widest
lanes checks every shorter one."""
import random
from typing import List

import frizbee_b200 as F
from frizbee_b200.types import Config, Scoring

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


def scorings(seed: int, count: int, max_needle: int) -> List[Scoring]:
    """The accepted edge cases, then random accepted scorings up to `count` in all."""
    out = [sc for sc in edge_cases(max_needle) if accepted(sc, max_needle)]
    rng = random.Random(seed)
    while len(out) < count:
        sc = _draw(rng)
        if accepted(sc, max_needle):
            out.append(sc)
    return out
