"""Host-side mirror of the reference's public types, plus their C-ABI (ctypes) layouts.

Reference: ``Match`` src/lib.rs:141-153, ``Config`` src/lib.rs:236-271, ``SortStrategy``
src/lib.rs:311-351, ``CaseMatching`` :353-377, ``UnicodeMatching`` :379-402, ``Matching``
:413-436, ``Scoring`` :439-478, ``Pattern``/``PatternConfig`` src/pattern.rs:9-18,230-246.
The C layouts are declared in include/frz_cuda.h.
"""
from __future__ import annotations

import ctypes as C
import enum
from dataclasses import dataclass, field, replace
from typing import Optional


class SortStrategy(enum.IntEnum):
    ScoreThenIndexAsc = 0
    ScoreThenIndexDesc = 1
    IndexAsc = 2
    IndexDesc = 3

    def reverse(self) -> "SortStrategy":  # src/lib.rs:325-332
        return {0: SortStrategy.ScoreThenIndexDesc, 1: SortStrategy.ScoreThenIndexAsc,
                2: SortStrategy.IndexDesc, 3: SortStrategy.IndexAsc}[int(self)]

    def is_reversed(self) -> bool:  # src/lib.rs:339-344
        return self in (SortStrategy.IndexDesc, SortStrategy.ScoreThenIndexDesc)

    def is_by_score(self) -> bool:  # src/lib.rs:347-352
        return self in (SortStrategy.ScoreThenIndexAsc, SortStrategy.ScoreThenIndexDesc)


class Order(enum.IntEnum):
    """How Matcher.match_list_ordered_array orders the matches by an attribute (FRZ_ORDER_*); rows without a value go
    last in every order."""
    AttrDesc = 0            # by value, largest first
    AttrAsc = 1             # by value, smallest first
    ScoreThenAttrDesc = 2   # by score (with the boost), then by value, largest first
    ScoreThenAttrAsc = 3    # by score (with the boost), then by value, smallest first


class CaseMatching(enum.IntEnum):
    Ignore = 0
    Smart = 1
    Respect = 2


class UnicodeMatching(enum.IntEnum):
    Ignore = 0
    Smart = 1
    Always = 2


class Matching(enum.IntEnum):
    Fuzzy = 0
    Exact = 1
    Prefix = 2
    Suffix = 3
    Substring = 4


@dataclass(frozen=True)
class Scoring:
    """src/lib.rs:439-478; defaults src/const.rs:1-10."""
    match_score: int = 12
    mismatch_penalty: int = 6
    gap_open_penalty: int = 5
    gap_extend_penalty: int = 1
    prefix_bonus: int = 12
    capitalization_bonus: int = 4
    matching_case_bonus: int = 4
    exact_match_bonus: int = 8
    delimiter_bonus: int = 4


@dataclass(frozen=True)
class Config:
    """src/lib.rs:236-271.  ``emulate_lanes`` is this repo's addition: which reference SIMD
    backend the integer results are bit-exact with (0 = the one the reference picks on this CPU)."""
    max_typos: Optional[int] = 0
    casing: CaseMatching = CaseMatching.Smart
    unicode: UnicodeMatching = UnicodeMatching.Smart
    matching: Matching = Matching.Fuzzy
    sort: SortStrategy = SortStrategy.ScoreThenIndexAsc
    scoring: Scoring = field(default_factory=Scoring)
    emulate_lanes: int = 0

    def with_(self, **kw) -> "Config":
        return replace(self, **kw)


@dataclass(frozen=True)
class Pattern:
    """src/pattern.rs:9-18 + PatternConfig :230-246 (None = inherit the matcher's Config)."""
    needle: str
    negated: bool = False
    max_typos: Optional[int] = None
    casing: Optional[CaseMatching] = None
    unicode: Optional[UnicodeMatching] = None
    matching: Optional[Matching] = None
    scoring: Optional[Scoring] = None
    pattern: Optional[str] = None  # raw atom text


@dataclass(frozen=True)
class Match:
    """src/lib.rs:141-153.  Ordering (src/lib.rs:172-185): score desc, then index asc; eq ignores exact."""
    score: int
    index: int
    exact: bool = False


# --------------------------------------------------------------------------- ctypes layouts

class CScoring(C.Structure):
    _fields_ = [(n, C.c_uint16) for n in (
        "match_score", "mismatch_penalty", "gap_open_penalty", "gap_extend_penalty", "prefix_bonus",
        "capitalization_bonus", "matching_case_bonus", "exact_match_bonus", "delimiter_bonus")]

    @staticmethod
    def of(s: Scoring) -> "CScoring":
        return CScoring(*(getattr(s, n) for n, _ in CScoring._fields_))


class CConfig(C.Structure):
    _fields_ = [("max_typos", C.c_int32), ("casing", C.c_uint8), ("unicode", C.c_uint8),
                ("matching", C.c_uint8), ("sort", C.c_uint8), ("scoring", CScoring),
                ("emulate_lanes", C.c_uint8), ("_pad", C.c_uint8)]

    @staticmethod
    def of(c: Config) -> "CConfig":
        return CConfig(-1 if c.max_typos is None else int(c.max_typos), int(c.casing), int(c.unicode),
                       int(c.matching), int(c.sort), CScoring.of(c.scoring), int(c.emulate_lanes), 0)


class CPattern(C.Structure):
    _fields_ = [("needle", C.c_char_p), ("needle_len", C.c_size_t), ("negated", C.c_uint8),
                ("has_scoring", C.c_uint8), ("casing", C.c_int8), ("unicode", C.c_int8),
                ("matching", C.c_int8), ("_pad", C.c_int8 * 3), ("max_typos", C.c_int32),
                ("scoring", CScoring)]

    @staticmethod
    def of(p: Pattern) -> "CPattern":
        raw = p.needle.encode("utf-8") if isinstance(p.needle, str) else bytes(p.needle)
        cp = CPattern()
        cp._keep = raw  # keep the bytes alive as long as the struct
        cp.needle = raw
        cp.needle_len = len(raw)
        cp.negated = 1 if p.negated else 0
        cp.has_scoring = 1 if p.scoring is not None else 0
        cp.casing = -1 if p.casing is None else int(p.casing)
        cp.unicode = -1 if p.unicode is None else int(p.unicode)
        cp.matching = -1 if p.matching is None else int(p.matching)
        cp.max_typos = -1 if p.max_typos is None else int(p.max_typos)
        cp.scoring = CScoring.of(p.scoring if p.scoring is not None else Scoring())
        return cp


class CMatch(C.Structure):
    _fields_ = [("index", C.c_uint32), ("score", C.c_uint16), ("exact", C.c_uint8), ("_pad", C.c_uint8)]


def pattern_array(patterns):
    """ctypes array of CPattern (keeps the needle byte strings alive via the returned list)."""
    cps = [CPattern.of(p) for p in patterns]
    arr = (CPattern * max(1, len(cps)))(*cps)
    arr._keep = cps
    return arr


def as_pattern(p) -> Pattern:
    """``impl From<&str> for Pattern`` (src/pattern.rs:22-38)."""
    if isinstance(p, Pattern):
        return p
    if isinstance(p, (bytes, bytearray)):
        p = bytes(p).decode("utf-8", "surrogateescape")
    return Pattern(needle=p, pattern=p)
