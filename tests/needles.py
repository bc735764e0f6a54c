"""Needle helpers shared by the prefilter tests: the distinct byte classes of a needle (which prefilter form the kernels
take for it) and haystacks with a needle planted in them."""
FRZ_MAX_NEEDLE = 64    # longest needle with per-position data in FrzPatternDev (frz_device.cuh)
MAX_DISTINCT = 16      # occurrence-mask rows (prefilter_masks.cuh: kMaxDistinct)


def case_sensitive(needle: bytes, casing) -> bool:
    """CaseMatching → case-sensitive for this byte needle (Smart: the needle holds an uppercase ASCII letter)."""
    from frizbee_b200.types import CaseMatching
    return casing == CaseMatching.Respect or (casing == CaseMatching.Smart and any(65 <= b <= 90 for b in needle))


def case_pairs(needle: bytes, cs: bool):
    """The case_needle pairs (c, flip) of host.cu: compile_pattern: flip is the other case of an ASCII letter when
    case-insensitive, else the byte itself."""
    flip = bytes(b if cs else b - 32 if 97 <= b <= 122 else b + 32 if 65 <= b <= 90 else b for b in needle)
    return needle, flip


def probes(needle: bytes, cs: bool):
    """Word-probe byte (om, tg) per needle position: byte b matches position i iff (b | om) == tg."""
    c, flip = case_pairs(needle, cs)
    return [(0x20, x | 0x20) if f != x else (0, x) for x, f in zip(c, flip)]


def n_distinct(needle: bytes, cs: bool) -> int:
    """FrzPatternDev.n_distinct as host.cu: compile_pattern counts it: the needle's distinct (om, tg) probe classes when
    there are at most 16 of them and the needle has at most 64 bytes (the occurrence-mask trackers of prefilter_masks.cuh),
    else 0 (the scanning forms of prefilter_scan.cuh)."""
    if len(needle) > FRZ_MAX_NEEDLE:
        return 0
    classes = set(probes(needle, cs))
    return len(classes) if len(classes) <= MAX_DISTINCT else 0


def plant(rng, needle: bytes, W: int, filler: bytes, drops: int = 0, spread: bool = False, flip_p: float = 0.1) -> bytes:
    """A haystack of W bytes of `filler` holding the needle with `drops` of its bytes deleted, ASCII letters case-flipped
    with probability flip_p, at contiguous positions or (spread) at sorted random ones."""
    nb = bytearray(b ^ 0x20 if (chr(b).isalpha() and b < 0x80 and rng.random() < flip_p) else b for b in needle)
    for _ in range(min(drops, len(nb))):
        del nb[rng.randrange(len(nb))]
    nb = nb[:W]
    out = bytearray(rng.choice(filler) for _ in range(W))
    if spread:
        pos = sorted(rng.sample(range(W), len(nb)))
    else:
        s = rng.randint(0, W - len(nb))
        pos = range(s, s + len(nb))
    for p, b in zip(pos, nb):
        out[p] = b
    return bytes(out)
