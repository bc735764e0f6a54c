"""GPU parity tests: the CUDA path (through the C ABI) vs the CPU oracle on the same inputs.
Bit-exact (score, index, exact) triples and ordering are required.  Needs a CUDA device."""
import random

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200 import synth
from frizbee_b200.types import (CaseMatching, Config, Match, Matching, Pattern, Scoring, SortStrategy,
                                UnicodeMatching)
from oracle import pyoracle as O
from scorings import edge_cases, scorings

pytestmark = pytest.mark.gpu


def gpu_vs_oracle(patterns, data, offsets, config, corpus=None):
    if isinstance(patterns, (str, Pattern)):
        patterns = [patterns]
    want = O.match_list_packed(patterns, config, data, offsets)
    own = corpus is None
    if own:
        corpus = F.Corpus.from_arrow(data, offsets)
    try:
        m = F.Matcher(patterns, config)
        got = m.match_list_array(corpus)
        m.close()
    finally:
        if own:
            corpus.close()
    assert len(got) == len(want), (len(got), len(want), patterns, config)
    for f in ("index", "score", "exact"):
        bad = np.nonzero(got[f] != want[f])[0]
        assert bad.size == 0, (f, bad[:5], got[bad[:5]], want[bad[:5]], patterns, config)
    return got


def from_list(hs):
    return O.pack(hs)


# ---------------------------------------------------------------- reference KATs through the GPU path
def test_config1_literal_haystacks():
    # BASELINE.json configs[0]: needle 'fBr' vs 5 literal haystacks, max_typos=0
    hay = ["fooBar", "foo_bar", "barfoo", "prelude", "println!"]
    for lanes in (16, 32, 64):
        got = F.Matcher("fBr", Config(emulate_lanes=lanes)).match_list(hay)
        assert got == [Match(score=53, index=0, exact=False)]


@pytest.mark.parametrize("lanes", [16, 32, 64])
def test_matcher_basic_kats(lanes):
    # src/matcher/mod.rs:533-593
    hay = ["deadbeef", "deadbf", "deadbeefg", "deadbe"]
    m = F.Matcher("deadbe", Config(max_typos=None, emulate_lanes=lanes)).match_list(hay)
    assert [(x.index, x.score) for x in m] == [(3, 116), (0, 108), (2, 108), (1, 87)]
    m0 = F.Matcher("deadbe", Config(max_typos=0, emulate_lanes=lanes)).match_list(hay)
    assert len(m0) == 3 and [x.index for x in m0 if x.exact] == [3]
    m1 = F.Matcher("1", Config(max_typos=2, emulate_lanes=lanes)).match_list(["1"])
    assert len(m1) == 1 and m1[0].exact


def test_case_modes_and_order():
    # src/matcher/mod.rs:618-654, src/matcher/algo.rs:443-456
    hay = ["foo", "FOO", "fOo", "xxfooxx"]
    idx = lambda ms: [m.index for m in ms]
    assert idx(F.Matcher("foo", Config(sort=SortStrategy.IndexAsc)).match_list(hay)) == [0, 1, 2, 3]
    assert idx(F.Matcher("foo", Config(sort=SortStrategy.IndexAsc, casing=CaseMatching.Respect)).match_list(hay)) == [0, 3]
    assert idx(F.Matcher("FoO", Config(sort=SortStrategy.IndexAsc)).match_list(["foo", "FOO", "FoO", "xxFoOxx"])) == [2, 3]
    assert idx(F.Matcher("foo", Config(sort=SortStrategy.IndexAsc)).match_list(["foo", "nomatch", "xfoo", "f_o_o", "bar"])) == [0, 2, 3]
    assert idx(F.Matcher("", Config()).match_list(["foo", "bar"])) == [0, 1]


SW_PAIRS = [
    ("a", "abc"), ("abc", "abc"), ("foo", "fooBar"), ("foo", "012345foo"), ("foo", "01234567foo"),
    ("foo", "0123456789foo"), ("foo", "0123456789012345foo"), ("foo", "0123456789012345678901234567foo"),
    ("test", "Utooooeoooosoooot"), ("test", "Utooooooeoooooosoooooot"), ("foo", "Ufooo"), ("foo", "Ufo"),
    ("hw", "hello_world"), ("fBr", "fooBar"), ("D", "FOR_DIST"), ("needle", "____________needle____________"),
    ("abcdefghij", "abcdefghij"), ("abcdefghijklmnopqrst", "abcdefghijklmnopqrst"),
    ("b", "a-b"), ("a", "-a--bc"), ("D", "forDist"), ("test", "Uteost"), ("test", "Uteoost"),
    ("babb0_", "Bab"), ("ab_", "-1Abb1-aabB1-bbaAa-_bb/b0ABB/-0/Aa-a0a/1_/"),
    ("eyqoof", "eA21viFrVA1k7gylcKJMa0amSvnEEVFU2YBOO9UgbFmrjkBzK0jo6ge"),
]


@pytest.mark.parametrize("lanes", [16, 32, 64])
def test_sw_kats_no_prefilter(lanes):
    # parity.rs:95-124 and mod.rs:208-299 pairs scored through match_list with max_typos=None
    # (NO_PREFILTER: whole haystack, include_prefix) — compared with the oracle at the same LANES
    for needle, hay in SW_PAIRS:
        data, off = from_list([hay])
        gpu_vs_oracle(needle, data, off, Config(max_typos=None, emulate_lanes=lanes, sort=SortStrategy.IndexAsc))


# ---------------------------------------------------------------- randomized parity, all typo modes
def dense_list(rng, n, max_len, pool=b"abAB_/-ab01"):
    return [bytes(rng.choice(pool) for _ in range(rng.randint(0, max_len))) for _ in range(n)]


@pytest.mark.parametrize("lanes", [16, 32, 64])
@pytest.mark.parametrize("max_typos", [0, 1, 2, 3, None])
def test_randomized_dense_alphabet(lanes, max_typos):
    # the adversarial 10-symbol alphabet of SURVEY.md §8(d): exposes lane dependence
    rng = random.Random(1000 + lanes + (max_typos or 7))
    hs = dense_list(rng, 6000, 70)
    data, off = from_list(hs)
    corpus = F.Corpus.from_arrow(data, off)
    for needle in ("ab", "aB_", "ab01", "b/a-", "abABab", "a_b-a/b0"):
        gpu_vs_oracle(needle, data, off, Config(max_typos=max_typos, emulate_lanes=lanes), corpus)
    corpus.close()


@pytest.mark.parametrize("lanes", [16, 32, 64])
def test_randomized_long_haystacks(lanes):
    # windows of 65..128 (wide register variant), 129..1024 (generic) and > 1024 (greedy fallback)
    rng = random.Random(77 + lanes)
    hs = []
    for _ in range(1500):
        ln = rng.choice([70, 100, 128, 129, 200, 400, 1023, 1024, 1025, 1500])
        hs.append(bytes(rng.choice(b"abcdefgh_-/AB01") for _ in range(rng.randint(ln // 2, ln))))
    data, off = from_list(hs)
    corpus = F.Corpus.from_arrow(data, off)
    for needle, k in (("abc", 0), ("deadbe", 1), ("a_b", 0), ("hgfedcba", 2), ("abcdefgh", None)):
        gpu_vs_oracle(needle, data, off, Config(max_typos=k, emulate_lanes=lanes), corpus)
    corpus.close()


@pytest.mark.parametrize("lanes", [16, 32, 64])
def test_u16_family_long_needles(lanes):
    # needles too long for u8 scores select the u16 backends (src/matcher/mod.rs:751-785)
    rng = random.Random(5)
    hs = dense_list(rng, 3000, 90, pool=b"abcdefghijklmnopqrstuvwxyz_-")
    hs += ["abcdefghijklmnopqrst", "xxabcdefghijklmnopqrstxx", "abcdefghij_klmnopqrst"]
    data, off = from_list(hs)
    for needle in ("abcdefghijklmnopqrst", "abcdefghijklmn", "zyxwvutsrqponmlkj"):
        for k in (0, 1, None):
            gpu_vs_oracle(needle, data, off, Config(max_typos=k, emulate_lanes=lanes))
    m = F.Matcher("abcdefghijklmnopqrst", Config(emulate_lanes=64))
    assert m.backend_info()["score_bits"] == 16 and m.backend_info()["lanes"] == 32
    assert F.Matcher("abc", Config(emulate_lanes=64)).backend_info() == {"lanes": 64, "score_bits": 8, "prefilter_lanes": 64, "literal": False}


def test_u8_wrap_emulation_adversarial_needle():
    # 13-byte needle whose true best score exceeds what the reference's u8 bound assumes
    # (DESIGN.md §5): the reference wraps; the GPU path must wrap identically (WRAP8 variant)
    hs = ["aB-cD-eF-gH-i", "aB-cD-eF-gH-iJ", "xaB-cD-eF-gH-i", "aB-cD-eF-gH-"] + ["aB-cD-eF-gH-i" * 3]
    data, off = from_list(hs)
    for lanes in (16, 32, 64):
        for k in (0, 1, None):
            gpu_vs_oracle("aB-cD-eF-gH-i", data, off, Config(max_typos=k, emulate_lanes=lanes))


def test_custom_scoring_configs():
    rng = random.Random(11)
    hs = dense_list(rng, 3000, 64)
    data, off = from_list(hs)
    for sc in (Scoring(0, 0, 0, 0, 0, 0, 0, 0, 0), Scoring(gap_open_penalty=1, gap_extend_penalty=5),
               Scoring(match_score=40, capitalization_bonus=40, mismatch_penalty=0, gap_open_penalty=0,
                       gap_extend_penalty=0, prefix_bonus=0, matching_case_bonus=0, exact_match_bonus=0, delimiter_bonus=0),
               Scoring(mismatch_penalty=260), Scoring(match_score=20, delimiter_bonus=9, prefix_bonus=30, gap_extend_penalty=2)):
        for needle in ("ab", "aB_b", "BBBB"):
            for k in (0, 1, None):
                gpu_vs_oracle(needle, data, off, Config(max_typos=k, scoring=sc, emulate_lanes=32))


SWEEP_NEEDLES = ("a_B", "ab0/", "abAB_-ab01ab")
SWEEP_SCORINGS = scorings(seed=5150, count=len(edge_cases(12)) + 3, max_needle=max(map(len, SWEEP_NEEDLES)))


def class_sweep_list(rng, per_class=250):
    """Haystacks whose whole-haystack windows fall into every Smith-Waterman work class: <= 40, 41-48, 49-56, 57-64
    (the column classes of k_sw64), 65-128 (k_sw), 129-1024 (k_sw_generic) and > 1024 bytes (the greedy scorer)."""
    spans = [(0, 40), (41, 48), (49, 56), (57, 64), (65, 128), (129, 1024), (1025, 1600)]
    counts = [per_class] * 5 + [per_class // 3, 12]
    pool = b"abAB_/-ab01"
    return [bytes(rng.choice(pool) for _ in range(rng.randint(lo, hi)))
            for (lo, hi), c in zip(spans, counts) for _ in range(c)]


@pytest.mark.parametrize("lanes", [16, 32, 64])
def test_scoring_sweep(lanes):
    """Generated scorings (tests/scorings.py, with its edge cases: gap_extend = 0 < gap_open, gap_open < gap_extend,
    constants >= 256, both sides of score_fits_in_u8, WRAP8 through the scoring, the signed 16-bit bounds) through every
    SW kernel the lane width reaches (k_sw64 in its column classes, WRAP8 and u16 forms, k_sw, k_sw_generic and the
    greedy scorer), typo modes 0, 1 and None."""
    rng = random.Random(11 + lanes)
    data, off = from_list(class_sweep_list(rng))
    corpus = F.Corpus.from_arrow(data, off)
    for sc in SWEEP_SCORINGS:
        for needle in SWEEP_NEEDLES:
            for k in (0, 1, None):
                gpu_vs_oracle(needle, data, off, Config(max_typos=k, scoring=sc, emulate_lanes=lanes), corpus)
    corpus.close()


def test_sort_strategies_across_score_bounds():
    """The counting sort picks its digit bins from the host's score bound: a scoring whose bound is <= 255 (one pass)
    and one whose bound is > 1023 (two passes), under every sort strategy."""
    rng = random.Random(12)
    data, off = from_list(class_sweep_list(rng, per_class=150))
    corpus = F.Corpus.from_arrow(data, off)
    low, high = Scoring(), Scoring(match_score=300, mismatch_penalty=10, gap_open_penalty=20, gap_extend_penalty=0)
    assert O.score_fits_in_u8(2, low) and not O.score_fits_in_u8(4, high)
    for sort in SortStrategy:
        for needle, sc in (("ab", low), ("ab0/", high)):
            got = gpu_vs_oracle(needle, data, off, Config(sort=sort, max_typos=1, scoring=sc), corpus)
            assert len(got) > 100
            if sc is high:
                assert got["score"].max() > 1023
    corpus.close()


def test_multi_pattern_per_atom_scoring():
    """One query whose atoms carry different Pattern.scoring values (one with gap_extend = 0 < gap_open)."""
    rng = random.Random(13)
    data, off = from_list(class_sweep_list(rng, per_class=150))
    pats = [Pattern("ab", scoring=Scoring(gap_open_penalty=7, gap_extend_penalty=0)),
            Pattern("B_a", scoring=Scoring(match_score=40, delimiter_bonus=0, gap_open_penalty=1, gap_extend_penalty=3)),
            Pattern("01")]
    for k in (0, 1, None):
        for lanes in (16, 32, 64):
            gpu_vs_oracle(pats, data, off, Config(max_typos=k, emulate_lanes=lanes))


def test_sort_strategies_and_radix_sort():
    rng = random.Random(3)
    hs = dense_list(rng, 5000, 40)
    data, off = from_list(hs)
    for sort in SortStrategy:
        gpu_vs_oracle("ab", data, off, Config(sort=sort, max_typos=1))
    arr = np.zeros(1 << 18, dtype=F.MATCH_DTYPE)
    arr["index"] = np.arange(len(arr))
    arr["score"] = np.random.default_rng(7).integers(0, 65536, len(arr))
    got = F.radix_sort_matches(arr)
    want = O.radix_sort_matches(arr)
    assert np.array_equal(got, want)


def test_literal_modes():
    rng = random.Random(21)
    hs = dense_list(rng, 4000, 50, pool=b"abAB_-fo") + ["foo", "foobar", "xfoo", "FOO", "barfoo", "foo_bar", "ab_ab"]
    data, off = from_list(hs)
    for mode in (Matching.Exact, Matching.Prefix, Matching.Suffix, Matching.Substring):
        for needle in ("foo", "ab", "a", "A_b", "bar"):
            for casing in CaseMatching:
                gpu_vs_oracle(needle, data, off, Config(matching=mode, casing=casing))


def test_multi_pattern():
    rng = random.Random(31)
    hs = dense_list(rng, 4000, 60, pool=b"abrfo_/BF") + ["foo/bar", "bar/foo", "foo", "foobar", "barfoo", "Foo BAR", "foo bar"]
    data, off = from_list(hs)
    P = Pattern
    sets = [
        [P("foo"), P("bar", negated=True, matching=Matching.Prefix)],          # 'foo !^bar'  (config 5)
        [P("foo"), P("bar", negated=True, matching=Matching.Substring)],
        [P("foo"), P("bar", negated=True, matching=Matching.Suffix)],
        [P("foo"), P("foo")],
        [P("foo", negated=True, matching=Matching.Substring)],
        [P("foo", negated=True, matching=Matching.Substring), P("ab", negated=True, matching=Matching.Substring)],
        [P("fo"), P("ba", max_typos=1), P("r")],
        [P("Foo"), P("bar")],
        [P("foo"), P("foo", negated=True, matching=Matching.Substring)],
    ]
    for pats in sets:
        for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexAsc, SortStrategy.IndexDesc):
            gpu_vs_oracle(pats, data, off, Config(sort=sort))
    # the product's own query parser end to end
    m = F.Matcher.from_query("foo !^bar", Config(sort=SortStrategy.IndexAsc))
    assert [x.index for x in m.match_list(["foo/bar", "bar/foo", "foo", "foobar"])] == [0, 2, 3]
    assert len(F.Matcher.from_query("foo !^bar").match_list(["foo", "barfoo", "foobar"])) == 2


def test_edge_shapes():
    # empty list, empty strings, single item, exactly one tile, tile boundary +-1
    for hs in ([], [""], ["a"], ["", "", "ab"], ["ab"] * 1024, ["ab"] * 1023 + ["ba"], ["xab"] * 1025):
        data, off = from_list(hs)
        for k in (0, 1, None):
            gpu_vs_oracle("ab", data, off, Config(max_typos=k))
    hs = ["x" * i + "ab" for i in range(0, 300)]
    data, off = from_list(hs)
    gpu_vs_oracle("ab", data, off, Config())


# ---------------------------------------------------------------- bench-shaped data (BASELINE.json configs)
@pytest.mark.parametrize("needle,n,mu,max_len,k", [
    ("deadbe", 200_000, 24, 32, 0),     # config 2 shape
    ("deadbeef", 300_000, 48, 64, 1),   # config 3 shape
    ("deadbeef", 300_000, 48, 64, 0),   # config 4 shape (one shard)
])
@pytest.mark.parametrize("lanes", [32, 64])
def test_bench_shaped_parity(needle, n, mu, max_len, k, lanes):
    data, off = synth.generate(needle, n, mu, max_len)
    gpu_vs_oracle(needle, data, off, Config(max_typos=k, emulate_lanes=lanes))


def test_full_size_properties():
    # BASELINE.json config 3 at full size (10M x <=64, k=1): size-independent properties —
    # ordering, index uniqueness/range, determinism across calls, and a 200k-prefix cross-check
    n = 10_000_000
    data, off = synth.generate("deadbeef", n, 48, 64)
    corpus = F.Corpus.from_arrow(data, off)
    m = F.Matcher("deadbeef", Config(max_typos=1))
    a = m.match_list_array(corpus).copy()
    b = m.match_list_array(corpus).copy()
    assert np.array_equal(a, b)
    key = (65535 - a["score"].astype(np.int64)) * (1 << 32) + a["index"]
    assert np.all(np.diff(key) > 0)
    assert a["index"].max() < n
    sub_n = 200_000
    want = O.match_list_packed(["deadbeef"], Config(max_typos=1), data[: int(off[sub_n])], off[: sub_n + 1])
    got = a[a["index"] < sub_n]
    assert np.array_equal(np.sort(got, order=["index"]), np.sort(want, order=["index"]))
    # end-to-end host call gives the same list
    c = m.match_list_host_array(data, off)
    assert np.array_equal(a, c)
    corpus.close()


def test_config5_mixed_unicode_multi_pattern():
    # BASELINE.json configs[4] shape: query 'foo !^bar' on mixed-unicode haystacks, len <= 128 bytes.
    # The needles are ASCII, so the reference takes the byte path (UnicodeMatching::Smart, src/lib.rs:394-399);
    # bytes >= 128 are "not delimiters" for the bonuses (src/smith_waterman/algo/ascii.rs:86-89).
    data, off = synth.generate("foo", 150_000, 96, 128, unicode_frac=0.3, prefix_frac=0.1)
    pats = [Pattern("foo"), Pattern("bar", negated=True, matching=Matching.Prefix)]
    for lanes in (32, 64):
        gpu_vs_oracle(pats, data, off, Config(emulate_lanes=lanes))
    m = F.Matcher.from_query("foo !^bar", Config())
    corpus = F.Corpus.from_arrow(data, off)
    got = m.match_list_array(corpus)
    want = O.match_list_packed(pats, Config(emulate_lanes=m.backend_info()["prefilter_lanes"]), data, off)
    assert np.array_equal(got, want)
    corpus.close()


def test_config2_and_config4_shapes_full_prefix():
    # configs[1]: needle len 6, 1M haystacks len <= 32, k = 0; configs[3] shard shape: len <= 64, k = 0
    data, off = synth.generate("deadbe", 1_000_000, 24, 32)
    gpu_vs_oracle("deadbe", data, off, Config(max_typos=0))


# ---------------------------------------------------------------- ingestion (SURVEY §8(f) rank 1)
def test_arrow_ingest_widths_slices_and_streaming():
    # Arrow Utf8 (32-bit offsets) vs LargeUtf8 (64-bit), a sliced array (offsets[0] != 0), and a list large
    # enough for the streamed ingest to split the value bytes into several H2D chunks (>= 8 MiB each)
    n = 600_000
    data, off = synth.generate("deadbeef", n, 48, 64, seed=777)
    cfg = Config(max_typos=1)
    want = O.match_list_packed(["deadbeef"], cfg, data, off)
    m = F.Matcher("deadbeef", cfg)
    for offsets in (off.astype(np.uint64), off.astype(np.uint32), off.astype(np.int32)):
        c = F.Corpus.from_arrow(data, offsets)
        got = m.match_list_array(c)
        assert np.array_equal(got, want), offsets.dtype
        c.close()
        e2e = m.match_list_host_array(data, offsets)
        assert np.array_equal(e2e, want), offsets.dtype
    # slice [lo, hi) of the same Arrow array: same value buffer, offsets start inside it
    lo, hi = 123_457, 523_461
    sl = off[lo: hi + 1]
    want_sl = O.match_list_packed(["deadbeef"], cfg, data[int(sl[0]): int(sl[-1])], sl - sl[0])
    for offsets in (sl.astype(np.uint64), sl.astype(np.uint32)):
        c = F.Corpus.from_arrow(data, offsets)
        assert len(c) == hi - lo and c.total_bytes == int(sl[-1] - sl[0])
        assert np.array_equal(m.match_list_array(c), want_sl)
        c.close()
        assert np.array_equal(m.match_list_host_array(data, offsets), want_sl)
    # the arena is reused by a second, smaller list and by an empty one
    small = off[: 1001]
    want_small = O.match_list_packed(["deadbeef"], cfg, data[: int(small[-1])], small)
    assert np.array_equal(m.match_list_host_array(data, small.astype(np.uint32)), want_small)
    assert len(m.match_list_host_array(data[:0], np.zeros(1, dtype=np.uint32))) == 0
    m.close()


def test_corpus_append_matches_one_shot_pack():
    # incremental ingestion: batches that end on / next to tile boundaries (1024), empty batches, both offset widths
    n = 150_000
    data, off = synth.generate("deadbeef", n, 40, 64, seed=4242)
    cfg = Config(max_typos=1)
    m = F.Matcher("deadbeef", cfg)
    want = O.match_list_packed(["deadbeef"], cfg, data, off)
    cuts = [0, 1, 1, 1023, 1024, 1025, 2048, 2050, 5000, 5000 + 1024 * 3, 70_001, 70_001, 149_999, n]
    c = F.Corpus.from_arrow(data[:0], np.zeros(1, dtype=np.uint64))
    for k, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
        sl = off[a: b + 1]
        offsets = sl.astype(np.uint32) if k % 2 else sl.astype(np.uint64)   # slices of the same value buffer
        c.append(data, offsets)
        assert len(c) == b and c.total_bytes == int(off[b])
        if b in (1, 1025, 5000, 70_001):
            got = m.match_list_array(c)
            assert np.array_equal(got, O.match_list_packed(["deadbeef"], cfg, data[: int(off[b])], off[: b + 1])), b
    got = m.match_list_array(c)
    assert np.array_equal(got, want)
    # long haystack crossing the re-bucketed tail, then more appends
    c.append_list([b"x" * 5000 + b"deadbeef", b"deadbeef"])
    got = m.match_list_array(c)
    assert {n, n + 1} <= set(got["index"].tolist())
    assert got[got["index"] == n + 1]["exact"][0] == 1
    c.close()
    m.close()


@pytest.mark.parametrize("n_runs", [2, 3, 8])
def test_device_k_merge_equals_single_list(n_runs):
    # frz_match_shard_device + frz_merge_runs_device on ONE GPU (no NCCL): shards are index ranges, each scored into a
    # locally ordered run; the device merge must reproduce Matcher::match_list on the whole list for every
    # SortStrategy (k_merge_matches_by_*, src/k_merge.rs:56-88), through the boundary-search merge (score bound
    # known) and through the concatenate + stable sort fallback (bound unknown → 0).
    import ctypes as C
    import torch
    from frizbee_b200 import parallel
    n = 120_011
    data, off = synth.generate("deadbeef", n, 40, 64, seed=99)
    full = F.Corpus.from_arrow(data, off)
    bounds = parallel.shard_bounds(n, n_runs)
    shards = [F.Corpus.from_arrow(data, off[lo: hi + 1]) for lo, hi in bounds]
    dev = torch.device("cuda", 0)
    for sort in SortStrategy:
        cfg = Config(max_typos=1, sort=sort)
        m = F.Matcher("deadbeef", cfg)
        want = m.match_list_array(full).copy()
        stride = max(hi - lo for lo, hi in bounds)
        runs = torch.zeros(n_runs * stride, dtype=torch.int64, device=dev)
        cnt = torch.zeros(1, dtype=torch.int64, device=dev)
        counts = np.zeros(n_runs, dtype=np.uint64)
        for r, ((lo, hi), sh) in enumerate(zip(bounds, shards)):
            view = runs[r * stride: (r + 1) * stride]
            F._check(F.lib().frz_match_shard_device(m._h, sh._h, lo, view.data_ptr(), stride, cnt.data_ptr(), None))
            counts[r] = int(cnt.item())
        total = int(counts.sum())
        assert total == len(want)
        for bound in (m.score_bound(), 0):
            out = torch.zeros(max(total, 1), dtype=torch.int64, device=dev)
            F._check(F.lib().frz_merge_runs_device(runs.data_ptr(), stride, counts.ctypes.data, n_runs, int(sort), bound,
                                                   out.data_ptr(), 0, None))
            torch.cuda.synchronize()
            got = out[:total].cpu().numpy().view(F.MATCH_DTYPE)
            assert np.array_equal(got, want), (sort, bound)
        m.close()
    for sh in shards:
        sh.close()
    full.close()


# ---------------------------------------------------------------- unicode-needle path (SURVEY §8(f) rank 4)
def _unicode_haystacks(rng, n):
    pools = ["aéAÉ_다", "abé✓😀", "éÉeE-/x", "нНaя_Я", "fooBar_/-é다😀"]
    out = []
    for _ in range(n):
        pool = rng.choice(pools)
        ln = rng.choice([0, 1, 2, 5, 9, 14, 20, 31, 40, 70, 130, 300])
        out.append("".join(rng.choice(pool) for _ in range(ln)))
    out += ["é다😀", "xxé__다__😀yy", "É다😀", "é다", "a-é-다-😀", "", "😀", "x" * 1100 + "é" + "y" * 50 + "다😀"]
    return out


@pytest.mark.parametrize("lanes", [16, 32, 64])
def test_unicode_needle_path(lanes):
    # UNICODE = true specialisations (src/matcher/mod.rs:58-73): unicode prefilters, per-scalar Smith-Waterman,
    # exact flag, all typo budgets; the same code is checked on the CPU by tests/test_unicode_device_code.py
    rng = random.Random(4100 + lanes)
    hs = _unicode_haystacks(rng, 6000)
    data, off = from_list(hs)
    corpus = F.Corpus.from_arrow(data, off)
    for needle in ["é다😀", "éa", "Я", "аб", "é", "😀x", "aÉ"]:
        for k in (0, 1, 2, 3, None):
            gpu_vs_oracle(needle, data, off, Config(max_typos=k, emulate_lanes=lanes), corpus)
    # UnicodeMatching::Always routes an ASCII needle through the unicode kernels too (src/lib.rs:394-401)
    gpu_vs_oracle("foo", data, off, Config(max_typos=1, unicode=UnicodeMatching.Always, emulate_lanes=lanes), corpus)
    gpu_vs_oracle("fB", data, off, Config(max_typos=0, unicode=UnicodeMatching.Always, casing=CaseMatching.Respect,
                                           emulate_lanes=lanes), corpus)
    # u16 family (needle > 13 bytes at the default scoring) and custom scoring
    gpu_vs_oracle("é다😀é다😀", data, off, Config(max_typos=2, emulate_lanes=lanes), corpus)
    gpu_vs_oracle("éa", data, off, Config(max_typos=1, emulate_lanes=lanes,
                                          scoring=Scoring(gap_open_penalty=2, gap_extend_penalty=2, delimiter_bonus=7)), corpus)
    corpus.close()


def test_unicode_literal_and_multi_pattern():
    rng = random.Random(777)
    hs = _unicode_haystacks(rng, 5000) + ["éab", "Éab", "xéa", "é", "a다", "다"]
    data, off = from_list(hs)
    corpus = F.Corpus.from_arrow(data, off)
    for mode in (Matching.Exact, Matching.Prefix, Matching.Suffix, Matching.Substring):
        for needle in ["éa", "다", "É", "aé"]:
            gpu_vs_oracle(Pattern(needle, matching=mode), data, off, Config(), corpus)
            gpu_vs_oracle(Pattern(needle, matching=mode), data, off, Config(casing=CaseMatching.Respect, sort=SortStrategy.IndexDesc), corpus)
    # multi-pattern with unicode atoms: fuzzy base + negated unicode prefix, unicode base + ASCII extra
    gpu_vs_oracle([Pattern("aé"), Pattern("é", negated=True, matching=Matching.Prefix)], data, off, Config(max_typos=1), corpus)
    gpu_vs_oracle([Pattern("다"), Pattern("a")], data, off, Config(max_typos=0), corpus)
    gpu_vs_oracle([Pattern("fo"), Pattern("é😀", max_typos=1)], data, off, Config(max_typos=0), corpus)
    corpus.close()


def test_match_indices_traceback():
    # frz_match_indices == Matcher::match_list_indices restricted to chosen haystacks (src/matcher/mod.rs:234-262):
    # scores/exact flags equal match_list, indices equal the oracle's traceback (AlignmentPathIter)
    rng = random.Random(31337)
    hs = [rand for rand in ("".join(rng.choice("abAB_/-ab01") for _ in range(rng.choice([0, 3, 9, 20, 40, 70, 140]))) for _ in range(1500))]
    hs += _unicode_haystacks(rng, 1500)
    hs += ["foo", "f_o_o", "xfoo", "FooBar", "x" * 1200 + "a" + "y" * 30 + "bc", "é다😀", "xxé__다__😀yy"]
    data, off = from_list(hs)
    corpus = F.Corpus.from_arrow(data, off)
    which = list(range(len(hs)))
    cases = [("ab", Config(max_typos=0)), ("ab_", Config(max_typos=1)), ("abA", Config(max_typos=None)), ("a/b01", Config(max_typos=2)),
             ("abc", Config(max_typos=1)), ("é다😀", Config(max_typos=1)), ("éa", Config(max_typos=0)),
             ("foo", Config(max_typos=1, unicode=UnicodeMatching.Always)),
             (Pattern("ab", matching=Matching.Substring), Config()), (Pattern("é", matching=Matching.Prefix), Config()),
             ("ab", Config(max_typos=1, emulate_lanes=16)), ("abAB_/-ab01abAB", Config(max_typos=3, emulate_lanes=32)),
             # multi-pattern queries: pooled, de-duplicated indices (match_one_indices_multi, src/matcher/multi.rs:56-79)
             ([Pattern("ab"), Pattern("ab")], Config(max_typos=0)),
             ([Pattern("ab"), Pattern("b0", negated=True, matching=Matching.Substring)], Config(max_typos=1)),
             ([Pattern("é"), Pattern("a"), Pattern("다", negated=True)], Config(max_typos=0))]
    for needle, cfg in cases:
        m = F.Matcher(needle, cfg)
        lanes = m.backend_info()["prefilter_lanes"]
        got = m.match_indices(corpus, which)
        want = O.match_indices(needle, cfg.with_(emulate_lanes=lanes), data, off, which)
        assert got == want, (needle, cfg, [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w][:3])
        ml = {int(x["index"]): x for x in m.match_list_array(corpus)}
        assert {i for i, g in enumerate(got) if g is not None} == set(ml)
        assert all(got[i][0] == int(ml[i]["score"]) and got[i][1] == bool(ml[i]["exact"]) for i in ml)
        m.close()
    corpus.close()
