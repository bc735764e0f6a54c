"""The whole-corpus byte-path prefilter, k_scan_window (prefilter.cu): one persistent kernel that scans the signatures
of its 128-slot chunks and windows its candidates in batches of 32.  These corpora place known numbers of candidates in
each chunk (partial batches, batches that close in the middle of a chunk, ring wrap-around), mix haystacks that take the
shared-memory unit stage with ones that do not, and give the warps of the grid unequal numbers of chunks.  Bit-exact
parity with the oracle.  Needs a CUDA device."""
import random

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200 import synth
from frizbee_b200.types import Config
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

CHUNK = 128   # slots per scan chunk; one tile is 8 chunks
NEEDLE = "ab0/"


def check(needle, config, data, off, corpus):
    want = O.match_list_packed([needle], config, data, off)
    m = F.Matcher(needle, config)
    try:
        got = m.match_list_array(corpus)
    finally:
        m.close()
    assert len(got) == len(want), (len(got), len(want), needle, config)
    for f in ("index", "score", "exact"):
        bad = np.nonzero(got[f] != want[f])[0]
        assert bad.size == 0, (f, bad[:5], got[bad[:5]], want[bad[:5]], needle, config)
    return got


def counted_chunks(rng, per_chunk, length, long_every=0):
    """One chunk of equal-length haystacks per entry of `per_chunk`, that many of them candidates of NEEDLE (they contain
    it, with noise around), the rest built from bytes the needle does not have (they fail the signature test at k <= 1).
    `long_every` > 0 makes every such haystack a 100-byte one, so that the corpus does not fit the four staged units."""
    hs = []
    i = 0
    for c in per_chunk:
        hit = set(rng.sample(range(CHUNK), c))
        for j in range(CHUNK):
            ln = 100 if long_every and i % long_every == 0 else length
            if j in hit:
                pos = rng.randint(0, ln - len(NEEDLE))
                noise = bytes(rng.choice(b"abAB0/_-") for _ in range(ln))
                hs.append(noise[:pos] + NEEDLE.encode() + noise[pos + len(NEEDLE):])
            else:
                hs.append(bytes(rng.choice(b"xyzXYZ12") for _ in range(ln)))
            i += 1
    return hs


@pytest.mark.parametrize("long_every", [0, 37])
@pytest.mark.parametrize("k", [0, 1])
def test_candidate_counts_per_chunk(k, long_every):
    """0, 1, 31, 32, 33, 63, 64, 65 and 128 candidates per chunk: batches that stay partial until the end, close inside a
    chunk, or close several times in one chunk."""
    rng = random.Random(31 + k + long_every)
    counts = [0, 1, 31, 32, 33, 63, 64, 65, 128, 0, 33, 1]
    data, off = O.pack(counted_chunks(rng, counts, 24, long_every))
    corpus = F.Corpus.from_arrow(data, off)
    try:
        for lanes in (16, 64):
            got = check(NEEDLE, Config(max_typos=k, emulate_lanes=lanes), data, off, corpus)
            assert len(got) >= sum(counts)
        # a single chunk holding exactly one batch, and one candidate alone
        for c in (1, 31, 32, 33):
            d1, o1 = O.pack(counted_chunks(rng, [c], 40, long_every))
            c1 = F.Corpus.from_arrow(d1, o1)
            try:
                assert len(check(NEEDLE, Config(max_typos=k), d1, o1, c1)) >= c
            finally:
                c1.close()
    finally:
        corpus.close()


@pytest.mark.parametrize("lanes", [16, 32, 64])
@pytest.mark.parametrize("max_typos", [0, 1, 2, 3, None])
def test_typo_modes_staged_and_unstaged(lanes, max_typos):
    """Every typo mode at every emulated lane width, on a corpus whose haystacks all fit the staged units (<= 64 bytes)
    and on the same corpus with one longer haystack (every candidate then reads the corpus).  At max_typos = None every
    haystack is a candidate (no signature test)."""
    rng = random.Random(500 + lanes + (max_typos if max_typos is not None else 9))
    hs = [bytes(rng.choice(b"abAB_/-ab01") for _ in range(rng.randint(0, 64))) for _ in range(5000)]
    for extra in ([], [b"ab_-" * 30]):
        data, off = O.pack(hs + extra)
        corpus = F.Corpus.from_arrow(data, off)
        try:
            for needle in ("ab", "aB_", "b/a-", "a_b-a/b0"):
                got = check(needle, Config(max_typos=max_typos, emulate_lanes=lanes), data, off, corpus)
                if max_typos is None:
                    assert len(got) == len(hs) + len(extra)
        finally:
            corpus.close()


@pytest.mark.parametrize("k", [0, 1])
def test_more_chunks_than_grid_warps(k):
    """700 001 haystacks: 684 tiles, 5 472 chunks, more than one per warp of the persistent grid and not a multiple of
    its warps, so warps end after different numbers of chunks."""
    data, off = synth.generate("deadbeef", 700_001, 48, 64, seed=77)
    corpus = F.Corpus.from_arrow(data, off)
    try:
        check("deadbeef", Config(max_typos=k, emulate_lanes=64), data, off, corpus)
    finally:
        corpus.close()
