"""The hand-off inside k_scan_window (prefilter.cu): a producer warp per block scans the signatures and fills the block's
candidate queue of 32-record batches, the window warps take the batches from it.  These corpora fill the queue faster than
the window warps drain it (every haystack a candidate), end on batches of 0, 31, 32 and 33 records, have one chunk, give the
streamed call tile ranges with fewer chunks than the grid has producers, hold removed slots, do not fit the staged units, and
overflow the first survivor lists.  Bit-exact parity with the oracle.  Needs a CUDA device."""
import random

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200 import synth
from frizbee_b200.types import Config
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

CHUNK = 128   # slots per scan chunk
NEEDLE = "ab0/"
NOISE = np.frombuffer(b"abAB0/_-", dtype=np.uint8)


def expect(got, want):
    assert len(got) == len(want), (len(got), len(want))
    for f in ("index", "score", "exact"):
        bad = np.nonzero(got[f] != want[f])[0]
        assert bad.size == 0, (f, bad[:5], got[bad[:5]], want[bad[:5]])


def oracle(m, cfg, needle, data, off):
    return O.match_list_packed([needle], cfg.with_(emulate_lanes=m.backend_info()["prefilter_lanes"]), data, off)


def all_candidates(n, length, seed, long_at=None):
    """n haystacks of `length` noise bytes with NEEDLE planted at a random position: every one passes the signature test.
    `long_at`: that haystack is 100 bytes long, so the corpus does not fit the four staged units."""
    rng = np.random.default_rng(seed)
    rows = NOISE[rng.integers(0, NOISE.size, size=(n, length))]
    pos = rng.integers(0, length - len(NEEDLE) + 1, size=n)
    for j, b in enumerate(NEEDLE.encode()):
        rows[np.arange(n), pos + j] = b
    hs = [r.tobytes() for r in rows]
    if long_at is not None:
        hs[long_at] = hs[long_at] + bytes(NOISE[rng.integers(0, NOISE.size, size=100 - length)])
    return hs


def counted_chunk(rng, c, length):
    """one chunk of equal-length haystacks, c of them candidates of NEEDLE, the rest without any of its bytes"""
    hit = set(rng.sample(range(CHUNK), c))
    return [(bytes(rng.choice(b"abAB0/_-") for _ in range(length - len(NEEDLE))) + NEEDLE.encode()) if j in hit
            else bytes(rng.choice(b"xyzXYZ12") for _ in range(length)) for j in range(CHUNK)]


@pytest.mark.parametrize("staged", [True, False])
@pytest.mark.parametrize("k", [0, 1])
def test_queue_full_and_survivor_overflow(k, staged):
    """400 000 candidates, about five chunks per block: every producer fills all queue slots and waits for the window warps.
    Every haystack survives, more than the first survivor lists hold (a quarter of the corpus), so the call runs again."""
    hs = all_candidates(400_000, 24, 7 + k, long_at=None if staged else 123_457)
    data, off = O.pack(hs)
    cfg = Config(max_typos=k)
    corpus = F.Corpus.from_arrow(data, off)
    m = F.Matcher(NEEDLE, cfg)
    try:
        got = m.match_list_array(corpus)
        want = oracle(m, cfg, NEEDLE, data, off)
        assert len(want) == len(hs)
        expect(got, want)
        # removed slots: every third haystack, and a whole chunk
        gone = np.unique(np.concatenate([np.arange(0, len(hs), 3), np.arange(5 * CHUNK, 6 * CHUNK)])).astype(np.uint32)
        corpus.remove(gone)
        got = m.match_list_array(corpus)
        expect(got, want[~np.isin(want["index"], gone)])
    finally:
        m.close()
        corpus.close()


@pytest.mark.parametrize("k", [0, 1])
def test_last_batch_sizes_and_one_chunk(k):
    """Corpora of one chunk whose producer ends on 0, 31, 32 or 33 records (no batch, a partial one, a full one and none
    left, a full one and one record), and a corpus of three haystacks."""
    rng = random.Random(40 + k)
    cfg = Config(max_typos=k)
    cases = [O.pack(counted_chunk(rng, c, 20)) for c in (0, 31, 32, 33)] + [O.pack([b"xx" + NEEDLE.encode(), b"zzz", NEEDLE.encode()])]
    for (data, off), c in zip(cases, (0, 31, 32, 33, 2)):
        corpus = F.Corpus.from_arrow(data, off)
        m = F.Matcher(NEEDLE, cfg)
        try:
            got = m.match_list_array(corpus)
            expect(got, oracle(m, cfg, NEEDLE, data, off))
            assert len(got) == c
        finally:
            m.close()
            corpus.close()


@pytest.mark.parametrize("k", [0, 1])
def test_streamed_ranges_with_fewer_chunks_than_producers(k):
    """The streamed end-to-end call prefilters tile ranges of a few tiles each (a tile is eight chunks), far fewer chunks
    than one producer per block of a full grid."""
    data, off = synth.generate("deadbeef", 70_000, 40, 56, 99 + k)
    cfg = Config(max_typos=k)
    m = F.Matcher("deadbeef", cfg)
    try:
        got = m.match_list_host_array(data, off)
        expect(got, oracle(m, cfg, "deadbeef", data, off))
        assert len(got) > 1000
    finally:
        m.close()
