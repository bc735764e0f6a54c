"""frz_subset_match without a GPU: frizbee_b200/csrc/subset_match_plan.cuh built for the CPU
(tests/harness/subset_match_harness.cpp) against numpy, the decomposition the device fill relies on (match_list's rows are
the AND / AND-NOT of each pattern's own rows) checked on the CPU oracle alone, and the argument checks of frz_subset_match
on zero-filled stand-in handles.  The behaviour on a real corpus is in tests/test_gpu_subset_match.py."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from cpu_harness import load
from frizbee_b200.types import Config, Pattern
from oracle import pyoracle as O

INVALID, NO_DEVICE = 1, 8
FIRST, AND, ANDNOT = 0, 1, 2
CHUNK = 1024
vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32


@pytest.fixture(scope="module")
def H():
    L = load("subset_match_harness")
    L.h_steps.argtypes = [vp, u32, vp, vp]
    L.h_steps.restype = u32
    L.h_masked.argtypes = [u32, C.c_int, u64, u64]
    L.h_masked.restype = C.c_int
    L.h_fold.argtypes = [u64, vp, u64, u32, vp, u64, vp, u32, vp, vp]
    L.h_fold.restype = None
    return L


def to_words(mask: np.ndarray, n_words: int, rng=None) -> np.ndarray:
    """bool per index → uint32 words (bit i of word w is index 32w + i); past the mask's end random bits when rng is given
    (the fold must not read them), else zeros"""
    w = np.zeros(n_words * 32, dtype=bool) if rng is None else rng.random(n_words * 32) < 0.5
    w[: len(mask)] = mask
    return np.packbits(w.reshape(-1, 8), axis=1, bitorder="little").reshape(-1).view(np.uint32).copy()


def from_words(words: np.ndarray, n: int) -> np.ndarray:
    return np.unpackbits(words.view(np.uint8), bitorder="little")[:n].astype(bool)


def steps(H, negated):
    k = len(negated) + 1
    pat, op = np.zeros(k, np.int32), np.zeros(k, np.uint32)
    flags = np.array(negated, dtype=np.uint8)
    m = H.h_steps(flags.ctypes.data if len(flags) else None, len(negated), pat.ctypes.data, op.ctypes.data)
    return list(zip(pat[:m].tolist(), op[:m].tolist()))


def test_steps(H):
    assert steps(H, []) == [(-1, FIRST)]
    assert steps(H, [False]) == [(0, FIRST)]
    assert steps(H, [True]) == [(-1, FIRST), (0, ANDNOT)]
    assert steps(H, [True, True]) == [(-1, FIRST), (0, ANDNOT), (1, ANDNOT)]
    assert steps(H, [True, False, True, False]) == [(1, FIRST), (0, ANDNOT), (2, ANDNOT), (3, AND)]
    assert steps(H, [False, False, True]) == [(0, FIRST), (1, AND), (2, ANDNOT)]


def test_masked_rule(H):
    # the first step: masked by a base that leaves rows out, else the corpus's own metadata
    assert H.h_masked(0, 1, 0, 1000) == 1 and H.h_masked(0, 1, 999, 1000) == 1
    assert H.h_masked(0, 1, 1000, 1000) == 0 and H.h_masked(0, 0, 0, 1000) == 0
    # every later step: masked by the members so far, whatever the base
    for has_base, members in ((0, 0), (1, 10), (1, 1000)):
        assert H.h_masked(1, has_base, members, 1000) == 1 and H.h_masked(3, has_base, members, 1000) == 1


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1023, 1024, 1025, 5000, 70_001])
def test_fold_against_numpy(H, n):
    rng = np.random.default_rng(n)
    n_words = (n + 31) // 32
    for trial in range(6):
        negs = [bool(x) for x in rng.random(int(rng.integers(0, 5))) < 0.4]
        plan = steps(H, negs)
        # each step's survivors: a pattern's bitmap over the tiles (garbage past n: a bitmap covers whole tiles), or the
        # live rows for a start without a non-negated pattern
        surv_words = ((n + CHUNK - 1) // CHUNK) * 32
        density = rng.choice([0.01, 0.3, 0.9, 1.0])
        masks = [rng.random(n) < density for _ in plan]
        survs = np.concatenate([to_words(mk, surv_words, rng) for mk in masks])
        has_base = trial % 2 == 1
        n_base = int(rng.integers(0, n + 40)) if has_base else 0   # shorter than the corpus, or longer
        base_mask = rng.random(max(n_base, 1))[:n_base] < 0.6
        base = to_words(base_mask, max(1, (n_base + 31) // 32), rng)   # bits past n_base are set: they must not count
        ops = np.array([op for _, op in plan], dtype=np.uint32)
        bits = rng.integers(0, 2**32, size=n_words, dtype=np.uint32)   # the first step must not read them
        counts = np.full((n + CHUNK - 1) // CHUNK, 0xDEAD, dtype=np.uint32)
        H.h_fold(n, base.ctypes.data, n_base, int(has_base), survs.ctypes.data, surv_words, ops.ctypes.data, len(ops),
                 bits.ctypes.data, counts.ctypes.data)
        want = masks[0].copy()
        if has_base:
            b = np.zeros(n, dtype=bool)
            b[: min(n, n_base)] = base_mask[: min(n, n_base)]
            want &= b
        for mk, op in zip(masks[1:], ops[1:]):
            want = want & mk if op == AND else want & ~mk
        got = from_words(bits, n_words * 32)
        assert np.array_equal(got[:n], want) and not got[n:].any(), (n, trial, plan)
        padded = np.zeros(len(counts) * CHUNK, dtype=bool)
        padded[:n] = want
        assert np.array_equal(counts, padded.reshape(-1, CHUNK).sum(axis=1)), (n, trial)
        assert counts.sum() == want.sum()


# ---------------------------------------------------------------------------------- the decomposition, on the oracle
def rand_corpus(rng, n):
    dirs = ["src", "lib", "test", "tests", "docs", "node_modules", "Src", "été", "데이터"]
    exts = ["rs", "py", "toml", "md", "RS", "txt", "é"]
    rows = []
    for _ in range(n):
        depth = int(rng.integers(0, 4))
        parts = [dirs[int(rng.integers(len(dirs)))] for _ in range(depth)]
        name = "".join(chr(int(c)) for c in rng.integers(97, 123, size=int(rng.integers(1, 9))))
        if rng.random() < 0.1:
            name += "x" * int(rng.integers(60, 90))   # long rows, for needles over 64 bytes
        rows.append("/".join(parts + [name + "." + exts[int(rng.integers(len(exts)))]]))
    return rows


ATOMS = ["src", "^src/", ".rs$", "'test", "!test", "!^docs", "!.md$", "rs", "lib/", "^tests/", "été", "!데이터", "srcmain",
         "'node_modules", "toml$", "x" * 70, "!" + "x" * 66, "src/" + "x" * 62, "^" + "lib/" + "x" * 65]


def index_set(patterns, cfg, data, off):
    return set(O.match_list_into_packed(patterns, cfg, data, off)["index"].tolist())


@pytest.mark.parametrize("typos", [0, 1, 2, 3, None])
def test_match_list_is_the_and_of_its_patterns(typos):
    rng = np.random.default_rng(7 if typos is None else typos)
    cfg = Config(max_typos=typos)
    checked = 0
    for trial in range(12):
        rows = rand_corpus(rng, 300)
        data, off = O.pack(rows)
        for _ in range(6):
            k = int(rng.integers(1, 5))
            query = " ".join(ATOMS[int(j)] for j in rng.choice(len(ATOMS), size=k, replace=False))
            pats = F.parse_query(query)
            if not pats:
                continue
            live = set(range(len(rows)))
            want = set(live)
            positive = False
            for p in pats:
                if not p.needle:   # compiled away: constrains nothing
                    continue
                own = index_set([Pattern(needle=p.needle, matching=p.matching)], cfg, data, off)
                if p.negated:
                    want -= own
                else:
                    want &= own
                    positive = True
            got = index_set(pats, cfg, data, off)
            assert got == want, (query, typos, positive)
            checked += 1
    assert checked >= 50


# ---------------------------------------------------------------------------------- argument checks
def test_argument_checks_and_no_device():
    import torch
    L = F.lib()
    fake = C.create_string_buffer(4096)            # a corpus of 0 haystacks; never written
    c = C.addressof(fake)
    mine = C.create_string_buffer(c.to_bytes(8, "little"), 256)    # a subset of the fake corpus
    other = C.create_string_buffer(256)            # a subset whose corpus (its first field) is NULL: another corpus
    matcher = C.create_string_buffer(4096)         # a stand-in matcher: the checks never read it
    # a corpus of 5 rows: frz_corpus_len finds where a corpus keeps its length
    longer = C.create_string_buffer(4096)
    for at in range(0, 4096 - 8, 8):
        C.memmove(C.addressof(longer) + at, (5).to_bytes(8, "little"), 8)
        if L.frz_corpus_len(C.addressof(longer)) == 5:
            break
        C.memmove(C.addressof(longer) + at, bytes(8), 8)
    assert L.frz_corpus_len(C.addressof(longer)) == 5
    s, m, oth, t5 = C.addressof(mine), C.addressof(matcher), C.addressof(other), C.addressof(longer)
    snaps = (fake.raw, mine.raw, other.raw, matcher.raw, longer.raw)
    fn = L.frz_subset_match
    # a NULL subset or matcher
    assert fn(None, m, None, None) == INVALID
    assert fn(s, None, None, None) == INVALID
    assert b"null" in L.frz_last_error()
    # a text corpus of another length, before the base check
    assert fn(s, m, t5, oth) == INVALID
    assert b"index space" in L.frz_last_error()
    # a base of another corpus
    assert fn(s, m, None, oth) == INVALID
    assert fn(s, m, c, oth) == INVALID
    assert b"base subset was made on another corpus" in L.frz_last_error()
    assert (fake.raw, mine.raw, other.raw, matcher.raw, longer.raw) == snaps
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    # every argument is valid: the call reaches the device check, the handles untouched
    for text, base in ((None, None), (c, None), (None, s), (c, s)):
        assert fn(s, m, text, base) == NO_DEVICE
    assert (fake.raw, mine.raw, other.raw, matcher.raw, longer.raw) == snaps
