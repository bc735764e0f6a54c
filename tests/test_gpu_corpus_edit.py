"""In-place corpus edits on the GPU (frz_corpus_remove / frz_corpus_replace).  Every test keeps a Python model of the list
(bytes per index, None for a removed one) and checks after every step:
  - matches: every call on the edited corpus equals the same call on a fresh corpus of the model's list (an empty string
    in place of a removed row) with the removed rows filtered out — four sorts, top-K below / at / above the live total,
    match_list_into with an index offset, match_indices on live and removed rows — for a multi-pattern query with a
    negated atom, an all-negated query, the empty matcher, max_typos=None, a unicode needle and an 80-byte needle; on
    small lists also against the oracle;
  - image: frz_corpus_debug_image decodes back to the model, live slots' unit ranges do not overlap, removed slots are
    FRZ_INVALID_SLOT with slot_of still pointing at them, every tile without removed rows is expected_image's tile up to a
    shift of its units, and an arena without dead space or removed rows is exactly expected_image."""
import ctypes as C

import numpy as np
import pytest
import torch

import frizbee_b200 as F
from frizbee_b200 import parallel
from frizbee_b200.types import Config, SortStrategy
from oracle import pyoracle as O
from test_gpu_ingest import GROUP, INVALID_SLOT, LANES, MAX_HAY, TILE, UNIT, expected_image, read_image

pytestmark = pytest.mark.gpu

INVALID_ARG, UNSUPPORTED = 1, 9
GROUPS = TILE // GROUP
LONG = b"the quick brown fox jumps over the lazy dog while the cat sleeps in the warm sun"   # 65..1024 bytes
assert 64 < len(LONG) <= 1024


def device_bytes():
    L = F.lib()
    L.frz_debug_device_bytes.restype = C.c_uint64
    L.frz_debug_device_bytes.argtypes = []
    return L.frz_debug_device_bytes()


# ---------------------------------------------------------------------------------------------------------- the model
class Model:
    def __init__(self, hs):
        self.hs = list(hs)

    def append(self, new):
        self.hs += list(new)

    def remove(self, which):
        for i in which:
            self.hs[int(i)] = None

    def replace(self, which, new):
        for i, h in zip(which, new):
            self.hs[int(i)] = h

    def arrow(self):
        return O.pack([b"" if h is None else h for h in self.hs])

    def removed_mask(self):
        return np.array([h is None for h in self.hs], dtype=bool)


def gen(n, seed, longest=40):
    """Short haystacks over a small alphabet: "ab", "zz", "é7" and LONG (with a typo or two) appear in some of them."""
    rng = np.random.default_rng(seed)
    pool = np.frombuffer(b"abzcxyQ7 -_/\xc3\xa9", dtype=np.uint8)
    out = []
    for i in range(n):
        h = bytearray(rng.choice(pool, int(rng.integers(0, longest))).tobytes())
        r = rng.random()
        if r < 0.03:
            ln = bytearray(LONG)
            for _ in range(int(rng.integers(0, 3))):
                ln[int(rng.integers(0, len(ln)))] = ord("q")
            h += ln
        elif r < 0.06:
            h += "é7".encode()
        out.append(bytes(h))
    return out


def fresh_strings(rng, n, lo=0, hi=60):
    pool = np.frombuffer(b"abzc7Q", dtype=np.uint8)
    return [rng.choice(pool, int(rng.integers(lo, hi))).tobytes() for _ in range(n)]


# ------------------------------------------------------------------------------------------------------- the queries
def cfg(sort, max_typos=0):
    return Config(max_typos=max_typos, sort=sort, emulate_lanes=LANES)


# (name, matcher factory, oracle patterns or None, match_indices supported)
QUERIES = [
    ("ab !zz", lambda s: F.Matcher.from_query("ab !zz", cfg(s, 1)), lambda: (F.parse_query("ab !zz"), 1), True),
    ("empty", lambda s: F.Matcher.from_query("", cfg(s)), None, False),
    ("!zz", lambda s: F.Matcher.from_query("!zz", cfg(s)), lambda: (F.parse_query("!zz"), 0), True),
    ("ab None", lambda s: F.Matcher("ab", cfg(s, None)), lambda: (["ab"], None), True),
    ("é7", lambda s: F.Matcher("é7", cfg(s, 1)), lambda: (["é7"], 1), True),
    ("long", lambda s: F.Matcher(LONG, cfg(s, 2)), lambda: ([LONG], 2), False),
]


class Matchers:
    """One matcher per query and sort, built once per test."""

    def __init__(self, queries=QUERIES, sorts=tuple(SortStrategy)):
        self.items = [(name, s, make(s), orc, idx) for name, make, orc, idx in queries for s in sorts]

    def close(self):
        for *_, m, _o, _i in self.items:
            m.close()


def live(arr, removed, offset=0):
    return arr[~removed[arr["index"].astype(np.int64) - offset]] if len(arr) else arr


def assert_same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for f in ("index", "score", "exact"):
        bad = np.nonzero(got[f] != want[f])[0]
        assert bad.size == 0, (what, f, bad[:5], got[bad[:5]], want[bad[:5]])


def check_matches(c, model, ms, oracle=False, indices=True):
    data, off = model.arrow()
    removed = model.removed_mask()
    n_live = int((~removed).sum())
    fresh = F.Corpus.from_arrow(data, off)
    rng = np.random.default_rng(len(model.hs))
    rem_idx, live_idx = np.nonzero(removed)[0], np.nonzero(~removed)[0]
    which = np.concatenate([rng.choice(live_idx, min(40, live_idx.size), replace=False) if live_idx.size else live_idx,
                            rem_idx[:20]]).astype(np.uint32)
    try:
        for name, sort, m, orc, idx_ok in ms.items:
            what = (name, sort.name)
            want = live(m.match_list_array(fresh), removed)
            got = m.match_list_array(c)
            assert_same(got, want, what)
            if name == "ab None":   # every live row matches, no removed one does
                assert sorted(got["index"].tolist()) == live_idx.tolist(), what
            if oracle and orc is not None and sort == SortStrategy.ScoreThenIndexAsc:
                pats, k = orc()
                assert_same(got, live(O.match_list_packed(pats, cfg(sort, k), data, off), removed), what + ("oracle",))
            for k in sorted({0, 1, n_live // 2, max(n_live - 1, 0), n_live, n_live + 3}):
                top, total = m.match_list_top_array(c, k)
                assert total == len(want), what + (k,)
                assert_same(top, want[:k], what + ("top", k))
            if sort == SortStrategy.IndexAsc:
                assert_same(m.match_list_into_array(c, index_offset=7), live(m.match_list_into_array(fresh, index_offset=7), removed, 7),
                            what + ("into",))
                if idx_ok and indices and which.size:
                    g, w = m.match_indices(c, which), m.match_indices(fresh, which)
                    for j, i in enumerate(which):
                        assert g[j] == (None if removed[i] else w[j]), what + ("indices", int(i))
    finally:
        fresh.close()


# ------------------------------------------------------------------------------------------------------------ the image
def tile_units(groups):
    last = groups.reshape(-1, GROUPS)[:, -1]
    return last["unit_off"].astype(np.int64) + last["gunits"].astype(np.int64) * GROUP


def check_image(c, model, restated=True):
    """The image decodes to the model and its invariants hold.  Returns (arena units, live units).  restated=False skips
    the comparison with expected_image (a Python loop per slot: too slow for millions of haystacks)."""
    img = read_image(c)
    data, off = model.arrow()
    removed = model.removed_mask()
    n = len(model.hs)
    n_tiles = -(-n // TILE)
    assert F.lib().frz_corpus_len(c._h) == n
    assert c.total_bytes == sum(len(h) for h in model.hs if h is not None)
    meta, slot_of, groups = img["slot_meta"], img["slot_of"], img["groups"]
    assert meta.size == n_tiles * TILE
    idx = np.arange(n)
    slot = (idx // TILE) * TILE + slot_of[:n].astype(np.int64)
    m = meta[slot]
    assert np.all((m == INVALID_SLOT) == removed), np.nonzero((m == INVALID_SLOT) != removed)[0][:8]
    lv = ~removed
    assert np.all((m[lv] & (TILE - 1)) == idx[lv] % TILE)
    lens = (m[lv] >> 10).astype(np.int64)
    assert np.all(lens == np.diff(off.astype(np.int64))[lv])
    g = slot[lv] // GROUP
    lane = slot[lv] % GROUP
    gun = groups["gunits"][g].astype(np.int64)
    start = groups["abs_off"][g].astype(np.int64) + lane * gun
    arena = img["units"].size // UNIT
    assert np.all(start + gun <= arena)
    # the bytes of every live haystack where its slot says
    src0 = off[:-1].astype(np.int64)[lv]
    total = int(lens.sum())
    if total:
        rep = np.repeat(np.arange(lens.size), lens)
        pos = np.arange(total) - np.repeat(np.cumsum(lens) - lens, lens)
        assert np.array_equal(img["units"][start[rep] * UNIT + pos], data[src0[rep] + pos])
    # live slots' unit ranges do not overlap
    used = gun > 0
    order = np.argsort(start[used], kind="stable")
    s, e = start[used][order], (start + gun)[used][order]
    assert np.all(s[1:] >= e[:-1])
    tu = tile_units(groups)
    live_units = int(tu.sum())
    assert arena - live_units <= live_units, (arena, live_units)   # dead space never outgrows the live data
    if not restated:
        return arena, live_units
    # tiles without removed rows: expected_image's tile, shifted
    want = expected_image(data, off)
    want_tu = tile_units(want["groups"])   # (a tile with removed rows keeps their units until it is re-packed)
    clean = ~np.pad(removed, (0, n_tiles * TILE - n)).reshape(n_tiles, TILE).any(axis=1)
    for t in np.nonzero(clean)[0]:
        assert tu[t] == want_tu[t], t
        sl, gs = slice(t * TILE, (t + 1) * TILE), slice(t * GROUPS, (t + 1) * GROUPS)
        for key in ("slot_meta", "slot_of", "slot_sig"):
            assert np.array_equal(img[key][sl], want[key][sl]), (t, key)
        for f in ("unit_off", "gunits"):
            assert np.array_equal(groups[f][gs], want["groups"][f][gs]), (t, f)
        tb, wb = int(img["tile_base"][t]), int(want["tile_base"][t])
        assert np.array_equal(groups["abs_off"][gs].astype(np.int64) - tb, want["groups"]["abs_off"][gs].astype(np.int64) - wb)
        assert np.array_equal(img["units"][tb * UNIT:(tb + tu[t]) * UNIT], want["units"][wb * UNIT:(wb + tu[t]) * UNIT]), t
    if arena == live_units and not removed.any():                    # no dead space: the image of a fresh pack
        for key in want:
            g_, w_ = img[key], want[key]
            same = np.array_equal(g_, w_) if g_.dtype.names is None else all(np.array_equal(g_[f], w_[f]) for f in g_.dtype.names)
            assert same, key
    return arena, live_units


def check(c, model, ms, oracle=True, indices=True):
    out = check_image(c, model)
    check_matches(c, model, ms, oracle=oracle, indices=indices)
    return out


@pytest.fixture(scope="module")
def matchers():
    ms = Matchers()
    yield ms
    ms.close()


# ---------------------------------------------------------------------------------------------------------------- cases
def test_edits_in_the_partial_last_tile_and_appends(matchers):
    """Removes and replaces in the partial last tile, then appends behind them, then more edits of the tiles the appends
    filled: the re-packed tail keeps its removed rows removed, and an append after a replace moved a tile to the arena's
    end re-packs the tail behind that tile."""
    rng = np.random.default_rng(1)
    model = Model(gen(2 * TILE + 333, seed=2))
    c = F.Corpus.from_list(model.hs)
    check(c, model, matchers)
    tail = np.arange(2 * TILE, len(model.hs))
    steps = [
        ("remove tail", lambda: rng.choice(tail, 40, replace=False), None),
        ("replace tail", lambda: rng.choice(tail, 25, replace=False), 25),
        ("append", None, 100),
        ("remove across", lambda: rng.choice(len(model.hs), 60, replace=False), None),
        ("replace tile 0", lambda: rng.choice(TILE, 30, replace=False), 30),   # tile 0 moves to the arena's end
        ("append", None, 500),                                                 # the tail no longer ends the arena
        ("append", None, 2000),
        ("replace new tiles", lambda: rng.choice(np.arange(3 * TILE, len(model.hs)), 50, replace=False), 50),
        ("remove new rows", lambda: np.arange(len(model.hs) - 700, len(model.hs) - 600), None),
        ("append", None, 1),
    ]
    for what, pick, k in steps:
        if pick is None:
            new = fresh_strings(rng, k)
            c.append_list(new)
            model.append(new)
        elif k is None:
            which = pick()
            c.remove(which)
            model.remove(which)
        else:
            which = pick()
            new = fresh_strings(rng, k)
            c.replace_list(which, new)
            model.replace(which, new)
        check(c, model, matchers, oracle=what.startswith("append"))
    c.close()


def test_remove_everything_and_revive(matchers):
    model = Model(gen(TILE + 77, seed=3))
    c = F.Corpus.from_list(model.hs)
    everything = np.arange(len(model.hs))
    c.remove(np.concatenate([everything, everything[::3]]))   # duplicates count once
    model.remove(everything)
    assert c.total_bytes == 0
    check(c, model, matchers)
    c.remove(everything[:10])                                 # removing removed rows is a no-op
    check(c, model, matchers, oracle=False)
    revive = np.array([0, 5, 1023, 1024, len(model.hs) - 1])
    new = [b"ab", b"", LONG, "é7".encode(), b"zz ab"]
    c.replace_list(revive, new)
    model.replace(revive, new)
    check(c, model, matchers)
    c.append_list([b"ab"] * 3)
    model.append([b"ab"] * 3)
    check(c, model, matchers)
    c.close()


def test_replace_with_empty_and_longest(matchers):
    """A row replaced by an empty string and one by a MAX_HAY-byte string (its group pads to 128 MiB), then shrunk back."""
    model = Model(gen(TILE + 500, seed=4))
    c = F.Corpus.from_list(model.hs)
    longest = b"ab" + b"x" * (MAX_HAY - 4) + b"zz"
    assert len(longest) == MAX_HAY
    which, new = np.array([3, TILE + 10]), [b"", longest]
    c.replace_list(which, new)
    model.replace(which, new)
    two_sorts = Matchers(sorts=(SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexAsc))   # scoring 4 MiB rows takes a while
    check(c, model, two_sorts, oracle=False)
    two_sorts.close()
    which, new = np.array([TILE + 10, 7]), [b"ab", b""]
    c.replace_list(which, new)
    model.replace(which, new)
    check(c, model, matchers)
    c.close()


def test_long_rows_into_a_corpus_of_short_rows(matchers):
    """A corpus of <= 64-byte rows (the kernels specialise on its longest group), then rows of 1-3 KB: the longest-group
    bound follows the replace, so windows of more than 128 bytes are scored and the staged prefilter is not used."""
    rng = np.random.default_rng(5)
    model = Model([h[:64] for h in gen(3 * TILE, seed=6, longest=30)])
    c = F.Corpus.from_list(model.hs)
    check(c, model, matchers, oracle=False)
    which = rng.choice(len(model.hs), 40, replace=False)
    new = [b"a" + bytes(rng.choice(np.frombuffer(b"xyc7", dtype=np.uint8), int(rng.integers(1100, 3000)))) + b"b" + LONG
           for _ in which]
    c.replace_list(which, new)
    model.replace(which, new)
    check(c, model, matchers)
    c.close()


def test_compaction_in_the_call_that_brings_long_rows(matchers):
    """One replace both raises the longest group (a row of about 1.2 KB into <= 64-byte rows) and compacts the arena:
    the bound is recounted before the compaction runs, and the compacted corpus scores the long rows."""
    rng = np.random.default_rng(15)
    model = Model([h[:64] for h in gen(3 * TILE, seed=16, longest=30)])
    c = F.Corpus.from_list(model.hs)
    rows = np.arange(len(model.hs))
    short = [h[::-1] for h in model.hs]
    c.replace_list(rows, short)   # dead space = the live data: not compacted yet
    model.replace(rows, short)
    arena, live_units = check_image(c, model)
    assert arena == 2 * live_units
    # one long row pads its group of 32 slots to ~40 KB: the live data (~140 KB) stays below the dead space (~200 KB)
    which = np.array([TILE + 700])
    new = [b"a" + bytes(rng.choice(np.frombuffer(b"xyc7", dtype=np.uint8), int(rng.integers(1100, 1200)))) + b"b" + LONG
           for _ in which]
    rest = np.setdiff1d(rows, which)
    which = np.concatenate([which, rest])
    new = new + [model.hs[i] for i in rest]
    c.replace_list(which, new)    # every tile again: the dead space passes the live data
    model.replace(which, new)
    arena, live_units = check(c, model, matchers)
    assert arena == live_units    # compacted in this call
    c.close()


def test_large_replace_gives_its_staging_back():
    """A replace whose staging passes 64 MiB (one tile of 64 haystacks of 2 MiB) does not keep it: afterwards the corpus
    owns its arena and metadata only."""
    big = [bytes([97 + i % 26]) * (2 << 20) for i in range(64)]
    torch.cuda.synchronize()
    base = device_bytes()
    c = F.Corpus.from_list(big)
    c.replace_list([5], [b"ab" * (1 << 20)])
    owned = device_bytes() - base
    # arena: 1.5 x its units after the growth of this call (the new tile goes to the arena's end); the staging (the tile's
    # 128 MiB of raw bytes and the new string) would add more than that
    assert owned <= 1.5 * c.device_bytes + (8 << 20), (owned, c.device_bytes)
    c.close()
    assert device_bytes() == base


def test_compaction_rounds(matchers):
    """Rounds of replacements over rotating tiles: the dead space passes the live data several times, and every compaction
    leaves the image a fresh pack of the list has."""
    rng = np.random.default_rng(7)
    model = Model(gen(5 * TILE + 200, seed=8))
    c = F.Corpus.from_list(model.hs)
    compactions, last_arena = 0, None
    for r in range(16):
        # every round re-packs three of the six tiles: the dead space grows by about half the live data
        which = np.concatenate([rng.choice(np.arange(t * TILE, min((t + 1) * TILE, len(model.hs))), 100, replace=False)
                                for t in range(r % 2, 6, 2)])
        new = fresh_strings(rng, which.size, 0, 30 + 10 * (r % 4))
        c.replace_list(which, new)
        model.replace(which, new)
        arena, live_units = check_image(c, model)
        if last_arena is not None and arena < last_arena:
            compactions += 1
            assert arena == live_units
        last_arena = arena
        if r % 4 == 3:
            check_matches(c, model, matchers, oracle=r == 15)
    assert compactions >= 3, compactions
    c.close()


def test_many_replacements_in_a_large_corpus():
    """50 000 replacements spread over 2 M haystacks: more than 1024 tiles in one batch, next to removals."""
    n = 2_000_000
    rng = np.random.default_rng(9)
    lens = rng.integers(0, 24, n)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum(lens)
    data = rng.choice(np.frombuffer(b"abzcxy7_-", dtype=np.uint8), int(off[-1]))
    c = F.Corpus.from_arrow(data, off)
    model = Model([data[off[i]:off[i + 1]].tobytes() for i in range(n)])
    removed = rng.choice(n, 20_000, replace=False)
    c.remove(removed)
    model.remove(removed)
    which = rng.choice(n, 50_000, replace=False)
    assert np.unique(which // TILE).size > 1024
    new = fresh_strings(rng, which.size, 0, 40)
    c.replace_list(which, new)
    model.replace(which, new)
    check_image(c, model, restated=False)
    ms = Matchers(queries=[q for q in QUERIES if q[0] in ("ab !zz", "!zz", "empty", "ab None")],
                  sorts=(SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexAsc, SortStrategy.IndexDesc))
    check_matches(c, model, ms)
    ms.close()
    c.close()


def test_refused_calls_change_nothing(matchers):
    model = Model(gen(TILE + 300, seed=10))
    c = F.Corpus.from_list(model.hs)
    c.remove([1, 2, TILE + 5])
    model.remove([1, 2, TILE + 5])
    before = read_image(c)
    L = F.lib()
    n = len(model.hs)
    over = b"ab" + b"x" * (MAX_HAY - 1)

    def refused(status, call):
        with pytest.raises(F.FrizbeeError) as e:
            call()
        assert e.value.status == status, e.value
        after = read_image(c)
        for key in before:
            assert np.array_equal(after[key].view(np.uint8), before[key].view(np.uint8)), key
        assert L.frz_corpus_len(c._h) == n

    refused(INVALID_ARG, lambda: c.remove([0, n]))
    refused(INVALID_ARG, lambda: c.remove([0xFFFFFFFF]))
    refused(INVALID_ARG, lambda: c.replace_list([4, n], [b"ab", b"ab"]))
    refused(INVALID_ARG, lambda: c.replace_list([4, 9, 4], [b"ab", b"zz", b"ab"]))      # a duplicate
    refused(UNSUPPORTED, lambda: c.replace_list([4, TILE + 1], [b"ab", over]))           # valid first, then too long
    refused(UNSUPPORTED, lambda: c.replace_list([TILE + 1, 4], [over, b"ab"]))
    w = np.array([4, 5], dtype=np.uint32)
    d = np.frombuffer(b"abab", dtype=np.uint8).copy()
    o = np.array([0, 2, 4], dtype=np.uint64)
    assert L.frz_corpus_replace(c._h, w.ctypes.data, 2, None, o.ctypes.data, 8) == INVALID_ARG   # NULL bytes, 4 bytes to read
    assert L.frz_corpus_replace(c._h, w.ctypes.data, 2, d.ctypes.data, o.ctypes.data, 5) == INVALID_ARG
    assert L.frz_corpus_remove(c._h, None, 3) == INVALID_ARG
    assert L.frz_corpus_remove(c._h, None, 0) == 0
    assert L.frz_corpus_replace(c._h, None, 0, None, None, 8) == 0
    check(c, model, matchers)
    # and it still takes edits
    c.replace_list([4, 1], [b"zz ab", b"ab"])
    model.replace([4, 1], [b"zz ab", b"ab"])
    check(c, model, matchers)
    c.close()


def test_match_list_parallel_on_edited_shards():
    """match_list_parallel and its top-K form on a one-GPU communicator over an edited shard equal the single-corpus calls.
    Only the one-GPU form is tested here; the two-GPU form, which runs the same shard calls once per GPU, has not been
    run on edited shards."""
    rng = np.random.default_rng(11)
    model = Model(gen(2 * TILE + 100, seed=12))
    c = F.Corpus.from_list(model.hs)
    c.remove(rng.choice(len(model.hs), 200, replace=False))
    which = rng.choice(len(model.hs), 150, replace=False)
    c.replace_list(which, fresh_strings(rng, which.size))
    comm = parallel.Comm.local(1)
    try:
        ms = Matchers(queries=[q for q in QUERIES if q[0] != "long"])
        for name, sort, m, *_ in ms.items:
            want = m.match_list_array(c)
            assert_same(comm.match_list_parallel(m, [c]), want, (name, sort.name))
            for k in (1, len(want), len(want) + 5):
                top, total = comm.match_list_parallel_top(m, [c], k)
                assert total == len(want)
                assert_same(top, want[:k], (name, sort.name, k))
        ms.close()
    finally:
        comm.close()
        c.close()


def test_edit_cycles_give_memory_back():
    """Replace / compact cycles on one corpus settle at one footprint, and a corpus destroyed after edits leaves the bytes
    the library holds where they were."""
    rng = np.random.default_rng(13)
    hs = gen(3 * TILE + 50, seed=14)
    rows = np.arange(len(hs))
    a, b = fresh_strings(rng, len(hs)), fresh_strings(rng, len(hs))
    for i in range(len(hs)):   # the same lengths, other bytes: every cycle leaves the same arena
        b[i] = bytes(reversed(a[i]))

    def edit(c):   # two full replacements per cycle: one of them leaves more dead space than live data and compacts
        c.replace_list(rows, a)
        c.remove(rows[::7])
        c.replace_list(rows, b)
    torch.cuda.synchronize()
    base = device_bytes()
    c = F.Corpus.from_list(hs)
    L = F.lib()
    L.frz_debug_device_bytes_peak.restype = C.c_uint64
    L.frz_debug_device_bytes_peak.argtypes = [C.c_int]
    held = device_bytes()
    assert L.frz_debug_device_bytes_peak(1) == held
    edit(c)
    assert L.frz_debug_device_bytes_peak(0) > max(held, device_bytes())   # the arena grew before a compaction freed it
    edit(c)
    settled = device_bytes()
    for _ in range(3):
        edit(c)
        assert device_bytes() == settled
    c.close()
    assert device_bytes() == base
    for _ in range(2):
        c = F.Corpus.from_list(hs)
        edit(c)
        c.append_list(a[:100])
        c.close()
        assert device_bytes() == base
