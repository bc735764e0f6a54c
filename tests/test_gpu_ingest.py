"""Corpus ingestion on the GPU (pack.cu), checked bit-exact: the packed image of every constructor against a numpy
restatement of the layout (DESIGN.md §3, frz_device.cuh), and match_list on it against the oracle.  Also the haystack
length limit, refused appends and end-to-end calls, the greedy scorer's gap clamp, and a corpus of more than
12 224 tiles (the global-memory walk of k_tile_scan, and more than 1 M candidates for the multi-pattern compaction)."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

import frizbee_b200 as F
from frizbee_b200.types import Config, Pattern, Scoring, SortStrategy
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

MAX_HAY = (1 << 22) - 2          # longest haystack the corpus accepts (4 MiB - 2)
TILE, GROUP, UNIT = 1024, 32, 16
INVALID_SLOT = 0xFFFFFFFF
GROUP_DTYPE = np.dtype([("abs_off", "<u8"), ("unit_off", "<u4"), ("gunits", "<u4")])
LANES = 32
UNSUPPORTED = 9


# ------------------------------------------------------------------------------------------- the layout, restated
def sig_bucket_table():
    """frz_sig_bucket for every byte: letters fold case into 26 classes, digits share 3, every other byte shares 3."""
    b = np.arange(256, dtype=np.int64)
    t = (b | 0x20) - ord("a")
    d = b - ord("0")
    return np.where((t >= 0) & (t < 26), t, np.where((d >= 0) & (d < 10), 26 + d % 3, 29 + (b + (b >> 5)) % 3))


SIG_BUCKET = sig_bucket_table()
BIT = np.uint64(1) << np.arange(32, dtype=np.uint64)


def expected_image(data, offsets):
    """The packed image of haystacks data[offsets[i], offsets[i + 1]), computed without the CUDA code."""
    off = np.asarray(offsets, dtype=np.int64)
    n = len(off) - 1
    lens = np.diff(off)
    n_tiles = -(-n // TILE)
    slots = n_tiles * TILE
    units = (lens + UNIT - 1) // UNIT
    idx = np.arange(n)
    order = np.lexsort((idx, units, idx // TILE))    # within each tile, a stable sort by unit count
    slot_meta = np.full(slots, INVALID_SLOT, dtype=np.uint32)
    slot_meta[:n] = (lens[order] << 10) | (order % TILE)
    slot_of = np.zeros(slots, dtype=np.uint16)       # local index -> slot; 0 past the end of the list
    slot_of[order] = idx % TILE
    slot_units = np.zeros(slots, dtype=np.int64)
    slot_units[:n] = units[order]
    gunits = slot_units.reshape(-1, GROUP).max(axis=1)             # groups of 32 slots, padded to their longest
    per_group = (gunits * GROUP).reshape(n_tiles, TILE // GROUP)   # slot-major: 32 runs of gunits units
    unit_off = np.cumsum(per_group, axis=1) - per_group
    tile_units = per_group.sum(axis=1)
    tile_base = np.cumsum(tile_units) - tile_units
    groups = np.zeros(n_tiles * (TILE // GROUP), dtype=GROUP_DTYPE)
    groups["abs_off"] = (tile_base[:, None] + unit_off).ravel()
    groups["unit_off"] = unit_off.ravel()
    groups["gunits"] = gunits
    packed = np.zeros(int(tile_units.sum()) * UNIT, dtype=np.uint8)  # zero padding after every haystack, unused slots zero
    slot_sig = np.zeros((slots, 2), dtype=np.uint32)
    for s in np.nonzero(slot_units)[0]:
        h = order[s]
        g, lane = divmod(int(s), GROUP)
        at = (int(groups["abs_off"][g]) + lane * int(gunits[g])) * UNIT
        hay = data[off[h]: off[h + 1]]
        packed[at: at + len(hay)] = hay
        cnt = np.bincount(SIG_BUCKET[hay], minlength=32)
        slot_sig[s] = (int(BIT[cnt >= 1].sum()), int(BIT[cnt >= 2].sum()))   # .x classes present, .y present twice
    return {"tile_base": tile_base.astype(np.uint64), "groups": groups, "slot_meta": slot_meta, "slot_of": slot_of,
            "slot_sig": slot_sig, "units": packed}


def read_image(corpus):
    """frz_corpus_debug_image → the same dict as expected_image."""
    L = F.lib()
    sizes = (C.c_uint64 * 6)()
    F._check(L.frz_corpus_debug_image(corpus._h, *[None] * 6, sizes))
    bufs = [np.zeros(max(int(s), 1), dtype=np.uint8) for s in sizes]
    F._check(L.frz_corpus_debug_image(corpus._h, *[b.ctypes.data for b in bufs], sizes))
    bufs = [b[: int(s)] for b, s in zip(bufs, sizes)]
    return {"tile_base": bufs[0].view("<u8"), "groups": bufs[1].view(GROUP_DTYPE), "slot_meta": bufs[2].view("<u4"),
            "slot_of": bufs[3].view("<u2"), "slot_sig": bufs[4].view("<u4").reshape(-1, 2), "units": bufs[5]}


def assert_image(corpus, want, what):
    got = read_image(corpus)
    for key in want:
        g, w = got[key], want[key]
        assert g.shape == w.shape, (what, key, g.shape, w.shape)
        bad = np.nonzero(g != w)[0] if g.dtype.names is None else np.nonzero(
            np.any([g[f] != w[f] for f in g.dtype.names], axis=0))[0]
        assert bad.size == 0, (what, key, bad[:8], g[bad[:4]], w[bad[:4]])


def assert_same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for f in ("index", "score", "exact"):
        bad = np.nonzero(got[f] != want[f])[0]
        assert bad.size == 0, (what, f, bad[:5], got[bad[:5]], want[bad[:5]])


def pack(hs):
    return O.pack(hs)


def corpus_len(c):
    return F.lib().frz_corpus_len(c._h)


@contextlib.contextmanager
def refused(what):
    with pytest.raises(F.FrizbeeError) as e:
        yield
    assert e.value.status == UNSUPPORTED, (what, e.value)


# ------------------------------------------------------------------------------------------------ constructors
NEEDLE = b"mQ7"
UNEEDLE = "é7"


def mixed_list(seed=11, n=2 * TILE + 333):
    """Lengths 0, 1, 15-17, 63-65, 127-129 and a few of 2-70 KB; NUL and bytes >= 0x80; every byte value once and twice
    in one haystack each; n a multiple of neither 32 nor 1024; the needle ends the list."""
    rng = np.random.default_rng(seed)
    pool = np.frombuffer(b"abcmqQ7M_-/ \x00\xc3\xa9x", dtype=np.uint8)
    special = [0, 1, 15, 16, 17, 63, 64, 65, 127, 128, 129, 2048, 5003, 40000, 70001]
    hs = []
    for i in range(n - 3):
        ln = special[i % len(special)] if i % 7 == 0 else int(rng.integers(0, 40))
        src = rng.integers(0, 256, ln, dtype=np.uint8) if i % 5 == 0 else rng.choice(pool, ln)
        h = bytearray(src.tobytes())
        if ln >= 3 and i % 4 == 0:
            at = int(rng.integers(0, ln - 2))
            h[at: at + 3] = NEEDLE if i % 8 else "é7".encode()
        hs.append(bytes(h))
    every = np.arange(256, dtype=np.uint8)
    hs.append(rng.permutation(every).tobytes())
    hs.append(rng.permutation(np.concatenate([every, every])).tobytes())
    hs.append(b"\x80xx\x00" + NEEDLE)
    return hs


def configs():
    return [Config(max_typos=k, emulate_lanes=LANES) for k in (0, 1, None)]


def matchers():
    ms = [(F.Matcher(Pattern(NEEDLE), cfg), [Pattern(NEEDLE)], cfg) for cfg in configs()]
    ucfg = Config(max_typos=1, emulate_lanes=LANES)
    ms.append((F.Matcher(UNEEDLE, ucfg), [UNEEDLE], ucfg))
    return ms


def c_corpus(fn, *args):
    h = C.c_void_p()
    F._check(fn(*args, 0, C.byref(h)))
    return F.Corpus(h, F.lib().frz_corpus_len(h))


def device_corpus(data, off, base, lead, stream=None):
    """frz_corpus_create_device on a torch buffer: the values start `base` bytes past an allocation (any alignment) and
    the offsets at d_offsets[0] = lead; the rest of the buffer is 0xEE."""
    n, total = len(off) - 1, int(off[-1] - off[0])
    ctx = torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext()
    if stream is not None:
        stream.wait_stream(torch.cuda.current_stream())
    with ctx:
        buf = torch.full((base + lead + total + 64,), 0xEE, dtype=torch.uint8, device="cuda")
        buf[base + lead: base + lead + total] = torch.from_numpy(np.ascontiguousarray(data[int(off[0]): int(off[-1])])).cuda()
        d_off = torch.from_numpy((off.astype(np.int64) - int(off[0]) + lead)).cuda()
        c = F.Corpus.from_device(buf.data_ptr() + base, d_off.data_ptr(), n, total, 0,
                                 stream.cuda_stream if stream is not None else 0)
        buf.fill_(0x55)   # the corpus is complete on return and must not read the buffers any more
        d_off.fill_(0)
    if stream is not None:
        stream.synchronize()
    return c


def test_every_constructor_packs_the_same_image():
    hs = mixed_list()
    data, off = pack(hs)
    n = len(hs)
    assert n % 32 and n % TILE and data[-1] == NEEDLE[-1]
    want_img = expected_image(data, off)
    ms = matchers()
    wants = [O.match_list_packed(p, cfg, data, off) for _, p, cfg in ms]
    # the same list as a slice of a longer Arrow array: offsets[0] > 0, values before and after it
    pre, post = pack([b"\xee" * 5, b"zz", b"\x00" * 33]), pack([b"tail" * 9, b"mQ"])
    big_data = np.concatenate([pre[0], data, post[0]])
    big_off = np.concatenate([pre[1], off[1:] + pre[1][-1], post[1][1:] + pre[1][-1] + off[-1]])
    sl = big_off[3: 3 + n + 1]
    L = F.lib()

    def built():
        yield "frz_corpus_create", c_corpus(L.frz_corpus_create, data.ctypes.data, off.ctypes.data, n)
        for dt in (np.uint32, np.int32, np.uint64):
            yield f"create_arrow {np.dtype(dt)}", F.Corpus.from_arrow(data, off.astype(dt))
            yield f"create_arrow {np.dtype(dt)} slice", F.Corpus.from_arrow(big_data, sl.astype(dt))
        ptrs = (C.c_void_p * n)(*[data.ctypes.data + int(o) for o in off[:-1]])
        lens = np.diff(off).astype(np.uint32)
        yield "create_ptrs", c_corpus(L.frz_corpus_create_ptrs, ptrs, lens.ctypes.data, n)
        side = torch.cuda.Stream()
        for base in range(4):
            for lead in (0, 5, 4 + base):
                yield f"create_device base {base} lead {lead}", device_corpus(data, off, base, lead)
        yield "create_device side stream", device_corpus(big_data, sl, 3, int(sl[0]), side)
        c = F.Corpus.from_list([])
        at = 0
        for k, step in enumerate((1, 30, 2, 1024, 999, 1, 7, n)):
            hi = min(n, at + step)
            if hi > at:
                c.append(big_data, (sl[at: hi + 1]).astype(np.uint32 if k % 2 else np.uint64))
            at = hi
        yield "append from empty", c

    for what, c in built():
        assert corpus_len(c) == n and c.total_bytes == int(off[-1]), what
        assert_image(c, want_img, what)
        for (m, p, cfg), want in zip(ms, wants):
            assert_same(m.match_list_array(c), want, (what, p, cfg.max_typos))
        c.close()
    for (m, p, cfg), want in zip(ms, wants):
        out = np.empty(n, dtype=F.MATCH_DTYPE)
        cnt = C.c_uint64()
        F._check(L.frz_match_list_host(m._h, data.ctypes.data, off.ctypes.data, n, 0, out.ctypes.data, n, C.byref(cnt)))
        assert_same(out[: cnt.value], want, ("frz_match_list_host", p, cfg.max_typos))
        assert_same(m.match_list_host_array(big_data, sl.astype(np.uint32)), want, ("match_list_host_arrow u32 slice", p))
        m.close()


def test_debug_image_checks_its_buffers():
    data, off = pack([b"abc", b"", b"x" * 40])
    c = F.Corpus.from_arrow(data, off)
    L = F.lib()
    sizes = (C.c_uint64 * 6)()
    F._check(L.frz_corpus_debug_image(c._h, *[None] * 6, sizes))
    assert list(sizes) == [8, 32 * 16, 1024 * 4, 1024 * 2, 1024 * 8, (32 * 3) * 16]
    bufs = [np.zeros(int(s) + 16, dtype=np.uint8) for s in sizes]
    ptrs = [b.ctypes.data for b in bufs]
    assert L.frz_corpus_debug_image(c._h, *ptrs[:5], None, sizes) == 1          # some buffers missing
    wrong = (C.c_uint64 * 6)(*sizes)
    wrong[2] += 4
    assert L.frz_corpus_debug_image(c._h, *ptrs, wrong) == 1                    # a wrong size
    assert L.frz_corpus_debug_image(c._h, *ptrs, None) == 1
    assert L.frz_corpus_debug_image(c._h, *ptrs, sizes) == 0
    empty = F.Corpus.from_list([])
    F._check(L.frz_corpus_debug_image(empty._h, *[None] * 6, sizes))
    assert list(sizes) == [0] * 6
    c.close()
    empty.close()


# ------------------------------------------------------------------------------------------ the length limit
@pytest.mark.parametrize("total", [65535, 65536, 70000, 1 << 20])
def test_greedy_scorer_long_gaps(total):
    """Windows over 1024 bytes go through a greedy scorer, which clamps a gap at 65 535 bytes: windows of `total` bytes
    with the needle's bytes up to `total` - 3 apart.  The byte path keeps every score below 2^15 (its kernels' cells are
    signed 16-bit), so a clamp anywhere at or above 32 767 scores alike there.  The unicode path's scores reach 65 535:
    with a match score of 20 000, "éc" scores above 40 000 before its last gap, and the clamp decides the result."""
    for needle, scorings in (("abc", (Scoring(), Scoring(match_score=8000))), ("éc", (Scoring(), Scoring(match_score=20000)))):
        a, c = needle[:-1].encode(), needle[-1].encode()
        hs = [a + b"x" * (total - len(a) - 1) + c, a + b"x" * 40000 + c + b"x" * (total - len(a) - 40001),
              a[:1] + b"x" * (total - len(a) - 1) + a[1:] + c, b"x" * (total - len(a) - 1) + a + c, a + c]
        data, off = pack(hs)
        corpus = F.Corpus.from_arrow(data, off)
        for sc in scorings:
            for k in (0, None):
                cfg = Config(max_typos=k, scoring=sc, emulate_lanes=LANES, sort=SortStrategy.IndexAsc)
                want = O.match_list_packed([needle], cfg, data, off)
                assert len(want) >= len(hs) - 1   # (the unicode path refuses the haystack that splits "é")
                m = F.Matcher(needle, cfg)
                assert_same(m.match_list_array(corpus), want, (needle, total, sc.match_score, k))
                m.close()
        corpus.close()


def short_list(n, seed=3):
    """Haystacks of 0-23 bytes without the needle "zq", but for two."""
    rng = np.random.default_rng(seed)
    pool = np.frombuffer(b"abcz_-/Q", dtype=np.uint8)
    hs = [rng.choice(pool, int(rng.integers(0, 24))).tobytes() for _ in range(n)]
    hs[5], hs[n - 1] = b"zq", b"a-zq"
    return hs


def longest_list(where, n=2 * TILE + 5):
    """short_list with MAX_HAY-byte haystacks at the local indices `where`: the needle as the first bytes of one and the
    last bytes of the other."""
    hs = short_list(n)
    hs[where[0]] = b"zq" + b"a" * (MAX_HAY - 2)
    hs[where[1]] = b"a" * (MAX_HAY - 2) + b"zq"
    return hs


@pytest.mark.parametrize("where", [(0, 1023), (TILE + 31, TILE + 32)])
def test_longest_haystacks(where):
    """Haystacks of exactly MAX_HAY bytes, at local index 0 and 1023 of a tile (1023 made the old length limit collide
    with the unused-slot sentinel) and at 31 / 32.  Two per corpus: each pads its group to 128 MiB."""
    hs = longest_list(where)
    data, off = pack(hs)
    want_img = expected_image(data, off)
    cfgs = [Config(max_typos=k, emulate_lanes=LANES) for k in (0, 1, None)]
    wants = [O.match_list_packed(["zq"], cfg, data, off) for cfg in cfgs]
    for want in wants:
        assert set(where) <= set(want["index"].tolist())
    c = F.Corpus.from_arrow(data, off)
    assert_image(c, want_img, "create_arrow")
    a = F.Corpus.from_arrow(data, off[: where[0] + 1])
    a.append(data, off[where[0]:])
    assert_image(a, want_img, "append")
    for cfg, want in zip(cfgs, wants):
        m = F.Matcher("zq", cfg)
        assert_same(m.match_list_array(c), want, ("create_arrow", cfg.max_typos))
        assert_same(m.match_list_array(a), want, ("append", cfg.max_typos))
        assert_same(m.match_list_host_array(data, off.astype(np.uint32)), want, ("end to end", cfg.max_typos))
        m.close()
    c.close()
    a.close()


def test_one_byte_over_the_limit_is_refused():
    """A haystack of MAX_HAY + 1 bytes is refused by every constructor, append and the end-to-end calls; afterwards the
    matcher, its end-to-end arena and the corpus that refused an append give the right lists."""
    over = b"zq" + b"a" * (MAX_HAY - 1)
    small = short_list(300)
    s_data, s_off = pack(small)
    cfg = Config(max_typos=1, emulate_lanes=LANES)
    want = O.match_list_packed(["zq"], cfg, s_data, s_off)
    m = F.Matcher("zq", cfg)
    L = F.lib()
    # a short list, and one long enough (>= 64 tiles) for the end-to-end call to take its streamed form
    for n_short in (7, 70 * TILE):
        hs = [b"zq"] * n_short + [over] + [b"q"]
        data, off = pack(hs)
        with refused("create_arrow"):
            F.Corpus.from_arrow(data, off)
        with refused("create_arrow u32"):
            F.Corpus.from_arrow(data, off.astype(np.uint32))
        with refused("create_device"):
            device_corpus(data, off, 1, 3)
        with refused("match_list_host_arrow"):
            m.match_list_host_array(data, off.astype(np.uint32))
        assert_same(m.match_list_host_array(s_data, s_off), want, "end to end after a refusal")
        out = np.empty(len(hs), dtype=F.MATCH_DTYPE)
        cnt = C.c_uint64()
        assert L.frz_match_list_host(m._h, data.ctypes.data, off.ctypes.data, len(hs), 0, out.ctypes.data, len(hs),
                                     C.byref(cnt)) == UNSUPPORTED
        assert_same(m.match_list_host_array(s_data, s_off.astype(np.uint32)), want, "end to end after a refusal")
    # a refused append leaves the corpus as it was: length and byte count first, then the image, then matches
    c = F.Corpus.from_arrow(s_data, s_off)
    before = read_image(c)
    extra, e_off = pack([b"zq", b"", over, b"zq"])
    with refused("append"):
        c.append(extra, e_off)
    assert corpus_len(c) == len(small) and c.total_bytes == int(s_off[-1])
    assert_image(c, before, "after a refused append")
    assert_same(m.match_list_array(c), want, "after a refused append")
    # and it still takes appends
    more = [b"zq", b"", b"x" * 5000 + b"zq"] * 400
    c.append_list(more)
    a_data, a_off = pack(small + more)
    assert corpus_len(c) == len(small) + len(more)
    assert_image(c, expected_image(a_data, a_off), "append after a refused append")
    assert_same(m.match_list_array(c), O.match_list_packed(["zq"], cfg, a_data, a_off), "append after a refused append")
    c.close()
    m.close()


# ---------------------------------------------------------------------------------------- past 12 224 tiles
# 12 288 tiles: k_tile_scan walks global memory above 12 224 tiles, and with 12 288 = 1024 * 12 the scan's last thread
# owns the last 12 tiles (with fewer tiles its run is empty and the total never passes through the per-tile loop)
N_LARGE = 12_288 * TILE - 333


def large_list():
    rng = np.random.default_rng(12224)
    n = N_LARGE
    lens = rng.integers(0, 9, n)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum(lens)
    data = rng.choice(np.frombuffer(b"cdefghijklmnoprstuvwxyz_-", dtype=np.uint8), int(off[-1]))
    start = off[:-1].astype(np.int64)
    # "ab" in about 1.4 M haystacks (every one of the last 2000), 'q' in a tenth of those, "é" in 100 k others
    pick = (rng.random(n) < 0.12) & (lens >= 2)
    pick[-2000:] = lens[-2000:] >= 2
    at = start[pick] + (rng.random(pick.sum()) * (lens[pick] - 1)).astype(np.int64)
    data[at], data[at + 1] = ord("a"), ord("b")
    q = pick & (lens >= 4) & (rng.random(n) < 0.1)
    data[start[q] + lens[q] - 1] = ord("q")
    data[start[q]] = ord("a")
    u = ~pick & (lens >= 3) & (rng.random(n) < 0.01)
    data[start[u]], data[start[u] + 1] = 0xC3, 0xA9
    return data, off


def test_past_12224_tiles():
    free, total = torch.cuda.mem_get_info()
    need = 8 << 30
    if free < need:
        pytest.skip(f"needs {need >> 20} MiB of free device memory, {free >> 20} of {total >> 20} MiB free")
    data, off = large_list()
    c = F.Corpus.from_arrow(data, off)
    assert corpus_len(c) == N_LARGE and -(-N_LARGE // TILE) > 12_224
    for sort in SortStrategy:
        cfg = Config(max_typos=0, sort=sort, emulate_lanes=LANES)
        want = O.match_list_packed(["ab"], cfg, data, off)
        assert len(want) > 1_000_000 and want["index"].max() >= N_LARGE - 2000
        m = F.Matcher("ab", cfg)
        assert_same(m.match_list_array(c), want, sort)
        top, n_total = m.match_list_top_array(c, 1000)
        assert n_total == len(want)
        assert_same(top, want[:1000], ("top", sort))
        if sort == SortStrategy.ScoreThenIndexAsc:
            assert_same(m.match_list_host_array(data, off), want, "end to end")
        m.close()
    cfg = Config(max_typos=0, emulate_lanes=LANES)
    m = F.Matcher.from_query("ab !q", cfg)
    pats = F.parse_query("ab !q")
    assert pats[1].negated
    assert_same(m.match_list_array(c), O.match_list_packed(pats, cfg, data, off), "ab !q")
    m.close()
    ucfg = Config(max_typos=0, emulate_lanes=LANES)
    m = F.Matcher("é", ucfg)
    want = O.match_list_packed(["é"], ucfg, data, off)
    assert 10_000 < len(want) < 1_000_000
    assert_same(m.match_list_array(c), want, "unicode")
    m.close()
    c.close()
