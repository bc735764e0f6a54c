"""Device memory is owned and given back: every cycle below (create objects, run calls, destroy everything) leaves the
bytes the library holds (frz_debug_device_bytes) where they were.  Each cycle runs once first, so that caches that
outlive it (the per-device merge scratch of frz_merge_runs_device) are in place before the count is taken.  The check
reads the library's own counter, not the card's free memory, which other processes change."""
import ctypes as C

import numpy as np
import pytest
import torch

import frizbee_b200 as F
from frizbee_b200 import parallel, synth
from frizbee_b200.types import Config, SortStrategy

pytestmark = pytest.mark.gpu

NEEDLE = "deadbeef"
LONG_NEEDLE = "the quick brown fox jumps over the lazy dog, then naps by the red barn at dusk"   # > 64 bytes
assert 64 < len(LONG_NEEDLE) <= 1024


def device_bytes():
    L = F.lib()
    L.frz_debug_device_bytes.restype = C.c_uint64
    L.frz_debug_device_bytes.argtypes = []
    return L.frz_debug_device_bytes()


def check_cycle(cycle, repeats=3):
    cycle()
    torch.cuda.synchronize()
    base = device_bytes()
    for _ in range(repeats):
        cycle()
    torch.cuda.synchronize()
    assert device_bytes() == base


def small_arrow(n=5_000, seed=3, needle=NEEDLE):
    mu, longest = (48, 64) if len(needle) <= 64 else (200, 600)
    return synth.generate(needle, n, mu, longest, seed=seed)


def test_corpus_constructors_and_append():
    data, off = small_arrow()
    n = len(off) - 1
    extra_d, extra_o = small_arrow(1_500, seed=4)
    L = F.lib()

    def cycle():
        held = device_bytes()
        corpora = []
        h = C.c_void_p()
        F._check(L.frz_corpus_create(data.ctypes.data, off.ctypes.data, n, 0, C.byref(h)))   # (synth offsets are u64)
        corpora.append(F.Corpus(h, n))
        corpora.append(F.Corpus.from_arrow(data, off.astype(np.uint32)))
        corpora.append(F.Corpus.from_list([b"foo", b"bar_baz", b"deadbeef"]))
        ptrs = (C.c_void_p * n)(*[data.ctypes.data + int(o) for o in off[:-1]])
        lens = np.diff(off).astype(np.uint32)
        h = C.c_void_p()
        F._check(L.frz_corpus_create_ptrs(ptrs, lens.ctypes.data, n, 0, C.byref(h)))
        corpora.append(F.Corpus(h, n))
        d_bytes = torch.from_numpy(np.ascontiguousarray(data)).cuda()
        d_off = torch.from_numpy(off.astype(np.int64)).cuda()
        corpora.append(F.Corpus.from_device(d_bytes.data_ptr(), d_off.data_ptr(), n, int(off[-1] - off[0])))
        corpora.append(F.Corpus.from_list([]))
        for c in corpora:   # the first append creates the corpus's staging arena, the second one reuses it
            c.append(extra_d, extra_o)
            c.append(extra_d, extra_o.astype(np.uint32))
        assert device_bytes() > held
        for c in corpora:
            c.close()

    check_cycle(cycle)


@pytest.mark.parametrize("case", ["single", "multi_negated", "long_needle", "unicode", "top_k"])
def test_matcher_calls(case):
    needle = LONG_NEEDLE if case == "long_needle" else NEEDLE
    data, off = small_arrow(needle=needle)
    uni = ["é다😀", "xxé__다__😀yy", "É다😀", "no match", "a-é-다-😀"] * 200

    def cycle():
        if case == "unicode":
            m = F.Matcher("é다😀", Config(max_typos=1))
            corpus = F.Corpus.from_list(uni)
        else:
            corpus = F.Corpus.from_arrow(data, off)
            if case == "multi_negated":
                m = F.Matcher.from_query("dead !zzz beef", Config(max_typos=1))
            else:
                m = F.Matcher(needle, Config(max_typos=1))
        for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexDesc):
            m.set_config(Config(max_typos=1, sort=sort))
            if case == "top_k":
                got, total = m.match_list_top_array(corpus, 10)
                assert len(got) == min(10, total)
            else:
                assert len(m.match_list_array(corpus)) > 0
        m.close()
        corpus.close()

    check_cycle(cycle)


@pytest.mark.parametrize("n", [5_000, 80_000])   # below and at >= 64 tiles (the streamed form)
def test_host_in_path(n):
    data, off = small_arrow(n)

    def cycle():
        m = F.Matcher(NEEDLE, Config(max_typos=1))
        assert len(m.match_list_host_array(data, off)) > 0
        assert len(m.match_list_host_array(data, off.astype(np.uint32))) > 0
        m.close()

    check_cycle(cycle)


def test_indices_sort_and_merge():
    data, off = small_arrow()
    rng = np.random.default_rng(7)
    arr = np.zeros(3_000, dtype=F.MATCH_DTYPE)
    arr["index"] = np.arange(len(arr))
    arr["score"] = rng.integers(0, 4000, len(arr))
    dev = torch.device("cuda", 0)

    def cycle():
        corpus = F.Corpus.from_arrow(data, off)
        for query in (NEEDLE, "dead !zzz beef"):
            m = F.Matcher.from_query(query, Config(max_typos=1))
            assert len(m.match_indices(corpus, np.arange(100))) == 100
            m.close()
        assert len(F.radix_sort_matches(arr)) == len(arr)
        m = F.Matcher(NEEDLE, Config(max_typos=1))
        # the two halves of a score-sorted list are two score-sorted runs
        runs = torch.from_numpy(m.match_list_array(corpus).view(np.int64).copy()).to(dev)
        half = len(runs) // 2
        assert half > 0
        counts = np.array([half, half], dtype=np.uint64)
        out = torch.zeros(2 * half, dtype=torch.int64, device=dev)
        for bound in (m.score_bound(), 0):   # the boundary-search merge and the concatenate + sort fallback
            F._check(F.lib().frz_merge_runs_device(runs.data_ptr(), half, counts.ctypes.data, 2,
                                                   int(SortStrategy.ScoreThenIndexAsc), bound, out.data_ptr(), 0, None))
        torch.cuda.synchronize()
        m.close()
        corpus.close()

    check_cycle(cycle)


def test_one_gpu_communicator():
    data, off = small_arrow(20_000)

    def cycle():
        comm = parallel.Comm.local(1)
        shards = comm.shard_arrow(data, off)
        m = F.Matcher(NEEDLE, Config(max_typos=1))
        assert len(comm.match_list_parallel(m, shards)) > 0
        top, total = comm.match_list_parallel_top(m, shards, 10)
        assert len(top) == min(10, total)
        m.close()
        for s in shards:
            s.close()
        comm.close()

    check_cycle(cycle)
