"""Top-K match_list on the GPU (frz_match_list_top, frz_match_list_parallel*_top): every call must return exactly the first
min(K, total) rows of the full call on the same matcher and corpus, and the full match count.  Needs a CUDA device."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200 import parallel, synth
from frizbee_b200.types import Config, Matching, Pattern, Scoring, SortStrategy

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEG = 2048   # elements per segment of the fused scatter (kFrzSortSegShift in frz_host.h)
LONG_NEEDLE = "abcdefghijklmnopqrstuvwxyzabcdefghijklmnopqrstuvwxyzabcdefgh"   # 60 bytes: score bound >= 1024
# FRZ_PARALLEL_EXCHANGE of the 2-GPU tests: unset (the default P2P placement), `slices` (the NCCL slice exchange), and
# two values that named removed forms, which communicator creation must refuse
EXCHANGES = [pytest.param(None, id="p2p"), "slices", "direct", "allgather"]
REFUSED = ("direct", "allgather")


def _gpus():
    import torch
    return torch.cuda.device_count()


def check_top(m, corpus, ks, full=None):
    """top == full[:K] and total == len(full) for every K; returns the full list."""
    if full is None:
        full = m.match_list_array(corpus).copy()
    for k in ks:
        top, total = m.match_list_top_array(corpus, k)
        assert total == len(full), (k, total, len(full))
        assert len(top) == min(k, total) and np.array_equal(top, full[:k]), (k, total)
    return full


def edge_ks(total):
    return sorted({0, 1, 2047, 2048, 2049, max(total - 1, 0), total, total + 1})


@pytest.fixture(scope="module")
def deadbeef():
    data, off = synth.generate("deadbeef", 200_000, 48, 64, seed=41, p_partial=0.3, p_full=0.1)
    corpus = F.Corpus.from_arrow(data, off)
    yield data, off, corpus
    corpus.close()


@pytest.mark.parametrize("lanes", [16, 32, 64])
@pytest.mark.parametrize("sort", list(SortStrategy))
def test_top_every_strategy_and_backend(deadbeef, sort, lanes):
    _, _, corpus = deadbeef
    m = F.Matcher("deadbeef", Config(max_typos=1, sort=sort, emulate_lanes=lanes))
    full = m.match_list_array(corpus).copy()
    assert len(full) > 3 * SEG
    check_top(m, corpus, edge_ks(len(full)) + [5000, len(full) // 2], full)
    m.close()


@pytest.mark.parametrize("sort", [SortStrategy.ScoreThenIndexAsc, SortStrategy.ScoreThenIndexDesc])
def test_top_cut_inside_a_block_of_tied_scores(sort):
    """Hundreds of matches share the score at position K, spread over several sort segments: index order decides."""
    rng = random.Random(3)
    hs = [bytes(rng.choice(b"xyz_-") for _ in range(rng.randint(0, 20))) for _ in range(30_000)]
    for i in range(0, 30_000, 37):
        hs[i] = b"qq_foo_qq"          # ~800 matches with one score
    for i in range(5, 30_000, 997):
        hs[i] = b"foo"                # ~30 exact matches above them
    data, off = F.pack_host(hs)
    corpus = F.Corpus.from_arrow(data, off)
    m = F.Matcher("foo", Config(max_typos=0, sort=sort))
    full = m.match_list_array(corpus).copy()
    scores = full["score"]
    n_top = int((scores == scores[0]).sum())
    assert n_top < 60 and int((scores == scores[n_top]).sum()) > 500
    check_top(m, corpus, [n_top - 1, n_top, n_top + 1, n_top + 250, n_top + 399, len(full) - 1], full)
    m.close(); corpus.close()


def _sweep(rng, per_class):
    spans = [(0, 40), (41, 64), (65, 128), (129, 600)]
    pool = b"abAB_/-ab01"
    return [bytes(rng.choice(pool) for _ in range(rng.randint(lo, hi))) for lo, hi in spans for _ in range(per_class)]


@pytest.mark.parametrize("match_score,bins", [(12, 256), (60, 512), (150, 1024), (300, 0)])
def test_top_fused_bins_and_two_pass(match_score, bins):
    """Each single-pass bin class (fused scatter) and the two-pass sort (bound >= 1024: histogram kernel, limit on the second
    pass only)."""
    if bins:
        cfg = Config(max_typos=1, scoring=Scoring(match_score=match_score))
    else:
        cfg = Config(max_typos=1, scoring=Scoring(match_score=300, mismatch_penalty=10, gap_open_penalty=20, gap_extend_penalty=0))
    data, off = F.pack_host(_sweep(random.Random(match_score), 3000))
    corpus = F.Corpus.from_arrow(data, off)
    for sort in SortStrategy:
        m = F.Matcher("ab0/", cfg.with_(sort=sort))
        if bins:
            assert bins // 2 <= m.score_bound() < bins or (bins == 256 and m.score_bound() < 256)
        else:
            assert m.score_bound() >= 1024
        full = check_top(m, corpus, [0, 1, 100, SEG, SEG + 1, 5 * SEG + 3])
        check_top(m, corpus, edge_ks(len(full)), full)
        m.close()
    corpus.close()


@pytest.mark.parametrize("case", ["multi", "unicode", "exact", "prefix", "suffix", "substring", "no_typo_limit", "empty_pattern"])
def test_top_other_pipelines(case):
    rng = random.Random(11)
    if case == "unicode":
        alphabet = ["é", "É", "다", "😀", "a", "-", "_", "x"]
        hs = ["".join(rng.choice(alphabet) for _ in range(rng.randint(0, 24))) for _ in range(30_000)]
        data, off = F.pack_host(hs)
    else:
        data, off = synth.generate("foo", 60_001, 40, 64, seed=13, prefix_frac=0.2, p_partial=0.3, p_full=0.1)
    corpus = F.Corpus.from_arrow(data, off)
    for sort in SortStrategy:
        if case == "multi":
            m = F.Matcher.from_query("foo !^bar", Config(max_typos=0, sort=sort))
        elif case == "unicode":
            m = F.Matcher("é다😀", Config(max_typos=1, sort=sort))
        elif case == "no_typo_limit":
            m = F.Matcher("foo", Config(max_typos=None, sort=sort))
        elif case == "empty_pattern":
            m = F.Matcher("", Config(sort=sort))   # every haystack, score 0 (k_fill_all)
        else:
            m = F.Matcher("foo", Config(sort=sort, matching=Matching[case.capitalize()]))
        full = check_top(m, corpus, [0, 1, 7, SEG + 1])
        assert len(full) > 0 or case == "exact", (case, len(full))
        check_top(m, corpus, edge_ks(len(full)), full)
        m.close()
    corpus.close()


def test_top_empty_corpus_and_no_matches():
    empty = F.Corpus.from_list([])
    none = F.Corpus.from_list(["xyz", "abc", ""] * 1000)
    for sort in SortStrategy:
        m = F.Matcher("foo", Config(max_typos=0, sort=sort))
        for corpus in (empty, none):
            for k in (0, 1, 10):
                top, total = m.match_list_top_array(corpus, k)
                assert len(top) == 0 and total == 0
        m.close()
    empty.close(); none.close()


def test_top_many_segments_retry_and_reuse():
    """> 2^21 matches (over a thousand sort segments, most of them past K), a first call whose survivor lists overflow
    (the call re-runs with worst-case lists), and top / full / top with another K on the same matcher: the fused histogram
    must be left clean by every call."""
    rng = np.random.default_rng(9)
    n = 2_300_000
    lens = rng.integers(2, 14, n)
    pool = np.frombuffer(b"abAB_/-ab01xyz", dtype=np.uint8)
    data = pool[rng.integers(0, len(pool), int(lens.sum()))]
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum(lens)
    corpus = F.Corpus.from_arrow(data, off)
    for k_typos in (None, 1):
        cfg = Config(max_typos=k_typos)
        want = F.Matcher("ab", cfg).match_list_array(corpus).copy()
        if k_typos is None:
            assert len(want) == n and n > (1 << 21)
        m = F.Matcher("ab", cfg)
        top, total = m.match_list_top_array(corpus, 100)   # first call on a fresh matcher
        assert total == len(want) and np.array_equal(top, want[:100])
        full = m.match_list_array(corpus)
        assert np.array_equal(full, want)
        check_top(m, corpus, [10, 5000, SEG * 300 + 5, len(want) - 1, len(want) + 1], want)
        assert np.array_equal(m.match_list_array(corpus), want)
        m.close()
    corpus.close()


def test_top_rows_compose_with_match_indices():
    """The rows a UI shows: their indices go to frz_match_indices, which returns the same Match for every row."""
    data, off = synth.generate("deadbeef", 50_000, 48, 64, seed=3)
    corpus = F.Corpus.from_arrow(data, off)
    m = F.Matcher("deadbeef", Config(max_typos=1))
    top, total = m.match_list_top_array(corpus, 50)
    assert len(top) == 50 and total > 50
    rows = m.match_indices(corpus, top["index"])
    for t, r in zip(top, rows):
        assert r is not None and r[0] == int(t["score"]) and r[1] == bool(t["exact"]) and len(r[2]) > 0
    m.close(); corpus.close()


@pytest.mark.parametrize("force_nccl", [0, 1])
def test_parallel_top_world1(force_nccl, monkeypatch):
    monkeypatch.setenv("FRZ_PARALLEL_FORCE_NCCL", str(force_nccl))
    comm = parallel.Comm.local(1)
    data, off = synth.generate("deadbeef", 120_001, 48, 64, seed=21)
    shards = comm.shard_arrow(data, off)
    whole = F.Corpus.from_arrow(data, off)
    for sort in SortStrategy:
        for k_typos in (1, None):
            m = F.Matcher("deadbeef", Config(max_typos=k_typos, sort=sort))
            full = comm.match_list_parallel(m, shards).copy()
            assert np.array_equal(full, m.match_list_array(whole))
            for k in edge_ks(len(full)):
                top, total = comm.match_list_parallel_top(m, shards, k)
                assert total == len(full) and np.array_equal(top, full[:k]), (sort, k_typos, k)
            m.close()
    for s in shards:
        s.close()
    whole.close(); comm.close()


@pytest.mark.parametrize("exchange", EXCHANGES)
def test_parallel_top_two_gpus_local(exchange, monkeypatch):
    """Both host-out exchange forms; a score bound >= 1024 (two-pass sort, no per-score table) takes the all-gather + merge.
    `direct` and `allgather` named removed forms: a two-GPU communicator must refuse them."""
    if _gpus() < 2:
        pytest.skip("needs >= 2 GPUs")
    if exchange is None:
        monkeypatch.delenv("FRZ_PARALLEL_EXCHANGE", raising=False)
    else:
        monkeypatch.setenv("FRZ_PARALLEL_EXCHANGE", exchange)
    if exchange in REFUSED:
        with pytest.raises(F.FrizbeeError) as e:
            parallel.Comm.local(2)
        assert e.value.status_name == "FRZ_ERR_INVALID_ARG"
        return
    comm = parallel.Comm.local(2)
    assert comm.exchange_mode() == (1 if exchange == "slices" else 2)
    data, off = synth.generate("deadbeef", 300_001, 48, 64, seed=33)
    shards = comm.shard_arrow(data, off)
    out = comm.host_alloc_matches(300_001)
    for sort in SortStrategy:
        for k_typos in (1, None):
            m = F.Matcher("deadbeef", Config(max_typos=k_typos, sort=sort))
            full = np.array(comm.match_list_parallel(m, shards, out))
            for k in edge_ks(len(full)) + [len(full) // 2 + 1]:
                top, total = comm.match_list_parallel_top(m, shards, k, out)
                assert total == len(full) and np.array_equal(np.array(top), full[:k]), (exchange, sort, k_typos, k)
            m.close()
    d2, o2 = synth.generate(LONG_NEEDLE, 20_001, 80, 128, seed=2, p_full=0.5)
    s2 = comm.shard_arrow(d2, o2)
    w2 = F.Corpus.from_arrow(d2, o2)
    for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.ScoreThenIndexDesc):
        m = F.Matcher(LONG_NEEDLE, Config(max_typos=None, sort=sort))
        assert m.score_bound() >= 1024
        full = m.match_list_array(w2).copy()
        for k in edge_ks(len(full)) + [len(full) // 2 + 1]:
            top, total = comm.match_list_parallel_top(m, s2, k, out)
            assert total == len(full) and np.array_equal(np.array(top), full[:k]), (exchange, "two-pass bound", sort, k)
        m.close()
    comm.host_free(out)
    for s in shards + s2:
        s.close()
    w2.close(); comm.close()


@pytest.mark.parametrize("exchange", EXCHANGES)
def test_parallel_top_two_gpus_torchrun(exchange):
    if _gpus() < 2:
        pytest.skip("needs >= 2 GPUs")
    env = dict(os.environ, FRZ_PARALLEL_TIMEOUT_S="60")
    env.pop("FRZ_PARALLEL_EXCHANGE", None)
    if exchange:
        env["FRZ_PARALLEL_EXCHANGE"] = exchange
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "tests", "_top_multi_gpu_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    sys.stdout.write(r.stdout[-4000:])
    sys.stderr.write(r.stderr[-4000:])
    assert r.returncode == 0
    assert "False" not in r.stdout and "differs" not in r.stdout
    if exchange in REFUSED:
        assert r.stdout.count("communicator refused with FRZ_ERR_INVALID_ARG: True") == 2


def test_parallel_rank_top_world1():
    """The multi-process form with one rank: host-out into the shared segment, and the device-only result."""
    comm = parallel.Comm.from_rank(parallel.Comm.unique_id(), 1, 0, 0)
    data, off = synth.generate("deadbeef", 60_000, 48, 64, seed=5)
    shard = F.Corpus.from_arrow(data, off)
    m = F.Matcher("deadbeef", Config(max_typos=1))
    out = comm.host_alloc_matches(60_000)
    total, _ = comm.match_list_parallel_rank(m, shard, 1000, out)
    full = np.array(out[:total])
    for k in edge_ks(total):
        n, t, _ = comm.match_list_parallel_rank_top(m, shard, 1000, k, out)
        assert t == total and n == min(k, total) and np.array_equal(np.array(out[:n]), full[:k]), k
    n, t, d = comm.match_list_parallel_rank_top(m, shard, 1000, 10, None)
    assert (n, t) == (10, total) and d != 0
    comm.host_free(out)
    shard.close(); m.close(); comm.close()


def test_top_output_buffer_holds_min_k_and_haystacks():
    """No more rows than haystacks can match, so a buffer of min(k, haystacks) rows is enough for any k — including
    k > total when every haystack matches (max_typos = None) — and a smaller one is refused before the library runs."""
    n = 5000
    data, off = synth.generate("deadbeef", n, 24, 32, seed=19)
    corpus = F.Corpus.from_arrow(data, off)
    m = F.Matcher("deadbeef", Config(max_typos=None))
    full = m.match_list_array(corpus).copy()
    assert len(full) == n
    for k in (n - 1, n, n + 1, 10 * n):
        out = np.empty(min(k, n), dtype=F.MATCH_DTYPE)
        top, total = m.match_list_top_array(corpus, k, out=out)
        assert total == n and np.array_equal(top, full[:k])
    with pytest.raises(ValueError):
        m.match_list_top_array(corpus, n + 1, out=np.empty(n - 1, dtype=F.MATCH_DTYPE))
    comm = parallel.Comm.local(1)
    shards = comm.shard_arrow(data, off)
    shared = comm.host_alloc_matches(n)
    for k in (n, n + 1, 10 * n):
        top, total = comm.match_list_parallel_top(m, shards, k, shared)
        assert total == n and np.array_equal(np.array(top), full[:k])
    with pytest.raises(ValueError):
        comm.match_list_parallel_top(m, shards, n + 1, np.empty(n - 1, dtype=F.MATCH_DTYPE))
    comm.host_free(shared)
    for s in shards:
        s.close()
    m.close(); corpus.close(); comm.close()
