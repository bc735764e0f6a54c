"""Ranks from keys on the device (frz_attr_rank) against the host path it replaces, and an ordered top-K on the rank.

  python tools/bench_rank.py [--flagship 10000000] [--paths 1000000] [--steps 10] [--warmup 2] [--host-steps 2] [--k 50]

Workloads:
  flagship  the flagship corpus (synth `deadbeef` haystacks, 24-64 bytes), ranked by its text, and by its text with
            fold_case;
  paths     path-like rows: a directory of 1-5 components from tools/bench_batch_columns.py's vocabulary, a slash and a
            synth file name; ranked by the text alone, and by a file-kind attribute (8 values) then the text.
For each the timed configurations are:
  device    Attr.rank refilling one attribute (host clock around the call, which ends in a synchronise);
  host      what a caller does without it: the rows as fixed-width byte strings (folded when asked), np.unique for the
            dense text ranks (with np.lexsort over (kind, text rank) for two keys), then Corpus.attr to upload the ranks.
The two results are compared before timing and must be equal.  Then, on the flagship corpus, the ordered top-K by
SCORE_THEN_ATTR_ASC on the rank (Matcher("deadbeef", max_typos = 1)) is timed against match_list_ranked_array at the same
K in the same run.  Configurations alternate step by step.  The card name, power limit and maximum SM clock are read with
nvidia-smi in the same run (queries only).  Prints one JSON object."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import frizbee_b200 as F   # noqa: E402
from bench_batch import card_info   # noqa: E402
from bench_batch_columns import directories   # noqa: E402
from frizbee_b200 import synth   # noqa: E402
from frizbee_b200.types import Config, Order   # noqa: E402

WIDTH = 64 + 1 + 64   # the longest path: a directory of at most 5 * 11 bytes, a slash, a synth name
FOLD = np.arange(256, dtype=np.uint8)
FOLD[65:91] += 32


def summarize(samples):
    ms = sorted(1e3 * s for s in samples)
    return {"median_ms": round(statistics.median(ms), 3), "min_ms": round(ms[0], 3), "n": len(ms)}


def fixed_width(data, off, width, fold):
    """The rows as an (n,) array of `width`-byte strings, zero padded (numpy orders them as memcmp does when no row holds
    a NUL)."""
    n = len(off) - 1
    out = np.zeros((n, width), np.uint8)
    col = np.arange(width)
    for a in range(0, n, 1 << 20):
        b = min(n, a + (1 << 20))
        start = off[a:b].astype(np.int64)
        lens = off[a + 1:b + 1].astype(np.int64) - start
        idx = start[:, None] + col
        keep = col < lens[:, None]
        block = np.where(keep, data[np.minimum(idx, len(data) - 1)], 0).astype(np.uint8)
        out[a:b] = FOLD[block] if fold else block
    return out.view(f"S{width}").ravel()


def host_rank(corpus, data, off, width, fold, kind=None):
    _, inv = np.unique(fixed_width(data, off, width, fold), return_inverse=True)
    inv = inv.astype(np.int64)
    if kind is not None:
        perm = np.lexsort((inv, kind))
        s_kind, s_inv = kind[perm], inv[perm]
        new = np.ones(len(perm), bool)
        new[1:] = (s_kind[1:] != s_kind[:-1]) | (s_inv[1:] != s_inv[:-1])
        inv = np.empty(len(perm), np.int64)
        inv[perm] = np.cumsum(new) - 1
    return corpus.attr(inv), inv


def time_pair(device_fn, host_fn, steps, warmup, host_steps):
    dev, host = [], []
    for i in range(warmup + steps):
        t = time.perf_counter()
        device_fn()
        if i >= warmup:
            dev.append(time.perf_counter() - t)
        if i < host_steps:
            t = time.perf_counter()
            h = host_fn()
            host.append(time.perf_counter() - t)
            h.close()
    return {"device": summarize(dev), "host": summarize(host)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--flagship", type=int, default=10_000_000)
    ap.add_argument("--paths", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-steps", type=int, default=2)
    ap.add_argument("--k", type=int, default=50)
    ap.add_argument("--seed", type=int, default=12345)
    args = ap.parse_args()
    result = {"card": card_info(0), "steps": args.steps, "results": {}}

    # flagship: text, text with fold_case
    data, off = synth.generate("deadbeef", args.flagship, 24, 64, args.seed)
    c = F.Corpus.from_arrow(data, off)
    a = c.attr()
    for fold in (False, True):
        a.rank(c.text(fold_case=fold))
        h, inv = host_rank(c, data, off, 64, fold)
        h.close()
        assert np.array_equal(a.values(), inv), ("flagship", fold)
        result["results"][f"flagship_text{'_fold' if fold else ''}"] = time_pair(
            lambda: a.rank(c.text(fold_case=fold)), lambda: host_rank(c, data, off, 64, fold)[0], args.steps, args.warmup,
            args.host_steps)
    # the ordered top-K on the rank against the ranked top-K
    a.rank(c.text())
    boost = c.boost()
    m = F.Matcher("deadbeef", Config(max_typos=1))
    ordered, ranked = [], []
    for i in range(args.warmup + args.steps):
        t = time.perf_counter()
        m.match_list_ordered_array(c, a, Order.ScoreThenAttrAsc, args.k)
        if i >= args.warmup:
            ordered.append(time.perf_counter() - t)
        t = time.perf_counter()
        m.match_list_ranked_array(c, boost, args.k)
        if i >= args.warmup:
            ranked.append(time.perf_counter() - t)
    result["results"]["flagship_top"] = {"k": args.k, "ordered_score_then_rank": summarize(ordered), "ranked": summarize(ranked)}
    for h in (m, boost, a, c):
        h.close()
    del data, off

    # paths: text, and a kind attribute then the text
    rng = np.random.default_rng(args.seed)
    names, noff = synth.generate("deadbeef", args.paths, 24, 64, args.seed + 1)
    dirs = directories(args.paths, args.seed)
    rows = [d.encode() + b"/" + names[noff[i]:noff[i + 1]].tobytes() for i, d in enumerate(dirs)]
    data, off = F.pack_host(rows)
    del rows
    c = F.Corpus.from_arrow(data, off)
    kind = rng.integers(0, 8, args.paths).astype(np.int64)
    ka = c.attr(kind)
    a = c.attr()
    for name, keys, kk in (("paths_text", lambda: [c.text()], None), ("paths_kind_then_text", lambda: [ka.asc(), c.text()], kind)):
        a.rank(*keys())
        h, inv = host_rank(c, data, off, WIDTH, False, kk)
        h.close()
        assert np.array_equal(a.values(), inv), name
        result["results"][name] = time_pair(lambda: a.rank(*keys()), lambda: host_rank(c, data, off, WIDTH, False, kk)[0],
                                            args.steps, args.warmup, args.host_steps)
    for h in (a, ka, c):
        h.close()
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
