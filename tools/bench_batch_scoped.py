"""Batched call with per-query subsets and boosts (frz_match_list_batch) against a loop of the single-query calls over the same
resident corpus.

  python tools/bench_batch_scoped.py [--sizes 100000,1000000] [--qs 8,64,512] [--scopes subset1,subset50,boost,both]
                                     [--rounds 3] [--seed 7]

Corpora: synth's flagship shape (needle `deadbeef`, mean length 48, at most 64 bytes) at each size, resident.  Queries: q
needles of 3-12 bytes cut from corpus rows (seeded), max_typos 0 and 1, k = 10.  Scopes, one per measured row:
  subset1 / subset50  every query its own random subset of 1 % / 50 % of the rows (frz_match_list_subset_top per query);
  boost               one boost drawn from 0..255, shared by every query (frz_match_list_ranked per query);
  both                every query its own 50 % subset and the shared boost (frz_match_list_ranked with the subset).
For every (size, typos, q, scope) four calls alternate over rounds: the loop of single-query calls, frz_match_list_batch
with its default limits ("batch"), the same with the limits lifted (F.batch_limits: every batch of two or more queries that
fits the scratch budget runs the batched kernels, "forced"), and, for reference, frz_match_list_batch_top of the same
matchers without scopes ("plain", default limits).  Before any is timed, both scoped batch calls' rows, n_out and n_total are
checked equal to the loop's, and the queries each answered on the batched kernels are recorded.  Host clock around each
call (every call ends in a synchronise).  The card name, power limit and maximum SM clock are read with nvidia-smi in the
same run (queries only).  Prints one JSON object."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import frizbee_b200 as F   # noqa: E402
from frizbee_b200 import synth   # noqa: E402
from frizbee_b200.types import Config   # noqa: E402
from tools.bench_batch import card_info, needles   # noqa: E402


def scopes(corpus, q, kind, boost, rng):
    """(subsets, boosts) for q queries of scope `kind`."""
    n = len(corpus)
    density = {"subset1": 0.01, "subset50": 0.5, "both": 0.5}.get(kind)
    subsets = [corpus.subset(np.flatnonzero(rng.random(n) < density)) for _ in range(q)] if density else [None] * q
    boosts = [boost] * q if kind in ("boost", "both") else [None] * q
    return subsets, boosts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100000,1000000")
    ap.add_argument("--qs", default="8,64,512")
    ap.add_argument("--typos", default="0,1")
    ap.add_argument("--scopes", default="subset1,subset50,boost,both")
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    k = args.k
    result = {"card": card_info(0), "k": k, "rows": []}
    for n in [int(x) for x in args.sizes.split(",")]:
        data, off = synth.generate("deadbeef", n, 48, 64, seed=args.seed)
        corpus = F.Corpus.from_arrow(data, off)
        rng = np.random.default_rng(args.seed)
        boost = corpus.boost(rng.integers(0, 256, n).astype(np.int16))
        for typos in [int(x) for x in args.typos.split(",")]:
            for q in [int(x) for x in args.qs.split(",")]:
                ms = [F.Matcher(s, Config(max_typos=typos)) for s in needles(data, off, q, args.seed + q)]
                outs = [np.empty(max(1, min(k, n)), dtype=F.MATCH_DTYPE) for _ in ms]
                for kind in args.scopes.split(","):
                    subsets, boosts = scopes(corpus, q, kind, boost, rng)

                    def loop():
                        res = []
                        for m, o, s, b in zip(ms, outs, subsets, boosts):
                            if b is not None:
                                res.append(m.match_list_ranked_array(corpus, b, k, subset=s, out=o))
                            else:
                                res.append(m.match_list_subset_top_array(corpus, s, k))
                        return res

                    def batch():
                        F.batch_limits()
                        return F.match_list_batch(ms, corpus, k, subsets=subsets, boosts=boosts)

                    def forced():
                        F.batch_limits(2**64 - 1, 2)
                        r = F.match_list_batch(ms, corpus, k, subsets=subsets, boosts=boosts)
                        F.batch_limits()
                        return r

                    def plain():
                        F.batch_limits()
                        return F.match_list_batch_top(ms, corpus, k)

                    want = [(top.copy(), total) for top, total in loop()]
                    batched = {}
                    for name, fn in (("batch", batch), ("forced", forced), ("plain", plain)):   # warm-up, and the check
                        rows, n_out, n_total = fn()
                        batched[name] = F.batch_last()["batched"]
                        if name == "plain":
                            continue
                        for j, (top, total) in enumerate(want):
                            assert n_total[j] == total and n_out[j] == len(top) and np.array_equal(rows[j, :len(top)], top), \
                                (name, n, typos, q, kind, j)
                    t = {"loop": [], "batch": [], "forced": [], "plain": []}
                    for _ in range(args.rounds):
                        for name, fn in (("loop", loop), ("batch", batch), ("forced", forced), ("plain", plain)):
                            t0 = time.perf_counter(); fn(); t[name].append(time.perf_counter() - t0)
                    med = {name: statistics.median(v) * 1e3 for name, v in t.items()}
                    result["rows"].append({"n": n, "max_typos": typos, "q": q, "scope": kind, "loop_ms": round(med["loop"], 3),
                                           "batch_ms": round(med["batch"], 3), "forced_ms": round(med["forced"], 3),
                                           "plain_batch_top_ms": round(med["plain"], 3),
                                           "batch_batched_queries": batched["batch"], "forced_batched_queries": batched["forced"],
                                           "plain_batched_queries": batched["plain"], "checked_equal": True})
                    print(json.dumps(result["rows"][-1]), file=sys.stderr, flush=True)
                    for s in subsets:
                        if s is not None:
                            s.close()
                for m in ms:
                    m.close()
        boost.close()
        corpus.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
