"""Batched collapsed call (frz_match_list_batch_collapsed) against a loop of frz_match_list_collapsed over the same resident
corpus, and against the ungrouped batched call.

  python tools/bench_batch_collapsed.py [--sizes 100000,1000000] [--qs 8,64,512] [--typos 0,1] [--shapes shared,perquery,own]
                                        [--per-group 1,3] [--rounds 3] [--seed 7]

Corpora: synth's flagship shape (needle `deadbeef`, mean length 48, at most 64 bytes) at each size, resident.  Queries: q
needles of 3-12 bytes cut from corpus rows (seeded), max_typos 0 and 1, k = 10.  Group shapes, one per measured row group:
  shared    1 000 groups (random ids), one handle shared by every query;
  perquery  every query its own handle of random ids below 1 000;
  own       every row its own group (n groups), one shared handle.
Each shape runs at per_group 1 and 3, with and without counts.  Four calls alternate over rounds: the loop of
frz_match_list_collapsed ("loop"), the batched call at its default limits ("batch"), the same with the limits lifted
(F.batch_limits: every batch of two or more queries that fits the scratch budget runs the batched kernels, "forced"), and
frz_match_list_batch of the same matchers without groups ("plain", default limits).  Before any is timed, both grouped
batch calls' rows, n_out, n_total and counts are checked equal to the loop's, and the queries each answered on the batched
kernels are recorded.  Host clock around each call (every call ends in a synchronise).  The card name, power limit and
maximum SM clock are read with nvidia-smi in the same run (queries only).  Prints one JSON object."""
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


def handles(corpus, q, shape, rng):
    """(groups per query, the handles to close) for q queries of group shape `shape`."""
    n = len(corpus)
    if shape == "shared":
        g = corpus.groups(rng.integers(0, 1000, n).astype(np.uint32), 1000)
        return [g] * q, [g]
    if shape == "own":
        g = corpus.groups(np.arange(n, dtype=np.uint32), n)
        return [g] * q, [g]
    gs = [corpus.groups(rng.integers(0, 1000, n).astype(np.uint32), 1000) for _ in range(q)]
    return gs, gs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100000,1000000")
    ap.add_argument("--qs", default="8,64,512")
    ap.add_argument("--typos", default="0,1")
    ap.add_argument("--shapes", default="shared,perquery,own")
    ap.add_argument("--per-group", default="1,3")
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
        for typos in [int(x) for x in args.typos.split(",")]:
            for q in [int(x) for x in args.qs.split(",")]:
                ms = [F.Matcher(s, Config(max_typos=typos)) for s in needles(data, off, q, args.seed + q)]
                outs = [np.empty(max(1, min(k, n)), dtype=F.MATCH_DTYPE) for _ in ms]
                for shape in args.shapes.split(","):
                    groups, owned = handles(corpus, q, shape, rng)
                    for pg in [int(x) for x in args.per_group.split(",")]:
                        for counts in (False, True):
                            def loop():
                                return [m.match_list_collapsed_array(corpus, g, k, per_group=pg, counts=counts, out=o)
                                        for m, o, g in zip(ms, outs, groups)]

                            def batch():
                                F.batch_limits()
                                return F.match_list_batch_collapsed(ms, corpus, k, groups, pg, counts=counts)

                            def forced():
                                F.batch_limits(2**64 - 1, 2)
                                r = F.match_list_batch_collapsed(ms, corpus, k, groups, pg, counts=counts)
                                F.batch_limits()
                                return r

                            def plain():
                                F.batch_limits()
                                return F.match_list_batch(ms, corpus, k)

                            want = [tuple(x.copy() if isinstance(x, np.ndarray) else x for x in r) for r in loop()]
                            batched = {}
                            for name, fn in (("batch", batch), ("forced", forced), ("plain", plain)):   # warm-up, and the check
                                res = fn()
                                batched[name] = F.batch_last()["batched"]
                                if name == "plain":
                                    continue
                                rows, n_out, n_total = res[:3]
                                for j, w in enumerate(want):
                                    top, total = w[0], w[1]
                                    assert n_total[j] == total and n_out[j] == len(top) and np.array_equal(rows[j, :len(top)], top), \
                                        (name, n, typos, q, shape, pg, j)
                                    assert not counts or np.array_equal(res[3][j], w[2]), (name, n, typos, q, shape, pg, j)
                            t = {"loop": [], "batch": [], "forced": [], "plain": []}
                            for _ in range(args.rounds):
                                for name, fn in (("loop", loop), ("batch", batch), ("forced", forced), ("plain", plain)):
                                    t0 = time.perf_counter(); fn(); t[name].append(time.perf_counter() - t0)
                            med = {name: statistics.median(v) * 1e3 for name, v in t.items()}
                            result["rows"].append({"n": n, "max_typos": typos, "q": q, "shape": shape, "per_group": pg, "counts": counts,
                                                   "loop_ms": round(med["loop"], 3), "batch_ms": round(med["batch"], 3),
                                                   "forced_ms": round(med["forced"], 3), "plain_batch_ms": round(med["plain"], 3),
                                                   "batch_batched_queries": batched["batch"],
                                                   "forced_batched_queries": batched["forced"],
                                                   "plain_batched_queries": batched["plain"], "checked_equal": True})
                            print(json.dumps(result["rows"][-1]), file=sys.stderr, flush=True)
                    for g in owned:
                        g.close()
                for m in ms:
                    m.close()
        corpus.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
