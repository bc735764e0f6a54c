"""Batched ordered call (frz_match_list_batch_ordered) against a loop of frz_match_list_ordered /
frz_match_list_ordered_collapsed over the same resident corpus.

  python tools/bench_batch_ordered.py [--sizes 100000,1000000] [--qs 8,64,512] [--typos 0,1] [--orders 0,2]
                                      [--attrs stamp,status] [--groups 0,1000] [--rounds 3] [--seed 7]

Corpora: synth's flagship shape (needle `deadbeef`, mean length 48, at most 64 bytes) at each size, resident.  Queries: q
needles of 3-12 bytes cut from corpus rows (seeded), max_typos 0 and 1, k = 10, every query ordered by one shared
attribute:
  stamp   a uniform timestamp (a permutation of the rows, scaled);
  status  a three-valued exit status (0, 1, 127).
Orders: 0 = ATTR_DESC, 2 = SCORE_THEN_ATTR_DESC.  Groups: 0 = none (frz_match_list_ordered per query), or that many groups
of random ids shared by every query at per_group 1 (frz_match_list_ordered_collapsed).  Three calls alternate over rounds:
the loop of single-query calls ("loop"), the batched call at its default limits ("batch"), and the same with the limits
lifted (F.batch_limits: every batch of two or more queries that fits the scratch budget runs the batched kernels,
"forced").  Before any is timed, both batched calls' rows, n_out and n_total are checked equal to the loop's, and the
queries each answered on the batched kernels, and those whose survivor lists overflowed, are recorded.  Host clock around
each call (every call ends in a synchronise).  The card name, power limit and maximum SM clock are read with nvidia-smi in
the same run (queries only).  Prints one JSON object."""
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
from frizbee_b200.types import Config, Order   # noqa: E402
from tools.bench_batch import card_info, needles   # noqa: E402


def attr_values(kind, n, rng):
    if kind == "stamp":
        return 1_600_000_000_000 + rng.permutation(n).astype(np.int64) * 7
    return rng.choice([0, 1, 127], n).astype(np.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100000,1000000")
    ap.add_argument("--qs", default="8,64,512")
    ap.add_argument("--typos", default="0,1")
    ap.add_argument("--orders", default="0,2")
    ap.add_argument("--attrs", default="stamp,status")
    ap.add_argument("--groups", default="0,1000")
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
        attrs = {kind: corpus.attr(attr_values(kind, n, rng)) for kind in args.attrs.split(",")}
        groups = {int(g): corpus.groups(rng.integers(0, int(g), n).astype(np.uint32), int(g)) if int(g) else None
                  for g in args.groups.split(",")}
        for typos in [int(x) for x in args.typos.split(",")]:
            for q in [int(x) for x in args.qs.split(",")]:
                ms = [F.Matcher(s, Config(max_typos=typos)) for s in needles(data, off, q, args.seed + q)]
                outs = [np.empty(max(1, min(k, n)), dtype=F.MATCH_DTYPE) for _ in ms]
                for kind, attr in attrs.items():
                    for order in [Order(int(x)) for x in args.orders.split(",")]:
                        for n_groups, g in groups.items():
                            gs = [g] * q if g is not None else None

                            def loop():
                                return [m.match_list_ordered_array(corpus, attr, order, k, out=o, groups=g, per_group=1)
                                        for m, o in zip(ms, outs)]

                            def batch():
                                F.batch_limits()
                                return F.match_list_batch_ordered(ms, corpus, k, attr, order, groups=gs)

                            def forced():
                                F.batch_limits(2**64 - 1, 2)
                                r = F.match_list_batch_ordered(ms, corpus, k, attr, order, groups=gs)
                                F.batch_limits()
                                return r

                            want = [(r[0].copy(), r[1]) for r in loop()]
                            last = {}
                            for name, fn in (("batch", batch), ("forced", forced)):   # warm-up, and the check
                                rows, n_out, n_total = fn()
                                last[name] = F.batch_last()
                                for j, (top, total) in enumerate(want):
                                    assert n_total[j] == total and n_out[j] == len(top) and np.array_equal(rows[j, :len(top)], top), \
                                        (name, n, typos, q, kind, order, n_groups, j)
                            t = {"loop": [], "batch": [], "forced": []}
                            for _ in range(args.rounds):
                                for name, fn in (("loop", loop), ("batch", batch), ("forced", forced)):
                                    t0 = time.perf_counter(); fn(); t[name].append(time.perf_counter() - t0)
                            med = {name: statistics.median(v) * 1e3 for name, v in t.items()}
                            result["rows"].append({"n": n, "max_typos": typos, "q": q, "attr": kind, "order": order.name,
                                                   "groups": n_groups, "loop_ms": round(med["loop"], 3),
                                                   "batch_ms": round(med["batch"], 3), "forced_ms": round(med["forced"], 3),
                                                   "batch_batched_queries": last["batch"]["batched"],
                                                   "forced_batched_queries": last["forced"]["batched"],
                                                   "forced_overflowed_queries": last["forced"]["overflowed"], "checked_equal": True})
                            print(json.dumps(result["rows"][-1]), file=sys.stderr, flush=True)
                for m in ms:
                    m.close()
        for a in attrs.values():
            a.close()
        for g in groups.values():
            if g is not None:
                g.close()
        corpus.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
