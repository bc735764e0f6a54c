"""Batched column calls (frz_match_list_batch_columns) against a loop of frz_match_list_columns over the same two columns.

  python tools/bench_batch_columns.py [--sizes 100000,1000000] [--qs 8,64,512] [--typos 0,1] [--rounds 3] [--seed 7]

Columns: a file-name-like column (synth's flagship shape: mean length 48, at most 64 bytes) and a directory-like column
(seeded paths of 1-5 components), both resident, of the same length.  Queries: q pairs of needles cut from the rows of
each column (3-10 bytes for the name, 2-6 for the directory), both at the given max_typos, ScoreThenIndexAsc, k = 10.  For
every (size, typos, q) three calls alternate over rounds: the loop, the batch call with its default limits ("batch"), and
the batch call with the limits lifted (F.batch_limits: every batch of two or more batched-class queries that fits the
scratch budget runs the batched kernels, "forced") — the evidence for the default limits.  Before any is timed, each batch
call's rows, n_out and n_total are checked equal to the loop's, and the queries each answered on the batched kernels are
recorded.  Host clock around each call (both end in a synchronise).  The card name, power limit and maximum SM clock are
read with nvidia-smi in the same run (queries only).  Prints one JSON object."""
import argparse
import json
import os
import random
import statistics
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import frizbee_b200 as F   # noqa: E402
from bench_batch import card_info   # noqa: E402
from frizbee_b200 import synth   # noqa: E402
from frizbee_b200.types import Config, SortStrategy   # noqa: E402

PARTS = ["src", "lib", "include", "tests", "docs", "build", "matcher", "prefilter", "core", "utils", "net", "io", "gpu",
         "kernels", "third_party", "tools", "examples", "bench"]


def directories(n, seed):
    rng = random.Random(seed)
    return ["/".join(rng.choice(PARTS) for _ in range(rng.randrange(1, 6))) for _ in range(n)]


def cut(rows, rng, lo, hi):
    while True:
        s = rows[rng.randrange(len(rows))]
        m = rng.randrange(lo, hi + 1)
        if len(s) >= m:
            a = rng.randrange(len(s) - m + 1)
            return s[a:a + m]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100000,1000000")
    ap.add_argument("--qs", default="8,64,512")
    ap.add_argument("--typos", default="0,1")
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    k = args.k
    sort = SortStrategy.ScoreThenIndexAsc
    result = {"card": card_info(0), "k": k, "rows": []}
    for n in [int(x) for x in args.sizes.split(",")]:
        data, off = synth.generate("deadbeef", n, 48, 64, seed=args.seed)
        names = [bytes(data[off[i]:off[i + 1]]).decode("utf-8", "replace") for i in range(min(n, 20000))]
        dirs = directories(n, args.seed)
        cols = [F.Corpus.from_arrow(data, off), F.Corpus.from_list(dirs)]
        for typos in [int(x) for x in args.typos.split(",")]:
            for q in [int(x) for x in args.qs.split(",")]:
                rng = random.Random(args.seed + q + typos)
                ms = [[F.Matcher(cut(names, rng, 3, 10), Config(max_typos=typos)), F.Matcher(cut(dirs, rng, 2, 6), Config(max_typos=typos))]
                      for _ in range(q)]
                outs = [np.empty(max(1, min(k, n)), dtype=F.MATCH_DTYPE) for _ in ms]

                def loop():
                    return [F.match_list_columns(mj, cols, k, sort, out=o) for mj, o in zip(ms, outs)]

                def batch():
                    F.batch_limits()
                    return F.match_list_batch_columns(ms, cols, k, sort)

                def forced():
                    F.batch_limits(2**64 - 1, 2)
                    r = F.match_list_batch_columns(ms, cols, k, sort)
                    F.batch_limits()
                    return r

                want = loop()
                batched = {}
                for name, fn in (("batch", batch), ("forced", forced)):   # warm-up, and the check
                    rows, n_out, n_total = fn()
                    last = F.batch_last()
                    batched[name] = last["batched"]
                    batched[name + "_overflowed"] = last["overflowed"]
                    for j, (top, total) in enumerate(want):
                        assert n_total[j] == total and n_out[j] == len(top) and np.array_equal(rows[j, :len(top)], top), (name, n, typos, q, j)
                t = {"loop": [], "batch": [], "forced": []}
                for _ in range(args.rounds):
                    for name, fn in (("loop", loop), ("batch", batch), ("forced", forced)):
                        t0 = time.perf_counter(); fn(); t[name].append(time.perf_counter() - t0)
                med = {name: statistics.median(v) * 1e3 for name, v in t.items()}
                result["rows"].append({"n": n, "max_typos": typos, "q": q, "loop_ms": round(med["loop"], 3),
                                       "batch_ms": round(med["batch"], 3), "forced_ms": round(med["forced"], 3),
                                       "batch_batched_queries": batched["batch"], "forced_batched_queries": batched["forced"],
                                       "forced_overflowed_queries": batched["forced_overflowed"], "checked_equal": True})
                print(json.dumps(result["rows"][-1]), file=sys.stderr, flush=True)
                for mj in ms:
                    for m in mj:
                        m.close()
        for c in cols:
            c.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
