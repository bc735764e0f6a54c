"""Batched top-K (frz_match_list_batch_top) against a loop of frz_match_list_top over the same resident corpus.

  python tools/bench_batch.py [--sizes 100000,1000000,10000000] [--qs 1,8,64,512] [--rounds 3] [--seed 7]

Corpora: synth's flagship shape (needle `deadbeef`, mean length 48, at most 64 bytes) at each size, resident.  Queries: q
needles of 3-12 bytes cut from corpus rows (seeded), max_typos 0 and 1, k = 10.  For every (size, typos, q) three calls
alternate over rounds: the loop, the batch call with its default limits ("batch", which batches only where that was measured
faster, DESIGN.md §4.11), and the batch call with the limits lifted (F.batch_limits: every batch of two or more queries that
fits the scratch budget runs the batched kernels, "forced") — the evidence for the default limits.  Before any is timed,
each batch call's rows, n_out and n_total are checked equal to the loop's, and the queries each answered on the batched
kernels are recorded.  Host clock around each call (both end in a synchronise).  The card name, power limit and maximum SM clock are read
with nvidia-smi in the same run (queries only).  Prints one JSON object."""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import frizbee_b200 as F   # noqa: E402
from frizbee_b200 import synth   # noqa: E402
from frizbee_b200.types import Config   # noqa: E402


def card_info(device: int) -> dict:
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(device), f"--query-gpu={q}", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clock}
    except Exception as e:   # noqa: BLE001 — the numbers are still reported, the card is "unknown"
        return {"name": "unknown", "error": str(e)}


def needles(data, off, q, seed):
    rng = random.Random(seed)
    out = []
    while len(out) < q:
        i = rng.randrange(len(off) - 1)
        s = bytes(data[off[i]:off[i + 1]]).decode("utf-8", "replace")
        n = rng.randrange(3, 13)
        if len(s) >= n:
            a = rng.randrange(len(s) - n + 1)
            out.append(s[a:a + n])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100000,1000000,10000000")
    ap.add_argument("--qs", default="1,8,64,512")
    ap.add_argument("--typos", default="0,1")
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--max-rows-x-queries", type=int, default=10_000_000 * 64)
    args = ap.parse_args()
    k = args.k
    result = {"card": card_info(0), "k": k, "rows": []}
    for n in [int(x) for x in args.sizes.split(",")]:
        data, off = synth.generate("deadbeef", n, 48, 64, seed=args.seed)
        corpus = F.Corpus.from_arrow(data, off)
        for typos in [int(x) for x in args.typos.split(",")]:
            for q in [int(x) for x in args.qs.split(",")]:
                if n * q > args.max_rows_x_queries:
                    # every matcher of the loop keeps its own single-query workspace (about 60 bytes per corpus row)
                    result["rows"].append({"n": n, "max_typos": typos, "q": q, "not_measured": "q single-query workspaces exceed the card"})
                    continue
                ms = [F.Matcher(s, Config(max_typos=typos)) for s in needles(data, off, q, args.seed + q)]
                outs = [np.empty(max(1, min(k, n)), dtype=F.MATCH_DTYPE) for _ in ms]

                def loop():
                    return [m.match_list_top_array(corpus, k, out=o) for m, o in zip(ms, outs)]

                def batch():
                    F.batch_limits()
                    return F.match_list_batch_top(ms, corpus, k)

                def forced():
                    F.batch_limits(2**64 - 1, 2)
                    r = F.match_list_batch_top(ms, corpus, k)
                    F.batch_limits()
                    return r

                want = loop()
                batched = {}
                for name, fn in (("batch", batch), ("forced", forced)):   # warm-up, and the check
                    rows, n_out, n_total = fn()
                    batched[name] = F.batch_last()["batched"]
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
                                       "checked_equal": True})
                print(json.dumps(result["rows"][-1]), file=sys.stderr, flush=True)
                for m in ms:
                    m.close()
        corpus.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
