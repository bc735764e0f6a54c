"""Filling a subset from attribute predicates on the device (frz_subset_where) against the host path it replaces, on the
flagship workload (synthetic `deadbeef` haystacks, max_typos = 1), on a resident corpus.

  python tools/bench_where.py [--sizes 1000000,10000000] [--steps 20] [--warmup 3] [--k 50] [--out FILE]

The corpus has three attribute columns, shaped like a shell history: a timestamp (uniform), a directory id (about 10 000
values, Zipf-skewed) and an exit status (mostly 0, some non-zero, some null).  Three predicates, each at time windows
that cover about 0.01 % to 100 % of the rows:
  time      ts in a window;
  time_exit ts in a window and exit != 0;
  dir_time  directory in a set of 20 ids, and ts in a window.
For each, the timed configurations are:
  where       Subset.where refilling one subset (host clock around the call, which ends in a read-back);
  host        the numpy predicate, np.flatnonzero, Corpus.subset and Subset.close (what a caller does without where);
  top@where / top@host        match_list_subset_top_array(K) over either subset;
  ranked@where / ranked@host  match_list_ranked_array(boost, K) over either subset.
The results over the two subsets are compared before timing and must be equal.  Configurations alternate step by step,
and each timed call follows an untimed call of the same configuration.  A
separate torch.profiler pass records the device time of k_where, k_scan_blocks and k_where_members at the largest size,
set against the bytes they must move.  The card name, power limit and maximum SM clock are read with nvidia-smi in the
same run (queries only).  Prints one JSON object (and writes it to --out when given)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

WINDOWS = [0.0001, 0.001, 0.01, 0.1, 0.5, 1.0]
TS_SPAN = 1_000_000_000


def card_info(device: int) -> dict:
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(device), f"--query-gpu={q}", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clock}
    except Exception as e:   # noqa: BLE001 — the numbers are still reported, the card is "unknown"
        return {"name": "unknown", "error": str(e)}


def summarize(samples):
    ms = sorted(1e3 * s for s in samples)
    return {"median_ms": round(statistics.median(ms), 4), "min_ms": round(ms[0], 4),
            "p90_ms": round(ms[min(len(ms) - 1, int(0.9 * len(ms)))], 4), "n": len(ms)}


def columns(n, rng):
    ts = rng.integers(0, TS_SPAN, n).astype(np.int64)
    dirs = (np.minimum(rng.zipf(1.2, n), 10_000) - 1).astype(np.int64)
    r = rng.random(n)
    ex = np.where(r < 0.88, 0, rng.integers(1, 256, n)).astype(np.int64)
    ex[r > 0.98] = np.iinfo(np.int64).min   # exit status unknown
    return ts, dirs, ex


def predicates(F, attrs, cols, window, rng):
    """name -> (the clauses for Subset.where, the numpy predicate)."""
    ts, dirs, ex = cols
    a_ts, a_dir, a_ex = attrs
    lo = int(rng.integers(0, int(TS_SPAN * (1 - window)) + 1))
    hi = lo + int(TS_SPAN * window) - 1
    pick = np.concatenate([np.arange(5), rng.choice(np.arange(5, 10_000), 15, replace=False)]).astype(np.int64)
    null = F.ATTR_NULL
    return {
        "time": ([a_ts.between(lo, hi)], lambda: (ts >= lo) & (ts <= hi)),
        "time_exit": ([a_ts.between(lo, hi), ~a_ex.isin([0])], lambda: (ts >= lo) & (ts <= hi) & (ex != 0) & (ex != null)),
        "dir_time": ([a_dir.isin(pick), a_ts.between(lo, hi)], lambda: np.isin(dirs, pick) & (ts >= lo) & (ts <= hi)),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,10000000")
    ap.add_argument("--steps", type=int, default=20, help="timed steps per configuration (>= 20)")
    ap.add_argument("--warmup", type=int, default=3, help="untimed steps per configuration (>= 3)")
    ap.add_argument("--k", type=int, default=50)
    ap.add_argument("--seed", type=int, default=12345)
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    args.steps, args.warmup = max(args.steps, 20), max(args.warmup, 3)

    import torch
    import frizbee_b200 as F
    from frizbee_b200 import synth
    from frizbee_b200.types import Config

    if not torch.cuda.is_available():
        raise SystemExit("bench_where.py measures on a CUDA device; none is available")
    result = {"card": card_info(0), "k": args.k, "steps": args.steps, "results": []}
    m = F.Matcher("deadbeef", Config(max_typos=1))
    sizes = [int(x) for x in args.sizes.split(",")]
    for n in sizes:
        rng = np.random.default_rng(args.seed)
        data, off = synth.generate("deadbeef", n, 24, 64, args.seed)
        corpus = F.Corpus.from_arrow(data, off)
        del data, off
        cols = columns(n, rng)
        attrs = [corpus.attr(c) for c in cols]
        boost = corpus.boost(rng.integers(0, 200, n).astype(np.int16))
        s = corpus.subset([])
        for window in WINDOWS:
            for name, (clauses, pred) in predicates(F, attrs, cols, window, rng).items():
                s.where(*clauses)
                h = corpus.subset(np.flatnonzero(pred()))
                assert len(h) == len(s), (n, name, window)
                a, ta = m.match_list_subset_top_array(corpus, s, args.k)
                b, tb = m.match_list_subset_top_array(corpus, h, args.k)
                assert ta == tb and np.array_equal(a, b), (n, name, window, "top")
                a, ta = m.match_list_ranked_array(corpus, boost, args.k, s)
                b, tb = m.match_list_ranked_array(corpus, boost, args.k, h)
                assert ta == tb and np.array_equal(a, b), (n, name, window, "ranked")

                def host_path():
                    corpus.subset(np.flatnonzero(pred())).close()

                confs = {
                    "where": lambda: s.where(*clauses),
                    "host": host_path,
                    "top@where": lambda: m.match_list_subset_top_array(corpus, s, args.k),
                    "top@host": lambda: m.match_list_subset_top_array(corpus, h, args.k),
                    "ranked@where": lambda: m.match_list_ranked_array(corpus, boost, args.k, s),
                    "ranked@host": lambda: m.match_list_ranked_array(corpus, boost, args.k, h),
                }
                times = {c: [] for c in confs}
                for _ in range(args.warmup):
                    for fn in confs.values():
                        fn()
                for _ in range(args.steps):   # alternated: drift hits every configuration alike
                    for c, fn in confs.items():
                        fn()   # untimed: no sample follows another configuration's idle or allocating step
                        t0 = time.perf_counter()
                        fn()
                        times[c].append(time.perf_counter() - t0)
                row = {"n": n, "predicate": name, "window": window, "members": len(s), "density": round(len(s) / n, 6),
                       "matches": int(ta)}
                row.update({c: summarize(t) for c, t in times.items()})
                row["where_speedup"] = round(row["host"]["median_ms"] / row["where"]["median_ms"], 2)
                result["results"].append(row)
                print(json.dumps({k: row[k] for k in ("n", "predicate", "window", "density")} |
                                 {c: row[c]["median_ms"] for c in confs}), file=sys.stderr, flush=True)
                h.close()
        if n == sizes[-1] and not args.no_profile:
            result["profile"] = profile(F, torch, s, attrs, cols, n, rng)
        s.close()
        boost.close()
        for a in attrs:
            a.close()
        corpus.close()
    text = json.dumps(result)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


def profile(F, torch, s, attrs, cols, n, rng):
    """Device time per kernel of the fill, for a sparse and a full one-clause and a two-clause predicate, against the
    bytes the kernels must move (k_where: 8 B per row and clause read, n / 8 B of bitmap written; k_where_members: the
    bitmap read, 4 B per member written)."""
    from torch.profiler import ProfilerActivity, profile as tprof
    out = {}
    reps = 20
    for label, window, pname in (("time@0.01%", 0.0001, "time"), ("time@100%", 1.0, "time"), ("time_exit@10%", 0.1, "time_exit")):
        clauses, _ = predicates(F, attrs, cols, window, rng)[pname]
        s.where(*clauses)
        with tprof(activities=[ProfilerActivity.CUDA]) as p:
            for _ in range(reps):
                s.where(*clauses)
            torch.cuda.synchronize()
        kern = {}
        for e in p.key_averages():
            for key in ("k_where_members", "k_scan_blocks", "k_where"):
                if key in e.key and not (key == "k_where" and "members" in e.key):
                    t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                    kern[key] = round(t / max(1, e.count), 2)
        members = len(s)
        bytes_where = 8 * n * len(clauses) + n // 8
        bytes_members = n // 8 + 4 * members
        row = {"members": members, "us": kern, "bytes_k_where": bytes_where, "bytes_k_where_members": bytes_members}
        if kern.get("k_where"):
            row["k_where_GBps"] = round(bytes_where / (kern["k_where"] * 1e-6) / 1e9, 1)
        if kern.get("k_where_members"):
            row["k_where_members_GBps"] = round(bytes_members / (kern["k_where_members"] * 1e-6) / 1e9, 1)
        out[label] = row
    return out


if __name__ == "__main__":
    main()
