"""Collapsed match_list against its baselines on the flagship workload (10 M haystacks, needle `deadbeef`, max_typos = 1), on
a resident corpus, results landed in pinned host memory, alternated in one process.

  python tools/bench_collapsed.py [--steps 20] [--warmup 3] [--rounds 3] [--profile-calls 10]

Group shapes (ids per corpus row):
  r1M    1 M random groups (a history with many executions of each command)
  g1000  1 000 random groups
  one    one group holding every row (every atomic of the count and max passes goes to one address)
  own    every row its own group (nothing is dropped, but every row is counted and tested)
Configurations, each timed in every round (rounds alternate them, so drift hits all alike; host clock around each call,
every call ends in a synchronise):
  top50                 frz_match_list_top, K = 50 (ScoreThenIndexAsc)
  ranked50              frz_match_list_ranked, K = 50, boost uniform in 0..255 (a recency prior)
  col_<shape>_<pg>      frz_match_list_collapsed with that boost, K = 50, per_group pg in 1, 3, 32, all (UINT64_MAX)
  plain_<shape>_1       the same without a boost (the score order of frz_match_list_top), per_group 1
  host_<shape>_1        today's workaround: the whole ranked list (frz_match_list_ranked, k = UINT64_MAX) and the collapse on
                        the host in numpy (tests/collapsing.py), cut at 50
  empty_<shape>_1       the empty matcher, ranked and collapsed, per_group 1: the "most recent distinct rows" screen
Every configuration's result is checked in every round against tests/collapsing.py's collapse of the uncollapsed call.
A separate pass under torch.profiler gives the device time per call of every kernel of some of the calls.  The card's
name, power limit and SM clocks are read with nvidia-smi in the same run (queries only).  Prints one JSON object."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

from collapsing import collapse  # noqa: E402

PER_GROUP = {"1": 1, "3": 3, "32": 32, "all": None}


def card_info(device: int) -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(device), f"--query-gpu={q}", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clock, clock_max = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock": clock, "sm_clock_max": clock_max}
    except Exception as e:   # noqa: BLE001 — the numbers are still reported, the card is "unknown"
        return {"name": "unknown", "error": str(e)}


def summarize(samples):
    ms = sorted(1e3 * s for s in samples)
    return {"median_ms": round(statistics.median(ms), 4), "min_ms": round(ms[0], 4),
            "p90_ms": round(ms[min(len(ms) - 1, int(0.9 * len(ms)))], 4), "n": len(ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="timed steps per configuration per round (>= 20)")
    ap.add_argument("--warmup", type=int, default=3, help="untimed steps before each configuration's timed steps (>= 3)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--seed", type=int, default=12345)
    ap.add_argument("--profile-calls", type=int, default=10)
    args = ap.parse_args()
    args.steps, args.warmup = max(args.steps, 20), max(args.warmup, 3)

    import torch
    import frizbee_b200 as F
    from frizbee_b200 import synth
    from frizbee_b200.types import Config, SortStrategy

    if not torch.cuda.is_available():
        raise SystemExit("bench_collapsed.py measures the GPU calls and needs a CUDA device")
    dev = torch.device("cuda", 0)
    n = args.n
    data, off = synth.generate("deadbeef", n, 48, 64, seed=args.seed)
    corpus = F.Corpus.from_arrow(data, off)
    m = F.Matcher("deadbeef", Config(max_typos=1, sort=SortStrategy.ScoreThenIndexAsc))
    empty = F.Matcher.from_query("", Config(sort=SortStrategy.ScoreThenIndexAsc))
    rng = np.random.default_rng(args.seed + 1)
    host_boost = rng.integers(0, 256, n).astype(np.int16)
    boost = corpus.boost(host_boost)
    ids = {"r1M": rng.integers(0, 1_000_000, n).astype(np.uint32), "g1000": rng.integers(0, 1000, n).astype(np.uint32),
           "one": np.zeros(n, np.uint32), "own": np.arange(n, dtype=np.uint32)}
    groups = {s: corpus.groups(v) for s, v in ids.items()}

    def pinned(k):
        return torch.empty(max(k, 1) * F.MATCH_DTYPE.itemsize, dtype=torch.uint8, pin_memory=True).numpy().view(F.MATCH_DTYPE)

    full_buf, top_buf = pinned(n), pinned(50)

    def host_collapse(s):
        rows = m.match_list_ranked_array(corpus, boost, out=full_buf)[0]
        return collapse(rows, ids[s], 1, len(groups[s]))[0][:50]

    runs = {"top50": lambda: m.match_list_top_array(corpus, 50, out=top_buf)[0],
            "ranked50": lambda: m.match_list_ranked_array(corpus, boost, 50, out=top_buf)[0]}
    for s in ids:
        for p, pg in PER_GROUP.items():
            runs[f"col_{s}_{p}"] = (lambda s=s, pg=pg: m.match_list_collapsed_array(corpus, groups[s], 50, per_group=pg, boost=boost,
                                                                                    out=top_buf)[0])
        runs[f"plain_{s}_1"] = lambda s=s: m.match_list_collapsed_array(corpus, groups[s], 50, out=top_buf)[0]
        runs[f"host_{s}_1"] = lambda s=s: host_collapse(s)
    for s in ("r1M", "g1000"):
        runs[f"empty_{s}_1"] = (lambda s=s: empty.match_list_collapsed_array(corpus, groups[s], 50, boost=boost, out=top_buf)[0])

    # the uncollapsed lists L, and each configuration's expected rows
    L = {"ranked": m.match_list_ranked_array(corpus, boost)[0].copy(), "plain": m.match_list_array(corpus).copy(),
         "empty": empty.match_list_ranked_array(corpus, boost)[0].copy()}
    want = {"top50": L["plain"][:50], "ranked50": L["ranked"][:50]}
    for c in runs:
        kind, _, rest = c.partition("_")
        if not rest:
            continue
        s, p = rest.rsplit("_", 1)
        src = {"col": "ranked", "host": "ranked", "plain": "plain", "empty": "empty"}[kind]
        want[c] = collapse(L[src], ids[s], PER_GROUP[p], len(groups[s]))[0][:50]

    def check(c):
        got = np.array(runs[c]())
        w = want[c]
        return len(got) == len(w) and all(np.array_equal(got[f], w[f]) for f in ("index", "score", "exact"))

    configs = list(runs)
    times = {c: [] for c in configs}
    parity = {c: True for c in configs}
    for c in configs:
        for _ in range(args.warmup):
            runs[c]()
    for _ in range(args.rounds):
        for c in configs:
            parity[c] = parity[c] and bool(check(c))
            for _ in range(args.warmup):
                runs[c]()
            torch.cuda.synchronize(dev)
            for _ in range(args.steps):
                t0 = time.perf_counter()
                runs[c]()
                times[c].append(time.perf_counter() - t0)

    # per-kernel device time, in a pass of its own
    from torch.profiler import ProfilerActivity, profile
    kernels = {}
    for c in ("ranked50", "col_r1M_1", "col_r1M_32", "col_one_1", "col_one_32", "col_own_1", "col_r1M_all", "empty_r1M_1"):
        runs[c]()
        torch.cuda.synchronize(dev)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.profile_calls):
                runs[c]()
            torch.cuda.synchronize(dev)
        per = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = getattr(e, "cuda_time_total", 0)
            if t <= 0 or not e.key.strip():
                continue
            per[e.key[:120]] = {"us_per_call": round(t / args.profile_calls, 2),
                                "launches_per_call": round(e.count / args.profile_calls, 2)}
        kernels[c] = dict(sorted(per.items(), key=lambda kv: -kv[1]["us_per_call"]))

    result = {"workload": {"needle": "deadbeef", "haystacks": n, "max_typos": 1, "seed": args.seed, "sort": "ScoreThenIndexAsc",
                           "boost": "uniform 0..255", "k": 50},
              "matches": len(L["plain"]), "kept_per_group_1": {s: len(collapse(L["ranked"], ids[s], 1, len(groups[s]))[0]) for s in ids},
              "steps_per_round": args.steps, "rounds": args.rounds, "warmup": args.warmup,
              "card": card_info(0), "configs": {}, "kernels_per_call": kernels}
    for c in configs:
        result["configs"][c] = dict(summarize(times[c]), parity=parity[c])
    for g in groups.values():
        g.close()
    boost.close()
    m.close()
    empty.close()
    corpus.close()
    print(json.dumps(result, indent=1))
    if not all(parity.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
