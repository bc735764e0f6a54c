"""Ranked match_list against its baselines on the flagship workload (10 M haystacks, needle `deadbeef`, max_typos = 1), on
a resident corpus, results landed in pinned host memory, alternated in one process.

  python tools/bench_ranked.py [--steps 20] [--warmup 3] [--rounds 3] [--profile-calls 20]

Configurations, each timed in every round (rounds alternate them, so drift hits all alike; host clock around each call,
every call ends in a synchronise):
  full              frz_match_list (ScoreThenIndexAsc)
  top50             frz_match_list_top, K = 50
  ranked50_b255     frz_match_list_ranked, K = 50, boost uniform in 0..255 (key bound below 1024: one sort pass)
  rankedall_b255    the same, the whole list
  ranked50_pm1000   K = 50, boost uniform in -1000..1000 (key bound >= 1024: two passes)
  rankedall_pm1000  the same, the whole list
  rerank_b255       frz_match_list, then the caller's re-rank on the host in numpy (keys, a partition, a sort of the
                    first 50 rows)
  rerank_pm1000     the same with the other boost
Before a configuration is timed its result is checked against tests/ranking.py's rank_by_boost applied to the GPU's
index-ordered list.  A separate pass under torch.profiler gives the device time per call of every kernel of the ranked
and top-K calls.  The card's name, power limit and SM clocks are read with nvidia-smi in the same run (queries only).
Prints one JSON object."""
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

from ranking import rank_by_boost  # noqa: E402


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
    ap.add_argument("--profile-calls", type=int, default=20)
    ap.add_argument("--trace-dir", default="", help="write the profiler pass's trace here (optional)")
    args = ap.parse_args()
    args.steps, args.warmup = max(args.steps, 20), max(args.warmup, 3)

    import torch
    import frizbee_b200 as F
    from frizbee_b200 import synth
    from frizbee_b200.types import Config, SortStrategy

    if not torch.cuda.is_available():
        raise SystemExit("bench_ranked.py measures the GPU calls and needs a CUDA device")
    dev = torch.device("cuda", 0)
    data, off = synth.generate("deadbeef", args.n, 48, 64, seed=args.seed)
    corpus = F.Corpus.from_arrow(data, off)
    m = F.Matcher("deadbeef", Config(max_typos=1, sort=SortStrategy.ScoreThenIndexAsc))
    rng = np.random.default_rng(args.seed + 1)
    host_boost = {"b255": rng.integers(0, 256, args.n).astype(np.int16),
                  "pm1000": rng.integers(-1000, 1001, args.n).astype(np.int16)}
    boost = {k: corpus.boost(v) for k, v in host_boost.items()}
    key_bound = {k: min(65535, m.score_bound() + max(0, int(v.max()))) for k, v in host_boost.items()}

    def pinned(n):
        return torch.empty(max(n, 1) * F.MATCH_DTYPE.itemsize, dtype=torch.uint8, pin_memory=True).numpy().view(F.MATCH_DTYPE)

    full_buf, top_buf = pinned(args.n), pinned(50)

    def rerank(rows, b, k):
        """The caller-side re-rank of match_list's output: one int64 per row, (65535 - key) << 32 | index, whose ascending
        order is descending key with ties in index order; a partition picks the first k, and only those are sorted."""
        idx = rows["index"]
        key = np.clip(rows["score"].astype(np.int32) + b[idx], 0, 65535)
        comp = ((65535 - key).astype(np.int64) << 32) | idx.astype(np.int64)
        part = np.argpartition(comp, k)[:k] if len(comp) > k else np.arange(len(comp))
        return rows[part[np.argsort(comp[part])]]

    runs = {
        "full": lambda: m.match_list_array(corpus, out=full_buf),
        "top50": lambda: m.match_list_top_array(corpus, 50, out=top_buf)[0],
    }
    for b in boost:
        runs[f"ranked50_{b}"] = (lambda b=b: m.match_list_ranked_array(corpus, boost[b], 50, out=top_buf)[0])
        runs[f"rankedall_{b}"] = (lambda b=b: m.match_list_ranked_array(corpus, boost[b], out=full_buf)[0])
        runs[f"rerank_{b}"] = (lambda b=b: rerank(m.match_list_array(corpus, out=full_buf), host_boost[b], 50))

    index_order = m.match_list_into_array(corpus).copy()
    want = {b: rank_by_boost(index_order, host_boost[b], False) for b in boost}
    full_want = m.match_list_array(corpus).copy()

    def check(c):
        got = np.array(runs[c]())
        if c == "full":
            return np.array_equal(got, full_want)
        if c == "top50":
            return np.array_equal(got, full_want[:50])
        b = c.split("_")[1]
        w = want[b] if c.startswith("rankedall") else want[b][:50]
        return len(got) == len(w) and all(np.array_equal(got[f], w[f]) for f in ("index", "score", "exact"))

    configs = list(runs)
    times = {c: [] for c in configs}
    stage = {c: [] for c in configs}
    parity = {c: True for c in configs}
    for _ in range(args.warmup):
        for c in configs:
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
                t = m.last_timings()
                stage[c].append({k: t[k] for k in ("prefilter_ms", "sw_ms", "sort_ms", "total_ms")})

    # per-kernel device time, in a pass of its own
    from torch.profiler import ProfilerActivity, profile
    kernels = {}
    for c in ("top50", "ranked50_b255", "ranked50_pm1000", "rankedall_b255", "rankedall_pm1000"):
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
            per[e.key[:120]] = {"us_per_call": round(t / args.profile_calls, 2), "launches_per_call": round(e.count / args.profile_calls, 2)}
        kernels[c] = dict(sorted(per.items(), key=lambda kv: -kv[1]["us_per_call"]))
        if args.trace_dir:
            os.makedirs(args.trace_dir, exist_ok=True)
            prof.export_chrome_trace(os.path.join(args.trace_dir, f"{c}.pt.trace.json"))

    result = {"workload": {"needle": "deadbeef", "haystacks": args.n, "max_typos": 1, "seed": args.seed,
                           "sort": "ScoreThenIndexAsc"},
              "matches": len(index_order), "score_bound": m.score_bound(),
              "key_bound": key_bound, "steps_per_round": args.steps, "rounds": args.rounds, "warmup": args.warmup,
              "card": card_info(0), "configs": {}, "kernels_per_call": kernels}
    for c in configs:
        st = {k: round(statistics.median(s[k] for s in stage[c]), 4) for k in stage[c][0]}
        result["configs"][c] = dict(summarize(times[c]), stages_median_ms=st, parity=parity[c])
    for b in boost.values():
        b.close()
    m.close()
    corpus.close()
    print(json.dumps(result, indent=1))
    if not all(parity.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
