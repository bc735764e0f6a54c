"""Ordered match_list against its baselines on the flagship workload (10 M haystacks, needle `deadbeef`, max_typos = 1),
on a resident corpus, results landed in pinned host memory, alternated in one process.

  python tools/bench_ordered.py [--steps 20] [--warmup 3] [--rounds 3] [--profile-calls 20]

Two attributes: `ts`, a uniform timestamp (high cardinality: the select narrows in its first passes), and `status`, an
exit status of 0, 1 or 127 (tie-heavy: the select narrows only in the score and index digits).  Configurations, each
timed in every round (rounds alternate them, so drift hits all alike; host clock around each call, every call ends in a
synchronise):
  attr50_<a>         frz_match_list_ordered, ATTR_DESC, K = 50
  attrall_<a>        the same, the whole list
  score50_<a>        SCORE_THEN_ATTR_DESC, K = 50
  scoreall_<a>       the same, the whole list
  where50_<a>        ATTR_DESC, K = 50, over a subset filled by Corpus.where (status != 0: about a third of the rows)
  ranked50           frz_match_list_ranked, K = 50 (boost uniform in 0..255): the nearest existing device call
  host50_<a>         frz_match_list, then the caller's ordering on the host in numpy: a host copy of the field gathered by
                     index, np.argpartition for the first 50 and np.lexsort of those (ATTR_DESC)
Before a configuration is timed its result is checked against tests/ordering.py's order_by_attr applied to the GPU's
index-ordered list.  A separate pass under torch.profiler gives the device time per call of every kernel and the launch
count per call.  The card's name, power limit and SM clocks are read with nvidia-smi in the same run (queries only).
Prints one JSON object."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

from bench_ranked import card_info, summarize  # noqa: E402
from ordering import order_by_attr  # noqa: E402
from ranking import rank_by_boost  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="timed steps per configuration per round (>= 20)")
    ap.add_argument("--warmup", type=int, default=3, help="untimed steps before each configuration's timed steps (>= 3)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--seed", type=int, default=12345)
    ap.add_argument("--profile-calls", type=int, default=20)
    args = ap.parse_args()
    args.steps, args.warmup = max(args.steps, 20), max(args.warmup, 3)

    import torch
    import frizbee_b200 as F
    from frizbee_b200 import synth
    from frizbee_b200.types import Config, Order, SortStrategy

    if not torch.cuda.is_available():
        raise SystemExit("bench_ordered.py measures the GPU calls and needs a CUDA device")
    dev = torch.device("cuda", 0)
    data, off = synth.generate("deadbeef", args.n, 48, 64, seed=args.seed)
    corpus = F.Corpus.from_arrow(data, off)
    m = F.Matcher("deadbeef", Config(max_typos=1, sort=SortStrategy.ScoreThenIndexAsc))
    rng = np.random.default_rng(args.seed + 1)
    host = {"ts": 1_700_000_000 + rng.integers(0, 30 * 86400, args.n).astype(np.int64),
            "status": rng.choice(np.array([0, 1, 127], np.int64), args.n, p=[0.7, 0.2, 0.1])}
    attr = {a: corpus.attr(v) for a, v in host.items()}
    bvals = rng.integers(0, 256, args.n).astype(np.int16)
    boost = corpus.boost(bvals)
    failed = corpus.where(~attr["status"].isin([0]))

    def pinned(n):
        return torch.empty(max(n, 1) * F.MATCH_DTYPE.itemsize, dtype=torch.uint8, pin_memory=True).numpy().view(F.MATCH_DTYPE)

    full_buf, top_buf = pinned(args.n), pinned(50)

    def host_order(rows, v, k):
        """The caller-side ordering of match_list's output by its own copy of the field (ATTR_DESC; the field has no
        nulls): the k-th largest value by a partition, then a lexsort by (value desc, score desc, index) of the rows at or
        above it (ties in the field make that more than k rows)."""
        val = v[rows["index"]]
        if len(val) > k:
            keep = np.nonzero(val >= np.partition(val, len(val) - k)[len(val) - k])[0]
        else:
            keep = np.arange(len(val))
        sub = rows[keep]
        return sub[np.lexsort((sub["index"], -sub["score"].astype(np.int64), -val[keep]))][:k]

    runs = {}
    for a in attr:
        runs[f"attr50_{a}"] = (lambda a=a: m.match_list_ordered_array(corpus, attr[a], Order.AttrDesc, 50, out=top_buf)[0])
        runs[f"attrall_{a}"] = (lambda a=a: m.match_list_ordered_array(corpus, attr[a], Order.AttrDesc, out=full_buf)[0])
        runs[f"score50_{a}"] = (lambda a=a: m.match_list_ordered_array(corpus, attr[a], Order.ScoreThenAttrDesc, 50, out=top_buf)[0])
        runs[f"scoreall_{a}"] = (lambda a=a: m.match_list_ordered_array(corpus, attr[a], Order.ScoreThenAttrDesc, out=full_buf)[0])
        runs[f"where50_{a}"] = (lambda a=a: m.match_list_ordered_array(corpus, attr[a], Order.AttrDesc, 50, subset=failed,
                                                                      out=top_buf)[0])
        runs[f"host50_{a}"] = (lambda a=a: host_order(m.match_list_array(corpus, out=full_buf), host[a], 50))
    runs["ranked50"] = lambda: m.match_list_ranked_array(corpus, boost, 50, out=top_buf)[0]

    index_order = m.match_list_into_array(corpus).copy()
    in_failed = index_order[host["status"][index_order["index"]] != 0]
    want = {}
    for a in attr:
        want[f"attr_{a}"] = order_by_attr(index_order, host[a], int(Order.AttrDesc), False)
        want[f"score_{a}"] = order_by_attr(index_order, host[a], int(Order.ScoreThenAttrDesc), False)
        want[f"where_{a}"] = order_by_attr(in_failed, host[a], int(Order.AttrDesc), False)
        want[f"host_{a}"] = want[f"attr_{a}"]
    want["ranked"] = rank_by_boost(index_order, bvals, False)

    def check(c):
        got = np.array(runs[c]())
        kind = c.split("_")[0]
        w = want[kind.replace("50", "").replace("all", "") + c[len(kind):]]
        if "50" in kind:
            w = w[:50]
        return len(got) == len(w) and all(np.array_equal(got[f], w[f]) for f in ("index", "score", "exact"))

    configs = list(runs)
    times = {c: [] for c in configs}
    launches = {c: [] for c in configs}
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
                launches[c].append(m.last_timings()["launches"])

    # per-kernel device time and launches per call, in a pass of its own
    from torch.profiler import ProfilerActivity, profile
    kernels = {}
    for c in configs:
        if c.startswith("host"):
            continue
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

    result = {"workload": {"needle": "deadbeef", "haystacks": args.n, "max_typos": 1, "seed": args.seed,
                           "sort": "ScoreThenIndexAsc"},
              "matches": len(index_order), "where_matches": len(in_failed), "steps_per_round": args.steps,
              "rounds": args.rounds, "warmup": args.warmup, "card": card_info(0), "configs": {}, "kernels_per_call": kernels}
    for c in configs:
        result["configs"][c] = dict(summarize(times[c]), launches=int(statistics.median(launches[c])), parity=parity[c])
    for h in list(attr.values()) + [boost, failed]:
        h.close()
    m.close()
    corpus.close()
    print(json.dumps(result, indent=1))
    if not all(parity.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
