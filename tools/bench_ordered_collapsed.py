"""Ordered collapsed and ordered column calls against their baselines on the flagship workload (10 M haystacks, needle
`deadbeef`, max_typos = 1, ScoreThenIndexAsc), on a resident corpus, results landed in pinned host memory, alternated in
one process.

  python tools/bench_ordered_collapsed.py [--steps 20] [--warmup 3] [--rounds 3] [--profile-calls 20]

The attribute is `ts`, a uniform timestamp over 30 days.  Group shapes (those of tools/bench_collapsed.py): `g1M`, 1 M
random groups; `g1000`, 1 000 random groups; `one`, every row in one group; `own`, every row its own group.
Configurations, each timed in every round (rounds alternate them; host clock around each call, every call ends in a
synchronise):
  oc50_<g>_p<P>      frz_match_list_ordered_collapsed, ATTR_DESC, K = 50, per_group P in 1, 3, 32 and no cap ("all")
  host50_<g>         what a caller does today: frz_match_list_ordered with the whole list, then tests/collapsing.py's
                     collapse in numpy (per_group 1), first 50 rows
  ordered50          frz_match_list_ordered, ATTR_DESC, K = 50 (no groups)
  collapsed50_<g>    frz_match_list_collapsed, per_group 1, K = 50 (by score)
  screen50_<g>       the empty matcher (all 10 M rows), per_group 1, K = 50: "each group's latest row, newest first", for
                     g1M and g1000
  cols50 / cols50_g1M  frz_match_list_columns_ordered over two columns of 10 M rows (`deadbeef` with one typo over the
                     flagship text, `dead` over a second copy of it), ATTR_DESC, K = 50, without and with the 1 M groups
                     (per_group 1)
  colshost50         the whole two-column list (frz_match_list_columns), then tests/ordering.py's order_by_attr in numpy
Before a configuration is timed its result is checked against the specification (collapse(order_by_attr(...)) over the
GPU's index-ordered list).  A separate pass under torch.profiler gives the device time per call of every kernel and the
launch count per call.  The card's name, power limit and SM clocks are read with nvidia-smi in the same run (queries
only).  Prints one JSON object."""
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
from collapsing import collapse  # noqa: E402
from columns import combine  # noqa: E402
from ordering import order_by_attr  # noqa: E402

PER_GROUP = {"p1": 1, "p3": 3, "p32": 32, "pall": None}


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
        raise SystemExit("bench_ordered_collapsed.py measures the GPU calls and needs a CUDA device")
    dev = torch.device("cuda", 0)
    n = args.n
    data, off = synth.generate("deadbeef", n, 48, 64, seed=args.seed)
    corpus = F.Corpus.from_arrow(data, off)
    second = F.Corpus.from_arrow(data, off)   # the second column: its own resident copy of the text
    sort = SortStrategy.ScoreThenIndexAsc
    m = F.Matcher("deadbeef", Config(max_typos=1, sort=sort))
    m2 = F.Matcher("dead", Config(max_typos=0, sort=sort))
    empty = F.Matcher.from_query("", Config(sort=sort))
    rng = np.random.default_rng(args.seed + 1)
    ts = 1_700_000_000 + rng.integers(0, 30 * 86400, n).astype(np.int64)
    attr = corpus.attr(ts)
    shapes = {"g1M": (rng.integers(0, 1_000_000, n).astype(np.uint32), 1_000_000),
              "g1000": (rng.integers(0, 1000, n).astype(np.uint32), 1000),
              "one": (np.zeros(n, np.uint32), 1),
              "own": (np.arange(n, dtype=np.uint32), n)}
    groups = {g: corpus.groups(ids, ng) for g, (ids, ng) in shapes.items()}

    def pinned(k):
        return torch.empty(max(k, 1) * F.MATCH_DTYPE.itemsize, dtype=torch.uint8, pin_memory=True).numpy().view(F.MATCH_DTYPE)

    full_buf, top_buf = pinned(n), pinned(50)
    AD = Order.AttrDesc

    runs, want = {}, {}
    index_order = m.match_list_into_array(corpus).copy()
    L = order_by_attr(index_order, ts, int(AD), False)
    for g, (ids, ng) in shapes.items():
        h = groups[g]
        for p, pg in PER_GROUP.items():
            runs[f"oc50_{g}_{p}"] = (lambda h=h, pg=pg: m.match_list_ordered_array(corpus, attr, AD, 50, groups=h, per_group=pg,
                                                                                    out=top_buf)[0])
            want[f"oc50_{g}_{p}"] = collapse(L, ids, pg, ng)[0][:50]
        runs[f"host50_{g}"] = (lambda ids=ids, ng=ng: collapse(m.match_list_ordered_array(corpus, attr, AD, out=full_buf)[0], ids, 1,
                                                               ng)[0][:50])
        want[f"host50_{g}"] = want[f"oc50_{g}_p1"]
        runs[f"collapsed50_{g}"] = (lambda h=h: m.match_list_collapsed_array(corpus, h, 50, out=top_buf)[0])
        want[f"collapsed50_{g}"] = collapse(index_order[np.argsort(-index_order["score"].astype(np.int64), kind="stable")], ids, 1,
                                            ng)[0][:50]
    runs["ordered50"] = lambda: m.match_list_ordered_array(corpus, attr, AD, 50, out=top_buf)[0]
    want["ordered50"] = L[:50]
    every = empty.match_list_into_array(corpus).copy()
    L_every = order_by_attr(every, ts, int(AD), False)
    for g in ("g1M", "g1000"):
        ids, ng = shapes[g]
        runs[f"screen50_{g}"] = (lambda h=groups[g]: empty.match_list_ordered_array(corpus, attr, AD, 50, groups=h, out=top_buf)[0])
        want[f"screen50_{g}"] = collapse(L_every, ids, 1, ng)[0][:50]
    L_cols = order_by_attr(combine([index_order, m2.match_list_into_array(second).copy()], n), ts, int(AD), False)
    runs["cols50"] = lambda: F.match_list_columns([m, m2], [corpus, second], 50, sort, attr=attr, out=top_buf)[0]
    want["cols50"] = L_cols[:50]
    runs["cols50_g1M"] = lambda: F.match_list_columns([m, m2], [corpus, second], 50, sort, groups=groups["g1M"], attr=attr,
                                                      out=top_buf)[0]
    want["cols50_g1M"] = collapse(L_cols, shapes["g1M"][0], 1, shapes["g1M"][1])[0][:50]
    runs["colshost50"] = lambda: order_by_attr(F.match_list_columns([m, m2], [corpus, second], None, SortStrategy.IndexAsc,
                                                                    out=full_buf)[0], ts, int(AD), False)[:50]
    want["colshost50"] = want["cols50"]

    def check(c):
        got = np.array(runs[c]())
        w = want[c]
        return len(got) == len(w) and all(np.array_equal(got[f], w[f]) for f in ("index", "score", "exact"))

    matcher_of = {c: (empty if c.startswith("screen") else m) for c in runs}
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
                launches[c].append(matcher_of[c].last_timings()["launches"])

    # per-kernel device time and launches per call, in a pass of its own
    from torch.profiler import ProfilerActivity, profile
    kernels = {}
    for c in configs:
        if "host" in c:
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

    result = {"workload": {"needle": "deadbeef", "haystacks": n, "max_typos": 1, "seed": args.seed, "sort": "ScoreThenIndexAsc",
                           "second_column": "dead, max_typos = 0"},
              "matches": len(index_order), "column_matches": len(L_cols), "steps_per_round": args.steps, "rounds": args.rounds,
              "warmup": args.warmup, "card": card_info(0), "configs": {}, "kernels_per_call": kernels}
    for c in configs:
        result["configs"][c] = dict(summarize(times[c]), launches=int(statistics.median(launches[c])), parity=parity[c])
    for h in list(groups.values()) + [attr]:
        h.close()
    for x in (m, m2, empty, corpus, second):
        x.close()
    print(json.dumps(result, indent=1))
    if not all(parity.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
