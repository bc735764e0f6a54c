"""Column calls (frz_match_list_columns) against today's host workaround, on a two-column synthetic table of 10 M rows,
resident corpora, results landed in pinned host memory, alternated in one process.

  python tools/bench_columns.py [--steps 20] [--warmup 3] [--rounds 3] [--profile-calls 10]

Columns (frizbee_b200/synth.py, different seeds):
  c0  short names (48 ± 12 bytes), queried with `deadbeef` at max_typos = 1 (the flagship query)
  c1  longer path-like rows (60 ± 15 bytes, lower case, digits and `/_.-`, 10 % starting with `src/`), queried with the
      short fuzzy needle `srcmn` (max_typos = 0), and separately with the literal `^src/` (Matching.Prefix)
Configurations, each timed in every round (rounds alternate them; host clock around each call, every call ends in a
synchronise), all ScoreThenIndexAsc, K = 50:
  cols_<q>       frz_match_list_columns over [c0, c1] with c1 queried by q (fuzzy or prefix)
  ranked_<q>     the same with a boost uniform in 0..255
  grouped_<q>    the same with 1 000 random groups, per_group 1
  swapped_<q>    the same call with the columns in the other order, [c1, c0]
  host_<q>       today's workaround, on index-ordered lists throughout: the full list of c0 (frz_match_list_into), a subset
                 of c1 built from its indices (frz_subset_create), the full subset list of c1 in index order
                 (frz_match_list_subset under IndexAsc), then numpy: find each c1 row in c0's list by binary search on the
                 uint32 index column, sum, stable sort by score, cut at 50.  Its time is also reported split into these
                 four stages.
  top50          a single-column frz_match_list_top on c0, for scale
Every configuration's result is checked in every round against tests/columns.py over the GPU's own per-column
match_list_into lists.  A separate pass under torch.profiler gives the device time per call of every kernel.  The card's
name, power limit and SM clocks are read with nvidia-smi in the same run (queries only).  Prints one JSON object."""
import argparse
import ctypes as C
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

from columns import match_list_columns as spec  # noqa: E402


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
    from frizbee_b200.types import Config, Matching, Pattern, SortStrategy

    if not torch.cuda.is_available():
        raise SystemExit("bench_columns.py measures the GPU calls and needs a CUDA device")
    dev = torch.device("cuda", 0)
    n, K, sort = args.n, 50, SortStrategy.ScoreThenIndexAsc
    d0, o0 = synth.generate("deadbeef", n, 48, 64, seed=args.seed)
    d1, o1 = synth.generate("srcmain", n, 60, 120, seed=args.seed + 1, p_partial=0.2, p_full=0.1,
                            alphabet=b"abcdefghijklmnopqrstuvwxyz0123456789/_.-", prefix_frac=0.1, prefixes=(b"src/", b"src/"))
    c0, c1 = F.Corpus.from_arrow(d0, o0), F.Corpus.from_arrow(d1, o1)
    m0 = F.Matcher("deadbeef", Config(max_typos=1, sort=sort))
    m1 = {"fuzzy": F.Matcher("srcmn", Config(max_typos=0, sort=sort)),
          "prefix": F.Matcher(Pattern("src/", matching=Matching.Prefix), Config(max_typos=0, sort=sort))}
    rng = np.random.default_rng(args.seed + 2)
    values = rng.integers(0, 256, n).astype(np.int16)
    ids = rng.integers(0, 1000, n).astype(np.uint32)
    boost, groups = c0.boost(values), c1.groups(ids, 1000)

    def pinned(k):
        return torch.empty(max(k, 1) * F.MATCH_DTYPE.itemsize, dtype=torch.uint8, pin_memory=True).numpy().view(F.MATCH_DTYPE)

    full0, full1, top_buf = pinned(n), pinned(n), pinned(K)

    # the workaround's c1 matchers list in index order, so that neither list needs a host sort
    m1_index = {"fuzzy": F.Matcher("srcmn", Config(max_typos=0, sort=SortStrategy.IndexAsc)),
                "prefix": F.Matcher(Pattern("src/", matching=Matching.Prefix), Config(max_typos=0, sort=SortStrategy.IndexAsc))}
    stages = {q: {"c0_list_into_ms": [], "c1_subset_create_ms": [], "c1_subset_list_ms": [], "numpy_ms": []} for q in m1}

    def host(q):
        t0 = time.perf_counter()
        cnt = C.c_uint64()
        F._check(F.lib().frz_match_list_into(m0._h, c0._h, 0, full0.ctypes.data, len(full0), C.byref(cnt)))   # index order
        a = full0[: cnt.value]
        t1 = time.perf_counter()
        sub = c1.subset(a["index"])
        t2 = time.perf_counter()
        b = m1_index[q].match_list_subset_array(c1, sub, out=full1)                                             # index order
        sub.close()
        t3 = time.perf_counter()
        # every row of c1's subset list is a member, so a row of c0's list: a binary search finds it there
        ia = np.searchsorted(a["index"], b["index"])
        score = np.minimum(a["score"][ia].astype(np.int32) + b["score"], 65535)
        top = np.argsort(-score, kind="stable")[:K]
        out = np.zeros(len(top), dtype=F.MATCH_DTYPE)
        out["index"], out["score"] = b["index"][top], score[top]
        out["exact"] = a["exact"][ia[top]] | b["exact"][top]
        t4 = time.perf_counter()
        st = stages[q]
        for key, dt in zip(st, (t1 - t0, t2 - t1, t3 - t2, t4 - t3)):
            st[key].append(1e3 * dt)
        return out

    runs = {"top50": lambda: m0.match_list_top_array(c0, K, out=top_buf)[0]}
    for q in m1:
        runs[f"cols_{q}"] = lambda q=q: F.match_list_columns([m0, m1[q]], [c0, c1], K, sort, out=top_buf)[0]
        runs[f"ranked_{q}"] = lambda q=q: F.match_list_columns([m0, m1[q]], [c0, c1], K, sort, boost=boost, out=top_buf)[0]
        runs[f"grouped_{q}"] = lambda q=q: F.match_list_columns([m0, m1[q]], [c0, c1], K, sort, groups=groups, out=top_buf)[0]
        runs[f"swapped_{q}"] = lambda q=q: F.match_list_columns([m1[q], m0], [c1, c0], K, sort, out=top_buf)[0]
        runs[f"host_{q}"] = lambda q=q: host(q)

    L0 = m0.match_list_into_array(c0).copy()
    L1 = {q: m.match_list_into_array(c1).copy() for q, m in m1.items()}
    want = {"top50": L0[np.argsort(-L0["score"].astype(np.int64), kind="stable")][:K]}
    for q in m1:
        lists = [L0, L1[q]]
        base = spec(lists, n, sort)[0]
        want[f"cols_{q}"] = want[f"swapped_{q}"] = want[f"host_{q}"] = base[:K]
        want[f"ranked_{q}"] = spec(lists, n, sort, boost=values)[0][:K]
        want[f"grouped_{q}"] = spec(lists, n, sort, group_of=ids, n_groups=1000)[0][:K]

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
    for c in ("top50", "cols_fuzzy", "swapped_fuzzy", "cols_prefix", "swapped_prefix", "grouped_fuzzy"):
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

    result = {"workload": {"rows": n, "seed": args.seed, "sort": "ScoreThenIndexAsc", "k": K,
                           "c0": "deadbeef, max_typos 1", "c1_fuzzy": "srcmn, max_typos 0", "c1_prefix": "^src/"},
              "matches": {"c0": len(L0), **{f"c1_{q}": len(v) for q, v in L1.items()},
                          **{f"both_{q}": len(spec([L0, L1[q]], n, sort)[0]) for q in m1}},
              "steps_per_round": args.steps, "rounds": args.rounds, "warmup": args.warmup,
              "card": card_info(0), "configs": {}, "kernels_per_call": kernels}
    for c in configs:
        result["configs"][c] = dict(summarize(times[c]), parity=parity[c])
    result["host_stages_median_ms"] = {q: {k: round(statistics.median(v), 4) for k, v in st.items()} for q, st in stages.items()}
    for x in (boost, groups, m0, *m1.values(), *m1_index.values(), c0, c1):
        x.close()
    print(json.dumps(result, indent=1))
    if not all(parity.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
