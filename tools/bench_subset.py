"""Subset match calls against the full-list calls on the flagship workload (10 M haystacks, needle `deadbeef`,
max_typos = 1), on a resident corpus, alternated in one process.

  python tools/bench_subset.py [--steps 20] [--warmup 3] [--rounds 3] [--k 50]

Configurations: frz_match_list (`full`), frz_match_list_top (`top`), frz_match_list followed by a numpy filter on the
host (`host_filter@d`: what a caller without subset calls does; it also stands for a filtered top-K, which needs the
whole list first), frz_match_list_subset (`subset[form]@d`) and frz_match_list_subset_top (`subset_top[form]@d`), for
random subsets of densities d, in both forms of a subset call.  The forms are build variants (VARIANTS below, built on
first use) loaded side by side, each holding its own corpus of the same list.  Every configuration is timed in every
round (rounds alternate the configurations, so drift hits all of them alike): host clock around each call (every call
ends in a synchronise).  Before a configuration is timed its result is checked against the full list filtered on the
host.  A separate torch.profiler pass then records the device time per kernel of each form's top-K call at the sparsest
and the densest subset.  The card name, power limit and maximum SM clock are read with nvidia-smi in the same run
(queries only).  Prints one JSON object."""
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

# the two forms of a subset call as build variants (frizbee_b200/build.py --variant NAME --define D)
VARIANTS = {"masked": "FRZ_SUBSET_LIST_PERMILLE=-1", "list": "FRZ_SUBSET_LIST_PERMILLE=1000"}


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="timed steps per configuration per round (>= 20)")
    ap.add_argument("--warmup", type=int, default=3, help="untimed steps before each configuration's timed steps (>= 3)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--seed", type=int, default=12345)
    ap.add_argument("--k", type=int, default=50)
    ap.add_argument("--densities", default="0.0001,0.001,0.01,0.1,0.5,1.0")
    args = ap.parse_args()
    args.steps, args.warmup = max(args.steps, 20), max(args.warmup, 3)
    dens = [float(x) for x in args.densities.split(",")]

    import torch
    import frizbee_b200 as F
    from frizbee_b200 import build, synth
    from frizbee_b200.types import Config

    # one library per form, loaded side by side; every call below first makes its form's library current
    libs = {}
    for v, define in VARIANTS.items():
        path = os.path.join(ROOT, "frizbee_b200", f"libfrz_cuda_{v}.so")
        if not os.path.exists(path):
            build.build(variant=v, defines=[define])
        F._lib = None
        os.environ["FRZ_LIB"] = path
        libs[v] = F.lib()
    os.environ.pop("FRZ_LIB")

    def use(v):
        F._lib = libs[v]

    torch.cuda.set_device(0)
    data, off = synth.generate("deadbeef", args.n, 48, 64, seed=args.seed)
    k = args.k
    rng = np.random.default_rng(args.seed + 1)
    perm = rng.permutation(args.n)
    which = {d: np.sort(perm[: max(1, int(round(d * args.n)))]).astype(np.uint32) for d in dens}
    masks = {}
    for d in dens:
        masks[d] = np.zeros(args.n, dtype=bool)
        masks[d][which[d]] = True
    corpus, m, subs = {}, {}, {}
    for v in VARIANTS:   # each form's library holds its own corpus of the same list
        use(v)
        corpus[v] = F.Corpus.from_arrow(data, off)
        m[v] = F.Matcher("deadbeef", Config(max_typos=1))
        subs[v] = {d: corpus[v].subset(which[d]) for d in dens}

    def pinned_matches(n):
        return torch.empty(max(n, 1) * F.MATCH_DTYPE.itemsize, dtype=torch.uint8, pin_memory=True).numpy().view(F.MATCH_DTYPE)

    full_buf = pinned_matches(args.n)   # pinned host memory, as bench.py's host-out step lands its list
    base = "masked"                     # the full-list calls are the same code in every form's library

    def run_full():
        use(base)
        return m[base].match_list_array(corpus[base], out=full_buf)

    def run_top():
        use(base)
        return m[base].match_list_top_array(corpus[base], k)[0]

    def run_host_filter(d):
        full = run_full()
        return full[masks[d][full["index"]]]

    def run_subset(v, d):
        use(v)
        return m[v].match_list_subset_array(corpus[v], subs[v][d], out=full_buf)

    def run_subset_top(v, d):
        use(v)
        return m[v].match_list_subset_top_array(corpus[v], subs[v][d], k)[0]

    configs = {"full": run_full, f"top{k}": run_top}
    for d in dens:
        configs[f"host_filter@{d:g}"] = lambda d=d: run_host_filter(d)
        for v in VARIANTS:
            configs[f"subset[{v}]@{d:g}"] = lambda d=d, v=v: run_subset(v, d)
            configs[f"subset_top{k}[{v}]@{d:g}"] = lambda d=d, v=v: run_subset_top(v, d)
    times = {c: [] for c in configs}
    parity = {c: True for c in configs}
    for _ in range(args.warmup):
        run_full()
    want_full = np.array(run_full())
    for rnd in range(args.rounds):
        for c, fn in configs.items():
            got = np.array(fn())   # parity first (same inputs), then warm-up and timed steps
            if c == "full":
                want = want_full
            elif c.startswith("top"):
                want = want_full[:k]
            else:
                d = float(c.split("@")[1])
                want = want_full[masks[d][want_full["index"]]]
                if c.startswith("subset_top"):
                    want = want[:k]
            parity[c] = parity[c] and len(got) == len(want) and bool(np.array_equal(got, want))
            for _ in range(args.warmup):
                fn()
            torch.cuda.synchronize()
            for _ in range(args.steps):
                t0 = time.perf_counter()
                fn()
                times[c].append(time.perf_counter() - t0)

    # per-kernel device time of a top-K subset call, from a profiler pass of its own: each form at the sparsest and the
    # densest subset (us per call, kernels over 1 us)
    from torch.profiler import ProfilerActivity, profile
    kernels = {}
    for v in VARIANTS:
        for d in (dens[0], dens[-1]):
            for _ in range(args.warmup):
                run_subset_top(v, d)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    run_subset_top(v, d)
                torch.cuda.synchronize()
            row = {}
            for e in prof.key_averages():
                us = (getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)) / args.steps
                if us >= 1.0:
                    row[e.key[:90]] = round(us, 2)
            kernels[f"{v}@{d:g}"] = dict(sorted(row.items(), key=lambda kv: -kv[1]))

    slots = -(-args.n // 1024) * 1024
    result = {"form": "frz_match_list_subset / _subset_top vs frz_match_list, _top and a host filter (one GPU, resident corpus)",
              "workload": {"needle": "deadbeef", "haystacks": args.n, "max_typos": 1, "seed": args.seed, "k": k},
              "matches_full": len(want_full), "steps_per_round": args.steps, "rounds": args.rounds, "warmup": args.warmup,
              "card": card_info(0),
              "variants": VARIANTS, "mask_bytes_per_call": 2 * 4 * slots,
              "kernels_us_per_call": kernels, "members": {f"{d:g}": len(which[d]) for d in dens}, "configs": {}}
    for c in configs:
        result["configs"][c] = dict(summarize(times[c]), parity=parity[c])
    for v in VARIANTS:
        use(v)
        for sub in subs[v].values():
            sub.close()
        m[v].close()
        corpus[v].close()
    print(json.dumps(result, indent=1))
    if not all(parity.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
