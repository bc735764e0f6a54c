"""Filling a subset from a text query on the device (frz_subset_match) against the host path it replaces, on a resident
corpus of seeded path-like rows.

  python tools/bench_subset_match.py [--sizes 1000000,10000000] [--steps 20] [--warmup 3] [--k 50] [--out FILE]

The rows are file paths: a top-level directory (src about 50 % of the rows, lib 10 %, docs 1 %, tools 0.1 %, the rest
spread over Zipf-skewed package directories), zero to three Zipf-skewed subdirectories (some named test or tests), and a
file name with an extension (rs about 30 %).  Beside the path corpus C, a directory corpus and a file-name corpus hold
the same rows' two halves, for the form whose text corpus T is not the subset's.  Scopes, with max_typos = 0:
  ^tools/ ^docs/ ^lib/ ^src/   prefix scopes at about 0.1 %, 1 %, 10 % and 50 % of the rows;
  .rs$, src !test, ^src/ .rs$ !test;
  names<-^src/                 the file-name corpus's subset filled from ^src/ over the directory corpus.
For each, the timed configurations are:
  fill        Subset.matching refilling one subset (host clock around the call, which ends in a read-back);
  host        match_list_into_array over T, Corpus.subset of its indices and Subset.close (what a caller does without
              the fill: Smith-Waterman, two PCIe copies and a host pass);
  top@fill / top@host  match_list_subset_top_array(K) of a fuzzy query ("main", max_typos = 1) over either subset.
A second table times `.rs$ !test` refined inside a base (a prefix scope's subset at each density) with the prefilter
reading T's own slot metadata (full) and metadata masked to the base's members (masked, k_subset_meta), and under the
rule the call applies.  Results over the compared subsets are checked equal before timing.  Configurations alternate
step by step, and each timed call follows an untimed call of the same configuration.  A separate torch.profiler pass
records the device time of the prefilter, k_subset_meta, k_subset_fold, k_scan_blocks and k_where_members at the
largest size, set against the bytes they must move.  The card name, power limit and maximum SM clock are read with
nvidia-smi in the same run (queries only).  Prints one JSON object (and writes it to --out when given)."""
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

SCOPES = ["^tools/", "^docs/", "^lib/", "^src/", ".rs$", "src !test", "^src/ .rs$ !test"]
BASES = ["^tools/", "^docs/", "^lib/", "^src/"]
REFINE = ".rs$ !test"


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


def path_rows(n, seed):
    """(paths, directories, file names) of n seeded rows."""
    rng = np.random.default_rng(seed)
    tops = np.array(["src", "lib", "docs", "tools"] + [f"pkg{j}" for j in range(2000)])
    p = np.concatenate([[0.5, 0.1, 0.01, 0.001], 0.389 / np.arange(1, 2001) ** 1.1 / np.sum(1 / np.arange(1, 2001) ** 1.1)])
    top = rng.choice(len(tops), n, p=p / p.sum())
    subs = np.array(["test", "tests", "core", "util", "matcher", "io"] + [f"m{j}" for j in range(5000)])
    depth = rng.integers(0, 4, n)
    sub = np.minimum(rng.zipf(1.4, (n, 3)) - 1, len(subs) - 1)
    exts = np.array(["rs", "py", "toml", "md", "c", "h", "ts", "json"])
    ext = rng.choice(len(exts), n, p=[0.3, 0.2, 0.05, 0.1, 0.1, 0.1, 0.1, 0.05])
    stem = rng.integers(0, 100_000, n)
    dirs, names = [], []
    for i in range(n):
        d = tops[top[i]]
        for j in range(depth[i]):
            d += "/" + subs[sub[i, j]]
        dirs.append(d + "/")
        names.append(f"f{stem[i]}.{exts[ext[i]]}")
    paths = [d + nm for d, nm in zip(dirs, names)]
    return paths, dirs, names


def timed(confs, steps, warmup):
    times = {c: [] for c in confs}
    for _ in range(warmup):
        for fn in confs.values():
            fn()
    for _ in range(steps):   # alternated: drift hits every configuration alike
        for c, fn in confs.items():
            fn()   # untimed: no sample follows another configuration's idle or allocating step
            t0 = time.perf_counter()
            fn()
            times[c].append(time.perf_counter() - t0)
    return {c: summarize(t) for c, t in times.items()}


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
    from frizbee_b200.types import Config

    if not torch.cuda.is_available():
        raise SystemExit("bench_subset_match.py measures on a CUDA device; none is available")
    result = {"card": card_info(0), "k": args.k, "steps": args.steps, "results": [], "refine": []}
    cfg = Config(max_typos=0)
    top_m = F.Matcher("main", Config(max_typos=1))
    sizes = [int(x) for x in args.sizes.split(",")]
    for n in sizes:
        paths, dirs, names = path_rows(n, args.seed)
        corpus, dcol, ncol = F.Corpus.from_list(paths), F.Corpus.from_list(dirs), F.Corpus.from_list(names)
        del paths, dirs, names
        s = corpus.subset([])
        for scope in SCOPES + ["names<-^src/"]:
            other = scope.startswith("names")
            m = F.Matcher.from_query(scope.split("<-")[-1], cfg)
            c, t = (ncol, dcol) if other else (corpus, corpus)
            sub = c.subset([]) if other else s
            sub.matching(m, text=t)
            h = c.subset(m.match_list_into_array(t)["index"])
            assert len(h) == len(sub), (n, scope)
            a, ta = top_m.match_list_subset_top_array(c, sub, args.k)
            b, tb = top_m.match_list_subset_top_array(c, h, args.k)
            assert ta == tb and np.array_equal(a, b), (n, scope, "top")

            def host_path():
                c.subset(m.match_list_into_array(t)["index"]).close()

            confs = {
                "fill": lambda: sub.matching(m, text=t),
                "host": host_path,
                "top@fill": lambda: top_m.match_list_subset_top_array(c, sub, args.k),
                "top@host": lambda: top_m.match_list_subset_top_array(c, h, args.k),
            }
            row = {"n": n, "scope": scope, "members": len(sub), "density": round(len(sub) / n, 6), "matches": int(ta)}
            row.update(timed(confs, args.steps, args.warmup))
            row["fill_speedup"] = round(row["host"]["median_ms"] / row["fill"]["median_ms"], 2)
            result["results"].append(row)
            print(json.dumps({k: row[k] for k in ("n", "scope", "density")} | {cf: row[cf]["median_ms"] for cf in confs}),
                  file=sys.stderr, flush=True)
            h.close()
            if other:
                sub.close()
        refine = F.Matcher.from_query(REFINE, cfg)
        for b_scope in BASES:
            base = corpus.matching(F.Matcher.from_query(b_scope, cfg))
            for force in ("full", "masked"):
                F.subset_match_debug(force)
                s.matching(refine, base=base)
                want = len(s)
                F.subset_match_debug("rule")
                s.matching(refine, base=base)
                assert len(s) == want, (n, b_scope, force)

            def forced(force):
                def run():
                    F.subset_match_debug(force)
                    s.matching(refine, base=base)
                return run

            confs = {"rule": forced("rule"), "full": forced("full"), "masked": forced("masked")}
            row = {"n": n, "base": b_scope, "base_density": round(len(base) / n, 6), "members": len(s)}
            row.update(timed(confs, args.steps, args.warmup))
            F.subset_match_debug("rule")
            s.matching(refine, base=base)
            row["rule_masked_steps"] = F.subset_match_debug()
            result["refine"].append(row)
            print(json.dumps({k: row[k] for k in ("n", "base", "base_density")} | {cf: row[cf]["median_ms"] for cf in confs}),
                  file=sys.stderr, flush=True)
            base.close()
        if n == sizes[-1] and not args.no_profile:
            result["profile"] = profile(F, torch, corpus, s, cfg, n)
        s.close()
        for x in (corpus, dcol, ncol):
            x.close()
    text = json.dumps(result)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


KERNELS = ["k_scan_window", "k_sig_scan", "k_unicode", "k_subset_meta", "k_subset_fold", "k_scan_blocks", "k_where_members"]


def profile(F, torch, corpus, s, cfg, n):
    """Device time per kernel of a fill, against the bytes the bitmap kernels must move (k_subset_fold: n / 8 B per bitmap
    read or written; k_where_members: the bitmap read, 4 B per member written; the prefilter streams 12 B of slot metadata
    and signature per row before it reads any haystack byte)."""
    from torch.profiler import ProfilerActivity, profile as tprof
    out = {}
    reps = 20
    base = corpus.matching(F.Matcher.from_query("^docs/", cfg))
    for label, query, b, force in (("^src/", "^src/", None, "rule"), (".rs$", ".rs$", None, "rule"),
                                   ("^src/ .rs$ !test", "^src/ .rs$ !test", None, "rule"),
                                   (".rs$ !test in ^docs/ (masked)", REFINE, base, "masked"),
                                   (".rs$ !test in ^docs/ (full)", REFINE, base, "full")):
        m = F.Matcher.from_query(query, cfg)
        F.subset_match_debug(force)
        s.matching(m, base=b)
        with tprof(activities=[ProfilerActivity.CUDA]) as p:
            for _ in range(reps):
                s.matching(m, base=b)
            torch.cuda.synchronize()
        F.subset_match_debug("rule")
        kern = {}
        for e in p.key_averages():
            for key in KERNELS:
                if key in e.key:
                    t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                    kern[key] = round(kern.get(key, 0) + t / reps, 2)
        members = len(s)
        steps = len(F.parse_query(query))
        bytes_fold = (n // 8) * (2 + 3 * (steps - 1)) + (n // 8 if b is not None else 0)
        bytes_members = n // 8 + 4 * members
        row = {"members": members, "us_per_fill": kern, "bytes_k_subset_fold": bytes_fold, "bytes_k_where_members": bytes_members}
        if kern.get("k_subset_fold"):
            row["k_subset_fold_GBps"] = round(bytes_fold / (kern["k_subset_fold"] * 1e-6) / 1e9, 1)
        if kern.get("k_where_members"):
            row["k_where_members_GBps"] = round(bytes_members / (kern["k_where_members"] * 1e-6) / 1e9, 1)
        out[label] = row
    base.close()
    return out


if __name__ == "__main__":
    main()
