"""Long-needle workload: 1 M haystacks from synth.generate(mu=220, max_len=600), whose lengths are normal(220, 55) clipped
to [1, 600] (1-478 bytes in practice, not a uniform 80-600), with a 100-byte and a 300-byte needle planted fully and
partially, matched at max_typos 0 and 1.  Prints one JSON line per configuration: step time of a resident
match_list call, the library's per-stage times (frz_matcher_last_timings), per-kernel times from torch.profiler
(k_sw_long_thread and k_sw_long among them; FRZ_LIB selects a build variant to compare), the
card and its power limit, and the result of an oracle check on a seeded sample (a mismatch fails the run).

    python tools/bench_long_needle.py [--n 1000000] [--steps 10] [--warmup 2] [--sample 3000]
"""
import argparse
import json
import os
import random
import re
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import frizbee_b200 as F  # noqa: E402
from frizbee_b200 import synth  # noqa: E402
from frizbee_b200.types import Config  # noqa: E402
from oracle import pyoracle as O  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def needle_of(n, seed):
    rng = random.Random(seed)
    words = ["src", "lib", "matcher", "prefilter", "smith", "waterman", "kernel", "warp", "needle", "haystack", "score"]
    s = ""
    while len(s) < n:
        s += rng.choice(words) + rng.choice(["_", "/", "-", ".", " "])
    return s[:n]


def kernel_ms(m, corpus, steps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            m.match_list_array(corpus)
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            hit = re.search(r"\b(k_\w+(?:<[^>]*>)?)", e.name)
            if hit:
                tot[hit.group(1)] = tot.get(hit.group(1), 0.0) + e.device_time / 1000.0
    return {k: v / steps for k, v in tot.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=3000)
    ap.add_argument("--no-profile", action="store_true")
    a = ap.parse_args()
    gpu = card()
    bad = 0
    for nlen in (100, 300):
        needle = needle_of(nlen, nlen)
        data, off = synth.generate(needle, a.n, 220, 600, seed=nlen)
        lens = np.diff(off.astype(np.int64))
        corpus = F.Corpus.from_arrow(data, off)
        rng = np.random.default_rng(nlen)
        pick = np.sort(rng.choice(a.n, size=min(a.sample, a.n), replace=False))
        sample = [bytes(data[off[i]:off[i + 1]]) for i in pick]
        for k in (0, 1):
            cfg = Config(max_typos=k)
            m = F.Matcher(needle, cfg)
            lanes = m.backend_info()["prefilter_lanes"]
            for _ in range(a.warmup):
                res = m.match_list_array(corpus)
            t0 = time.perf_counter()
            for _ in range(a.steps):
                res = m.match_list_array(corpus)
            step_ms = (time.perf_counter() - t0) * 1000 / a.steps
            stages = m.last_timings()
            got = m.match_list_array(sample)
            sd, so = O.pack(sample)
            want = O.match_list_packed([needle], cfg.with_(emulate_lanes=lanes), sd, so)
            ok = len(got) == len(want) and all(np.array_equal(got[f], want[f]) for f in ("index", "score", "exact"))
            bad += not ok
            kern = {} if a.no_profile else kernel_ms(m, corpus, 3)
            print(json.dumps({"needle_bytes": nlen, "max_typos": k, "haystacks": a.n, "min_len": int(lens.min()),
                              "max_len": int(lens.max()), "matches": int(len(res)), "step_ms": round(step_ms, 3),
                              "stage_ms": stages, "kernel_ms": {kk: round(v, 4) for kk, v in kern.items()},
                              "oracle_sample": len(sample), "oracle_ok": bool(ok), "gpu": gpu}), flush=True)
            m.close()
        corpus.close()
    if bad:
        sys.exit(f"{bad} configuration(s) differ from the oracle")


if __name__ == "__main__":
    main()
