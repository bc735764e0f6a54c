"""Filling a boost from attribute rules on the device (frz_boost_where: Boost.where; frz_boost_where_batch:
F.boost_where_batch) against evaluating the same rules in numpy and uploading the boost, alone and in front of a ranked
top-k call, on the flagship workload (synthetic `deadbeef` haystacks) on a resident corpus.

  python tools/bench_boost_where.py [--sizes 1000000,10000000] [--batch-sizes 100000,1000000] [--queries 8,64]
                                    [--steps 20] [--warmup 3] [--k 50] [--out FILE]

Attributes as in bench_where.py: a timestamp, a Zipf directory id, and a pin flag (1 % pinned, 2 % null).  Rule sets:
  one       the last day +20;
  ladder4   a recency ladder over the timestamp: last hour +30, day +20, week +10, month +5;
  eight3    the ladder, the caller's directory +15, two other directories +5, pinned +50 and not pinned -5
            (8 rules over 3 attributes);
each without a base and with a frecency base.  The timed configurations, per (rows, rule set, base):
  fill          Boost.where (host clock around the call, which ends in its read-back of the key bound);
  host_set      the rules in numpy, then Boost.set of every row;
  host_create   the rules in numpy, then a fresh Corpus.boost (closed again);
  *_rank        the same, then match_list_ranked_array top-k.
Batched fills: for q queries on each --batch-sizes corpus, each query with its own `now` and directory, one
F.boost_where_batch against a loop of Boost.where.  Before timing, the values and the ranked top-k of each
configuration are checked equal.  Configurations alternate step by step.  A separate torch.profiler pass gives
k_boost_where's device time against the bytes it must move: 8 B per row and distinct attribute, and per row and query
2 B written and 2 B of base read.  The card name, power limit and maximum SM clock are read with nvidia-smi in the same
run.  Prints one JSON object (and writes it to --out when given)."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

from bench_where import TS_SPAN, card_info, summarize  # noqa: E402

NOW = TS_SPAN
MONTH = TS_SPAN // 12
WEEK, DAY, HOUR = MONTH // 4, MONTH // 30, MONTH // 720
HBM_BPS = 3.35e12   # H100 SXM data sheet


def columns(n, rng):
    ts = rng.integers(0, TS_SPAN, n).astype(np.int64)
    dirs = (np.minimum(rng.zipf(1.2, n), 10_000) - 1).astype(np.int64)
    pin = (rng.random(n) < 0.01).astype(np.int64)
    pin[rng.random(n) < 0.02] = np.iinfo(np.int64).min
    return ts, dirs, pin


def rule_set(name, attrs, cols, now=NOW, here=0):
    """(rules, numpy evaluation of their sum, distinct attributes) of one rule set."""
    a_ts, a_dir, a_pin = attrs
    ts, dirs, pin = cols
    ladder = [(HOUR, 30), (DAY, 20), (WEEK, 10), (MONTH, 5)]
    if name == "one":
        spec = [(a_ts.between(now - DAY, now), lambda: (ts >= now - DAY) & (ts <= now), 20)]
    else:
        spec = [(a_ts.between(now - w, now), lambda w=w: (ts >= now - w) & (ts <= now), add) for w, add in ladder]
    if name == "eight3":
        null = np.iinfo(np.int64).min
        spec += [(a_dir.isin([here]), lambda: dirs == here, 15),
                 (a_dir.isin([here + 1, here + 2]), lambda: np.isin(dirs, [here + 1, here + 2]), 5),
                 (a_pin.isin([1]), lambda: pin == 1, 50),
                 (~a_pin.isin([1]), lambda: (pin != 1) & (pin != null), -5)]

    def host(base):
        acc = base.astype(np.int32) if base is not None else np.zeros(len(ts), np.int32)
        for _, pred, add in spec:
            acc += np.where(pred(), np.int32(add), np.int32(0))
        return np.clip(acc, -32768, 32767).astype(np.int16)

    return [w.add(add) for w, _, add in spec], host, (1 if name != "eight3" else 3)


def run_alternating(confs, steps, warmup):
    samples = {k: [] for k in confs}
    for _ in range(warmup):
        for f in confs.values():
            f()
    for _ in range(steps):
        for k, f in confs.items():
            t0 = time.perf_counter()
            f()
            samples[k].append(time.perf_counter() - t0)
    return {k: summarize(v) for k, v in samples.items()}


def kernel_us(torch, call, reps=20):
    from torch.profiler import ProfilerActivity, profile as tprof
    call()
    with tprof(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    for e in p.key_averages():
        if "k_boost_where" in e.key:
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            return t / max(1, e.count)
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,10000000")
    ap.add_argument("--batch-sizes", default="100000,1000000")
    ap.add_argument("--queries", default="8,64")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--k", type=int, default=50)
    ap.add_argument("--seed", type=int, default=12345)
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    import torch
    import frizbee_b200 as F
    from frizbee_b200 import synth
    from frizbee_b200.types import Config

    if not torch.cuda.is_available():
        raise SystemExit("bench_boost_where.py measures on a CUDA device; none is available")
    result = {"card": card_info(0), "k": args.k, "steps": args.steps, "single": [], "batch": [], "profile": []}
    m = F.Matcher("deadbeef", Config(max_typos=1))
    sizes = sorted({int(x) for x in args.sizes.split(",")} | {int(x) for x in args.batch_sizes.split(",")})
    for n in sizes:
        rng = np.random.default_rng(args.seed)
        data, off = synth.generate("deadbeef", n, 24, 64, args.seed)
        corpus = F.Corpus.from_arrow(data, off)
        del data, off
        cols = columns(n, rng)
        attrs = [corpus.attr(c) for c in cols]
        frec_host = rng.integers(0, 200, n).astype(np.int16)
        frec = corpus.boost(frec_host)
        b, hb = corpus.boost(), corpus.boost()
        all_rows = np.arange(n, dtype=np.uint32)
        if str(n) in args.sizes.split(","):
            for name in ("one", "ladder4", "eight3"):
                rules, host, n_attrs = rule_set(name, attrs, cols)
                for with_base in (False, True):
                    base, base_host = (frec, frec_host) if with_base else (None, None)
                    want = host(base_host)
                    assert np.array_equal(b.where(*rules, base=base).values(), want), (n, name, with_base)
                    hb.set(all_rows, want)
                    x, tx = m.match_list_ranked_array(corpus, b, args.k)
                    y, ty = m.match_list_ranked_array(corpus, hb, args.k)
                    assert tx == ty and np.array_equal(x, y), (n, name, with_base)

                    def fresh():
                        corpus.boost(host(base_host)).close()

                    def fresh_rank():
                        t = corpus.boost(host(base_host))
                        m.match_list_ranked_array(corpus, t, args.k)
                        t.close()

                    confs = {
                        "fill": lambda: b.where(*rules, base=base),
                        "host_set": lambda: hb.set(all_rows, host(base_host)),
                        "host_create": fresh,
                        "fill_rank": lambda: (b.where(*rules, base=base), m.match_list_ranked_array(corpus, b, args.k)),
                        "host_set_rank": lambda: (hb.set(all_rows, host(base_host)), m.match_list_ranked_array(corpus, hb, args.k)),
                        "host_create_rank": fresh_rank,
                    }
                    row = {"rows": n, "rules": name, "base": with_base, "ms": run_alternating(confs, args.steps, args.warmup)}
                    ms = row["ms"]
                    best_host = min(ms["host_set"]["median_ms"], ms["host_create"]["median_ms"])
                    row["host_over_fill"] = round(best_host / ms["fill"]["median_ms"], 2)
                    result["single"].append(row)
                    print(json.dumps(row), file=sys.stderr)
                    if not args.no_profile:
                        us = kernel_us(torch, lambda: b.where(*rules, base=base))
                        by = n * (8 * n_attrs + 2 + (2 if with_base else 0))
                        prow = {"rows": n, "rules": name, "base": with_base, "q": 1, "k_boost_where_us": us and round(us, 2),
                                "bytes": by}
                        if us:
                            prow["GBps"] = round(by / (us * 1e-6) / 1e9, 1)
                            prow["share_of_hbm"] = round(by / (us * 1e-6) / HBM_BPS, 3)
                        result["profile"].append(prow)
        if str(n) in args.batch_sizes.split(","):
            for q in (int(x) for x in args.queries.split(",")):
                boosts = [corpus.boost() for _ in range(q)]
                twins = [corpus.boost() for _ in range(q)]
                sets = [rule_set(("one", "ladder4", "eight3")[j % 3], attrs, cols, NOW - j * HOUR, here=j % 50) for j in range(q)]
                rules = [s[0] for s in sets]
                bases = [frec if j % 2 else None for j in range(q)]
                F.boost_where_batch(boosts, rules, bases)
                for t, r, bs in zip(twins, rules, bases):
                    t.where(*r, base=bs)
                for j in range(q):
                    assert np.array_equal(boosts[j].values(), twins[j].values()), (n, q, j)
                    assert np.array_equal(boosts[j].values(), sets[j][1](frec_host if j % 2 else None)), (n, q, j)

                def loop():
                    for t, r, bs in zip(twins, rules, bases):
                        t.where(*r, base=bs)

                confs = {"loop": loop, "batch": lambda: F.boost_where_batch(boosts, rules, bases)}
                row = {"rows": n, "q": q, "ms": run_alternating(confs, args.steps, args.warmup)}
                row["loop_over_batch"] = round(row["ms"]["loop"]["median_ms"] / row["ms"]["batch"]["median_ms"], 2)
                result["batch"].append(row)
                print(json.dumps(row), file=sys.stderr)
                if not args.no_profile:
                    us = kernel_us(torch, lambda: F.boost_where_batch(boosts, rules, bases))
                    by = n * (8 * 3 + q * 2 + (q // 2) * 2)
                    prow = {"rows": n, "q": q, "k_boost_where_us": us and round(us, 2), "bytes": by}
                    if us:
                        prow["GBps"] = round(by / (us * 1e-6) / 1e9, 1)
                        prow["share_of_hbm"] = round(by / (us * 1e-6) / HBM_BPS, 3)
                    result["profile"].append(prow)
                for h in boosts + twins:
                    h.close()
        for h in attrs + [frec, b, hb]:
            h.close()
        corpus.close()
    m.close()
    result["card_after"] = card_info(0)
    out = json.dumps(result)
    print(out)
    if args.out:
        with open(args.out, "w") as f:
            f.write(out + "\n")


if __name__ == "__main__":
    main()
