"""Filling many subsets from attribute filters in one call (frz_subset_where_batch, F.where_batch) against a loop of
Subset.where, alone and in front of a batched ordered match call, on the flagship workload (synthetic `deadbeef`
haystacks) on a resident corpus.

  python tools/bench_where_batch.py [--sizes 100000,1000000,10000000] [--queries 8,64,512] [--steps 10] [--warmup 2]
                                    [--e2e-max-rows 1000000] [--k 10] [--out FILE]

The corpus has bench_where.py's three attribute columns (timestamp, directory id, exit status).  Query j gets its own
filter in one of bench_where.py's three shapes, in turn: a time window; a time window and exit != 0; a set of 20
directories and a time window.  Every query's window sits at its own place, and covers 0.1 %, 1 % or 10 % of the
timestamps.  The timed configurations, per (rows, queries):
  loop        Subset.where for every query's subset (host clock around the loop; each call ends in a read-back);
  batch       one F.where_batch over the same subsets and filters;
  batch_kernels   (q <= 2) the same with the batched kernels forced (F.where_batch_debug), the other side of the
              call's rule, which runs the loop for one query and for two over more than 2^22 rows;
  e2e_loop / e2e_batch   the fills, then match_list_batch_ordered over those subsets (k, by timestamp, one matcher per
              query), up to --e2e-max-rows rows.
Before timing, each configuration's subsets are checked equal (len and the ordered batch's rows).  Configurations
alternate step by step, and each timed step follows an untimed step of the same configuration.  A separate
torch.profiler pass records the device time of k_where_batch, k_scan_blocks_batch and k_where_members_batch, with the
bytes k_where_batch reads.  The card name, power limit and maximum SM clock are read with nvidia-smi in the same run.
Prints one JSON object (and writes it to --out when given)."""
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

from bench_where import TS_SPAN, card_info, columns, summarize  # noqa: E402

WINDOWS = [0.001, 0.01, 0.1]
STAGED = 4   # kFrzWhereBatchStaged
NEEDLES = ["deadbeef", "dead", "beef", "adbe", "eadb", "deadbe", "dbeef", "deab"]


def filters(F, attrs, cols, q, rng):
    """q (clauses, numpy predicate) pairs, the shapes in turn, each window at its own place."""
    ts, dirs, ex = cols
    a_ts, a_dir, a_ex = attrs
    out = []
    for j in range(q):
        w = WINDOWS[(j // 3) % len(WINDOWS)]
        lo = int(rng.integers(0, int(TS_SPAN * (1 - w)) + 1))
        hi = lo + int(TS_SPAN * w) - 1
        shape = j % 3
        if shape == 0:
            out.append(([a_ts.between(lo, hi)], lambda lo=lo, hi=hi: (ts >= lo) & (ts <= hi)))
        elif shape == 1:
            out.append(([a_ts.between(lo, hi), ~a_ex.isin([0])],
                        lambda lo=lo, hi=hi: (ts >= lo) & (ts <= hi) & (ex != 0) & (ex != F.ATTR_NULL)))
        else:
            pick = np.concatenate([np.arange(5), rng.choice(np.arange(5, 10_000), 15, replace=False)]).astype(np.int64)
            out.append(([a_dir.isin(pick), a_ts.between(lo, hi)],
                        lambda lo=lo, hi=hi, pick=pick: np.isin(dirs, pick) & (ts >= lo) & (ts <= hi)))
    return out


def k_where_batch_bytes(n, q, n_staged, n_sms):
    """What k_where_batch reads: each of its grid rows stages every chunk's values of the staged attributes (8 B per row
    and attribute; launch_where_batch's split of the queries over y), plus the bitmaps it writes (q * n / 8 B)."""
    n_chunks = (n + 1023) // 1024
    ys = min(q, max(1, -(-(n_sms * 4) // n_chunks)))
    per = -(-q // ys)
    ys = -(-q // per)
    return {"read": 8 * n * n_staged * ys, "written": q * ((n + 31) // 32) * 4, "grid_rows": ys}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100000,1000000,10000000")
    ap.add_argument("--queries", default="8,64,512")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--e2e-max-rows", type=int, default=1_000_000)
    ap.add_argument("--seed", type=int, default=12345)
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    import torch
    import frizbee_b200 as F
    from frizbee_b200 import synth
    from frizbee_b200.types import Config, Order

    if not torch.cuda.is_available():
        raise SystemExit("bench_where_batch.py measures on a CUDA device; none is available")
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    result = {"card": card_info(0), "sms": n_sms, "k": args.k, "steps": args.steps, "results": [], "profile": {}}
    sizes = [int(x) for x in args.sizes.split(",")]
    qs = [int(x) for x in args.queries.split(",")]
    for n in sizes:
        rng = np.random.default_rng(args.seed)
        data, off = synth.generate("deadbeef", n, 24, 64, args.seed)
        corpus = F.Corpus.from_arrow(data, off)
        del data, off
        cols = columns(n, rng)
        attrs = [corpus.attr(c) for c in cols]
        for q in qs:
            fl = filters(F, attrs, cols, q, rng)
            clauses = [c for c, _ in fl]
            looped = [corpus.subset([]) for _ in range(q)]
            batched = [corpus.subset([]) for _ in range(q)]
            ms = [F.Matcher(NEEDLES[j % len(NEEDLES)], Config(max_typos=j % 2)) for j in range(q)]

            def loop():
                for s, c in zip(looped, clauses):
                    s.where(*c)

            def batch():
                F.where_batch(batched, clauses)

            def e2e(fill, subs):
                fill()
                return F.match_list_batch_ordered(ms, corpus, args.k, attrs[0], Order.AttrDesc, subsets=subs)

            loop()
            batch()
            for j, (_, pred) in enumerate(fl[: min(q, 16)]):   # the loop itself against numpy, for a few queries
                assert len(looped[j]) == int(pred().sum()), (n, q, j)
            assert [len(s) for s in looped] == [len(s) for s in batched], (n, q)
            def batch_kernels():   # the batched kernels where the call's rule would run the loop
                F.where_batch_debug(True)
                batch()
                F.where_batch_debug(False)

            confs = {"loop": loop, "batch": batch}
            if q <= 2:
                confs["batch_kernels"] = batch_kernels
            if n <= args.e2e_max_rows:
                a, b = e2e(loop, looped), e2e(batch, batched)
                assert all(np.array_equal(x, y) for x, y in zip(a, b)), (n, q, "e2e")
                confs["e2e_loop"] = lambda: e2e(loop, looped)
                confs["e2e_batch"] = lambda: e2e(batch, batched)
            times = {c: [] for c in confs}
            for _ in range(args.warmup):
                for fn in confs.values():
                    fn()
            for _ in range(args.steps):   # alternated: drift hits every configuration alike
                for c, fn in confs.items():
                    fn()   # untimed
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    times[c].append(time.perf_counter() - t0)
            row = {"n": n, "q": q, "members_mean": round(float(np.mean([len(s) for s in batched])), 1)}
            row.update({c: summarize(t) for c, t in times.items()})
            row["fill_speedup"] = round(row["loop"]["median_ms"] / row["batch"]["median_ms"], 2)
            if "e2e_loop" in row:
                row["e2e_speedup"] = round(row["e2e_loop"]["median_ms"] / row["e2e_batch"]["median_ms"], 2)
            result["results"].append(row)
            print(json.dumps({"n": n, "q": q} | {c: row[c]["median_ms"] for c in confs}), file=sys.stderr, flush=True)
            if not args.no_profile and q in (64, qs[-1]):
                result["profile"][f"{n}x{q}"] = profile(torch, batch, n, q, n_sms)
            for s in looped + batched:
                s.close()
        for a in attrs:
            a.close()
        corpus.close()
    text = json.dumps(result)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


def profile(torch, batch, n, q, n_sms):
    """Device time per kernel of the batched fill (its own profiler run), against the bytes k_where_batch moves."""
    from torch.profiler import ProfilerActivity, profile as tprof
    reps = 10
    batch()
    with tprof(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(reps):
            batch()
        torch.cuda.synchronize()
    kern = {}
    for e in p.key_averages():
        for key in ("k_where_members_batch", "k_scan_blocks_batch", "k_where_batch"):
            if key in e.key and not (key == "k_where_batch" and "members" in e.key):
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                kern[key] = round(t / max(1, e.count), 2)
    by = k_where_batch_bytes(n, q, min(3, STAGED), n_sms)
    row = {"us": kern, "bytes_k_where_batch": by}
    if kern.get("k_where_batch"):
        row["k_where_batch_GBps"] = round((by["read"] + by["written"]) / (kern["k_where_batch"] * 1e-6) / 1e9, 1)
    return row


if __name__ == "__main__":
    main()
