"""Full match_list vs top-K match_list on the flagship workload (10 M haystacks, needle `deadbeef`, max_typos = 1), on a
resident corpus, alternated in one process.

  python tools/bench_top.py [--steps 20] [--warmup 3] [--rounds 3]
  torchrun --nproc-per-node N tools/bench_top.py --gpus N      (the one-rank-per-process form, N GPUs)

One GPU: frz_match_list against frz_match_list_top at every K of --ks.  Under torchrun: frz_match_list_parallel_rank
against frz_match_list_parallel_rank_top, both into the shared pinned host buffer, each rank holding --n haystacks.
Every configuration is timed in every round (rounds alternate the configurations, so drift hits all of them alike):
host clock around each call (every call ends in a synchronise), plus the library's per-stage device timings.  Before
a configuration is timed its result is checked: top == full[:K] and the reported total == len(full).  The card name,
power limit and maximum SM clock are read with nvidia-smi in the same run (queries only).  Prints one JSON object."""
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
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20, help="timed steps per configuration per round (>= 20)")
    ap.add_argument("--warmup", type=int, default=3, help="untimed steps before each configuration's timed steps (>= 3)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--n", type=int, default=10_000_000, help="haystacks (per GPU under torchrun)")
    ap.add_argument("--seed", type=int, default=12345)
    ap.add_argument("--ks", default="10,100,10000,1000000")
    args = ap.parse_args()
    args.steps, args.warmup = max(args.steps, 20), max(args.warmup, 3)
    ks = [int(x) for x in args.ks.split(",")]

    import torch
    import frizbee_b200 as F
    from frizbee_b200 import parallel, synth
    from frizbee_b200.types import Config

    rank, world, local = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus:
        raise SystemExit(f"--gpus {args.gpus} needs a world of that size (torchrun --nproc-per-node {args.gpus}); have {world}")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)

    data, off = synth.generate("deadbeef", args.n, 48, 64, seed=args.seed + rank)
    corpus = F.Corpus.from_arrow(data, off, device=local)
    m = F.Matcher("deadbeef", Config(max_typos=1))
    index_offset = rank * args.n

    def pinned_matches(n):
        return torch.empty(max(n, 1) * F.MATCH_DTYPE.itemsize, dtype=torch.uint8, pin_memory=True).numpy().view(F.MATCH_DTYPE)

    if world == 1:
        full_buf = pinned_matches(args.n)   # pinned host memory, as bench.py's host-out step lands its list
        top_buf = pinned_matches(max(ks))

        def run_full():
            return m.match_list_array(corpus, out=full_buf)

        def run_top(k):
            return m.match_list_top_array(corpus, k, out=top_buf)   # (rows, total)

        def stages():
            t = m.last_timings()
            return {k: t[k] for k in ("prefilter_ms", "sw_ms", "sort_ms", "total_ms")}
        form = "frz_match_list vs frz_match_list_top (one GPU, resident corpus)"
    else:
        comm = parallel.Comm.from_torch_distributed(local)
        out_h = comm.host_alloc_matches(world * args.n)

        def run_full():
            total, _ = comm.match_list_parallel_rank(m, corpus, index_offset, out_h)
            return out_h[:total]

        def run_top(k):
            kept, total, _ = comm.match_list_parallel_rank_top(m, corpus, index_offset, k, out_h)
            return out_h[:kept], total

        def stages():
            t = comm.last_timings(0)
            return {k: t.get(k, 0.0) for k in ("local_ms", "gather_merge_ms", "d2h_ms", "total_ms", "sort_ms")}
        form = f"frz_match_list_parallel_rank vs frz_match_list_parallel_rank_top ({world} GPUs, {args.n} haystacks per GPU)"

    configs = ["full"] + [f"top{k}" for k in ks]
    times = {c: [] for c in configs}
    stage = {c: [] for c in configs}
    parity = {c: True for c in configs}
    total_matches = None
    for _ in range(args.warmup):
        run_full()
    for rnd in range(args.rounds):
        want = np.array(run_full())   # the reference list of this round, outside any timed region
        total_matches = len(want)
        for c in configs:
            k = None if c == "full" else int(c[3:])
            # parity first (same inputs), then warm-up and timed steps
            if k is not None:
                rows, total = run_top(k)
                ok = total == len(want) and len(rows) == min(k, total) and np.array_equal(np.array(rows), want[:k])
                parity[c] = parity[c] and bool(ok)
            for _ in range(args.warmup):
                run_full() if k is None else run_top(k)
            barrier()
            for _ in range(args.steps):
                if world > 1:
                    dist.barrier()
                t0 = time.perf_counter()
                run_full() if k is None else run_top(k)
                times[c].append(time.perf_counter() - t0)
                stage[c].append(stages())
    barrier()
    result = {"form": form, "workload": {"needle": "deadbeef", "haystacks": args.n * world, "max_typos": 1, "seed": args.seed},
              "matches": total_matches, "steps_per_round": args.steps, "rounds": args.rounds, "warmup": args.warmup,
              "card": card_info(local), "configs": {}}
    for c in configs:
        st = {k: round(statistics.median(s[k] for s in stage[c]), 4) for k in stage[c][0]}
        result["configs"][c] = dict(summarize(times[c]), stages_median_ms=st, parity_top_equals_full_prefix=parity[c])
    if world > 1:
        comm.host_free(out_h)
        comm.close()
        dist.destroy_process_group()
    if rank == 0:
        print(json.dumps(result, indent=1))
    if not all(parity.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
