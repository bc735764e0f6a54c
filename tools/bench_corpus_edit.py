"""In-place corpus edits on the bench list (synth, 10 M haystacks, needle "deadbeef", max_typos 1 — bench.py's workload).
Prints one JSON line per measurement:
  - frz_corpus_remove and frz_corpus_replace of 1, 1 000 and 100 000 random indices (replacements drawn from the same
    generator), wall time of the synchronous call followed by a device synchronise, median of --reps calls on fresh
    index sets; whether a call compacted the arena;
  - a full rebuild with frz_corpus_create_arrow from pinned host memory, for comparison;
  - the resident match step (frz_match_list, host out) on the edited corpus and on a fresh corpus of the edited list
    (removed rows as empty strings), whose lists must be identical once the removed rows are dropped (a mismatch fails
    the run);
  - the device memory of every replace: the library's high-water mark during the call (frz_debug_device_bytes_peak)
    over what it held before; for the first call that compacts the arena also the bytes held before and after it.  That
    call grows the arena (the new tiles go to its end), stages the touched tiles and then compacts, so its peak covers
    all three;
and the card's name and power limit, read in the same run.

    python tools/bench_corpus_edit.py [--n 10000000] [--reps 3] [--steps 20] [--warmup 3]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import frizbee_b200 as F  # noqa: E402
from frizbee_b200 import synth  # noqa: E402
from frizbee_b200.types import Config  # noqa: E402

NEEDLE, MU, MAX_LEN, SEED = "deadbeef", 48, 64, 12345


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def device_bytes():
    L = F.lib()
    L.frz_debug_device_bytes.restype = C.c_uint64
    L.frz_debug_device_bytes.argtypes = []
    return int(L.frz_debug_device_bytes())


def peak_reset():
    """frz_debug_device_bytes_peak: the library's high-water mark since the last call, then reset to what it holds now."""
    L = F.lib()
    L.frz_debug_device_bytes_peak.restype = C.c_uint64
    L.frz_debug_device_bytes_peak.argtypes = [C.c_int]
    peak = int(L.frz_debug_device_bytes_peak(0))
    L.frz_debug_device_bytes_peak(1)
    return peak


class EditedList:
    """The list as the corpus holds it: every index points at bytes in a pool (the original buffer, then every
    replacement buffer); a removed index has length 0 and is flagged."""

    def __init__(self, data, off):
        self.pools = [data]
        self.pool_len = len(data)
        self.start = off[:-1].astype(np.int64)
        self.lens = np.diff(off).astype(np.int64)
        self.removed = np.zeros(len(off) - 1, dtype=bool)

    def remove(self, which):
        self.removed[which] = True
        self.lens[which] = 0

    def replace(self, which, data, off):
        self.start[which] = self.pool_len + off[:-1].astype(np.int64)
        self.lens[which] = np.diff(off).astype(np.int64)
        self.removed[which] = False
        self.pools.append(data)
        self.pool_len += len(data)

    def arrow(self):
        pool = np.concatenate(self.pools)
        off = np.zeros(len(self.lens) + 1, dtype=np.uint64)
        np.cumsum(self.lens, out=off[1:])
        total = int(off[-1])
        src = np.repeat(self.start - off[:-1].astype(np.int64), self.lens) + np.arange(total)
        return pool[src], off


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def match_ms(m, corpus, steps, warmup):
    for _ in range(warmup):
        m.match_list_array(corpus)
    ts = [timed(lambda: m.match_list_array(corpus)) for _ in range(steps)]
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    gpu = card()
    out = lambda d: print(json.dumps({"card": gpu, **d}), flush=True)   # noqa: E731
    data, off = synth.generate(NEEDLE, a.n, MU, MAX_LEN, SEED)
    # pinned copies for the rebuild
    p_data = torch.empty(len(data), dtype=torch.uint8, pin_memory=True).numpy()
    p_off = torch.empty(len(off), dtype=torch.int64, pin_memory=True).numpy().view(np.uint64)
    p_data[:] = data
    p_off[:] = off
    rebuild = []
    for _ in range(a.reps + 1):
        t = timed(lambda: F.Corpus.from_arrow(p_data, p_off).close())
        rebuild.append(t)
    out({"what": "rebuild frz_corpus_create_arrow (pinned)", "n": a.n, "bytes": int(off[-1]),
         "ms_median": float(np.median(rebuild[1:])), "ms_all": rebuild})

    corpus = F.Corpus.from_arrow(p_data, p_off)
    model = EditedList(data, off)
    rng = np.random.default_rng(7)
    m = F.Matcher(NEEDLE, Config(max_typos=1))
    m.match_list_array(corpus)   # warm the matcher's workspace before any edit is timed
    compaction = None
    gen_seed = 100
    for k in (1, 1000, 100_000):
        rem_t, rep_t, compacted, peaks = [], [], [], []
        for r in range(a.reps + 1):   # the first call of each size is a warm-up (small staging buffers grow and are kept)
            which = rng.choice(a.n, k, replace=False).astype(np.uint32)
            t = timed(lambda: corpus.remove(which))
            model.remove(which)
            if r:
                rem_t.append(t)
            which = rng.choice(a.n, k, replace=False).astype(np.uint32)
            gen_seed += 1
            r_data, r_off = synth.generate(NEEDLE, k, MU, MAX_LEN, gen_seed)
            held, arena = device_bytes(), corpus.device_bytes
            peak_reset()
            t = timed(lambda: corpus.replace(which, r_data, r_off))
            peak = peak_reset()   # the high-water mark of the call (reset to the current value for the next one)
            model.replace(which, r_data, r_off)
            shrunk = corpus.device_bytes < arena
            if shrunk and compaction is None:
                compaction = {"what": "compacting replace", "replace_k": k, "call_ms": t, "held_before": held,
                              "held_after": device_bytes(), "peak_bytes_measured": peak, "peak_over_before": peak - held,
                              "corpus_device_bytes_before": arena, "corpus_device_bytes_after": corpus.device_bytes}
            if r:
                rep_t.append(t)
                compacted.append(bool(shrunk))
                peaks.append(peak - held)
        out({"what": "remove", "k": k, "ms_median": float(np.median(rem_t)), "ms_all": rem_t})
        out({"what": "replace", "k": k, "ms_median": float(np.median(rep_t)), "ms_all": rep_t, "compacted": compacted,
             "peak_over_held_before_bytes": peaks})
    out(compaction or {"what": "compacting replace", "note": "no call compacted the arena"})

    # the match step on the edited corpus against a fresh corpus of the edited list
    f_data, f_off = model.arrow()
    fresh = F.Corpus.from_arrow(f_data, f_off)
    got = m.match_list_array(corpus)
    want = m.match_list_array(fresh)
    want = want[~model.removed[want["index"]]]
    same = len(got) == len(want) and all(np.array_equal(got[f], want[f]) for f in ("index", "score", "exact"))
    edited = match_ms(m, corpus, a.steps, a.warmup)
    fresh_t = match_ms(m, fresh, a.steps, a.warmup)
    out({"what": "match step (frz_match_list, host out)", "matches": len(got), "identical": bool(same),
         "removed": int(model.removed.sum()), "edited_ms": edited[0], "edited_min_max": edited[1:],
         "fresh_ms": fresh_t[0], "fresh_min_max": fresh_t[1:]})
    m.close()
    fresh.close()
    corpus.close()
    if not same:
        sys.exit("the edited corpus's matches differ from the fresh corpus's")


if __name__ == "__main__":
    main()
