"""torchrun worker (one rank per GPU) for the top-K form of match_list_parallel: every rank runs
frz_match_list_parallel_rank_top on its shard, and rank 0 checks that the first min(K, total) rows in the shared host
buffer equal the full parallel call's first rows — for every sort strategy, K at the slice seams, a match-everything
query, empty shards and a multi-pattern query.  The device-only form is checked against the host result on every rank."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np
import torch
import torch.distributed as dist

import frizbee_b200 as F
from frizbee_b200 import parallel, synth
from frizbee_b200.types import Config, SortStrategy


def run_case(comm, rank, world, local, make_matcher, data, off, label):
    n = len(off) - 1
    lo, hi = parallel.shard_bounds(n, world)[rank]
    shard = F.Corpus.from_arrow(data[int(off[lo]):int(off[hi])], (off[lo:hi + 1] - off[lo]).astype(np.uint64), device=local)
    m = make_matcher()
    out = comm.host_alloc_matches(max(n, 1) + 1)
    total, _ = comm.match_list_parallel_rank(m, shard, lo, out)
    full = np.array(out[:total])
    ok = True
    for k in sorted({0, 1, 2, total // 2, total // 2 + 1, max(total - 1, 0), total, total + 1}):
        kept, t, _ = comm.match_list_parallel_rank_top(m, shard, lo, k, out)
        good = t == total and kept == min(k, total) and np.array_equal(np.array(out[:kept]), full[:k])
        if rank == 0 and not good:
            print(f"{label}: top-{k} differs (kept {kept}, total {t} vs {total})", flush=True)
        ok = ok and good
        kept2, t2, d_ptr = comm.match_list_parallel_rank_top(m, shard, lo, k, None)
        if kept2:
            import cuda.bindings.runtime as rt
            dev_host = np.empty(kept2, dtype=F.MATCH_DTYPE)
            err, = rt.cudaMemcpy(dev_host.ctypes.data, d_ptr, kept2 * 8, rt.cudaMemcpyKind.cudaMemcpyDeviceToHost)
            assert int(err) == 0, err
            if not (t2 == total and np.array_equal(dev_host, full[:kept2])):
                print(f"{label}: rank {rank} device-resident top-{k} differs", flush=True)
                ok = False
    if rank == 0:
        print(f"{label}: {total} matches, top-K == full[:K]: {ok}", flush=True)
    comm.barrier()
    comm.host_free(out)
    shard.close()
    m.close()
    return ok


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    comm = parallel.Comm.from_torch_distributed(local)
    data, off = synth.generate("deadbeef", 400_003, 48, 64, seed=7)
    ok = True
    for sort in SortStrategy:
        for k in (1, 0):
            ok = run_case(comm, rank, world, local, lambda: F.Matcher("deadbeef", Config(max_typos=k, sort=sort)), data, off,
                          f"sort={sort.name} k={k}") and ok
    d2, o2 = synth.generate("deadbeef", 10_001, 24, 32, seed=9)
    for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexDesc):
        ok = run_case(comm, rank, world, local, lambda: F.Matcher("deadbeef", Config(max_typos=None, sort=sort)), d2, o2,
                      f"all-match sort={sort.name}") and ok
    for n3 in (1, 0):
        d3, o3 = synth.generate("deadbeef", n3, 24, 32, seed=3, p_full=1.0, p_partial=0.0)
        ok = run_case(comm, rank, world, local, lambda: F.Matcher("deadbeef", Config(max_typos=0)), d3, o3, f"tiny n={n3}") and ok
    d4, o4 = synth.generate("foo", 50_001, 40, 64, seed=11, prefix_frac=0.2)
    ok = run_case(comm, rank, world, local, lambda: F.Matcher.from_query("foo !^bar", Config(max_typos=0)), d4, o4,
                  "multi-pattern 'foo !^bar'") and ok
    flag = torch.tensor([0 if ok else 1], device=torch.device("cuda", local))
    dist.all_reduce(flag)
    comm.close()
    dist.barrier()
    dist.destroy_process_group()
    if int(flag.item()) != 0:
        sys.exit(1)


if __name__ == "__main__":
    try:
        main()
    except BaseException:
        import traceback
        sys.stderr.write(f"[rank {os.environ.get('RANK')}] {traceback.format_exc()}\n")
        sys.stderr.flush()
        os._exit(1)
