"""torchrun worker (one rank per GPU): shards a list over WORLD_SIZE GPUs, runs Matcher::match_list_parallel through the
C ABI (frz_comm_create_rank + frz_match_list_parallel_rank: NCCL all-gather + device merge + per-rank slice copy into
the shared host buffer) and checks on rank 0 that the result equals the single-GPU match_list (parallel == sequential,
src/matcher/parallel.rs:104-130) — for every sort strategy, for shard sizes that do not divide evenly, for a
match-everything query (another rank's run longer than the last rank's whole shard), for a score bound that needs the
two-pass sort and for lists shorter than the number of ranks (empty shards).  With FRZ_PARALLEL_EXCHANGE set to a value
other than `slices`, it checks instead that every rank's communicator creation refuses it."""
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


def run_case(comm, rank, world, local, needle, cfg, data, off, label):
    n = len(off) - 1
    lo, hi = parallel.shard_bounds(n, world)[rank]
    sdata = data[int(off[lo]):int(off[hi])]
    soff = (off[lo:hi + 1] - off[lo]).astype(np.uint64)
    shard = F.Corpus.from_arrow(sdata, soff, device=local)
    m = F.Matcher(needle, cfg)
    out = comm.host_alloc_matches(max(n, 1))
    total, d_ptr = comm.match_list_parallel_rank(m, shard, lo, out)
    ok = True
    if rank == 0:
        got = np.array(out[:total])
        full = F.Corpus.from_arrow(data, off, device=local)
        want = F.Matcher(needle, cfg).match_list_array(full, device=local)
        ok = len(got) == len(want) and np.array_equal(got, want)
        print(f"{label}: {total} matches, parallel == single-GPU: {ok}", flush=True)
        full.close()
    # the device-resident form leaves the same list on every rank
    total2, d_ptr2 = comm.match_list_parallel_rank(m, shard, lo, None)
    if total2:
        import cuda.bindings.runtime as rt   # cuda-python: a plain cudaMemcpy from the raw device pointer
        dev_host = np.empty(total2, dtype=F.MATCH_DTYPE)
        err, = rt.cudaMemcpy(dev_host.ctypes.data, d_ptr2, total2 * 8, rt.cudaMemcpyKind.cudaMemcpyDeviceToHost)
        assert int(err) == 0, err
        if not (total2 == total and np.array_equal(dev_host, np.array(out[:total]))):
            print(f"{label}: rank {rank} device-resident result differs from the host result", flush=True)
            ok = False
    comm.barrier()
    comm.host_free(out)
    shard.close()
    m.close()
    return ok


def refused_exchange(local):
    """FRZ_PARALLEL_EXCHANGE set to anything but `slices` (or nothing): this rank's communicator creation must fail with
    FRZ_ERR_INVALID_ARG.  Returns None when the variable is unset or `slices`, else whether the creation was refused."""
    value = os.environ.get("FRZ_PARALLEL_EXCHANGE", "")
    if value in ("", "slices"):
        return None
    try:
        parallel.Comm.from_torch_distributed(local).close()
        refused = False
    except F.FrizbeeError as e:
        refused = e.status_name == "FRZ_ERR_INVALID_ARG"
    print(f"FRZ_PARALLEL_EXCHANGE={value}: communicator refused with FRZ_ERR_INVALID_ARG: {refused}", flush=True)
    return refused


def finish(local, ok, comm=None):
    """Every rank learns whether all ranks passed; exits with 1 if one did not."""
    flag = torch.tensor([0 if ok else 1], device=torch.device("cuda", local))
    dist.all_reduce(flag)
    if comm is not None:
        comm.close()
    dist.barrier()
    dist.destroy_process_group()
    if int(flag.item()) != 0:
        sys.exit(1)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    refused = refused_exchange(local)
    if refused is not None:
        return finish(local, refused)
    comm = parallel.Comm.from_torch_distributed(local)
    assert comm.world == world and comm.rank == rank
    n = 400_003
    data, off = synth.generate("deadbeef", n, 48, 64, seed=7)
    ok = True
    for sort in SortStrategy:
        for k in (0, 1):
            ok = run_case(comm, rank, world, local, "deadbeef", Config(max_typos=k, sort=sort), data, off, f"sort={sort.name} k={k}") and ok
    # everything matches (max_typos=None), n % world != 0: every other rank's run is longer than the last rank's shard
    n2 = 10_001 if world == 2 else 1000 * world + 1
    d2, o2 = synth.generate("deadbeef", n2, 24, 32, seed=9)
    for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexDesc):
        ok = run_case(comm, rank, world, local, "deadbeef", Config(max_typos=None, sort=sort), d2, o2, f"all-match sort={sort.name} n={n2}") and ok
    # a score bound >= 1024 sorts in two passes, which publish no per-score table: host-out calls take the all-gather + merge
    long_needle = "abcdefghijklmnopqrstuvwxyzabcdefghijklmnopqrstuvwxyzabcdefgh"   # 60 bytes
    d5, o5 = synth.generate(long_needle, 20_001, 80, 128, seed=2, p_full=0.5)
    for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.ScoreThenIndexDesc):
        ok = run_case(comm, rank, world, local, long_needle, Config(max_typos=None, sort=sort), d5, o5, f"two-pass bound sort={sort.name}") and ok
    # fewer haystacks than ranks (empty shards), and the empty list
    for n3 in (1, 0):
        d3, o3 = synth.generate("deadbeef", n3, 24, 32, seed=3, p_full=1.0, p_partial=0.0)
        ok = run_case(comm, rank, world, local, "deadbeef", Config(max_typos=0), d3, o3, f"tiny n={n3}") and ok
    # multi-pattern query through the parallel path (count published at the end of the local pipeline)
    d4, o4 = synth.generate("foo", 50_001, 40, 64, seed=11, prefix_frac=0.2)
    m_ok = True
    lo, hi = parallel.shard_bounds(50_001, world)[rank]
    shard = F.Corpus.from_arrow(d4[int(o4[lo]):int(o4[hi])], (o4[lo:hi + 1] - o4[lo]).astype(np.uint64), device=local)
    mq = F.Matcher.from_query("foo !^bar", Config(max_typos=0))
    out = comm.host_alloc_matches(50_001)
    total, _ = comm.match_list_parallel_rank(mq, shard, lo, out)
    if rank == 0:
        full = F.Corpus.from_arrow(d4, o4, device=local)
        want = F.Matcher.from_query("foo !^bar", Config(max_typos=0)).match_list_array(full, device=local)
        m_ok = total == len(want) and np.array_equal(np.array(out[:total]), want)
        print(f"multi-pattern 'foo !^bar': {total} matches, parallel == single-GPU: {m_ok}", flush=True)
        full.close()
    comm.barrier()
    comm.host_free(out)
    shard.close(); mq.close()
    finish(local, ok and m_ok, comm)


if __name__ == "__main__":
    try:
        main()
    except BaseException:
        import traceback
        sys.stderr.write(f"[rank {os.environ.get('RANK')}] {traceback.format_exc()}\n")
        sys.stderr.flush()
        os._exit(1)
