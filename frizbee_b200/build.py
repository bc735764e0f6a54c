"""Builds libfrz_cuda.so (sm_90a only) in-tree with nvcc.  Used by __graft_entry__.build()."""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libfrz_cuda.so")
SOURCES = ["pack.cu", "prefilter.cu", "sw.cu", "sort.cu", "unicode.cu", "host.cu", "merge.cu", "parallel.cu", "batch.cu", "collapse.cu",
           "batch_columns.cu", "where.cu", "order.cu", "rank.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]
# A/B hook (compile-time, the default binary is untouched): extra -D flags from the environment, e.g. FRZ_NVCC_DEFINES="NAME=1"
# (force a rebuild: `python frizbee_b200/build.py --force`); `--variant NAME --define D` builds libfrz_cuda_NAME.so beside the default
FLAGS += ["-D" + d for d in os.environ.get("FRZ_NVCC_DEFINES", "").split()]


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False, variant: str = "", defines=()) -> str:
    """variant/defines: an A/B build (`libfrz_cuda_<variant>.so`, own object directory) with extra -D flags; load it with
    FRZ_LIB=<path> (frizbee_b200.lib_path).  The default build is untouched."""
    headers = [os.path.join(CSRC, h) for h in ("frz_device.cuh", "frz_host.h", "unicode_path.cuh", "unicode_needle.h", "unicode_case.inc", "indices_path.cuh", "sw_core.cuh", "sw_generic.cuh", "sw_wave.cuh", "prefilter_masks.cuh", "prefilter_scan.cuh", "merge_plan.cuh", "batch_plan.cuh", "collapse_plan.cuh", "batch_collapse_plan.cuh", "batch_columns_plan.cuh", "where_plan.cuh", "order_plan.cuh", "batch_order_plan.cuh", "rank_plan.cuh")] + \
              [os.path.join(HERE, "..", "include", "frz_cuda.h")]
    objdir = os.path.join(HERE, "build" + ("_" + variant if variant else ""))
    out = OUT if not variant else os.path.join(HERE, f"libfrz_cuda_{variant}.so")
    flags = FLAGS + ["-D" + d for d in defines]
    os.makedirs(objdir, exist_ok=True)
    jobs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src.replace(".cu", ".o"))
        if force or _stale(o, [s] + headers):
            cmd = [NVCC] + flags + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        return cmd, r

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        for cmd, r in ex.map(run, jobs):
            if verbose or r.returncode != 0:
                sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
            if r.returncode != 0:
                raise RuntimeError("nvcc failed for " + cmd[-3])
    objs = [os.path.join(objdir, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or _stale(out, objs):
        # no NCCL on the link line: parallel.cu resolves libnccl.so.2 with dlopen at the first multi-GPU call
        cmd = [NVCC, "-shared", "-o", out] + objs + ["-Xcompiler", "-fPIC", "-ldl", "-lpthread"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return out


if __name__ == "__main__":
    variant, defines = "", []
    for i, a in enumerate(sys.argv):
        if a == "--variant":
            variant = sys.argv[i + 1]
        if a == "--define":
            defines.append(sys.argv[i + 1])
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, variant=variant, defines=defines))
