"""Builds libfrz_cuda.so (sm_90a only) in-tree with nvcc.  Used by __graft_entry__.build()."""
from __future__ import annotations

import os
import re
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libfrz_cuda.so")
SOURCES = ["pack.cu", "prefilter.cu", "sw.cu", "sort.cu", "unicode.cu", "host.cu", "merge.cu", "parallel.cu", "batch.cu", "collapse.cu",
           "batch_columns.cu", "where.cu", "order.cu", "rank.cu", "boost_where.cu",
           "subset_match.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]
# A/B hook (compile-time, the default binary is untouched): extra -D flags from the environment, e.g. FRZ_NVCC_DEFINES="NAME=1";
# `--variant NAME --define D` builds libfrz_cuda_NAME.so beside the default
FLAGS += ["-D" + d for d in os.environ.get("FRZ_NVCC_DEFINES", "").split()]


def depfile_deps(text: str) -> list[str]:
    """The prerequisites of a make rule the compiler wrote with -MMD: `target: dep dep \\` continuation lines, spaces in
    a path escaped as `\\ `."""
    deps = []
    for line in text.replace("\\\n", " ").splitlines():
        deps += [w.replace("\\ ", " ") for w in re.findall(r"(?:\\ |\S)+", line.partition(":")[2])]
    return deps


def _outdated(out: str, deps) -> bool:
    if not os.path.exists(out):
        return True
    t = os.stat(out).st_mtime_ns
    return any(not os.path.exists(d) or os.stat(d).st_mtime_ns > t for d in deps)


def stale(cmd: list[str], out: str) -> bool:
    """Whether rebuild(cmd, out) has to run: out, its depfile or its recorded command is missing, the command differs,
    or a file the depfile names is gone or newer than out."""
    base = os.path.splitext(out)[0]
    try:
        with open(base + ".cmd") as f:
            if f.read() != "\n".join(cmd):
                return True
        with open(base + ".d") as f:
            return _outdated(out, depfile_deps(f.read()))
    except FileNotFoundError:
        return True


def _tmp(out: str) -> str:
    base, ext = os.path.splitext(out)
    return f"{base}.tmp{os.getpid()}{ext}"


def rebuild(cmd: list[str], out: str) -> str:
    """Runs the compiler command cmd (without -o) to build out, with the depfile <out without extension>.d, and records
    cmd beside it in <...>.cmd.  out is written under a temporary name and moved into place, and the record is removed
    first and written last, so an interrupted or failed build never leaves an out that stale() takes as current.
    Returns the compiler's messages; raises RuntimeError with them when it fails."""
    base, tmp = os.path.splitext(out)[0], _tmp(out)
    if os.path.exists(base + ".cmd"):
        os.remove(base + ".cmd")
    try:
        r = subprocess.run(cmd + ["-MMD", "-MF", base + ".d", "-o", tmp], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        os.replace(tmp, out)
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)
    with open(base + ".cmd", "w") as f:
        f.write("\n".join(cmd))
    return r.stdout + r.stderr


def build(force: bool = False, verbose: bool = False, variant: str = "", defines=()) -> str:
    """variant/defines: an A/B build (`libfrz_cuda_<variant>.so`, own object directory) with extra -D flags; load it with
    FRZ_LIB=<path> (frizbee_b200.lib_path).  The default build is untouched."""
    objdir = os.path.join(HERE, "build" + ("_" + variant if variant else ""))
    out = OUT if not variant else os.path.join(HERE, f"libfrz_cuda_{variant}.so")
    flags = FLAGS + ["-D" + d for d in defines] + (["-Xptxas", "-v"] if verbose else [])
    os.makedirs(objdir, exist_ok=True)
    objs = [os.path.join(objdir, s.replace(".cu", ".o")) for s in SOURCES]
    jobs = [([NVCC] + flags + ["-c", os.path.join(CSRC, s)], o) for s, o in zip(SOURCES, objs)]
    jobs = [(cmd, o) for cmd, o in jobs if force or stale(cmd, o)]

    def run(job):
        cmd, o = job
        msg = rebuild(cmd, o)
        if verbose:
            sys.stderr.write(" ".join(cmd) + "\n" + msg)

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        list(ex.map(run, jobs))
    if force or jobs or _outdated(out, objs):
        # no NCCL on the link line: parallel.cu resolves libnccl.so.2 with dlopen at the first multi-GPU call
        tmp = _tmp(out)
        cmd = [NVCC, "-shared", "-o", tmp] + objs + ["-Xcompiler", "-fPIC", "-ldl", "-lpthread"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
        os.replace(tmp, out)
    return out


if __name__ == "__main__":
    variant, defines = "", []
    for i, a in enumerate(sys.argv):
        if a == "--variant":
            variant = sys.argv[i + 1]
        if a == "--define":
            defines.append(sys.argv[i + 1])
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, variant=variant, defines=defines))
