"""Builds and loads the g++ harnesses of tests/harness/, which compile the library's host/device headers for the CPU.  A
harness is rebuilt when a file its depfile names changes or its command line does (frizbee_b200/build.py's rule)."""
import ctypes
import os

import pytest

from frizbee_b200.build import rebuild, stale

HARNESS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "harness")
CUDA_INC = "/usr/local/cuda/include"


def load(name: str, opt: str = "-O2", cuda_include: bool = False) -> ctypes.CDLL:
    """lib<name>.so built from <name>.cpp, both in tests/harness/; name may also be the path of a .cpp elsewhere.
    cuda_include: the harness includes CUDA headers (skips the test when they are not installed)."""
    src = name if name.endswith(".cpp") else os.path.join(HARNESS, name + ".cpp")
    if cuda_include and not os.path.isdir(CUDA_INC):
        pytest.skip("CUDA headers not found")
    folder, file = os.path.split(src)
    lib = os.path.join(folder, "lib" + file[:-len(".cpp")] + ".so")
    cmd = ["g++", opt, "-std=c++17"] + (["-I" + CUDA_INC] if cuda_include else []) + ["-fPIC", "-shared", src]
    if stale(cmd, lib):
        rebuild(cmd, lib)
    return ctypes.CDLL(lib)
