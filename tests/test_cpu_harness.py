"""The harness loader (tests/cpu_harness.py) rebuilds a library when a header it includes changes, and only then; the
depfile parser it shares with frizbee_b200/build.py reads the rules g++ and nvcc write."""
import _ctypes
import os

from cpu_harness import load
from frizbee_b200.build import depfile_deps


def _value(path):
    L = load(path)
    value = L.value()
    _ctypes.dlclose(L._handle)   # dlopen hands back a library it already holds: close it so the next load maps the rebuilt one
    return value


def test_rebuilds_when_an_included_header_changes(tmp_path):
    src, hdr, lib = tmp_path / "toy.cpp", tmp_path / "toy.h", tmp_path / "libtoy.so"
    src.write_text('#include "toy.h"\nextern "C" int value() { return toy_value(); }\n')
    hdr.write_text("inline int toy_value() { return 1; }\n")
    assert _value(str(src)) == 1
    hdr.write_text("inline int toy_value() { return 2; }\n")
    built = os.stat(lib).st_mtime_ns
    os.utime(hdr, ns=(built + 1, built + 1))   # newer than the library even on a coarse file clock
    assert _value(str(src)) == 2
    rebuilt = os.stat(lib).st_mtime_ns
    assert rebuilt > built
    assert _value(str(src)) == 2
    assert os.stat(lib).st_mtime_ns == rebuilt


def test_depfile_continuation_lines():
    text = "/o/a.o: /s/a.cu \\\n  /s/a.cuh \\\n  /s/b.cuh\n"
    assert depfile_deps(text) == ["/s/a.cu", "/s/a.cuh", "/s/b.cuh"]


def test_depfile_escaped_space():
    text = "a.o : /my\\ dir/a\\ b.cu \\\n    /my\\ dir/h.cuh\n"
    assert depfile_deps(text) == ["/my dir/a b.cu", "/my dir/h.cuh"]


def test_depfile_one_line():
    assert depfile_deps("libx.so: x.cpp x.h y.h\n") == ["x.cpp", "x.h", "y.h"]
