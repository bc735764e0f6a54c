"""CPU-only tests of the product's host logic (no GPU compute): the C-ABI library loads and exports
every symbol include/frz_cuda.h declares, the query parser matches the reference's own parser tests
(src/pattern.rs:296-383), and backend selection / guards mirror the reference."""
import ctypes
import os
import re

import pytest

import frizbee_b200 as F
from frizbee_b200.types import CaseMatching, Config, Matching, Pattern, Scoring, UnicodeMatching

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "frz_cuda.h")).read()
    names = set(re.findall(r"\b(frz_[a-z0-9_]+)\s*\(", hdr))
    names -= {"frz_status"}
    lib = ctypes.CDLL(F.lib_path())
    missing = [n for n in sorted(names) if not hasattr(lib, n)]
    assert not missing, missing
    assert F.lib().frz_abi_version() == 3


def test_corpus_debug_image_argument_checks():
    """frz_corpus_debug_image (a test aid) refuses a null corpus or a null size array before it touches a device; the
    size and buffer checks on a real corpus are in tests/test_gpu_ingest.py."""
    L = F.lib()
    sizes = (ctypes.c_uint64 * 6)()
    bufs = [ctypes.create_string_buffer(16) for _ in range(6)]
    assert L.frz_corpus_debug_image(None, *[None] * 6, sizes) == 1   # FRZ_ERR_INVALID_ARG
    assert L.frz_corpus_debug_image(None, *[ctypes.addressof(b) for b in bufs], sizes) == 1
    assert L.frz_corpus_debug_image(None, *[None] * 6, None) == 1
    assert b"null" in L.frz_last_error()


def test_parse_atom_reference_vectors():
    def check(atom, needle, matching, negated):
        p = F.parse_atom(atom)
        assert (p.needle, p.matching, p.negated) == (needle, matching, negated), atom
    check("foo", "foo", None, False)
    check("^foo", "foo", Matching.Prefix, False)
    check("foo$", "foo", Matching.Suffix, False)
    check("'foo", "foo", Matching.Substring, False)
    check("^foo$", "foo", Matching.Exact, False)
    check("!foo", "foo", Matching.Substring, True)
    check("!^foo", "foo", Matching.Prefix, True)
    check("!foo$", "foo", Matching.Suffix, True)
    check("!'foo", "foo", Matching.Substring, True)
    check("!^foo$", "foo", Matching.Exact, True)
    check("\\^foo", "^foo", None, False)
    check("foo\\$", "foo$", None, False)
    check("\\'foo", "'foo", None, False)
    check("\\!foo", "!foo", None, False)
    check("foo\\ bar", "foo bar", None, False)
    check("!\\^foo", "^foo", Matching.Substring, True)
    check("!\\!foo", "!foo", Matching.Substring, True)
    check("foo\\\\$", "foo\\\\", Matching.Suffix, False)
    check("foo\\bar", "foo\\bar", None, False)
    check("foo\\", "foo\\", None, False)
    check("a\\\\\\ b", "a\\\\ b", None, False)


def test_parse_query_reference_vectors():
    ps = F.parse_query("foo !^bar")
    assert [(p.needle, p.matching, p.negated) for p in ps] == [("foo", None, False), ("bar", Matching.Prefix, True)]
    assert [p.needle for p in F.parse_query("  foo \t bar  ")] == ["foo", "bar"]
    assert [p.needle for p in F.parse_query("foo\\ bar baz")] == ["foo bar", "baz"]
    assert [p.needle for p in F.parse_query("foo\\\\ bar")] == ["foo\\\\", "bar"]
    assert F.parse_query("") == [] and F.parse_query("   ") == [] and F.parse_query("! ^$ '") == []
    assert [p.needle for p in F.parse_query("é다 😀x")] == ["é다", "😀x"]


def test_backend_selection_mirrors_get_backend():
    # src/matcher/mod.rs:448-498, :751-785; src/smith_waterman/mod.rs:522-532
    for em, (l8, l16) in {64: (64, 32), 32: (32, 16), 16: (16, 8)}.items():
        assert F.Matcher("abc", Config(emulate_lanes=em)).backend_info() == \
            {"lanes": l8, "score_bits": 8, "prefilter_lanes": em, "literal": False}
        assert F.Matcher("a" * 13, Config(emulate_lanes=em)).backend_info()["score_bits"] == 8
        info = F.Matcher("abcdefghijklmnopqrst", Config(emulate_lanes=em)).backend_info()
        assert info == {"lanes": l16, "score_bits": 16, "prefilter_lanes": em, "literal": False}
    assert F.Matcher("abcd", Config(scoring=Scoring(gap_extend_penalty=8), emulate_lanes=64)).backend_info()["score_bits"] == 16
    auto = F.Matcher("abc", Config()).backend_info()
    flags = open("/proc/cpuinfo").read()
    if all(f in flags for f in ("avx512f", "avx512bw", "avx512vbmi", "bmi1", "bmi2")):
        assert auto["lanes"] == 64 and auto["prefilter_lanes"] == 64
    elif "avx2" in flags:
        assert auto["lanes"] == 32
    assert F.Matcher("foo", Config(matching=Matching.Prefix)).backend_info()["literal"]


def test_build_patterns_and_guards():
    assert F.Matcher("", Config()).num_patterns() == 0
    assert F.Matcher.from_query("! ^$", Config()).num_patterns() == 0
    assert F.Matcher.from_query("foo !^bar", Config()).num_patterns() == 2
    # huge_bonuses_report_descriptive_overflow_error (src/matcher/algo.rs:370-378)
    with pytest.raises(F.FrizbeeError) as e:
        F.Matcher("f", Config(scoring=Scoring(capitalization_bonus=60000, matching_case_bonus=40000)))
    assert e.value.status_name == "FRZ_ERR_NEEDLE_TOO_LONG" and "needle too long" in str(e.value)
    # non-ASCII needles build (the unicode path, unicode.cu); malformed UTF-8 on that path is an argument error
    F.Matcher("é다😀", Config()).close()
    F.Matcher("é", Config(unicode=UnicodeMatching.Ignore, casing=CaseMatching.Ignore)).close()
    with pytest.raises(F.FrizbeeError) as e:
        F.Matcher([Pattern(b"\xff\xfe")], Config(unicode=UnicodeMatching.Always))
    assert e.value.status_name == "FRZ_ERR_INVALID_ARG"


def test_no_cpu_fallback_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(F.FrizbeeError) as e:
        F.Matcher("foo", Config()).match_list(["foo", "bar"])
    assert e.value.status_name in ("FRZ_ERR_NO_DEVICE", "FRZ_ERR_CUDA")


def _build_ffi_demo(tmp_path):
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    F.lib()   # make sure libfrz_cuda.so exists
    exe = str(tmp_path / "ffi_demo")
    libdir = os.path.join(root, "frizbee_b200")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(root, "include"),
                    os.path.join(root, "examples", "ffi_demo.c"), "-L" + libdir, "-lfrz_cuda", "-Wl,-rpath," + libdir, "-o", exe],
                   check=True)
    return exe


def test_c_abi_from_plain_c(tmp_path):
    """examples/ffi_demo.c uses only include/frz_cuda.h (C11, no CUDA headers, no torch types): it must compile and
    link warning-free; without a GPU it reports the missing device instead of falling back."""
    import subprocess
    import torch
    exe = _build_ffi_demo(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    if torch.cuda.is_available():
        assert r.returncode == 0 and "Match { score: 53, index: 0, exact: false }" in r.stdout, (r.stdout, r.stderr)
    else:
        assert r.returncode == 3 and "no CPU fallback" in r.stderr, (r.stdout, r.stderr)


def test_host_entry_points_survive_random_input():
    """Parser and pattern compilation are host code fed by user input: random byte strings (valid UTF-8 or not, NULs,
    operators, escapes) must produce a status, never a crash, and compiled matchers must report sane backends."""
    import random
    rng = random.Random(20260923)
    L = F.lib()
    alphabet = [b"a", b"B", b" ", b"!", b"^", b"$", b"'", b"\\", b"\x00", b"\xc3\xa9", b"\xf0\x9f\x98\x80", b"\xff", b"\t", b"\xe2\x80\x83", b"0"]
    for _ in range(3000):
        q = b"".join(rng.choice(alphabet) for _ in range(rng.randint(0, 12)))
        h = ctypes.c_void_p()
        assert L.frz_parse_query(q, len(q), ctypes.byref(h)) == 0
        n = L.frz_query_len(h)
        assert 0 <= n <= len(q)
        L.frz_query_destroy(h)
        cfg = F.types.CConfig.of(Config(max_typos=rng.choice([None, 0, 1, 2, 5]), unicode=rng.choice(list(UnicodeMatching)),
                                        casing=rng.choice(list(CaseMatching))))
        m = ctypes.c_void_p()
        st = L.frz_matcher_from_query(q, len(q), ctypes.byref(cfg), ctypes.byref(m))
        assert 0 <= st <= 10, st   # a status, whatever it is
        if st == 0:
            for i in range(L.frz_matcher_num_patterns(m)):
                lanes, bits, pf, lit = ctypes.c_int(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
                assert L.frz_matcher_backend_info(m, i, ctypes.byref(lanes), ctypes.byref(bits), ctypes.byref(pf), ctypes.byref(lit)) == 0
                assert lanes.value in (8, 16, 32, 64) and bits.value in (8, 16) and pf.value in (16, 32, 64)
            L.frz_matcher_destroy(m)


def test_parallel_entry_points_argument_errors_without_a_device():
    """frz_comm_* / frz_match_list_parallel* (src/matcher/parallel.rs:18-89 behind the C ABI): argument errors mirror the
    reference's panics (threads == 0 → "threads must be positive", parallel.rs:24), and without a device the
    communicator constructors fail with FRZ_ERR_NO_DEVICE — never a CPU fallback."""
    import torch
    from frizbee_b200 import parallel
    with pytest.raises(F.FrizbeeError) as e:
        parallel.Comm.local(0)
    assert e.value.status_name == "FRZ_ERR_THREADS_ZERO" and "threads must be positive" in str(e.value)
    with pytest.raises(F.FrizbeeError) as e:
        parallel.Comm.local(65)
    assert e.value.status_name == "FRZ_ERR_INVALID_ARG"
    with pytest.raises(F.FrizbeeError) as e:
        parallel.Comm.from_rank(b"\0" * 128, 2, 5, 0)
    assert e.value.status_name == "FRZ_ERR_INVALID_ARG"
    L = parallel.plib()
    n = ctypes.c_uint64()
    assert L.frz_match_list_parallel(None, None, 0, None, None, 0, ctypes.byref(n)) == 1          # FRZ_ERR_INVALID_ARG
    assert L.frz_match_list_parallel_rank(None, None, 0, None, None, 0, ctypes.byref(n), None) == 1
    assert L.frz_comm_world(None) == 0 and L.frz_comm_rank(None) == -1
    assert L.frz_comm_exchange_mode(None) == -1
    assert L.frz_match_list_parallel_rank_host(None, None, None, 4, 0, 0, None, None, 0, ctypes.byref(n)) == 1
    if not torch.cuda.is_available():
        with pytest.raises(F.FrizbeeError) as e:
            parallel.Comm.local(1)
        assert e.value.status_name == "FRZ_ERR_NO_DEVICE" and "no CPU fallback" in str(e.value)
    m = F.Matcher("foo", Config())
    clone = ctypes.c_void_p()
    assert L.frz_matcher_clone(m._h, ctypes.byref(clone)) == 0 and clone.value
    assert F.lib().frz_matcher_score_bound(clone) == m.score_bound()
    F.lib().frz_matcher_destroy(clone)
    m.close()
