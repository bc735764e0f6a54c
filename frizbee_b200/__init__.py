"""frizbee_b200 — H100-native `match_list` path of saghen/frizbee behind a C ABI.

This Python layer is a thin ctypes binding over ``libfrz_cuda.so`` (include/frz_cuda.h); it mirrors
the reference's public names (``Matcher``, ``Pattern``, ``Config``, ``Scoring``, ``Match``,
``radix_sort_matches``; src/lib.rs:120-122) so the parity tests read like the reference's own tests.
There is no CPU fallback: if the CUDA library or a device is missing, calls raise ``FrizbeeError``.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Iterable, List, Optional, Sequence, Tuple, Union

import numpy as np

from .types import (CaseMatching, CConfig, CMatch, Config, CPattern, Match, Matching, Pattern, Scoring,
                    SortStrategy, UnicodeMatching, as_pattern, pattern_array)

__all__ = ["Matcher", "Corpus", "Pattern", "Config", "Scoring", "Match", "SortStrategy", "CaseMatching",
           "UnicodeMatching", "Matching", "FrizbeeError", "parse_query", "parse_atom", "radix_sort_matches",
           "MATCH_DTYPE", "lib", "lib_path"]

_HERE = os.path.dirname(os.path.abspath(__file__))
MATCH_DTYPE = np.dtype([("index", "<u4"), ("score", "<u2"), ("exact", "u1"), ("_pad", "u1")])

STATUS_NAMES = {0: "FRZ_OK", 1: "FRZ_ERR_INVALID_ARG", 2: "FRZ_ERR_NEEDLE_TOO_LONG", 3: "FRZ_ERR_GAP_OVERFLOW",
                4: "FRZ_ERR_TOO_MANY_ITEMS", 5: "FRZ_ERR_THREADS_ZERO", 6: "FRZ_ERR_CAPACITY", 7: "FRZ_ERR_CUDA",
                8: "FRZ_ERR_NO_DEVICE", 9: "FRZ_ERR_UNSUPPORTED", 10: "FRZ_ERR_OOM", 11: "FRZ_ERR_NCCL"}


class FrizbeeError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"{STATUS_NAMES.get(status, status)}: {message}")
        self.status = status
        self.status_name = STATUS_NAMES.get(status, str(status))


def lib_path() -> str:
    """libfrz_cuda.so next to this file; FRZ_LIB names an A/B build instead (frizbee_b200/build.py --variant)."""
    return os.environ.get("FRZ_LIB") or os.path.join(_HERE, "libfrz_cuda.so")


_lib = None


def lib():
    """Loads libfrz_cuda.so.  Raises (never falls back) when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise FrizbeeError(8, f"{path} is missing — run `python -c 'import __graft_entry__ as g; g.build()'`; "
                              "there is no CPU fallback")
    L = C.CDLL(path)
    vp, u8p, sz, u64, u32 = C.c_void_p, C.c_char_p, C.c_size_t, C.c_uint64, C.c_uint32
    L.frz_last_error.restype = C.c_char_p
    L.frz_status_str.restype = C.c_char_p
    L.frz_status_str.argtypes = [C.c_int]
    L.frz_abi_version.restype = C.c_int
    L.frz_config_default.argtypes = [C.POINTER(CConfig)]
    L.frz_parse_query.argtypes = [u8p, sz, C.POINTER(vp)]
    L.frz_parse_atom.argtypes = [u8p, sz, C.POINTER(vp)]
    L.frz_query_len.restype = sz
    L.frz_query_len.argtypes = [vp]
    L.frz_query_get.argtypes = [vp, sz, C.POINTER(CPattern)]
    L.frz_query_destroy.argtypes = [vp]
    L.frz_query_destroy.restype = None
    L.frz_corpus_create.argtypes = [vp, vp, u64, C.c_int, C.POINTER(vp)]
    L.frz_corpus_create_arrow.argtypes = [vp, vp, C.c_int, u64, C.c_int, C.POINTER(vp)]
    L.frz_corpus_append.argtypes = [vp, vp, vp, C.c_int, u64]
    L.frz_corpus_create_ptrs.argtypes = [vp, vp, u64, C.c_int, C.POINTER(vp)]
    L.frz_corpus_create_device.argtypes = [vp, vp, u64, u64, C.c_int, vp, C.POINTER(vp)]
    for fn in (L.frz_corpus_len, L.frz_corpus_total_bytes, L.frz_corpus_device_bytes):
        fn.restype = u64
        fn.argtypes = [vp]
    L.frz_corpus_device.argtypes = [vp]
    L.frz_corpus_destroy.argtypes = [vp]
    L.frz_corpus_destroy.restype = None
    L.frz_matcher_create.argtypes = [vp, sz, C.POINTER(CConfig), C.POINTER(vp)]
    L.frz_matcher_from_query.argtypes = [u8p, sz, C.POINTER(CConfig), C.POINTER(vp)]
    L.frz_matcher_set_config.argtypes = [vp, C.POINTER(CConfig)]
    L.frz_matcher_destroy.argtypes = [vp]
    L.frz_matcher_destroy.restype = None
    L.frz_matcher_num_patterns.restype = sz
    L.frz_matcher_num_patterns.argtypes = [vp]
    L.frz_matcher_backend_info.argtypes = [vp, sz] + [C.POINTER(C.c_int)] * 4
    L.frz_matcher_last_timings.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(u64)]
    L.frz_match_list.argtypes = [vp, vp, vp, u64, C.POINTER(u64)]
    L.frz_match_list_top.argtypes = [vp, vp, u64, vp, C.POINTER(u64), C.POINTER(u64)]
    L.frz_match_list_into.argtypes = [vp, vp, u32, vp, u64, C.POINTER(u64)]
    L.frz_match_list_host.argtypes = [vp, vp, vp, u64, C.c_int, vp, u64, C.POINTER(u64)]
    L.frz_match_list_host_arrow.argtypes = [vp, vp, vp, C.c_int, u64, C.c_int, vp, u64, C.POINTER(u64)]
    L.frz_match_indices.argtypes = [vp, vp, vp, u64, vp, vp, u32, vp]
    L.frz_match_shard_device.argtypes = [vp, vp, u32, vp, u64, vp, vp]
    L.frz_matcher_wait_count.argtypes = [vp, vp]
    L.frz_merge_runs_device.argtypes = [vp, u64, vp, C.c_int, C.c_uint8, u32, vp, C.c_int, vp]
    L.frz_matcher_score_bound.restype = u32
    L.frz_matcher_score_bound.argtypes = [vp]
    L.frz_radix_sort_matches.argtypes = [vp, u64, C.c_int]
    _lib = L
    return L


def _check(status: int):
    if status != 0:
        raise FrizbeeError(status, lib().frz_last_error().decode("utf-8", "replace"))


def _arrow_offsets(offsets: np.ndarray):
    """(contiguous offsets, width in bytes): 32-bit integer arrays stay 32-bit (Arrow Utf8), the rest become uint64."""
    offsets = np.asarray(offsets)
    if offsets.dtype in (np.dtype(np.uint32), np.dtype(np.int32)):
        return np.ascontiguousarray(offsets), 4
    return np.ascontiguousarray(offsets, dtype=np.uint64), 8


def _b(x) -> bytes:
    return x.encode("utf-8") if isinstance(x, str) else bytes(x)


def _patterns_from_query(handle) -> List[Pattern]:
    L = lib()
    out = []
    for i in range(L.frz_query_len(handle)):
        cp = CPattern()
        _check(L.frz_query_get(handle, i, C.byref(cp)))
        needle = C.string_at(cp.needle, cp.needle_len).decode("utf-8", "surrogateescape") if cp.needle_len else ""
        out.append(Pattern(needle=needle, negated=bool(cp.negated),
                           matching=None if cp.matching < 0 else Matching(cp.matching)))
    return out


def parse_query(query: str) -> List[Pattern]:
    """Pattern::parse_query (src/pattern.rs:190-222)."""
    L = lib()
    h = C.c_void_p()
    q = _b(query)
    _check(L.frz_parse_query(q, len(q), C.byref(h)))
    try:
        return _patterns_from_query(h)
    finally:
        L.frz_query_destroy(h)


def parse_atom(atom: str) -> Pattern:
    """Pattern::parse (src/pattern.rs:100-165)."""
    L = lib()
    h = C.c_void_p()
    a = _b(atom)
    _check(L.frz_parse_atom(a, len(a), C.byref(h)))
    try:
        p = _patterns_from_query(h)[0]
        return Pattern(needle=p.needle, negated=p.negated, matching=p.matching, pattern=atom)
    finally:
        L.frz_query_destroy(h)


def pack_host(haystacks: Sequence) -> Tuple[np.ndarray, np.ndarray]:
    """List of str/bytes → Arrow-style (bytes u8[], offsets u64[n+1])."""
    raw = [_b(h) for h in haystacks]
    offsets = np.zeros(len(raw) + 1, dtype=np.uint64)
    if raw:
        offsets[1:] = np.cumsum([len(r) for r in raw], dtype=np.uint64)
    data = np.frombuffer(b"".join(raw), dtype=np.uint8).copy() if raw else np.zeros(0, dtype=np.uint8)
    return data, offsets


class Corpus:
    """A haystack list packed and resident in HBM (frz_corpus)."""

    def __init__(self, handle, n: int):
        self._h = handle
        self.n = n

    @classmethod
    def from_list(cls, haystacks: Sequence, device: int = 0) -> "Corpus":
        data, offsets = pack_host(haystacks)
        return cls.from_arrow(data, offsets, device)

    @classmethod
    def from_arrow(cls, data: np.ndarray, offsets: np.ndarray, device: int = 0) -> "Corpus":
        """Arrow value bytes + offsets (uint32/int32 = Utf8, otherwise 64-bit = LargeUtf8; offsets[0] may be > 0)."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        offsets, width = _arrow_offsets(offsets)
        h = C.c_void_p()
        n = len(offsets) - 1
        _check(lib().frz_corpus_create_arrow(data.ctypes.data if data.size else None, offsets.ctypes.data, width, n, device,
                                             C.byref(h)))
        return cls(h, n)

    @classmethod
    def from_device(cls, d_bytes_ptr: int, d_offsets_ptr: int, n: int, total_bytes: int, device: int = 0,
                    stream: int = 0) -> "Corpus":
        h = C.c_void_p()
        _check(lib().frz_corpus_create_device(d_bytes_ptr, d_offsets_ptr, n, total_bytes, device, stream, C.byref(h)))
        return cls(h, n)

    def append(self, data: np.ndarray, offsets: np.ndarray) -> "Corpus":
        """Appends haystacks (Arrow value bytes + offsets); their indices continue at len(self)."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        offsets, width = _arrow_offsets(offsets)
        n_new = len(offsets) - 1
        _check(lib().frz_corpus_append(self._h, data.ctypes.data if data.size else None, offsets.ctypes.data, width, n_new))
        self.n += n_new
        return self

    def append_list(self, haystacks: Sequence) -> "Corpus":
        data, offsets = pack_host(haystacks)
        return self.append(data, offsets)

    def __len__(self):
        return self.n

    @property
    def total_bytes(self) -> int:
        return lib().frz_corpus_total_bytes(self._h)

    @property
    def device_bytes(self) -> int:
        return lib().frz_corpus_device_bytes(self._h)

    def close(self):
        if self._h:
            lib().frz_corpus_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _to_matches(arr: np.ndarray) -> List[Match]:
    return [Match(score=int(s), index=int(i), exact=bool(e)) for i, s, e in zip(arr["index"], arr["score"], arr["exact"])]


class Matcher:
    """`Matcher` (src/matcher/mod.rs:76-222), GPU-backed."""

    def __init__(self, pattern: Union[str, Pattern, Sequence[Pattern]], config: Config = Config()):
        if isinstance(pattern, (str, bytes, Pattern)):
            pattern = [pattern]
        self._patterns = [as_pattern(p) for p in pattern]
        self.config = config
        self._h = C.c_void_p()
        arr = pattern_array(self._patterns)
        cfg = CConfig.of(config)
        _check(lib().frz_matcher_create(C.cast(arr, C.c_void_p), len(self._patterns), C.byref(cfg), C.byref(self._h)))

    @classmethod
    def from_patterns(cls, patterns: Sequence[Pattern], config: Config = Config()) -> "Matcher":
        return cls(list(patterns), config)

    @classmethod
    def from_query(cls, query: str, config: Config = Config()) -> "Matcher":
        self = cls.__new__(cls)
        self._patterns = None
        self.config = config
        self._h = C.c_void_p()
        q = _b(query)
        cfg = CConfig.of(config)
        _check(lib().frz_matcher_from_query(q, len(q), C.byref(cfg), C.byref(self._h)))
        return self

    def set_config(self, config: Config):
        cfg = CConfig.of(config)
        _check(lib().frz_matcher_set_config(self._h, C.byref(cfg)))
        self.config = config

    def backend_info(self, i: int = 0) -> dict:
        lanes, bits, pf, lit = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        _check(lib().frz_matcher_backend_info(self._h, i, C.byref(lanes), C.byref(bits), C.byref(pf), C.byref(lit)))
        return {"lanes": lanes.value, "score_bits": bits.value, "prefilter_lanes": pf.value, "literal": bool(lit.value)}

    def score_bound(self) -> int:
        return lib().frz_matcher_score_bound(self._h)

    def num_patterns(self) -> int:
        return lib().frz_matcher_num_patterns(self._h)

    def last_timings(self) -> dict:
        ms = (C.c_float * 4)()
        launches = C.c_uint64()
        _check(lib().frz_matcher_last_timings(self._h, ms, C.byref(launches)))
        return {"prefilter_ms": ms[0], "sw_ms": ms[1], "sort_ms": ms[2], "total_ms": ms[3], "launches": launches.value}

    # ---- match_list ----
    def _corpus(self, haystacks, device):
        if isinstance(haystacks, Corpus):
            return haystacks, False
        return Corpus.from_list(haystacks, device), True

    def match_list_array(self, haystacks, device: int = 0, out: Optional[np.ndarray] = None) -> np.ndarray:
        """Matcher::match_list → structured numpy array (MATCH_DTYPE)."""
        corpus, owned = self._corpus(haystacks, device)
        try:
            if out is None:
                out = np.empty(max(1, corpus.n), dtype=MATCH_DTYPE)
            n = C.c_uint64()
            _check(lib().frz_match_list(self._h, corpus._h, out.ctypes.data, len(out), C.byref(n)))
            return out[: n.value]
        finally:
            if owned:
                corpus.close()

    def match_list(self, haystacks, device: int = 0) -> List[Match]:
        return _to_matches(self.match_list_array(haystacks, device))

    def match_list_top_array(self, haystacks, k: int, device: int = 0, out: Optional[np.ndarray] = None) -> Tuple[np.ndarray, int]:
        """Matcher::match_list truncated to its first k rows (frz_match_list_top): (array of min(k, total) matches, total).
        `out` (optional) needs room for min(k, len(corpus)) matches: no more rows can match."""
        corpus, owned = self._corpus(haystacks, device)
        try:
            need = min(int(k), corpus.n)
            if out is None:
                out = np.empty(max(1, need), dtype=MATCH_DTYPE)
            elif len(out) < need:
                raise ValueError(f"out holds {len(out)} matches; a top-{k} call on {corpus.n} haystacks needs {need}")
            n, total = C.c_uint64(), C.c_uint64()
            _check(lib().frz_match_list_top(self._h, corpus._h, int(k), out.ctypes.data, C.byref(n), C.byref(total)))
            return out[: n.value], total.value
        finally:
            if owned:
                corpus.close()

    def match_list_into_array(self, haystacks, index_offset: int = 0, device: int = 0) -> np.ndarray:
        """Specialized::match_list / Matcher::match_list_into: index order, unsorted."""
        corpus, owned = self._corpus(haystacks, device)
        try:
            out = np.empty(max(1, corpus.n), dtype=MATCH_DTYPE)
            n = C.c_uint64()
            _check(lib().frz_match_list_into(self._h, corpus._h, index_offset, out.ctypes.data, len(out), C.byref(n)))
            return out[: n.value]
        finally:
            if owned:
                corpus.close()

    def match_indices(self, corpus: "Corpus", which, stride: int = 128):
        """Matcher::match_list_indices for the chosen haystacks: list of None (no match) or (score, exact, indices)."""
        which = np.ascontiguousarray(which, dtype=np.uint32)
        n = len(which)
        out_m = np.zeros(max(n, 1), dtype=MATCH_DTYPE)
        out_idx = np.zeros((max(n, 1), stride), dtype=np.uint32)
        out_cnt = np.zeros(max(n, 1), dtype=np.uint32)
        _check(lib().frz_match_indices(self._h, corpus._h, which.ctypes.data, n, out_m.ctypes.data, out_idx.ctypes.data, stride,
                                       out_cnt.ctypes.data))
        res = []
        for j in range(n):
            if out_cnt[j] == 0xFFFFFFFF:
                res.append(None)
            else:
                res.append((int(out_m[j]["score"]), bool(out_m[j]["exact"]), out_idx[j, : min(int(out_cnt[j]), stride)].tolist()))
        return res

    def match_list_host_array(self, data: np.ndarray, offsets: np.ndarray, device: int = 0,
                              out: Optional[np.ndarray] = None) -> np.ndarray:
        """End-to-end: host Arrow buffers in, host matches out (pack + H2D + match + D2H)."""
        n_items = len(offsets) - 1
        if out is None:
            out = np.empty(max(1, n_items), dtype=MATCH_DTYPE)
        n = C.c_uint64()
        if offsets.dtype.itemsize == 4 and offsets.flags.c_contiguous:
            width = 4
        else:
            offsets, width = _arrow_offsets(offsets)
        _check(lib().frz_match_list_host_arrow(self._h, data.ctypes.data if data.size else None, offsets.ctypes.data, width,
                                               n_items, device, out.ctypes.data, len(out), C.byref(n)))
        return out[: n.value]

    def close(self):
        if getattr(self, "_h", None):
            lib().frz_matcher_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def radix_sort_matches(arr: np.ndarray, device: int = 0) -> np.ndarray:
    """radix_sort_matches (src/sort.rs:6-40) on the GPU: stable, descending score."""
    arr = np.ascontiguousarray(arr, dtype=MATCH_DTYPE).copy()
    _check(lib().frz_radix_sort_matches(arr.ctypes.data, len(arr), device))
    return arr
