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

from .types import (CaseMatching, CConfig, CMatch, Config, CPattern, Match, Matching, Order, Pattern, Scoring,
                    SortStrategy, UnicodeMatching, as_pattern, pattern_array)

__all__ = ["Matcher", "Corpus", "Subset", "Boost", "Groups", "GROUP_NONE", "Attr", "Where", "where_batch", "BoostRule", "boost_where_batch", "BOOST_MAX_RULES", "ATTR_NULL", "RankKey", "RANK_MAX_KEYS", "Pattern", "Config", "Scoring", "Match", "SortStrategy", "Order", "CaseMatching",
           "UnicodeMatching", "Matching", "FrizbeeError", "parse_query", "parse_atom", "radix_sort_matches",
           "MATCH_DTYPE", "lib", "lib_path"]

_HERE = os.path.dirname(os.path.abspath(__file__))
GROUP_NONE = 0xFFFFFFFF   # FRZ_GROUP_NONE: a row in no group
ATTR_NULL = -(2**63)      # FRZ_ATTR_NULL: a row with no value for an attribute
RANK_MAX_KEYS = 4         # FRZ_RANK_MAX_KEYS: keys of one Corpus.rank / Attr.rank
BOOST_MAX_RULES = 8       # FRZ_BOOST_MAX_RULES: rules of one Boost.where
_U64_MAX = 0xFFFFFFFFFFFFFFFF   # UINT64_MAX: no k limit / no per-group cap
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
    L.frz_corpus_remove.argtypes = [vp, vp, u64]
    L.frz_corpus_replace.argtypes = [vp, vp, u64, vp, vp, C.c_int]
    L.frz_corpus_create_ptrs.argtypes = [vp, vp, u64, C.c_int, C.POINTER(vp)]
    L.frz_corpus_create_device.argtypes = [vp, vp, u64, u64, C.c_int, vp, C.POINTER(vp)]
    for fn in (L.frz_corpus_len, L.frz_corpus_total_bytes, L.frz_corpus_device_bytes):
        fn.restype = u64
        fn.argtypes = [vp]
    L.frz_corpus_device.argtypes = [vp]
    L.frz_corpus_destroy.argtypes = [vp]
    L.frz_corpus_destroy.restype = None
    L.frz_corpus_debug_image.argtypes = [vp] * 7 + [C.POINTER(u64)]
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
    L.frz_match_list_batch_top.argtypes = [vp, u64, vp, u64, vp, vp, vp]
    L.frz_match_list_batch.argtypes = [vp, u64, vp, vp, vp, u64, vp, vp, vp]
    L.frz_match_list_batch_collapsed.argtypes = [vp, u64, vp, vp, vp, vp, vp, u64, vp, vp, vp, vp]
    L.frz_match_list_batch_ordered.argtypes = [vp, u64, vp, vp, vp, vp, vp, vp, vp, u64, vp, vp, vp, vp]
    L.frz_debug_batch_limits.argtypes = [u64, u64]
    L.frz_debug_batch_limits.restype = None
    L.frz_debug_batch_last.argtypes = [vp]
    L.frz_debug_batch_last.restype = None
    L.frz_subset_create.argtypes = [vp, vp, u64, C.POINTER(vp)]
    L.frz_subset_len.restype = u64
    L.frz_subset_len.argtypes = [vp]
    L.frz_subset_destroy.argtypes = [vp]
    L.frz_subset_destroy.restype = None
    L.frz_match_list_subset.argtypes = [vp, vp, vp, vp, u64, C.POINTER(u64)]
    L.frz_match_list_subset_top.argtypes = [vp, vp, vp, u64, vp, C.POINTER(u64), C.POINTER(u64)]
    L.frz_attr_create.argtypes = [vp, vp, u64, C.POINTER(vp)]
    L.frz_attr_set.argtypes = [vp, vp, vp, u64]
    L.frz_attr_destroy.argtypes = [vp]
    L.frz_attr_destroy.restype = None
    L.frz_subset_where.argtypes = [vp, vp, u64, vp]
    L.frz_subset_where_batch.argtypes = [vp, u64, vp, vp, vp]
    L.frz_debug_where_batch.argtypes = [C.c_int]
    L.frz_subset_match.argtypes = [vp, vp, vp, vp]
    L.frz_debug_subset_match.argtypes = [C.c_int]
    L.frz_debug_subset_match.restype = u32
    L.frz_attr_rank.argtypes = [vp, vp, u64]
    L.frz_attr_get.argtypes = [vp, vp, u64]
    L.frz_boost_create.argtypes = [vp, vp, u64, C.POINTER(vp)]
    L.frz_boost_set.argtypes = [vp, vp, vp, u64]
    L.frz_boost_destroy.argtypes = [vp]
    L.frz_boost_get.argtypes = [vp, vp, u64]
    L.frz_boost_where.argtypes = [vp, vp, u64, vp]
    L.frz_boost_where_batch.argtypes = [vp, u64, vp, vp, vp]
    L.frz_boost_destroy.restype = None
    L.frz_match_list_ranked.argtypes = [vp, vp, vp, vp, u64, vp, C.POINTER(u64), C.POINTER(u64)]
    L.frz_match_list_ordered.argtypes = [vp, vp, vp, vp, vp, u32, u64, vp, C.POINTER(u64), C.POINTER(u64)]
    L.frz_match_list_ordered_collapsed.argtypes = [vp, vp, vp, vp, vp, u32, vp, u64, u64, vp, C.POINTER(u64), C.POINTER(u64), vp]
    L.frz_groups_create.argtypes = [vp, vp, u64, u64, C.POINTER(vp)]
    L.frz_groups_set.argtypes = [vp, vp, vp, u64]
    L.frz_groups_count.restype = u64
    L.frz_groups_count.argtypes = [vp]
    L.frz_groups_destroy.argtypes = [vp]
    L.frz_groups_destroy.restype = None
    L.frz_match_list_collapsed.argtypes = [vp, vp, vp, vp, vp, u64, u64, vp, C.POINTER(u64), C.POINTER(u64), vp]
    L.frz_match_list_columns.argtypes = [vp, vp, u64, C.c_uint8, vp, vp, vp, u64, u64, vp, C.POINTER(u64), C.POINTER(u64), vp]
    L.frz_match_list_columns_ordered.argtypes = [vp, vp, u64, C.c_uint8, vp, vp, vp, u32, vp, u64, u64, vp, C.POINTER(u64),
                                                 C.POINTER(u64), vp]
    L.frz_match_list_batch_columns.argtypes = [vp, u64, vp, u64, C.c_uint8, vp, vp, vp, vp, u64, vp, vp, vp, vp]
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

    def remove(self, which) -> "Corpus":
        """Haystacks `which` stop matching; indices do not move (len(self) is unchanged).  Duplicates are allowed."""
        which = np.ascontiguousarray(which, dtype=np.uint32)
        _check(lib().frz_corpus_remove(self._h, which.ctypes.data if which.size else None, len(which)))
        return self

    def replace(self, which, data: np.ndarray, offsets: np.ndarray) -> "Corpus":
        """Haystack which[j] becomes data[offsets[j], offsets[j + 1]) (Arrow value bytes + offsets); a removed one comes
        back.  Only the tiles holding `which` are re-packed."""
        which = np.ascontiguousarray(which, dtype=np.uint32)
        data = np.ascontiguousarray(data, dtype=np.uint8)
        offsets, width = _arrow_offsets(offsets)
        if len(offsets) != len(which) + 1:
            raise ValueError(f"{len(which)} indices need {len(which) + 1} offsets, got {len(offsets)}")
        _check(lib().frz_corpus_replace(self._h, which.ctypes.data if which.size else None, len(which),
                                        data.ctypes.data if data.size else None, offsets.ctypes.data, width))
        return self

    def replace_list(self, which, haystacks: Sequence) -> "Corpus":
        data, offsets = pack_host(haystacks)
        return self.replace(which, data, offsets)

    def subset(self, which) -> "Subset":
        """The rows `which` (any order, duplicates allowed) as a resident subset for Matcher.match_list_subset_array and
        match_list_subset_top_array.  Close it before the corpus."""
        which = np.ascontiguousarray(which, dtype=np.uint32)
        h = C.c_void_p()
        _check(lib().frz_subset_create(self._h, which.ctypes.data if which.size else None, len(which), C.byref(h)))
        return Subset(h, self)

    def attr(self, values=None) -> "Attr":
        """A resident int64 attribute per row for Corpus.where / Subset.where: values[i] is the value of row i, rows past
        len(values) (and values equal to ATTR_NULL) have none; at most len(self) values.  Close it before the corpus."""
        values = np.ascontiguousarray(np.zeros(0, np.int64) if values is None else values, dtype=np.int64)
        h = C.c_void_p()
        _check(lib().frz_attr_create(self._h, values.ctypes.data if values.size else None, len(values), C.byref(h)))
        return Attr(h, self)

    def where(self, *clauses: "Where", base: Optional["Subset"] = None) -> "Subset":
        """A new subset of the rows for which every clause holds (and which are members of `base`, when given), filled on
        the device (frz_subset_where).  Close it before the corpus."""
        return self.subset([]).where(*clauses, base=base)

    def matching(self, matcher: "Matcher", text: Optional["Corpus"] = None, base: Optional["Subset"] = None) -> "Subset":
        """A new subset of the rows of matcher.match_list_into over `text` (this corpus when None; another corpus must have
        as many rows), restricted to `base` when given, filled on the device from the prefilter stage alone
        (frz_subset_match).  Close it before the corpus."""
        return self.subset([]).matching(matcher, text=text, base=base)

    def text(self, desc: bool = False, fold_case: bool = False) -> "RankKey":
        """The rows' haystacks as a key of Corpus.rank / Attr.rank: bytewise (memcmp) order, a proper prefix first; desc
        reverses it, fold_case compares ASCII A-Z as a-z."""
        return RankKey(text=self, desc=desc, fold_case=fold_case)

    def rank(self, *keys: "RankKey") -> "Attr":
        """A new attribute holding each row's dense rank in the lexicographic order of `keys` (at most RANK_MAX_KEYS, each
        Attr.asc() / Attr.desc() or Corpus.text(...) of a corpus with as many rows), filled on the device
        (frz_attr_rank).  Rows removed here or in a text key's corpus have no value.  Close it before the corpus."""
        return self.attr().rank(*keys)

    def boost(self, values=None) -> "Boost":
        """A resident per-row boost for Matcher.match_list_ranked_array: values[i] (int16) is the boost of row i, rows
        past len(values) have 0; at most len(self) values.  Close it before the corpus."""
        values = np.ascontiguousarray(np.zeros(0, np.int16) if values is None else values, dtype=np.int16)
        h = C.c_void_p()
        _check(lib().frz_boost_create(self._h, values.ctypes.data if values.size else None, len(values), C.byref(h)))
        return Boost(h, self)

    def groups(self, ids=None, n_groups: Optional[int] = None) -> "Groups":
        """A resident group id per row for Matcher.match_list_collapsed_array: ids[i] (uint32) is the group of row i, or
        GROUP_NONE; rows past len(ids) are in no group; at most len(self) ids.  n_groups defaults to one more than the
        largest id that is not GROUP_NONE (1 when there is none).  Close it before the corpus."""
        ids = np.ascontiguousarray(np.zeros(0, np.uint32) if ids is None else ids, dtype=np.uint32)
        if n_groups is None:
            real = ids[ids != GROUP_NONE]
            n_groups = int(real.max()) + 1 if real.size else 1
        h = C.c_void_p()
        _check(lib().frz_groups_create(self._h, ids.ctypes.data if ids.size else None, len(ids), int(n_groups), C.byref(h)))
        return Groups(h, self)

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


class Subset:
    """A chosen set of rows of one resident Corpus (frz_subset); membership is by index and survives corpus edits."""

    def __init__(self, handle, corpus: Corpus):
        self._h = handle
        self.corpus = corpus

    def __len__(self):
        return lib().frz_subset_len(self._h)

    def where(self, *clauses: "Where", base: Optional["Subset"] = None) -> "Subset":
        """Refills this subset with the rows of its corpus for which every clause holds and which are members of `base`
        (when given; it may be this subset), on the device (frz_subset_where).  Returns self."""
        _check(lib().frz_subset_where(self._h, _where_clauses(clauses) if clauses else None, len(clauses),
                                      base._h if base is not None else None))
        return self

    def matching(self, matcher: "Matcher", text: Optional[Corpus] = None, base: Optional["Subset"] = None) -> "Subset":
        """Refills this subset with the indices of the rows of matcher.match_list_into over `text` (its corpus when None;
        another corpus must have as many rows) that are members of `base` (when given; it may be this subset), on the
        device from the prefilter stage alone (frz_subset_match).  For example
        Matcher.from_query("^src/ .rs$ !test", cfg) keeps the Rust files under src/ outside test paths; the matcher's
        config decides case, unicode and typos.  Returns self."""
        _check(lib().frz_subset_match(self._h, matcher._h, text._h if text is not None else None,
                                      base._h if base is not None else None))
        return self

    def close(self):
        if self._h:
            lib().frz_subset_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _RowValues:
    """A value per row of one resident Corpus, kept by index across corpus edits: the part Boost, Attr and Groups share."""
    _dtype, _what, _set_fn, _destroy_fn = None, "values", "", ""

    def __init__(self, handle, corpus: Corpus):
        self._h = handle
        self.corpus = corpus

    def _set(self, which, values):
        which = np.ascontiguousarray(which, dtype=np.uint32)
        values = np.ascontiguousarray(values, dtype=self._dtype)
        if len(values) != len(which):
            raise ValueError(f"{len(which)} indices need {len(which)} {self._what}, got {len(values)}")
        _check(getattr(lib(), self._set_fn)(self._h, which.ctypes.data if which.size else None,
                                            values.ctypes.data if values.size else None, len(which)))
        return self

    def close(self):
        if self._h:
            getattr(lib(), self._destroy_fn)(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Boost(_RowValues):
    """A signed 16-bit boost per row of one resident Corpus (frz_boost), kept by index across corpus edits."""
    _dtype, _set_fn, _destroy_fn = np.int16, "frz_boost_set", "frz_boost_destroy"

    def set(self, which, values) -> "Boost":
        """boost[which[j]] = values[j]; any row below len(corpus), appended ones included, each at most once."""
        return self._set(which, values)

    def where(self, *rules: "BoostRule", base: Optional["Boost"] = None) -> "Boost":
        """Refills this boost on the device (frz_boost_where): row i's boost becomes base's boost of i (0 without a base;
        it may be this boost) plus the add of every rule whose clause holds for i, clamped to int16.  At most
        BOOST_MAX_RULES rules.  Returns self."""
        _check(lib().frz_boost_where(self._h, _boost_rules(rules) if rules else None, len(rules),
                                     base._h if base is not None else None))
        return self

    def values(self) -> np.ndarray:
        """The boost of every row below len(corpus), 0 where there is none (frz_boost_get)."""
        out = np.empty(max(1, self.corpus.n), np.int16)
        _check(lib().frz_boost_get(self._h, out.ctypes.data, self.corpus.n))
        return out[: self.corpus.n]


class _CWhereClause(C.Structure):
    _fields_ = [("attr", C.c_void_p), ("lo", C.c_int64), ("hi", C.c_int64), ("in_", C.c_void_p), ("n_in", C.c_uint64),
                ("negate", C.c_int32)]


def _where_clauses(clauses):
    """frz_where_clause records of a sequence of Where (their set values stay owned by the Where objects)."""
    arr = (_CWhereClause * max(1, len(clauses)))()
    for j, w in enumerate(clauses):
        arr[j].attr = w.attr._h
        arr[j].lo, arr[j].hi = w.lo, w.hi
        arr[j].in_ = w.values.ctypes.data if w.values is not None and w.values.size else None
        arr[j].n_in = 0 if w.values is None else len(w.values)
        arr[j].negate = int(w.negate)
    return arr


class Where:
    """One clause of Corpus.where / Subset.where (frz_where_clause): lo <= v <= hi, or v in values, v being a row's value in
    `attr`; ~clause holds where the test fails.  A row without a value fails every clause, negated or not."""

    def __init__(self, attr: "Attr", lo: int = 0, hi: int = -1, values=None, negate: bool = False):
        self.attr, self.lo, self.hi, self.negate = attr, int(lo), int(hi), bool(negate)
        self.values = None if values is None else np.ascontiguousarray(values, dtype=np.int64)

    def __invert__(self) -> "Where":
        return Where(self.attr, self.lo, self.hi, self.values, not self.negate)

    def add(self, n: int) -> "BoostRule":
        """The rule of Boost.where that adds n (-65535 .. 65535) to the boost of every row for which this clause holds."""
        return BoostRule(self, n)


class BoostRule:
    """One rule of Boost.where / boost_where_batch (frz_boost_rule): `add` for every row for which `when` holds."""

    def __init__(self, when: Where, add: int):
        self.when, self.add = when, int(add)


class _CBoostRule(C.Structure):
    _fields_ = [("when", _CWhereClause), ("add", C.c_int32)]


def _boost_rules(rules):
    """frz_boost_rule records of a sequence of BoostRule (their set values stay owned by the Where objects)."""
    clauses = _where_clauses([r.when for r in rules])
    arr = (_CBoostRule * max(1, len(rules)))()
    for j, r in enumerate(rules):
        arr[j].when = clauses[j]
        arr[j].add = r.add
    return arr


class Attr(_RowValues):
    """A signed 64-bit value per row of one resident Corpus (frz_attr), kept by index across corpus edits."""
    _dtype, _set_fn, _destroy_fn = np.int64, "frz_attr_set", "frz_attr_destroy"

    def set(self, which, values) -> "Attr":
        """value[which[j]] = values[j] (ATTR_NULL clears it); any row below len(corpus), appended ones included, each at
        most once."""
        return self._set(which, values)

    def between(self, lo: int, hi: int) -> Where:
        """The clause lo <= v <= hi (it holds for no value when lo > hi)."""
        return Where(self, lo, hi)

    def isin(self, values) -> Where:
        """The clause "v is one of values" (any order, duplicates allowed; an empty list holds for no value)."""
        values = np.ascontiguousarray(values, dtype=np.int64)
        return Where(self, values=values) if values.size else Where(self, 0, -1)

    def values(self) -> np.ndarray:
        """The value of every row below len(corpus), ATTR_NULL where there is none (frz_attr_get)."""
        out = np.empty(max(1, self.corpus.n), np.int64)
        _check(lib().frz_attr_get(self._h, out.ctypes.data, self.corpus.n))
        return out[: self.corpus.n]

    def asc(self) -> "RankKey":
        """This attribute as a key of Corpus.rank / Attr.rank, smaller values first (a row without a value last)."""
        return RankKey(attr=self)

    def desc(self) -> "RankKey":
        """This attribute as a key of Corpus.rank / Attr.rank, larger values first (a row without a value last)."""
        return RankKey(attr=self, desc=True)

    def rank(self, *keys: "RankKey") -> "Attr":
        """Refills this attribute with each row's dense rank in the lexicographic order of `keys` (Corpus.rank); it may
        be one of the keys.  Returns self."""
        arr = (_CRankKey * max(1, len(keys)))()
        for j, k in enumerate(keys):
            arr[j].attr = k.attr._h if k.attr is not None else None
            arr[j].text = k.text._h if k.text is not None else None
            arr[j].desc, arr[j].fold_case = int(k.desc), int(k.fold_case)
        _check(lib().frz_attr_rank(self._h, arr if keys else None, len(keys)))
        return self


class _CRankKey(C.Structure):
    _fields_ = [("attr", C.c_void_p), ("text", C.c_void_p), ("desc", C.c_uint32), ("fold_case", C.c_uint32)]


class RankKey:
    """One key of Corpus.rank / Attr.rank (frz_rank_key): an attribute (Attr.asc / Attr.desc) or the haystacks of a corpus
    (Corpus.text)."""

    def __init__(self, attr: Optional["Attr"] = None, text: Optional[Corpus] = None, desc: bool = False, fold_case: bool = False):
        self.attr, self.text, self.desc, self.fold_case = attr, text, bool(desc), bool(fold_case)


class Groups(_RowValues):
    """A group id per row of one resident Corpus (frz_groups), kept by index across corpus edits."""
    _dtype, _what, _set_fn, _destroy_fn = np.uint32, "ids", "frz_groups_set", "frz_groups_destroy"

    def set(self, which, ids) -> "Groups":
        """group[which[j]] = ids[j] (an id below len(self), or GROUP_NONE); any row below len(corpus), appended ones
        included, each at most once."""
        return self._set(which, ids)

    def __len__(self):
        return lib().frz_groups_count(self._h)


def _top_out(out: Optional[np.ndarray], k: Optional[int], n: int, subset: Optional["Subset"], what: str):
    """(k, out) for a call that returns the first k rows of n (and of the subset's members): k=None is every row; `out`, when
    given, must hold min(k, n, len(subset)) matches (`what` names the call in the error), else a new array that does."""
    k = _U64_MAX if k is None else int(k)
    need = min(k, n, len(subset) if subset is not None else n)
    if out is None:
        return k, np.empty(max(1, need), dtype=MATCH_DTYPE)
    if len(out) < need:
        raise ValueError(f"out holds {len(out)} matches; {what} needs {need}")
    return k, out


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
            k, out = _top_out(out, k, corpus.n, None, f"a top-{k} call on {corpus.n} haystacks")
            n, total = C.c_uint64(), C.c_uint64()
            _check(lib().frz_match_list_top(self._h, corpus._h, k, out.ctypes.data, C.byref(n), C.byref(total)))
            return out[: n.value], total.value
        finally:
            if owned:
                corpus.close()

    def match_list_subset_array(self, corpus: Corpus, subset: Subset, out: Optional[np.ndarray] = None) -> np.ndarray:
        """match_list_array(corpus) restricted to the subset's members (frz_match_list_subset), in the same order."""
        if out is None:
            out = np.empty(max(1, len(subset)), dtype=MATCH_DTYPE)
        n = C.c_uint64()
        _check(lib().frz_match_list_subset(self._h, corpus._h, subset._h, out.ctypes.data, len(out), C.byref(n)))
        return out[: n.value]

    def match_list_subset_top_array(self, corpus: Corpus, subset: Subset, k: int) -> Tuple[np.ndarray, int]:
        """The first k rows of match_list_subset_array (frz_match_list_subset_top): (array of min(k, total) matches, total)."""
        k, out = _top_out(None, k, corpus.n, subset, "")
        n, total = C.c_uint64(), C.c_uint64()
        _check(lib().frz_match_list_subset_top(self._h, corpus._h, subset._h, k, out.ctypes.data, C.byref(n), C.byref(total)))
        return out[: n.value], total.value

    def match_list_ranked_array(self, corpus: Corpus, boost: Boost, k: Optional[int] = None, subset: Optional[Subset] = None,
                                out: Optional[np.ndarray] = None) -> Tuple[np.ndarray, int]:
        """The rows of match_list_array(corpus) (or of its subset), ranked by clamp(score + boost[index], 0, 65535), ties in
        the strategy's index order, truncated to the first k (frz_match_list_ranked): (array of min(k, total) rows, total).
        k=None ranks the whole list.  `out` (optional) needs room for min(k, len(corpus), len(subset)) rows."""
        k, out = _top_out(out, k, corpus.n, subset, "this ranked call")
        n, total = C.c_uint64(), C.c_uint64()
        _check(lib().frz_match_list_ranked(self._h, corpus._h, subset._h if subset is not None else None, boost._h, k,
                                           out.ctypes.data, C.byref(n), C.byref(total)))
        return out[: n.value], total.value

    def match_list_ordered_array(self, corpus: Corpus, attr: Attr, order: Order = Order.AttrDesc, k: Optional[int] = None,
                                 subset: Optional[Subset] = None, boost: Optional[Boost] = None,
                                 out: Optional[np.ndarray] = None, groups: Optional[Groups] = None,
                                 per_group: Optional[int] = 1, counts: bool = False):
        """The rows of match_list_array(corpus) (or of its subset) ordered by attr (frz_match_list_ordered): by value
        (Order.AttrDesc / AttrAsc) or by score, clamp(score + boost[index], 0, 65535) with a boost, then by value
        (ScoreThenAttrDesc / Asc); rows without a value go last, and remaining ties keep the strategy's index order.
        Truncated to the first k: (array of min(k, total) rows, total).  k=None orders the whole list.  `out` (optional)
        needs room for min(k, len(corpus), len(subset)) rows.
        With groups, the ordered list is collapsed first (frz_match_list_ordered_collapsed): in its order, the rows in no
        group and the first per_group rows of each group are kept (per_group 1..32, or None for no cap), so per_group=1
        gives each group's first row by the attribute, e.g. its newest.  Returns (rows, total), total counting the kept
        rows, or (rows, total, counts) with counts=True: the ordered list's rows per group, before collapsing."""
        k, out = _top_out(out, k, corpus.n, subset, "this ordered call")
        n, total = C.c_uint64(), C.c_uint64()
        sh, bh = subset._h if subset is not None else None, boost._h if boost is not None else None
        if groups is None:
            if counts:
                raise ValueError("counts=True needs groups")
            _check(lib().frz_match_list_ordered(self._h, corpus._h, sh, bh, attr._h, int(order), k, out.ctypes.data, C.byref(n),
                                                C.byref(total)))
            return out[: n.value], total.value
        per_group = _U64_MAX if per_group is None else int(per_group)
        cnt = np.zeros(len(groups), dtype=np.uint32) if counts else None
        _check(lib().frz_match_list_ordered_collapsed(self._h, corpus._h, sh, bh, attr._h, int(order), groups._h, per_group, k,
                                                      out.ctypes.data, C.byref(n), C.byref(total),
                                                      cnt.ctypes.data if counts else None))
        if counts:
            return out[: n.value], total.value, cnt
        return out[: n.value], total.value

    def match_list_collapsed_array(self, corpus: Corpus, groups: Groups, k: Optional[int] = None,
                                   per_group: Optional[int] = 1, subset: Optional[Subset] = None, boost: Optional[Boost] = None,
                                   counts: bool = False, out: Optional[np.ndarray] = None):
        """The rows of the uncollapsed list L (match_list_ranked_array(corpus, boost, subset=subset) with a boost, else
        match_list_subset_array with a subset, else match_list_array), keeping in L's order the rows in no group and the
        first per_group rows of each group, truncated to the first k (frz_match_list_collapsed).  Returns (rows, total), or
        (rows, total, counts) with counts=True: the rows of L per group (uint32, len(groups) entries), before collapsing.
        k=None returns every kept row; per_group is 1..32, or None for no cap.  `out` (optional) needs room for
        min(k, len(corpus), len(subset)) rows."""
        k, out = _top_out(out, k, corpus.n, subset, "this collapsed call")
        per_group = _U64_MAX if per_group is None else int(per_group)
        cnt = np.zeros(len(groups), dtype=np.uint32) if counts else None
        n, total = C.c_uint64(), C.c_uint64()
        _check(lib().frz_match_list_collapsed(self._h, corpus._h, subset._h if subset is not None else None,
                                              boost._h if boost is not None else None, groups._h, per_group, k, out.ctypes.data,
                                              C.byref(n), C.byref(total), cnt.ctypes.data if counts else None))
        if counts:
            return out[: n.value], total.value, cnt
        return out[: n.value], total.value

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


class _BatchArgs:
    """The per-query arrays of a batched call: one handle or NULL per query for subsets / boosts (NULL for None), and the
    (q, k) rows, n_out and n_total; grouped() adds those of a call that may collapse."""

    def __init__(self, q: int, k: int, subsets=None, boosts=None):
        self.q = q
        self.hs, self.hb = _handles(subsets, q, "subsets"), _handles(boosts, q, "boosts")
        self.counts = None
        self.out = np.zeros((q, k), dtype=MATCH_DTYPE)
        self.n_out = np.zeros(q, dtype=np.uint64)
        self.n_total = np.zeros(q, dtype=np.uint64)

    def grouped(self, groups, per_group, counts: bool, who: str) -> "_BatchArgs":
        """groups (None, or one Groups / None per query), per_group (an int, None for no cap, or one such value per query) as
        uint64, and with counts=True a count array per query with groups and their pointers.  who: the queries' name in
        the errors."""
        q = self.q
        groups = list(groups) if groups is not None else [None] * q
        self.hg = _handles(groups, q, "groups")
        if per_group is None or isinstance(per_group, (int, np.integer)):
            per_group = [per_group] * q
        per_group = list(per_group)
        if len(per_group) != q:
            raise ValueError(f"{q} {who} need {q} per_group values, got {len(per_group)}")
        self.pg = np.array([_U64_MAX if p is None else int(p) for p in per_group] or [1], dtype=np.uint64)
        self.counts = [np.zeros(len(g), dtype=np.uint32) if g is not None else None for g in groups] if counts else None
        self.hc = (C.c_void_p * max(q, 1))(*[c.ctypes.data if c is not None else None for c in self.counts]) if counts else None
        return self

    def outputs(self):
        """out (NULL when q * k = 0), n_out, n_total."""
        return self.out.ctypes.data if self.out.size else None, self.n_out.ctypes.data, self.n_total.ctypes.data

    def result(self):
        """(rows, n_out, n_total), and the counts with counts=True."""
        r = (self.out, self.n_out.astype(np.int64), self.n_total.astype(np.int64))
        return r + (self.counts,) if self.counts is not None else r


def _handles(xs, q: int, what: str):
    """One handle (or NULL) per query of a batched call, or NULL for xs = None."""
    if xs is None:
        return None
    xs = list(xs)
    if len(xs) != q:
        raise ValueError(f"{q} matchers need {q} {what}, got {len(xs)}")
    return (C.c_void_p * max(q, 1))(*[x._h.value if x is not None else None for x in xs])


def _matcher_array(matchers):
    return (C.c_void_p * max(len(matchers), 1))(*[m._h.value for m in matchers])


def match_list_batch_top(matchers, corpus: Corpus, k: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """frz_match_list_batch_top: every matcher's match_list_top_array(corpus, k) in one call.  Returns a (q, k) array of
    MATCH_DTYPE (row j's first n_out[j] entries are matcher j's rows; the rest are zero), n_out and n_total (int64, length q)."""
    q, k = len(matchers), int(k)
    b = _BatchArgs(q, k)
    _check(lib().frz_match_list_batch_top(_matcher_array(matchers), q, corpus._h, k, *b.outputs()))
    return b.result()


def match_list_batch(matchers, corpus: Corpus, k: int, subsets=None, boosts=None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """frz_match_list_batch: match_list_batch_top where query j may have its own subset and boost.  subsets / boosts: None,
    or one Subset / Boost / None per matcher.  Query j's rows are those of matcher j's match_list_ranked_array(corpus,
    boosts[j], k, subsets[j]) when it has a boost, else of match_list_subset_top_array(corpus, subsets[j], k) when it has
    a subset, else of match_list_top_array(corpus, k).  Returns the (q, k) rows, n_out and n_total as match_list_batch_top."""
    q, k = len(matchers), int(k)
    b = _BatchArgs(q, k, subsets, boosts)
    _check(lib().frz_match_list_batch(_matcher_array(matchers), q, corpus._h, b.hs, b.hb, k, *b.outputs()))
    return b.result()


def match_list_batch_collapsed(matchers, corpus: Corpus, k: int, groups, per_group=1, subsets=None, boosts=None, counts: bool = False):
    """frz_match_list_batch_collapsed: match_list_batch where query j may also collapse its rows by groups[j].  groups: one
    Groups or None per matcher; per_group: an int (1..32), None (no cap), or one such value per matcher.  Query j's rows are
    those of matcher j's match_list_collapsed_array(corpus, groups[j], k, per_group[j], subsets[j], boosts[j]) when it has
    groups, else those of match_list_batch.  Returns the (q, k) rows, n_out and n_total as match_list_batch_top, and with
    counts=True also a list of each query's rows per group (uint32, len(groups[j]) entries; None for a query without groups)."""
    q, k = len(matchers), int(k)
    b = _BatchArgs(q, k, subsets, boosts).grouped(groups, per_group, counts, "matchers")
    _check(lib().frz_match_list_batch_collapsed(_matcher_array(matchers), q, corpus._h, b.hs, b.hb, b.hg, b.pg.ctypes.data, k,
                                                *b.outputs(), b.hc))
    return b.result()


def match_list_batch_ordered(matchers, corpus: Corpus, k: int, attrs, order=Order.AttrDesc, subsets=None, boosts=None, groups=None,
                             per_group=1, counts: bool = False):
    """frz_match_list_batch_ordered: match_list_batch_collapsed where query j may also order its rows by attrs[j].  attrs:
    one Attr for every query, or one Attr or None per matcher; order: one Order, or one per matcher.  Query j's rows are
    those of matcher j's match_list_ordered_array(corpus, attrs[j], order[j], k, subsets[j], boosts[j], groups=groups[j],
    per_group=per_group[j]) when it has an attribute, else those of match_list_batch_collapsed.  Returns the (q, k) rows,
    n_out and n_total as match_list_batch_top, and with counts=True also a list of each query's rows per group (uint32,
    len(groups[j]) entries; None for a query without groups)."""
    q, k = len(matchers), int(k)
    if attrs is None or isinstance(attrs, Attr):
        attrs = [attrs] * q
    if isinstance(order, (int, np.integer)):
        order = [order] * q
    order = list(order)
    if len(order) != q:
        raise ValueError(f"{q} matchers need {q} orders, got {len(order)}")
    b = _BatchArgs(q, k, subsets, boosts).grouped(groups, per_group, counts, "matchers")
    ha = _handles(attrs, q, "attrs")
    orders = np.array([int(o) for o in order] or [0], dtype=np.uint32)
    _check(lib().frz_match_list_batch_ordered(_matcher_array(matchers), q, corpus._h, b.hs, b.hb, ha, orders.ctypes.data, b.hg,
                                              b.pg.ctypes.data, k, *b.outputs(), b.hc))
    return b.result()


def where_batch(subsets, clauses, bases=None):
    """frz_subset_where_batch: subsets[j].where(*clauses[j], base=bases[j]) for every j in one call, each subset bit for
    bit what its own call leaves.  subsets: distinct Subset objects of one corpus; clauses: one sequence of Where per
    subset; bases: None, or one Subset or None per subset (a subset's own handle refines it in place; another query's
    subset is refused).  Returns subsets."""
    subsets = list(subsets)
    clauses = [list(c) for c in clauses]
    q = len(subsets)
    if len(clauses) != q:
        raise ValueError(f"{q} subsets need {q} clause lists, got {len(clauses)}")
    flat = [w for c in clauses for w in c]
    counts = np.array([len(c) for c in clauses] or [0], dtype=np.uint64)
    hs = (C.c_void_p * max(q, 1))(*[s._h.value for s in subsets])
    hb = None
    if bases is not None:
        bases = list(bases)
        if len(bases) != q:
            raise ValueError(f"{q} subsets need {q} bases, got {len(bases)}")
        hb = (C.c_void_p * max(q, 1))(*[b._h.value if b is not None else None for b in bases])
    _check(lib().frz_subset_where_batch(hs, q, _where_clauses(flat) if flat else None, counts.ctypes.data, hb))
    return subsets


def boost_where_batch(boosts, rules, bases=None):
    """frz_boost_where_batch: boosts[j].where(*rules[j], base=bases[j]) for every j in one call, each boost bit for bit
    what its own call leaves (values and key bound).  boosts: distinct Boost objects of one corpus; rules: one sequence of
    BoostRule per boost; bases: None, or one Boost or None per boost (a boost's own handle adds to it in place; another
    query's boost is refused).  Returns boosts."""
    boosts = list(boosts)
    rules = [list(r) for r in rules]
    q = len(boosts)
    if len(rules) != q:
        raise ValueError(f"{q} boosts need {q} rule lists, got {len(rules)}")
    flat = [r for rs in rules for r in rs]
    counts = np.array([len(r) for r in rules] or [0], dtype=np.uint64)
    hs = (C.c_void_p * max(q, 1))(*[b._h.value for b in boosts])
    hb = None
    if bases is not None:
        bases = list(bases)
        if len(bases) != q:
            raise ValueError(f"{q} boosts need {q} bases, got {len(bases)}")
        hb = (C.c_void_p * max(q, 1))(*[b._h.value if b is not None else None for b in bases])
    _check(lib().frz_boost_where_batch(hs, q, _boost_rules(flat) if flat else None, counts.ctypes.data, hb))
    return boosts


def match_list_columns(matchers, columns, k: Optional[int] = None, sort: SortStrategy = SortStrategy.ScoreThenIndexAsc,
                       subset: Optional[Subset] = None, boost: Optional[Boost] = None, groups: Optional[Groups] = None,
                       per_group: Optional[int] = 1, counts: bool = False, out: Optional[np.ndarray] = None,
                       attr: Optional[Attr] = None, order: Order = Order.AttrDesc):
    """frz_match_list_columns: rows with several text fields, matcher j searching columns[j] (Corpus objects of one length:
    row i is haystack i of every column).  A row matches when it matches in every column; its score is the saturating sum
    of the column scores and its exact flag their OR.  The list is ordered by `sort` (the matchers' own sort settings are
    not read), ranked by boost when one is given, collapsed by groups when they are given (per_group 1..32, or None for no
    cap), and truncated to the first k rows.  With attr, the list is instead ordered by the attribute as
    Matcher.match_list_ordered_array orders its list (`order`; the boost, when given, goes into the score), then collapsed
    in that order when groups are given (frz_match_list_columns_ordered).  subset / boost / groups / attr may be handles of
    any of the columns.  Returns (rows, total), or (rows, total, counts) with counts=True (the list's rows per group, before
    collapsing).  k=None returns every row; `out` (optional) needs room for min(k, len(columns[0]), len(subset)) rows.  Put
    the most selective column first: the order changes only the speed."""
    matchers, columns = list(matchers), list(columns)
    if len(matchers) != len(columns):
        raise ValueError(f"{len(matchers)} matchers for {len(columns)} columns")
    k, out = _top_out(out, k, columns[0].n if columns else 0, subset, "this columns call")
    per_group = _U64_MAX if per_group is None else int(per_group)
    if counts and groups is None:
        raise ValueError("counts=True needs groups")
    cnt = np.zeros(len(groups), dtype=np.uint32) if counts else None
    q = len(matchers)
    cs = (C.c_void_p * max(q, 1))(*[c._h.value for c in columns])
    n_out, total = C.c_uint64(), C.c_uint64()
    sh, bh, gh = (h._h if h is not None else None for h in (subset, boost, groups))
    tail = (per_group, k, out.ctypes.data, C.byref(n_out), C.byref(total), cnt.ctypes.data if counts else None)
    if attr is None:
        _check(lib().frz_match_list_columns(_matcher_array(matchers), cs, q, int(sort), sh, bh, gh, *tail))
    else:
        _check(lib().frz_match_list_columns_ordered(_matcher_array(matchers), cs, q, int(sort), sh, bh, attr._h, int(order), gh,
                                                    *tail))
    if counts:
        return out[: n_out.value], total.value, cnt
    return out[: n_out.value], total.value


def match_list_batch_columns(matchers, columns, k: int, sort: SortStrategy = SortStrategy.ScoreThenIndexAsc, subsets=None,
                             boosts=None, groups=None, per_group=1, counts: bool = False):
    """frz_match_list_batch_columns: match_list_columns for many queries over the same columns in one call.  matchers: q
    sequences of len(columns) matchers, matchers[j][c] searching columns[c].  subsets / boosts / groups: None, or one handle
    (of any column) or None per query; per_group: an int (1..32), None (no cap), or one such value per query.  Query j's
    rows are those of match_list_columns(matchers[j], columns, k, sort, subsets[j], boosts[j], groups[j], per_group[j]).
    Returns the (q, k) rows, n_out and n_total as match_list_batch_top, and with counts=True also a list of each query's
    rows per group (uint32, len(groups[j]) entries; None for a query without groups)."""
    matchers, columns = [list(m) for m in matchers], list(columns)
    q, k, n_cols = len(matchers), int(k), len(columns)
    for j, mj in enumerate(matchers):
        if len(mj) != n_cols:
            raise ValueError(f"query {j} has {len(mj)} matchers for {n_cols} columns")
    b = _BatchArgs(q, k, subsets, boosts).grouped(groups, per_group, counts, "queries")
    cs = (C.c_void_p * max(n_cols, 1))(*[c._h.value for c in columns])
    _check(lib().frz_match_list_batch_columns(_matcher_array([m for mj in matchers for m in mj]), q, cs, n_cols, int(sort), b.hs, b.hb,
                                              b.hg, b.pg.ctypes.data, k, *b.outputs(), b.hc))
    return b.result()


def batch_last() -> dict:
    """Test aid (frz_debug_batch_last): what this thread's last batched call (match_list_batch_top, match_list_batch,
    match_list_batch_collapsed, match_list_batch_ordered or match_list_batch_columns) did."""
    v = np.zeros(4, dtype=np.uint64)
    lib().frz_debug_batch_last(v.ctypes.data)
    return {"batched": int(v[0]), "overflowed": int(v[1]), "sub_batches": int(v[2]), "launches": int(v[3])}


def batch_limits(max_rows: int = 0, min_queries: int = 0):
    """Test aid (frz_debug_batch_limits): the batched path's corpus-size and query-count limits; 0 restores a default."""
    lib().frz_debug_batch_limits(int(max_rows), int(min_queries))


def subset_match_debug(force: Optional[str] = None) -> int:
    """Test aid (frz_debug_subset_match): force="masked" prefilters every pattern of Subset.matching after the first (and
    the first with a base) through slot metadata masked to the members so far, "full" never does, "rule" restores the
    rule, None changes nothing.  Returns how many patterns this thread's last fill prefiltered masked."""
    code = {None: -1, "rule": 0, "masked": 1, "full": 2}[force]
    return int(lib().frz_debug_subset_match(code))


def where_batch_debug(force: Optional[bool] = None) -> bool:
    """Test aid (frz_debug_where_batch): force=True runs where_batch's batched kernels at every shape, False restores the
    rule, None changes nothing.  Returns whether this thread's last where_batch ran the batched kernels."""
    return bool(lib().frz_debug_where_batch(-1 if force is None else int(force)))


def radix_sort_matches(arr: np.ndarray, device: int = 0) -> np.ndarray:
    """radix_sort_matches (src/sort.rs:6-40) on the GPU: stable, descending score."""
    arr = np.ascontiguousarray(arr, dtype=MATCH_DTYPE).copy()
    _check(lib().frz_radix_sort_matches(arr.ctypes.data, len(arr), device))
    return arr
