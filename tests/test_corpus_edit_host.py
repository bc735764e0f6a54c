"""Argument checks of the in-place corpus edits (frz_corpus_remove / frz_corpus_replace), which run on the host before
anything touches a device or the corpus.  A zero-filled block stands in for the corpus handle: the checks below must
return before the corpus is read, and on a machine without a GPU any CUDA call would fail with FRZ_ERR_NO_DEVICE, so an
FRZ_OK for n == 0 shows that no CUDA call was made.  The behaviour on a real corpus is in tests/test_gpu_corpus_edit.py."""
import ctypes

import numpy as np

import frizbee_b200 as F

INVALID_ARG = 1


def test_corpus_edit_argument_checks():
    L = F.lib()
    fake = ctypes.create_string_buffer(4096)          # never read by the checks below
    c = ctypes.addressof(fake)
    which = np.array([0, 1], dtype=np.uint32)
    data = np.frombuffer(b"abcd", dtype=np.uint8).copy()
    off64 = np.array([0, 2, 4], dtype=np.uint64)
    off32 = off64.astype(np.uint32)
    w, d, o = which.ctypes.data, data.ctypes.data, off64.ctypes.data

    # a NULL corpus
    assert L.frz_corpus_remove(None, w, 2) == INVALID_ARG
    assert L.frz_corpus_remove(None, None, 0) == INVALID_ARG
    assert L.frz_corpus_replace(None, w, 2, d, o, 8) == INVALID_ARG
    assert L.frz_corpus_replace(None, None, 0, None, None, 8) == INVALID_ARG
    assert b"null" in L.frz_last_error()
    # NULL arrays with n > 0
    assert L.frz_corpus_remove(c, None, 1) == INVALID_ARG
    assert L.frz_corpus_replace(c, None, 2, d, o, 8) == INVALID_ARG
    assert L.frz_corpus_replace(c, w, 2, d, None, 8) == INVALID_ARG
    assert b"null" in L.frz_last_error()
    # a bad offset width, with and without work to do
    for width in (0, 2, 3, 7, 16, -4):
        assert L.frz_corpus_replace(c, w, 2, d, off32.ctypes.data, width) == INVALID_ARG
        assert L.frz_corpus_replace(c, None, 0, None, None, width) == INVALID_ARG
    assert b"offset_width" in L.frz_last_error()
    # n == 0 is a no-op: OK without a device, the corpus untouched (NULL arrays are fine then)
    assert L.frz_corpus_remove(c, None, 0) == 0
    assert L.frz_corpus_remove(c, w, 0) == 0
    for width, off in ((8, o), (4, off32.ctypes.data), (8, None)):
        assert L.frz_corpus_replace(c, None, 0, None, off, width) == 0
        assert L.frz_corpus_replace(c, w, 0, d, off, width) == 0
    assert fake.raw == b"\0" * 4096


def test_corpus_edit_python_wrappers_check_their_shapes():
    """Corpus.replace refuses offsets that do not match the index count before it calls the library."""
    corpus = F.Corpus(None, 0)
    try:
        corpus.replace([0, 1], np.zeros(4, dtype=np.uint8), np.array([0, 4], dtype=np.uint64))
    except ValueError as e:
        assert "offsets" in str(e)
    else:
        raise AssertionError("a replace with too few offsets was accepted")
