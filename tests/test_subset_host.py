"""Argument checks of the subset calls (frz_subset_create, frz_match_list_subset, frz_match_list_subset_top), which run on
the host before anything touches a device.  A zero-filled block stands in for the corpus and matcher handles: the checks
below return before either is read.  The behaviour on a real corpus is in tests/test_gpu_subset.py."""
import ctypes

import numpy as np

import frizbee_b200 as F

INVALID_ARG = 1


def test_subset_argument_checks():
    L = F.lib()
    fake = ctypes.create_string_buffer(4096)          # never read by the checks below
    c = ctypes.addressof(fake)
    which = np.array([0, 1], dtype=np.uint32)
    h = ctypes.c_void_p()
    n, total = ctypes.c_uint64(), ctypes.c_uint64()
    # frz_subset_create: NULL corpus, NULL out, NULL indices with n > 0
    assert L.frz_subset_create(None, which.ctypes.data, 2, ctypes.byref(h)) == INVALID_ARG
    assert L.frz_subset_create(c, which.ctypes.data, 2, None) == INVALID_ARG
    assert L.frz_subset_create(c, None, 1, ctypes.byref(h)) == INVALID_ARG
    assert b"null" in L.frz_last_error() and not h.value
    # the match calls: a NULL matcher, corpus or subset
    for args in ((None, c, c), (c, None, c), (c, c, None)):
        assert L.frz_match_list_subset(*args, None, 0, ctypes.byref(n)) == INVALID_ARG
        assert L.frz_match_list_subset_top(*args, 0, None, ctypes.byref(n), ctypes.byref(total)) == INVALID_ARG
    # NULL handles are harmless for the length and destroy calls
    assert L.frz_subset_len(None) == 0
    L.frz_subset_destroy(None)
    assert fake.raw == b"\0" * 4096
