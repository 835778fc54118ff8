"""Multi-stream entry points of include/rwkv_b200.h without a GPU: declared by the Python binding, and safe to call
with a NULL handle (non-zero return and a message, no crash)."""
import ctypes

import numpy as np

NEW = ("rwkv_b200_forward_streams", "rwkv_b200_sample_typical_streams", "rwkv_b200_slot_zero", "rwkv_b200_slot_copy",
       "rwkv_b200_slot_upload", "rwkv_b200_slot_download")


def test_binding_declares_the_multi_stream_entry_points(pkg):
    lib = pkg.load_library()
    assert set(NEW) <= set(lib._declared)
    assert lib.rwkv_b200_abi_version() == 2


def test_null_handle_is_refused(pkg):
    lib = pkg.load_library()
    P = ctypes.POINTER(ctypes.c_ulonglong)
    D = ctypes.POINTER(ctypes.c_double)
    toks = np.array([1, 2], np.uint64)
    one = np.array([0], np.uint64)
    two = np.array([2], np.uint64)
    u = np.array([0.5])
    out = np.zeros(1, np.uint64)
    st = np.zeros(4, np.float64)
    calls = [
        lambda: lib.rwkv_b200_forward_streams(None, toks.ctypes.data_as(P), 2, one.ctypes.data_as(P), two.ctypes.data_as(P), 1, None,
                                              out.ctypes.data_as(P)),
        lambda: lib.rwkv_b200_sample_typical_streams(None, 1, 1.0, u.ctypes.data_as(D), out.ctypes.data_as(P), None),
        lambda: lib.rwkv_b200_slot_zero(None, 0),
        lambda: lib.rwkv_b200_slot_copy(None, 0, 1),
        lambda: lib.rwkv_b200_slot_upload(None, 0, st.ctypes.data_as(D), None, None, None, None),
        lambda: lib.rwkv_b200_slot_download(None, 0, st.ctypes.data_as(D), None, None, None, None),
    ]
    for call in calls:
        assert call() != 0
        assert b"null model handle" in lib.rwkv_b200_last_error()
