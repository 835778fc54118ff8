"""rwkv_b200_generate_streams without a GPU: declared by the Python binding, added without an ABI version change, and
safe to call with a NULL handle (non-zero return and a message, no crash)."""
import ctypes

import numpy as np


def test_binding_declares_generate_streams(pkg):
    lib = pkg.load_library()
    assert "rwkv_b200_generate_streams" in lib._declared
    assert lib.rwkv_b200_abi_version() == 2


def test_null_handle_is_refused(pkg):
    lib = pkg.load_library()
    P = ctypes.POINTER(ctypes.c_ulonglong)
    slots = np.array([0], np.uint64)
    first = np.array([4118], np.uint64)
    out = np.zeros(4, np.uint64)
    lens = np.zeros(1, np.uint64)
    rc = lib.rwkv_b200_generate_streams(None, slots.ctypes.data_as(P), first.ctypes.data_as(P), 1, 4, None, None, 0, None, None, 0,
                                        1.0, None, out.ctypes.data_as(P), lens.ctypes.data_as(P))
    assert rc != 0
    assert b"null model handle" in lib.rwkv_b200_last_error()
