"""rwkv_b200_beam_search without a GPU: declared by the Python binding, added without an ABI version change, and safe to
call with a NULL handle."""
import ctypes

import numpy as np


def test_binding_declares_beam_search(pkg):
    lib = pkg.load_library()
    assert "rwkv_b200_beam_search" in lib._declared
    assert lib.rwkv_b200_abi_version() == 2


def test_null_handle_is_refused(pkg):
    lib = pkg.load_library()
    P = ctypes.POINTER(ctypes.c_ulonglong)
    D = ctypes.POINTER(ctypes.c_double)
    slots, first = np.array([0, 1], np.uint64), np.array([4118], np.uint64)
    toks, lens = np.zeros(4, np.uint64), np.zeros(1, np.uint64)
    lp, scores, fin = np.zeros(1, np.float64), np.zeros(1, np.float64), np.zeros(1, np.uint8)
    rc = lib.rwkv_b200_beam_search(None, slots.ctypes.data_as(P), first.ctypes.data_as(P), 1, 2, 4, None, 0, 1.0, 1,
                                   toks.ctypes.data_as(P), lens.ctypes.data_as(P), lp.ctypes.data_as(D),
                                   scores.ctypes.data_as(D), fin.ctypes.data_as(ctypes.POINTER(ctypes.c_ubyte)), None)
    assert rc != 0 and b"null model handle" in lib.rwkv_b200_last_error()
