"""Continuous batching (rwkv_b200_batcher_*) without a GPU: declared by the Python binding, added without an ABI version
change, and a NULL model or batcher handle is refused with a message, no crash."""
import ctypes

import numpy as np

NAMES = ("open", "submit", "run", "read", "cancel", "release", "close")


def test_binding_declares_batcher(pkg):
    lib = pkg.load_library()
    for n in NAMES:
        assert "rwkv_b200_batcher_" + n in lib._declared
    assert lib.rwkv_b200_abi_version() == 2


def test_null_model_is_refused(pkg):
    lib = pkg.load_library()
    h = ctypes.c_void_p()
    assert lib.rwkv_b200_batcher_open(None, 4, 16, ctypes.byref(h)) != 0
    assert b"null model handle" in lib.rwkv_b200_last_error()
    assert not h.value


def test_null_batcher_is_refused(pkg):
    lib = pkg.load_library()
    P = ctypes.c_ulonglong
    prompt = np.array([4118, 15], np.uint64)
    req = pkg.engine.Request(0, prompt.ctypes.data_as(ctypes.POINTER(P)), 2, 4, pkg.Sampler(temperature=0.0), None, None, 0)
    rid, n, st = P(), P(), ctypes.c_int()
    calls = [
        lambda: lib.rwkv_b200_batcher_submit(None, ctypes.byref(req), ctypes.byref(rid)),
        lambda: lib.rwkv_b200_batcher_run(None, 16, ctypes.byref(n)),
        lambda: lib.rwkv_b200_batcher_read(None, 1, None, 0, ctypes.byref(n), ctypes.byref(st)),
        lambda: lib.rwkv_b200_batcher_cancel(None, 1),
        lambda: lib.rwkv_b200_batcher_release(None, 1),
    ]
    for call in calls:
        assert call() != 0
        assert b"null batcher handle" in lib.rwkv_b200_last_error()
    lib.rwkv_b200_batcher_close(None)  # ignored
