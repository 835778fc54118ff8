"""Batcher requests with overrides, automata and log-probabilities (rwkv_b200_batcher_submit_ex / read_ex) without a
GPU: declared by the Python binding, added without an ABI version change, NULL batcher handles refused with a message,
and the ctypes RequestEx laid out as rwkv_b200_request_ex in the header."""
import ctypes
import os
import re

import numpy as np


def test_binding_declares_ex(pkg):
    lib = pkg.load_library()
    for n in ("submit_ex", "read_ex"):
        assert "rwkv_b200_batcher_" + n in lib._declared
    assert lib.rwkv_b200_abi_version() == 2


def test_null_batcher_is_refused(pkg):
    lib = pkg.load_library()
    P = ctypes.c_ulonglong
    prompt = np.array([4118, 15], np.uint64)
    req = pkg.engine.Request(0, prompt.ctypes.data_as(ctypes.POINTER(P)), 2, 4, pkg.Sampler(temperature=0.0), None, None, 0)
    x = pkg.engine.RequestEx(None, None, 0, pkg.engine.NO_CONSTRAINT, 0, 1, pkg.engine.LOGPROBS_RAW, 5)
    rid, n, state, st = P(), P(), P(), ctypes.c_int()
    calls = [
        lambda: lib.rwkv_b200_batcher_submit_ex(None, ctypes.byref(req), ctypes.byref(x), ctypes.byref(rid)),
        lambda: lib.rwkv_b200_batcher_submit_ex(None, ctypes.byref(req), None, ctypes.byref(rid)),
        lambda: lib.rwkv_b200_batcher_read_ex(None, 1, 0, None, None, None, None, None, ctypes.byref(state), ctypes.byref(n),
                                              ctypes.byref(st)),
    ]
    for call in calls:
        assert call() != 0
        assert b"null batcher handle" in lib.rwkv_b200_last_error()


def test_request_ex_layout(pkg):
    """Field offsets and size of rwkv_b200_request_ex on LP64: three pointers-or-counts of 8 bytes, two 8-byte ids,
    then int logprobs, int logprob_mode and unsigned top_n, padded to 8."""
    R = pkg.engine.RequestEx
    want = {"override_tokens": 0, "override_values": 8, "n_override": 16, "constraint_id": 24, "start_state": 32,
            "logprobs": 40, "logprob_mode": 44, "top_n": 48}
    assert [f for f, _ in R._fields_] == list(want)
    for f, off in want.items():
        assert getattr(R, f).offset == off, f
    assert ctypes.sizeof(R) == 56


def test_header_declares_the_struct_in_this_order(pkg):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    text = open(os.path.join(root, "include", "rwkv_b200.h")).read()
    body = re.search(r"typedef struct rwkv_b200_request_ex \{(.*?)\} rwkv_b200_request_ex;", text, re.S).group(1)
    names = re.findall(r"(\w+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [f for f, _ in pkg.engine.RequestEx._fields_]
