"""rwkv_b200_generate_streams_logprobs without a GPU: declared by the Python binding, added without an ABI version
change, the header's mode constants equal the Python ones, and safe to call with a NULL handle."""
import ctypes
import os
import re

import numpy as np

from util import INCLUDE


def test_binding_declares_generate_streams_logprobs(pkg):
    lib = pkg.load_library()
    assert "rwkv_b200_generate_streams_logprobs" in lib._declared
    assert lib.rwkv_b200_abi_version() == 2


def test_header_mode_constants_match_python(pkg):
    with open(os.path.join(INCLUDE, "rwkv_b200.h")) as f:
        hdr = f.read()
    raw = re.search(r"#define RWKV_B200_LOGPROBS_RAW\s+(\d+)", hdr)
    processed = re.search(r"#define RWKV_B200_LOGPROBS_PROCESSED\s+(\d+)", hdr)
    assert raw and int(raw.group(1)) == pkg.engine.LOGPROBS_RAW == 0
    assert processed and int(processed.group(1)) == pkg.engine.LOGPROBS_PROCESSED == 1


def test_null_handle_is_refused(pkg):
    lib = pkg.load_library()
    P = ctypes.POINTER(ctypes.c_ulonglong)
    D = ctypes.POINTER(ctypes.c_double)
    slots, first = np.array([0], np.uint64), np.array([4118], np.uint64)
    out, lens = np.zeros(4, np.uint64), np.zeros(1, np.uint64)
    lp, ranks = np.zeros(4, np.float64), np.zeros(4, np.uint64)
    rc = lib.rwkv_b200_generate_streams_logprobs(None, slots.ctypes.data_as(P), first.ctypes.data_as(P), 1, 4, None, None, 0,
                                                 None, None, 0, None, None, out.ctypes.data_as(P), lens.ctypes.data_as(P),
                                                 pkg.engine.LOGPROBS_RAW, 0, lp.ctypes.data_as(D), ranks.ctypes.data_as(P),
                                                 None, None)
    assert rc != 0 and b"null model handle" in lib.rwkv_b200_last_error()
