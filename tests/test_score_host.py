"""rwkv_b200_score_streams without a GPU: declared by the Python binding, added without an ABI version change, the
header's constants equal the Python ones, and safe to call with a NULL handle."""
import ctypes
import os
import re

import numpy as np

from util import INCLUDE


def test_binding_declares_score_streams(pkg):
    lib = pkg.load_library()
    assert "rwkv_b200_score_streams" in lib._declared
    assert lib.rwkv_b200_abi_version() == 2


def test_header_constants_match_python(pkg):
    with open(os.path.join(INCLUDE, "rwkv_b200.h")) as f:
        hdr = f.read()
    no_target = re.search(r"#define RWKV_B200_NO_TARGET (0x[0-9A-Fa-f]+)ULL", hdr)
    top_n = re.search(r"#define RWKV_B200_MAX_TOP_N (\d+)", hdr)
    assert no_target and int(no_target.group(1), 16) == pkg.engine.NO_TARGET == 2 ** 64 - 1
    assert top_n and int(top_n.group(1)) == pkg.engine.MAX_TOP_N


def test_null_handle_is_refused(pkg):
    lib = pkg.load_library()
    P = ctypes.POINTER(ctypes.c_ulonglong)
    D = ctypes.POINTER(ctypes.c_double)
    toks, slots, lens = np.array([4118, 11], np.uint64), np.array([0], np.uint64), np.array([2], np.uint64)
    tgt = np.array([11, pkg.engine.NO_TARGET], np.uint64)
    lp, ranks = np.zeros(2, np.float64), np.zeros(2, np.uint64)
    rc = lib.rwkv_b200_score_streams(None, toks.ctypes.data_as(P), 2, slots.ctypes.data_as(P), lens.ctypes.data_as(P), 1,
                                     tgt.ctypes.data_as(P), 0, lp.ctypes.data_as(D), ranks.ctypes.data_as(P), None, None)
    assert rc != 0 and b"null model handle" in lib.rwkv_b200_last_error()
