"""State indexes (rwkv_b200_index_*) without a GPU: declared by the Python binding without an ABI version change, the
header's constants equal the Python ones, every entry point refuses a NULL model handle with a message, and the Python
argument errors are raised before any call into the library."""
import ctypes
import os
import re

import numpy as np
import pytest

from util import INCLUDE

NAMES = ("create", "free", "add_slots", "upload", "download", "remove", "search")


def test_binding_declares_the_index_entry_points(pkg):
    lib = pkg.load_library()
    for n in NAMES:
        assert "rwkv_b200_index_" + n in lib._declared
    assert lib.rwkv_b200_abi_version() == 2


def test_header_constants(pkg):
    with open(os.path.join(INCLUDE, "rwkv_b200.h")) as f:
        hdr = f.read()
    E = pkg.engine
    define = lambda name: re.search(r"#define RWKV_B200_%s\s+(0x[0-9A-F]+ULL|\d+)" % name, hdr).group(1)
    assert int(define("INDEX_L1")) == E.INDEX_L1 == 0
    assert int(define("INDEX_L2")) == E.INDEX_L2 == 1
    assert int(define("MAX_NEIGHBOURS")) == E.MAX_NEIGHBOURS == 256
    assert int(define("NO_ENTRY")[:-3], 16) == E.NO_ENTRY == 2 ** 64 - 1


def test_null_model_is_refused(pkg):
    lib = pkg.load_library()
    P, D = ctypes.POINTER(ctypes.c_ulonglong), ctypes.POINTER(ctypes.c_double)
    ids, vec = np.zeros(4, np.uint64), np.zeros(4096)
    l1, l2, found = np.zeros(4), np.zeros(4), np.zeros(1, np.uint64)
    iid = ctypes.c_ulonglong()
    p, d = (lambda a: a.ctypes.data_as(P)), (lambda a: a.ctypes.data_as(D))
    calls = [
        lambda: lib.rwkv_b200_index_create(None, 0, 1, 4, ctypes.byref(iid)),
        lambda: lib.rwkv_b200_index_free(None, 1),
        lambda: lib.rwkv_b200_index_add_slots(None, 1, p(ids), 1, p(ids)),
        lambda: lib.rwkv_b200_index_upload(None, 1, d(vec), 1, p(ids)),
        lambda: lib.rwkv_b200_index_download(None, 1, p(ids), 1, d(vec)),
        lambda: lib.rwkv_b200_index_remove(None, 1, p(ids), 1),
        lambda: lib.rwkv_b200_index_search(None, 1, p(ids), 1, 1, 4, p(ids), d(l1), d(l2), p(found)),
    ]
    for call in calls:
        assert call() != 0
        assert b"null model handle" in lib.rwkv_b200_last_error()


class NoCalls:
    """A library stand-in that fails the test on any call."""

    def __getattr__(self, name):
        raise AssertionError("library called: %s" % name)


@pytest.fixture
def engine(pkg):
    e = object.__new__(pkg.Engine)
    e.lib, e.h = NoCalls(), None
    e.n_layers, e.n_embed, e.max_gpt = 3, 64, 4
    return e


def test_python_argument_errors_before_any_call(pkg, engine):
    with pytest.raises(pkg.EngineError, match="consecutive layers"):
        engine.create_index(4, layers=[0, 2])
    with pytest.raises(pkg.EngineError, match="consecutive layers"):
        engine.create_index(4, layers=range(0))
    idx = object.__new__(pkg.StateIndex)
    idx.engine, idx.lib, idx.h, idx.D = engine, NoCalls(), 1, 128
    with pytest.raises(pkg.EngineError, match=r"expected \(n, 128\)"):
        idx.upload(np.zeros((2, 64)))
    with pytest.raises(pkg.EngineError, match="metric must be 'l1' or 'l2'"):
        idx.search([0], 3, metric="cosine")
    with pytest.raises(pkg.EngineError, match="document 1 has no tokens"):
        engine.embed([[1, 2], []], [0, 1], idx)
    with pytest.raises(pkg.EngineError, match="a slot appears twice"):
        engine.embed([[1, 2]], [0, 0], idx)
