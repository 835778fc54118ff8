"""Speculative generation with log-probabilities and token automata (rwkv_b200_generate_streams_speculative_constrained)
without a GPU: declared by the Python binding without an ABI version change, a NULL model handle refused with a
message, and Engine.generate_speculative's argument errors raised before any call into the library."""
import ctypes

import numpy as np
import pytest

NAME = "rwkv_b200_generate_streams_speculative_constrained"


def test_binding_declares_the_call(pkg):
    lib = pkg.load_library()
    assert NAME in lib._declared
    assert lib.rwkv_b200_abi_version() == 2


def test_null_model_is_refused(pkg):
    lib = pkg.load_library()
    P = ctypes.c_ulonglong
    slots = np.arange(4, dtype=np.uint64)
    first = np.array([5], np.uint64)
    out, lens, steps, states = np.zeros(8, np.uint64), np.zeros(1, np.uint64), np.zeros(1, np.uint64), np.zeros(1, np.uint64)
    lp = np.zeros(8)
    ids = np.array([1], np.uint64)
    p = lambda a: a.ctypes.data_as(ctypes.POINTER(P))
    rc = getattr(lib, NAME)(None, p(slots), p(first), 1, 8, None, None, 0, None, None, 0, None, None, p(out), p(lens), 3, 3,
                            None, None, p(steps), pkg.engine.LOGPROBS_RAW, 0,
                            lp.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), None, None, None, p(ids), None, p(states),
                            None)
    assert rc != 0
    assert b"null model handle" in lib.rwkv_b200_last_error()


class NoCalls:
    """A library stand-in that fails the test on any call."""

    def __getattr__(self, name):
        raise AssertionError("library called: %s" % name)


@pytest.fixture
def engine(pkg):
    e = object.__new__(pkg.Engine)
    e.lib, e.h = NoCalls(), None
    return e


def test_bad_logprobs_mode_before_any_call(pkg, engine):
    with pytest.raises(pkg.EngineError, match="logprobs must be 'raw' or 'processed'"):
        engine.generate_speculative([([0, 1, 2, 3], 5)], 8, 3, logprobs="scaled")


def test_constraint_count_before_any_call(pkg, engine):
    streams = [([0, 1, 2, 3], 5), ([4, 5, 6, 7], 6)]
    with pytest.raises(pkg.EngineError, match="generate_speculative: 3 constraints for 2 streams"):
        engine.generate_speculative(streams, 8, 3, constraints=[1, None, 1])
    with pytest.raises(pkg.EngineError, match="generate_speculative: 1 constraints for 2 streams"):
        engine.generate_speculative(streams, 8, 3, logprobs="raw", constraints=[1])
