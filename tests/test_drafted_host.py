"""rwkv_b200_generate_streams_drafted without a GPU: the binding and the drafter struct, the refusals that need no device,
and the Python plumbing of Engine.generate_speculative(drafter=...) against a recording stand-in for the library."""
import ctypes
import importlib

import numpy as np
import pytest

eng_mod = importlib.import_module("rwkv-cpp-accelerated_b200.engine")
P = ctypes.POINTER(ctypes.c_ulonglong)


def test_symbol_declared_and_exported(pkg):
    lib = pkg.load_library()
    assert "rwkv_b200_generate_streams_drafted" in lib._declared
    assert lib.rwkv_b200_generate_streams_drafted.restype is ctypes.c_int
    assert len(lib.rwkv_b200_generate_streams_drafted.argtypes) == 28
    assert lib.rwkv_b200_abi_version() == 2


def test_struct_matches_the_header():
    d = eng_mod.Drafter
    assert [f for f, _ in d._fields_] == ["model", "slots"]
    assert d.model.offset == 0 and d.slots.offset == ctypes.sizeof(ctypes.c_void_p)
    assert ctypes.sizeof(d) == 2 * ctypes.sizeof(ctypes.c_void_p)


def _call(lib, m, drafter):
    slots, first = np.array([0, 1, 2], np.uint64), np.array([4118], np.uint64)
    toks, lens, steps = np.zeros(4, np.uint64), np.zeros(1, np.uint64), np.zeros(1, np.uint64)
    return lib.rwkv_b200_generate_streams_drafted(m, slots.ctypes.data_as(P), first.ctypes.data_as(P), 1, 4, None, None, 0,
                                                  None, None, 0, None, None, toks.ctypes.data_as(P), lens.ctypes.data_as(P),
                                                  2, drafter, steps.ctypes.data_as(P), 0, 0, None, None, None, None, None,
                                                  None, None, None)


def test_null_handles_are_refused(pkg):
    lib = pkg.load_library()
    dslots = np.array([0, 1], np.uint64)
    d = eng_mod.Drafter(None, dslots.ctypes.data_as(P))
    assert _call(lib, None, ctypes.byref(d)) != 0 and b"null model handle" in lib.rwkv_b200_last_error()
    assert _call(lib, None, None) != 0 and b"null model handle" in lib.rwkv_b200_last_error()


def _unloaded_engine(pkg):
    e = object.__new__(pkg.Engine)
    e.lib, e.h = pkg.load_library(), None
    return e


def test_python_refusals(pkg):
    e, other = _unloaded_engine(pkg), _unloaded_engine(pkg)
    streams = [([0, 1, 2], 5), ([3, 4, 5], 6)]
    pairs = [(0, 1), (2, 3)]
    E = pkg.EngineError
    with pytest.raises(E, match="neither context nor ngram"):
        e.generate_speculative(streams, 4, draft=2, context=[[1], [2]], drafter=(other, pairs))
    with pytest.raises(E, match="neither context nor ngram"):
        e.generate_speculative(streams, 4, draft=2, ngram=2, drafter=(other, pairs))
    with pytest.raises(E, match="one \\(D0, D1\\) slot pair per stream"):
        e.generate_speculative(streams, 4, draft=2, drafter=(other, pairs[:1]))
    with pytest.raises(E, match="one \\(D0, D1\\) slot pair per stream"):
        e.generate_speculative(streams, 4, draft=2, drafter=(other, [(0, 1, 2), (3,)]))
    with pytest.raises(E, match="the draft engine is the target engine"):
        e.generate_speculative(streams, 4, draft=2, drafter=(e, pairs))
    # past the Python checks the library refuses the unloaded handle
    with pytest.raises(E, match="null model handle"):
        e.generate_speculative(streams, 4, draft=2, drafter=(other, pairs))


class _Recorder:
    """A stand-in for the library: records each entry point called and its arguments, returns 0."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            return 0
        return fn


def _recorded(pkg, **kw):
    e = object.__new__(pkg.Engine)
    e.lib, e.h = _Recorder(), ctypes.c_void_p(1)
    e.generate_speculative([([0, 1, 2], 5), ([3, 4, 5], 6)], 4, draft=2, **kw)
    assert len(e.lib.calls) == 1
    return e.lib.calls[0]


@pytest.mark.parametrize("kw, name", [
    ({}, "rwkv_b200_generate_streams_speculative"),
    ({"context": [[1, 2], None], "ngram": 4}, "rwkv_b200_generate_streams_speculative"),
    ({"logprobs": "raw"}, "rwkv_b200_generate_streams_speculative_constrained"),
])
def test_prompt_lookup_plumbing_unchanged(pkg, kw, name):
    got, args = _recorded(pkg, **kw)
    assert got == name
    # model, ten lead arguments, sampler, u, tokens, lengths, draft, ngram, context_start, context, steps_out
    assert args[15] == 2 and args[16] == kw.get("ngram", 3)
    assert (args[17] is None) == ("context" not in kw)


def test_drafted_plumbing(pkg):
    other = object.__new__(pkg.Engine)
    other.h = ctypes.c_void_p(1234)
    got, args = _recorded(pkg, drafter=(other, [(7, 8), (9, 10)]), logprobs="processed", top_n=2)
    assert got == "rwkv_b200_generate_streams_drafted"
    assert len(args) == 28
    assert args[15] == 2
    d = args[16]._obj
    assert d.model == 1234 and [d.slots[i] for i in range(4)] == [7, 8, 9, 10]
    assert args[18] == eng_mod.LOGPROBS_PROCESSED and args[19] == 2
