"""Speculative batcher requests (rwkv_b200_batcher_submit_spec / read_spec) without a GPU: the library exports both
symbols and the header declares them, the ctypes RequestSpec is laid out as rwkv_b200_request_spec, NULL batcher handles
and Python argument errors are refused before any C call, and engine.speculative_steps with the batcher's lookup context
(context ++ prompt[:-1], first token prompt[-1]) matches a brute-force restatement of the steps rule."""
import ctypes
import importlib
import os
import re

import numpy as np
import pytest

eng_mod = importlib.import_module("rwkv-cpp-accelerated_b200.engine")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_and_header_declares(pkg):
    lib = pkg.load_library()
    raw = ctypes.CDLL(pkg.lib_path())
    text = open(os.path.join(ROOT, "include", "rwkv_b200.h")).read()
    for n in ("rwkv_b200_batcher_submit_spec", "rwkv_b200_batcher_read_spec"):
        assert n in lib._declared
        assert hasattr(raw, n)
        assert re.search(r"\bint %s\(" % n, text), n
    assert lib.rwkv_b200_abi_version() == 2


def test_request_spec_layout(pkg):
    R = pkg.engine.RequestSpec
    want = {"spare_slots": 0, "draft": 8, "ngram": 12, "context": 16, "n_context": 24}
    assert [f for f, _ in R._fields_] == list(want)
    for f, off in want.items():
        assert getattr(R, f).offset == off, f
    assert ctypes.sizeof(R) == 32
    text = open(os.path.join(ROOT, "include", "rwkv_b200.h")).read()
    body = re.search(r"typedef struct rwkv_b200_request_spec \{(.*?)\} rwkv_b200_request_spec;", text, re.S).group(1)
    assert re.findall(r"(\w+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S)) == list(want)


def test_null_batcher_is_refused(pkg):
    lib = pkg.load_library()
    P = ctypes.c_ulonglong
    prompt = np.array([4118, 15], np.uint64)
    spares = np.array([1, 2], np.uint64)
    req = pkg.engine.Request(0, prompt.ctypes.data_as(ctypes.POINTER(P)), 2, 4, pkg.Sampler(temperature=0.0), None, None, 0)
    spec = pkg.engine.RequestSpec(spares.ctypes.data_as(ctypes.POINTER(P)), 2, 3, None, 0)
    rid, steps = P(), P()
    for call in (lambda: lib.rwkv_b200_batcher_submit_spec(None, ctypes.byref(req), None, pkg.engine.NO_STOP_SET, 0,
                                                           ctypes.byref(spec), ctypes.byref(rid)),
                 lambda: lib.rwkv_b200_batcher_submit_spec(None, ctypes.byref(req), None, pkg.engine.NO_STOP_SET, 0, None,
                                                           ctypes.byref(rid)),
                 lambda: lib.rwkv_b200_batcher_read_spec(None, 1, ctypes.byref(steps))):
        assert call() != 0
        assert b"null batcher handle" in lib.rwkv_b200_last_error()


def _unopened_batcher(pkg):
    """A Batcher whose handle is NULL: Python-side errors must be raised before the C call would refuse it."""
    bat = object.__new__(pkg.engine.Batcher)
    e = object.__new__(pkg.Engine)
    e.lib, e.h = pkg.load_library(), None
    bat.engine, bat.lib, bat.h = e, e.lib, None
    bat._ext, bat._stop, bat._spec = {}, set(), set()
    return bat


def test_python_argument_errors(pkg):
    bat = _unopened_batcher(pkg)
    with pytest.raises(pkg.EngineError, match="needs 2 spare slots, got 1"):
        bat.submit(0, [1, 2], 4, draft=2, spare_slots=[5])
    with pytest.raises(pkg.EngineError, match="needs 1 spare slots, got 0"):
        bat.submit(0, [1, 2], 4, draft=1)
    with pytest.raises(pkg.EngineError, match="needs 0 spare slots, got 1"):
        bat.submit(0, [1, 2], 4, spare_slots=[5])
    with pytest.raises(pkg.EngineError, match="lookup context needs draft > 0"):
        bat.submit(0, [1, 2], 4, context=[7])
    with pytest.raises(pkg.EngineError, match="draft -1 < 0"):
        bat.submit(0, [1, 2], 4, draft=-1, spare_slots=[5])
    with pytest.raises(pkg.EngineError, match="u has shape"):
        bat.submit(0, [1, 2], 4, draft=1, spare_slots=[5], u=np.zeros(3))
    with pytest.raises(pkg.EngineError, match="null batcher handle"):  # well-formed: reaches the C refusal
        bat.submit(0, [1, 2], 4, draft=1, spare_slots=[5], context=[7, 8])


def brute_steps(context, prompt, tokens, k, ngram):
    """The steps rule restated: each step looks up the drafts of the whole history (context ++ prompt ++ emitted) by
    trying every start position, then emits p_0 and each further token while it equals the previous draft."""
    h = list(context) + list(prompt)
    t, pos, steps = list(tokens), 0, 0
    while pos < len(t):
        L, prop = len(h), None
        for n in range(ngram, 0, -1):
            if n >= L:
                continue
            js = [j for j in range(L - n) if h[j:j + n] == h[L - n:]]
            if js:
                j = max(js)
                prop = h[j + n:min(j + n + k, L)]
                break
        d = [h[-1]] * k if prop is None else [prop[min(i, len(prop) - 1)] for i in range(k)]
        c = 1
        while c <= k and pos + c < len(t) and d[c - 1] == t[pos + c - 1]:
            c += 1
        h += t[pos:pos + c]
        pos += c
        steps += 1
    return steps


def test_speculative_steps_with_batcher_context():
    rng = np.random.default_rng(5)
    for trial in range(300):
        V = int(rng.integers(2, 6))  # small vocabularies: many matches
        ctx = [int(x) for x in rng.integers(0, V, size=int(rng.integers(0, 6)))]
        prompt = [int(x) for x in rng.integers(0, V, size=int(rng.integers(1, 8)))]
        if trial % 3 == 0:  # the ceiling: the output copies the context
            toks = (ctx + prompt)[: int(rng.integers(1, 12))] or [0]
        else:
            toks = [int(x) for x in rng.integers(0, V, size=int(rng.integers(1, 20)))]
        k, ng = int(rng.integers(1, 6)), int(rng.integers(1, 4))
        want = brute_steps(ctx, prompt, toks, k, ng)
        assert eng_mod.speculative_steps(ctx + prompt[:-1], prompt[-1], toks, k, ng) == want, (ctx, prompt, toks, k, ng)
        assert 1 <= want <= len(toks)


def test_ceiling_takes_few_steps():
    """A request whose output repeats its prompt emits k + 1 tokens per step once the lookup locks on."""
    prompt = list(range(100, 140))
    toks = prompt[1:] + prompt
    steps = eng_mod.speculative_steps(prompt[:-1], prompt[-1], toks, 4, 3)
    assert steps == brute_steps([], prompt, toks, 4, 3)
    assert steps <= len(toks) // 4
