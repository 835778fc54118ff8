"""rwkv_b200_generate_streams_speculative without a GPU: the binding, the refusals that need no device, and the Python
restatement of the draft rule (engine.lookup_drafts) and of steps_out (engine.speculative_steps) on hand-made histories."""
import ctypes
import importlib

import numpy as np
import pytest

eng_mod = importlib.import_module("rwkv-cpp-accelerated_b200.engine")
drafts = eng_mod.lookup_drafts
steps_of = eng_mod.speculative_steps


def test_binding_declares_speculative(pkg):
    lib = pkg.load_library()
    assert "rwkv_b200_generate_streams_speculative" in lib._declared
    assert lib.rwkv_b200_abi_version() == 2


def test_null_handle_is_refused(pkg):
    lib = pkg.load_library()
    P = ctypes.POINTER(ctypes.c_ulonglong)
    slots, first = np.array([0, 1], np.uint64), np.array([4118], np.uint64)
    toks, lens, steps = np.zeros(4, np.uint64), np.zeros(1, np.uint64), np.zeros(1, np.uint64)
    rc = lib.rwkv_b200_generate_streams_speculative(None, slots.ctypes.data_as(P), first.ctypes.data_as(P), 1, 4, None, None,
                                                    0, None, None, 0, None, None, toks.ctypes.data_as(P),
                                                    lens.ctypes.data_as(P), 1, 3, None, None, steps.ctypes.data_as(P))
    assert rc != 0 and b"null model handle" in lib.rwkv_b200_last_error()


def _unloaded_engine(pkg):
    e = object.__new__(pkg.Engine)
    e.lib, e.h = pkg.load_library(), None
    return e


def test_python_refusals(pkg):
    e = _unloaded_engine(pkg)
    with pytest.raises(pkg.EngineError, match="draft \\+ 1 = 3 slots"):
        e.generate_speculative([([0, 1], 5)], 4, draft=2)
    with pytest.raises(pkg.EngineError, match="2 contexts for 1 streams"):
        e.generate_speculative([([0, 1, 2], 5)], 4, draft=2, context=[[1], [2]])
    with pytest.raises(pkg.EngineError, match="u has shape"):
        e.generate_speculative([([0, 1, 2], 5)], 4, draft=2, u=np.zeros((3, 1)))
    with pytest.raises(pkg.EngineError, match="null model handle"):
        e.generate_speculative([([0, 1, 2], 5)], 4, draft=2, context=[[1, 2, 3]])


def test_no_match_pads_with_last_token():
    assert drafts([7], 3, 3) == [7, 7, 7]             # L = 1: no n < L
    assert drafts([1, 2, 3, 4], 2, 3) == [4, 4]       # no earlier 4
    assert drafts([5, 6, 5], 4, 1) == [6, 5, 5, 5]    # n = 1: j = 0, proposal [6, 5], padded with 5


def test_longest_ngram_wins_over_later_shorter_match():
    # n = 2 matches "1 2" at j = 0 (-> 3); n = 1 alone would pick the later 2 at j = 4 (-> 9)
    h = [1, 2, 3, 0, 2, 9, 1, 2]
    assert drafts(h, 2, 2) == [3, 0]
    assert drafts(h, 2, 1) == [9, 1]
    assert drafts([4, 2, 9, 8, 2], 2, 1) == [9, 8]
    assert drafts([4, 2, 9, 8, 2], 2, 3) == [9, 8]    # n = 3, 2 find nothing; n = 1 does


def test_largest_j_and_overlapping_continuation():
    # a run: the match at the largest j overlaps the suffix, and the proposal ends at h[L - 1]
    assert drafts([3, 3, 3, 3], 4, 2) == [3, 3, 3, 3]
    h = [1, 2, 1, 2, 1, 2]
    assert drafts(h, 5, 2) == [1, 2, 2, 2, 2]         # n = 2: j = 2, proposal h[4:6] = [1, 2], padded
    assert drafts(h, 1, 3) == [1]                     # n = 3: j = 1 ("2 1 2"), proposal h[4:5]
    assert drafts([9, 1, 2, 1, 2], 3, 2) == [1, 2, 2] # n = 2: j = 1, proposal h[3:5] = [1, 2] reaches the end


def _drafts_brute(h, k, ngram):
    """The rule read literally: every (n, j) pair, then the first n in descending order and the largest j."""
    L = len(h)
    hits = {n: [j for j in range(0, L - n) if h[j:j + n] == h[L - n:]] for n in range(1, ngram + 1) if n < L}
    for n in sorted(hits, reverse=True):
        if hits[n]:
            j = max(hits[n])
            prop = h[j + n:min(j + n + k, L)]
            return (prop + [prop[-1]] * k)[:k]
    return [h[-1]] * k


@pytest.mark.parametrize("seed", range(4))
def test_random_histories_match_the_literal_rule(seed):
    rng = np.random.default_rng(seed)
    for _ in range(300):
        L = int(rng.integers(1, 40))
        h = [int(x) for x in rng.integers(0, 1 + int(rng.integers(1, 6)), size=L)]
        k, n = int(rng.integers(1, 16)), int(rng.integers(1, 9))
        assert drafts(h, k, n) == _drafts_brute(h, k, n), (h, k, n)


def test_steps_restatement():
    # steps 1-3 find no useful match and emit one token each; step 4 accepts all three drafts [2, 3, 1] (4 tokens);
    # step 5 emits the last token
    assert steps_of([], 1, [2, 3, 1, 2, 3, 1, 2, 3], 3, 2) == 5
    # the same tokens with the text in the context: every step accepts every draft
    assert steps_of([1, 2, 3, 1, 2, 3, 1, 2, 3], 1, [2, 3, 1, 2, 3, 1, 2, 3], 3, 2) == 2
    # a stream that stopped inside a step: the tokens after the stop were dropped, so its last step is short
    assert steps_of([1, 2, 3, 1, 2, 3, 1, 2, 3], 1, [2, 3], 3, 2) == 1
    assert steps_of([], 5, [], 2, 3) == 0
