"""Device-resident multi-stream generation (rwkv_b200_generate_streams) against the host loop it replaces.

The oracle is a second engine that starts from the same state and runs, through the existing API and on the same
forward path, the loop the call promises to be equal to: feed every live stream its current token, pick the next one
(the device arg-max or the per-stream sampler), append it, stop on a stop token or the budget. A stream's arithmetic
depends only on its own row on either path, so the tokens and every named slot must match bit for bit, whatever the
group boundaries and the compaction of finished streams. Slots the call does not name must not change at all."""
import numpy as np
import pytest

from decoding import SHAPES, check_generated, engine_pair, host_loop, rand_tokens, stops_at

pytestmark = pytest.mark.gpu


def unconstrained(a, streams, max_new, max_gpt, **kw):
    """What a stream emits without stop tokens or budgets; a's state is restored afterwards."""
    st = a.state_download(max_gpt)
    seqs = a.generate_streams(streams, max_new, **kw)
    a.state_upload(st, max_gpt)
    return [[int(x) for x in s] for s in seqs]


@pytest.mark.parametrize("L,E", SHAPES)
def test_one_stream_decode_kernel_greedy(pkg, make_model, L, E):
    """One stream on slot 0 equals a forward_greedy loop, including a stop token hit mid-way: the stream's frozen rows
    run on the scratch slot until the group ends, and slot 0 stays where the loop left it."""
    max_gpt, max_new = 4, 40
    a, b = engine_pair(pkg, make_model(L, E), max_gpt, tc=False)
    streams = [(0, 4118)]
    seq = unconstrained(a, streams, max_new, max_gpt)[0]
    fresh = [i for i in range(max_new - 1) if seq[i] not in seq[:i]]  # positions where a stop token ends the stream
    at = min(fresh, key=lambda i: abs(i - 21))
    stop = [seq[at]]
    before = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, stop=stop)
    want = host_loop(b, streams, max_new, stop=stop, greedy_api=True)
    assert len(want[0]) == at + 1 < max_new
    check_generated(a, b, before, streams, got, want, max_gpt)
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", SHAPES)
def test_tensor_cores_twelve_streams_with_budgets_and_stops(pkg, make_model, L, E):
    max_gpt, max_new = 16, 40
    a, b = engine_pair(pkg, make_model(L, E), max_gpt, tc=True)
    slots = [9, 0, 3, 12, 5, 1, 14, 7, 2, 11, 6, 10]
    streams = [(s, t) for s, t in zip(slots, rand_tokens(12, 7))]
    seqs = unconstrained(a, streams, max_new, max_gpt)
    stop = stops_at(seqs, {0: 0, 1: 20, 2: 35}, prefer_unique=True)
    budgets = [40, 7, 40, 16, 33, 17, 1, 40, 25, 40, 9, 40]
    before = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, budgets=budgets, stop=stop)
    want = host_loop(b, streams, max_new, budgets=budgets, stop=stop, pad_slot=15)
    assert len(want[0]) == 1 and len({len(w) for w in want}) >= 4, [len(w) for w in want]
    check_generated(a, b, before, streams, got, want, max_gpt)
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", SHAPES)
def test_decode_kernel_three_streams(pkg, make_model, L, E):
    """prefill = 0: three streams through the decode kernel, ending at different steps (stop tokens and budgets)."""
    max_gpt, max_new = 6, 36
    a, b = engine_pair(pkg, make_model(L, E), max_gpt, tc=False)
    streams = [(4, 11), (1, 4118), (2, 777)]
    seqs = unconstrained(a, streams, max_new, max_gpt)
    stop = stops_at(seqs, {1: 5}, prefer_unique=True)
    budgets = [20, 36, 36]
    before = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, budgets=budgets, stop=stop)
    want = host_loop(b, streams, max_new, budgets=budgets, stop=stop)
    check_generated(a, b, before, streams, got, want, max_gpt)
    a.close()
    b.close()


def test_more_streams_than_one_pass(pkg, make_model):
    """150 streams: each step is a 128-row pass and a 22-row pass; budgets shrink the rows below one pass later."""
    max_gpt, max_new, S = 256, 20, 150
    a, b = engine_pair(pkg, make_model(3, 768), max_gpt, tc=True)
    perm = [int(x) for x in np.random.default_rng(3).permutation(max_gpt)]
    streams = [(s, t) for s, t in zip(perm[:S], rand_tokens(S, 8))]
    budgets = [20 if i % 5 == 0 else 1 + (7 * i) % 16 for i in range(S)]
    before = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, budgets=budgets)
    want = host_loop(b, streams, max_new, budgets=budgets, pad_slot=perm[S])
    check_generated(a, b, before, streams, got, want, max_gpt)
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", SHAPES)
@pytest.mark.parametrize("S,temp", [(1, 1.0), (10, 0.5)])
def test_typical_sampling(pkg, make_model, L, E, S, temp):
    """S = 1 runs on the decode kernel, S = 10 on the tensor cores; the loop samples with the same uniforms."""
    max_gpt, max_new = 12, 34
    a, b = engine_pair(pkg, make_model(L, E), max_gpt, tc=S >= 8)
    streams = [(s, t) for s, t in zip(range(S - 1, -1, -1), rand_tokens(S, 9))]
    u = np.random.default_rng(10).random((max_new, S))
    budgets = [max_new - (3 * i) % 20 for i in range(S)]
    before = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, budgets=budgets, temp=temp, u=u)
    want = host_loop(b, streams, max_new, budgets=budgets, temp=temp, u=u, pad_slot=max_gpt - 1)
    check_generated(a, b, before, streams, got, want, max_gpt)
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", SHAPES)
@pytest.mark.parametrize("S", [3, 9])
def test_overrides(pkg, make_model, L, E, S):
    """Each stream's unconstrained first pick is overridden to -99 before every pick; the loop does the same to its
    host logits and takes np.argmax (first index on ties)."""
    max_gpt, max_new = 12, 20
    a, b = engine_pair(pkg, make_model(L, E), max_gpt, tc=S >= 8)
    streams = [(5 * s % 11, t) for s, t in zip(range(S), rand_tokens(S, 11))]
    tops = [seq[0] for seq in unconstrained(a, streams, 1, max_gpt)]
    overrides = {t: -99.0 for t in tops}
    before = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, overrides=overrides)
    want = host_loop(b, streams, max_new, overrides=overrides, pad_slot=max_gpt - 1)
    assert all(w[0] != t for w, t in zip(want, tops))
    check_generated(a, b, before, streams, got, want, max_gpt)
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", SHAPES)
def test_continuation(pkg, make_model, L, E):
    """generate, then forward_streams from the last emitted token: one uninterrupted host loop."""
    max_gpt, first, more = 12, 18, 6
    a, b = engine_pair(pkg, make_model(L, E), max_gpt, tc=True)
    streams = [(s, t) for s, t in zip(range(9), rand_tokens(9, 12))]
    before = a.state_download(max_gpt)
    got = [[int(x) for x in g] for g in a.generate_streams(streams, first)]
    for _ in range(more):
        _, nxt = a.forward_streams([(slot, [g[-1]]) for (slot, _), g in zip(streams, got)], want_logits=False, want_next=True)
        for g, x in zip(got, nxt):
            g.append(int(x))
    want = host_loop(b, streams, first + more)
    a.forward_streams([(slot, [g[-1]]) for (slot, _), g in zip(streams, got)], want_logits=False)  # feed the last picks
    b.forward_streams([(slot, [w[-1]]) for (slot, _), w in zip(streams, want)], want_logits=False)
    check_generated(a, b, before, streams, got, want, max_gpt)
    a.close()
    b.close()


def test_rejected_inputs_leave_the_state_untouched(pkg, make_model):
    import ctypes
    path = make_model(2, 768)
    a = pkg.Engine(path, max_gpt=8)
    a.forward(rand_tokens(8, 70), mode=0, want_logits=False)
    before = a.state_download(8)
    ok = [(0, 5), (1, 6)]
    bad = [
        (dict(streams=[], max_new=4), "no streams"),
        (dict(streams=[(1, 5), (1, 6)], max_new=4), "slot 1 appears twice"),
        (dict(streams=[(8, 5)], max_new=4), "slot 8 >= max_gpt"),
        (dict(streams=[(0, 5), (1, 50277)], max_new=4), "first token 50277"),
        (dict(streams=ok, max_new=4, stop=[3, 50277]), "stop token 50277"),
        (dict(streams=ok, max_new=4, overrides={50277: 1.0}), "override token 50277"),
        (dict(streams=ok, max_new=0), "max_new is 0"),
        (dict(streams=ok, max_new=4, budgets=[4, 0]), "budget 0 of stream 1"),
        (dict(streams=ok, max_new=4, budgets=[5, 4]), "budget 5 of stream 0"),
        (dict(streams=ok, max_new=2, u=[[0.1, 0.2], [1.0, 0.5]]), r"u\[2\] = 1 is outside \[0, 1\)"),
        (dict(streams=ok, max_new=1, u=[[0.3, -0.25]]), r"u\[1\] = -0.25"),
        (dict(streams=ok, max_new=1, u=[[float("nan"), 0.5]]), r"u\[0\] = nan"),
    ]
    for kw, msg in bad:
        with pytest.raises(pkg.EngineError, match=msg):
            a.generate_streams(**kw)
    P = ctypes.POINTER(ctypes.c_ulonglong)
    slots, first = np.array([0, 1], np.uint64), np.array([5, 6], np.uint64)
    out, lens = np.zeros(8, np.uint64), np.zeros(2, np.uint64)
    raw = [
        (lambda: a.lib.rwkv_b200_generate_streams(a.h, None, first.ctypes.data_as(P), 2, 4, None, None, 0, None, None, 0, 1.0, None,
                                                  out.ctypes.data_as(P), lens.ctypes.data_as(P)), b"null argument"),
        (lambda: a.lib.rwkv_b200_generate_streams(a.h, slots.ctypes.data_as(P), first.ctypes.data_as(P), 2, 4, None, None, 1, None,
                                                  None, 0, 1.0, None, out.ctypes.data_as(P), lens.ctypes.data_as(P)), b"n_stop = 1"),
        (lambda: a.lib.rwkv_b200_generate_streams(a.h, slots.ctypes.data_as(P), first.ctypes.data_as(P), 2, 4, None, None, 0,
                                                  first.ctypes.data_as(P), None, 2, 1.0, None, out.ctypes.data_as(P),
                                                  lens.ctypes.data_as(P)), b"n_override = 2"),
    ]
    for call, msg in raw:
        assert call() != 0 and msg in a.lib.rwkv_b200_last_error()
    after = a.state_download(8)
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    # a successful call leaves no per-stream logits behind
    a.forward_streams(ok, want_next=True)
    a.generate_streams(ok, 3)
    with pytest.raises(pkg.EngineError, match="no per-stream logits"):
        a.sample_typical_streams(1.0, [0.5, 0.5])
    a.close()
    t = pkg.Engine(path, max_gpt=4, tp_rank=0, tp_size=2)
    with pytest.raises(pkg.EngineError, match="not supported with tensor parallelism"):
        t.generate_streams([(0, 5)], 4)
    t.close()
