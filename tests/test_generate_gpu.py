"""Device-resident multi-stream generation (rwkv_b200_generate_streams) against the host loop it replaces.

The oracle is a second engine that starts from the same state and runs, through the existing API and on the same
forward path, the loop the call promises to be equal to: feed every live stream its current token, pick the next one
(the device arg-max or the per-stream sampler), append it, stop on a stop token or the budget. A stream's arithmetic
depends only on its own row on either path, so the tokens and every named slot must match bit for bit, whatever the
group boundaries and the compaction of finished streams. Slots the call does not name must not change at all."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

V = 50277
KEYS = ("xy", "aa", "bb", "dd")
SHAPES = [(3, 768), (2, 2048)]


def rand_tokens(n, seed):
    return [int(x) for x in np.random.default_rng(seed).integers(0, V, size=n)]


def slot_of(state, slot, n):
    return {k: state[k][slot * n:(slot + 1) * n] for k in state}


def engines(pkg, path, max_gpt, tc, seed=99):
    """(a, b): a runs generate_streams, b the host loop on the same path, both from the same non-trivial state."""
    a = pkg.Engine(path, max_gpt=max_gpt)
    b = pkg.Engine(path, max_gpt=max_gpt)
    if tc:
        b.set_option("prefill_min", 2)  # the loop's calls shrink below 8 streams as streams finish
    else:
        a.set_option("prefill", 0)
        b.set_option("prefill", 0)
    for i in range(0, max_gpt, 128):
        n = min(128, max_gpt - i)
        a.forward_streams([(i + j, [t]) for j, t in enumerate(rand_tokens(n, seed + i))], want_logits=False)
    b.state_upload(a.state_download(max_gpt), max_gpt)
    return a, b


def host_loop(eng, streams, max_new, budgets=None, stop=(), overrides=None, temp=1.0, u=None, pad_slot=None, greedy_api=False):
    """The loop generate_streams stands for, one forward_streams call per step over the live streams. pad_slot: a
    spare slot that keeps a lone live stream on the tensor cores (rows are independent, so the pad changes nothing)."""
    S = len(streams)
    budgets = list(budgets) if budgets is not None else [max_new] * S
    cur = [int(t) for _, t in streams]
    out = [[] for _ in range(S)]
    live = list(range(S))
    for step in range(max_new):
        if not live:
            break
        call = [(streams[s][0], [cur[s]]) for s in live]
        us = [float(u[step][s]) for s in live] if u is not None else None
        if pad_slot is not None and len(call) == 1:
            call.append((pad_slot, [cur[live[0]]]))
            us = us + [0.5] if us is not None else None
        if greedy_api:
            picks = [int(eng.forward_greedy(cur[live[0]]))]
        elif overrides:
            logits, _ = eng.forward_streams(call)
            for tok, val in overrides.items():
                logits[:, tok] = val
            picks = [int(np.argmax(r)) for r in logits]
        elif u is None:
            _, nxt = eng.forward_streams(call, want_logits=False, want_next=True)
            picks = [int(x) for x in nxt]
        else:
            eng.forward_streams(call, want_logits=False, want_next=True)
            toks, _ = eng.sample_typical_streams(temp, us)
            picks = [int(x) for x in toks]
        for i, s in enumerate(live):
            out[s].append(picks[i])
            cur[s] = picks[i]
        live = [s for s in live if len(out[s]) < budgets[s] and out[s][-1] not in stop]
    return out


def check(a, b, before, streams, got, want, max_gpt, what=""):
    n = a.n_layers * a.n_embed
    assert [len(x) for x in got] == [len(x) for x in want], what + ": lengths"
    for s, (g, w) in enumerate(zip(got, want)):
        assert [int(x) for x in g] == w, what + ": tokens of stream %d" % s
    sa, sb = a.state_download(max_gpt), b.state_download(max_gpt)
    named = {slot for slot, _ in streams}
    for slot in range(max_gpt):
        if slot in named:
            for k in KEYS:
                assert np.array_equal(slot_of(sa, slot, n)[k], slot_of(sb, slot, n)[k]), what + ": slot %d state %s" % (slot, k)
        else:
            for k in ("xy", "aa", "bb", "pp", "dd"):
                assert np.array_equal(slot_of(sa, slot, n)[k], slot_of(before, slot, n)[k]), what + ": slot %d was touched" % slot


def unconstrained(a, streams, max_new, max_gpt, **kw):
    """What a stream emits without stop tokens or budgets; a's state is restored afterwards."""
    st = a.state_download(max_gpt)
    seqs = a.generate_streams(streams, max_new, **kw)
    a.state_upload(st, max_gpt)
    return [[int(x) for x in s] for s in seqs]


def stops_at(seqs, targets):
    """Stop tokens that end stream j near step targets[j]: the first token at or after the target that the stream has
    not emitted before, preferring one that no other stream emits."""
    stop = []
    for j, t in targets.items():
        seq = seqs[j]
        fresh = [i for i in range(t, len(seq)) if seq[i] not in seq[:i]]
        alone = [i for i in fresh if all(seq[i] not in other for k, other in enumerate(seqs) if k != j)]
        if alone or fresh:
            stop.append(seq[(alone or fresh)[0]])
    return stop


@pytest.mark.parametrize("L,E", SHAPES)
def test_one_stream_decode_kernel_greedy(pkg, make_model, L, E):
    """One stream on slot 0 equals a forward_greedy loop, including a stop token hit mid-way: the stream's frozen rows
    run on the scratch slot until the group ends, and slot 0 stays where the loop left it."""
    max_gpt, max_new = 4, 40
    a, b = engines(pkg, make_model(L, E), max_gpt, tc=False)
    streams = [(0, 4118)]
    seq = unconstrained(a, streams, max_new, max_gpt)[0]
    fresh = [i for i in range(max_new - 1) if seq[i] not in seq[:i]]  # positions where a stop token ends the stream
    at = min(fresh, key=lambda i: abs(i - 21))
    stop = [seq[at]]
    before = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, stop=stop)
    want = host_loop(b, streams, max_new, stop=stop, greedy_api=True)
    assert len(want[0]) == at + 1 < max_new
    check(a, b, before, streams, got, want, max_gpt)
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", SHAPES)
def test_tensor_cores_twelve_streams_with_budgets_and_stops(pkg, make_model, L, E):
    max_gpt, max_new = 16, 40
    a, b = engines(pkg, make_model(L, E), max_gpt, tc=True)
    slots = [9, 0, 3, 12, 5, 1, 14, 7, 2, 11, 6, 10]
    streams = [(s, t) for s, t in zip(slots, rand_tokens(12, 7))]
    seqs = unconstrained(a, streams, max_new, max_gpt)
    stop = stops_at(seqs, {0: 0, 1: 20, 2: 35})
    budgets = [40, 7, 40, 16, 33, 17, 1, 40, 25, 40, 9, 40]
    before = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, budgets=budgets, stop=stop)
    want = host_loop(b, streams, max_new, budgets=budgets, stop=stop, pad_slot=15)
    assert len(want[0]) == 1 and len({len(w) for w in want}) >= 4, [len(w) for w in want]
    check(a, b, before, streams, got, want, max_gpt)
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", SHAPES)
def test_decode_kernel_three_streams(pkg, make_model, L, E):
    """prefill = 0: three streams through the decode kernel, ending at different steps (stop tokens and budgets)."""
    max_gpt, max_new = 6, 36
    a, b = engines(pkg, make_model(L, E), max_gpt, tc=False)
    streams = [(4, 11), (1, 4118), (2, 777)]
    seqs = unconstrained(a, streams, max_new, max_gpt)
    stop = stops_at(seqs, {1: 5})
    budgets = [20, 36, 36]
    before = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, budgets=budgets, stop=stop)
    want = host_loop(b, streams, max_new, budgets=budgets, stop=stop)
    check(a, b, before, streams, got, want, max_gpt)
    a.close()
    b.close()


def test_more_streams_than_one_pass(pkg, make_model):
    """150 streams: each step is a 128-row pass and a 22-row pass; budgets shrink the rows below one pass later."""
    max_gpt, max_new, S = 256, 20, 150
    a, b = engines(pkg, make_model(3, 768), max_gpt, tc=True)
    perm = [int(x) for x in np.random.default_rng(3).permutation(max_gpt)]
    streams = [(s, t) for s, t in zip(perm[:S], rand_tokens(S, 8))]
    budgets = [20 if i % 5 == 0 else 1 + (7 * i) % 16 for i in range(S)]
    before = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, budgets=budgets)
    want = host_loop(b, streams, max_new, budgets=budgets, pad_slot=perm[S])
    check(a, b, before, streams, got, want, max_gpt)
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", SHAPES)
@pytest.mark.parametrize("S,temp", [(1, 1.0), (10, 0.5)])
def test_typical_sampling(pkg, make_model, L, E, S, temp):
    """S = 1 runs on the decode kernel, S = 10 on the tensor cores; the loop samples with the same uniforms."""
    max_gpt, max_new = 12, 34
    a, b = engines(pkg, make_model(L, E), max_gpt, tc=S >= 8)
    streams = [(s, t) for s, t in zip(range(S - 1, -1, -1), rand_tokens(S, 9))]
    u = np.random.default_rng(10).random((max_new, S))
    budgets = [max_new - (3 * i) % 20 for i in range(S)]
    before = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, budgets=budgets, temp=temp, u=u)
    want = host_loop(b, streams, max_new, budgets=budgets, temp=temp, u=u, pad_slot=max_gpt - 1)
    check(a, b, before, streams, got, want, max_gpt)
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", SHAPES)
@pytest.mark.parametrize("S", [3, 9])
def test_overrides(pkg, make_model, L, E, S):
    """Each stream's unconstrained first pick is overridden to -99 before every pick; the loop does the same to its
    host logits and takes np.argmax (first index on ties)."""
    max_gpt, max_new = 12, 20
    a, b = engines(pkg, make_model(L, E), max_gpt, tc=S >= 8)
    streams = [(5 * s % 11, t) for s, t in zip(range(S), rand_tokens(S, 11))]
    tops = [seq[0] for seq in unconstrained(a, streams, 1, max_gpt)]
    overrides = {t: -99.0 for t in tops}
    before = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, overrides=overrides)
    want = host_loop(b, streams, max_new, overrides=overrides, pad_slot=max_gpt - 1)
    assert all(w[0] != t for w, t in zip(want, tops))
    check(a, b, before, streams, got, want, max_gpt)
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", SHAPES)
def test_continuation(pkg, make_model, L, E):
    """generate, then forward_streams from the last emitted token: one uninterrupted host loop."""
    max_gpt, first, more = 12, 18, 6
    a, b = engines(pkg, make_model(L, E), max_gpt, tc=True)
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
    check(a, b, before, streams, got, want, max_gpt)
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
