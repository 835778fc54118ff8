"""Multi-stream serving (rwkv_b200_forward_streams, the slot operations, the per-stream arg-max and sampler).

A token's arithmetic in a ragged pass depends only on its own row and on its own stream's predecessors: the GEMMs
are exact integers and every layernorm / mix reduction is per row. So each stream of a ragged pass must match, bit
for bit, the same stream run alone on the tensor-core path (GPT mode on slot 0 of a second engine with
prefill_min = 2). A stream of one token runs alone through the decode kernel, which agrees with the tensor cores
to 2e-5 (tests/test_prefill_gpu.py)."""
import time

import numpy as np
import pytest

from test_sampler_gpu import host_pick

pytestmark = pytest.mark.gpu

V = 50277
KEYS = ("xy", "aa", "bb", "dd")


def rel_err(got, ref):
    return float(np.abs(got.astype(np.float64) - ref.astype(np.float64)).max() / max(np.abs(ref).max(), 1e-6))


def rand_tokens(n, seed):
    return [int(x) for x in np.random.default_rng(seed).integers(0, V, size=n)]


def slot_of(state, slot, n):
    return {k: state[k][slot * n:(slot + 1) * n] for k in state}


def solo(eng, toks, start=None):
    """Logits of the last token and the state after running `toks` alone in GPT mode on slot 0 from `start`."""
    if start is None:
        eng.state_zero()
    else:
        eng.state_upload(start)
    last = eng.forward(toks, mode=1)[-1]
    return last, eng.state_download()


def check_against_solo(got_logits, got_state, ref_logits, ref_state, length, what):
    n = ref_state["xy"].size
    if length > 1:
        assert np.array_equal(got_logits, ref_logits), what + ": logits differ from the solo run"
        for k in KEYS:
            assert np.array_equal(got_state[k], ref_state[k][:n]), what + ": state " + k
    else:
        assert rel_err(got_logits, ref_logits) < 2e-5, what
        for k in KEYS:
            assert rel_err(got_state[k], ref_state[k][:n]) < 2e-5, what + ": state " + k


def run_ragged_vs_solo(pkg, path, max_gpt, streams):
    a = pkg.Engine(path, max_gpt=max_gpt)
    n = a.n_layers * a.n_embed
    a.forward(rand_tokens(min(max_gpt, 128), 99), mode=0, want_logits=False)  # every slot holds some state
    before = a.state_download(max_gpt)
    logits, nxt = a.forward_streams(streams, want_next=True)
    after = a.state_download(max_gpt)
    named = {s for s, _ in streams}
    for slot in range(max_gpt):
        if slot not in named:
            for k in ("xy", "aa", "bb", "pp", "dd"):
                assert np.array_equal(slot_of(after, slot, n)[k], slot_of(before, slot, n)[k]), "slot %d was touched" % slot
    assert [int(x) for x in nxt] == [int(np.argmax(r)) for r in logits]
    b = pkg.Engine(path, max_gpt=max(len(t) for _, t in streams))
    b.set_option("prefill_min", 2)
    for i, (slot, toks) in enumerate(streams):
        ref, sb = solo(b, toks, slot_of(before, slot, n))
        check_against_solo(logits[i], slot_of(after, slot, n), ref, sb, len(toks), "stream %d (slot %d, %d tokens)" % (i, slot, len(toks)))
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", [(3, 768), (2, 2048)])
def test_ragged_pass_matches_each_stream_alone(pkg, make_model, L, E):
    lens, slots = [1, 7, 16, 33, 60], [9, 0, 3, 12, 5]
    streams = [(s, rand_tokens(n, 10 + i)) for i, (s, n) in enumerate(zip(slots, lens))]
    run_ragged_vs_solo(pkg, make_model(L, E), 128, streams)


def test_stream_crossing_the_128_token_pass_boundary(pkg, make_model):
    lens, slots = [20, 150, 25, 5], [7, 2, 200, 0]
    streams = [(s, rand_tokens(n, 30 + i)) for i, (s, n) in enumerate(zip(slots, lens))]
    run_ragged_vs_solo(pkg, make_model(3, 768), 256, streams)


def test_gpt_and_parralel_are_special_cases(pkg, make_model):
    path = make_model(2, 2048)
    a, b = pkg.Engine(path, max_gpt=64), pkg.Engine(path, max_gpt=64)
    toks = rand_tokens(40, 1)
    got, _ = a.forward_streams([(0, toks)])
    ref = b.forward(toks, mode=1)
    assert np.array_equal(got[0], ref[-1])
    sa, sb = a.state_download(64), b.state_download(64)
    for k in KEYS:
        assert np.array_equal(sa[k], sb[k]), k
    T = 16
    for seed in (2, 3):  # two steps: the second continues from the slots the first left
        toks = rand_tokens(T, seed)
        got, _ = a.forward_streams([(i, [t]) for i, t in enumerate(toks)])
        ref = b.forward(toks, mode=0)
        assert np.array_equal(got, ref)
    sa, sb = a.state_download(64), b.state_download(64)
    for k in KEYS:
        assert np.array_equal(sa[k], sb[k]), k
    a.close()
    b.close()


def test_short_calls_run_through_the_decode_kernel(pkg, make_model):
    """Under prefill_min tokens, and with prefill = 0, a stream is the decode kernel on its own slot: the same bits
    as the decode kernel on slot 0."""
    path = make_model(3, 768)
    a = pkg.Engine(path, max_gpt=32)
    b = pkg.Engine(path, max_gpt=32)
    b.set_option("prefill", 0)
    n = a.n_layers * a.n_embed
    calls = [[(3, rand_tokens(2, 40)), (1, rand_tokens(1, 41)), (6, rand_tokens(2, 42))]]  # 5 tokens
    calls.append([(6, rand_tokens(9, 43)), (0, rand_tokens(11, 44))])                     # 20 tokens, prefill = 0
    for step, streams in enumerate(calls):
        if step == 1:
            a.set_option("prefill", 0)
        before = a.state_download(32)
        logits, nxt = a.forward_streams(streams, want_next=True)
        after = a.state_download(32)
        assert [int(x) for x in nxt] == [int(np.argmax(r)) for r in logits]
        for i, (slot, toks) in enumerate(streams):
            ref, sb = solo(b, toks, slot_of(before, slot, n))
            assert np.array_equal(logits[i], ref), (step, i)
            for k in KEYS:
                assert np.array_equal(slot_of(after, slot, n)[k], sb[k][:n]), (step, i, k)
    a.close()
    b.close()


def test_graph_replay_follows_the_slots_of_each_call(pkg, make_model):
    """Two calls of the same shape (8 streams x 2 tokens) on different slot sets replay one recorded graph; both must
    match solo runs, which they would not if the first call's layout were part of the graph."""
    path = make_model(2, 2048)
    a = pkg.Engine(path, max_gpt=64)
    b = pkg.Engine(path, max_gpt=8)
    b.set_option("prefill_min", 2)
    n = a.n_layers * a.n_embed
    for slots in ([0, 1, 2, 3, 4, 5, 6, 7], [40, 3, 17, 9, 63, 22, 1, 50]):
        streams = [(s, rand_tokens(2, 100 + s)) for s in slots]
        before = a.state_download(64)
        logits, nxt = a.forward_streams(streams, want_next=True)
        after = a.state_download(64)
        assert [int(x) for x in nxt] == [int(np.argmax(r)) for r in logits]
        for i, (slot, toks) in enumerate(streams):
            ref, sb = solo(b, toks, slot_of(before, slot, n))
            check_against_solo(logits[i], slot_of(after, slot, n), ref, sb, 2, "slots %s stream %d" % (slots[:3], i))
    a.close()
    b.close()


def test_continuous_batching(pkg, make_model):
    """Six requests on three slots: each joins when a slot is free (after slot_zero), prefills its prompt in the same
    call as the others' next tokens, decodes 20 teacher-forced tokens and leaves."""
    path = make_model(3, 768)
    prompts = [rand_tokens(n, 200 + i) for i, n in enumerate([12, 3, 20, 1, 9, 30])]
    decode = [rand_tokens(20, 300 + i) for i in range(6)]
    arrive = [0, 0, 2, 5, 9, 12]
    a = pkg.Engine(path, max_gpt=64)
    free, active, waiting, got = [0, 1, 2], {}, list(range(6)), {r: [] for r in range(6)}
    step = 0
    while waiting or active:
        joining = [r for r in waiting if arrive[r] <= step][:len(free)]
        for r in joining:
            waiting.remove(r)
            active[r] = [free.pop(0), 0]  # slot, decode tokens fed so far
            a.slot_zero(active[r][0])
        streams, owners = [], []
        for r, (slot, fed) in sorted(active.items(), key=lambda kv: kv[1][0]):
            streams.append((slot, prompts[r] if r in joining else [decode[r][fed - 1]]))
            owners.append(r)
        if not streams:
            step += 1
            continue
        logits, _ = a.forward_streams(streams)
        for i, r in enumerate(owners):
            got[r].append(logits[i])
            active[r][1] += 1
            if active[r][1] > 20:
                free.append(active.pop(r)[0])
        step += 1
    b = pkg.Engine(path, max_gpt=64)
    for r in range(6):
        b.state_zero()
        ref = [b.forward(prompts[r], mode=1)[-1]] + [b.forward([t])[0] for t in decode[r][:20]]
        assert len(got[r]) == 21
        worst = max(rel_err(g, w) for g, w in zip(got[r], ref))
        assert worst < 2e-5, "request %d: %g" % (r, worst)
    a.close()
    b.close()


def test_slot_operations(pkg, make_model):
    path = make_model(3, 768)
    a = pkg.Engine(path, max_gpt=16)
    n = a.n_layers * a.n_embed
    toks = rand_tokens(12, 5)
    a.forward_streams([(2, toks)], want_logits=False)
    a.slot_copy(2, 5)
    logits, _ = a.forward_streams([(2, [4118]), (5, [4118])])
    assert np.array_equal(logits[0], logits[1])
    assert all(np.array_equal(a.slot_download(2)[k], a.slot_download(5)[k]) for k in KEYS)
    rng = np.random.default_rng(6)
    st = {k: rng.standard_normal(n) for k in ("xy", "aa", "bb", "pp", "dd")}
    a.slot_upload(7, st)
    back = a.slot_download(7)
    assert all(np.array_equal(back[k], st[k]) for k in st)
    assert np.array_equal(a.state_download(16)["aa"][7 * n:8 * n], st["aa"])
    a.slot_zero(2)
    got, _ = a.forward_streams([(2, toks)])
    fresh = pkg.Engine(path, max_gpt=16)
    ref, _ = fresh.forward_streams([(2, toks)])
    assert np.array_equal(got, ref)
    a.close()
    fresh.close()


@pytest.mark.parametrize("temp", [1.0, 0.5])
def test_sampler_per_stream(pkg, make_model, temp):
    a = pkg.Engine(make_model(2, 768), max_gpt=16)
    streams = [(s, rand_tokens(1 + s % 3, 60 + s)) for s in (4, 0, 9, 2, 11, 7)]
    logits, _ = a.forward_streams(streams)
    rng = np.random.default_rng(8)
    checked = 0
    for _ in range(20):
        us = rng.random(len(streams))
        toks, margins = a.sample_typical_streams(temp, us)
        for s in range(len(streams)):
            want, _ = host_pick(logits[s], temp, us[s])
            if margins[s] >= 1e-9:
                assert int(toks[s]) == want, (s, us[s])
                checked += 1
    assert checked >= 100
    a.close()


def test_rejected_calls_leave_the_state_untouched(pkg, make_model):
    import ctypes
    path = make_model(2, 768)
    a = pkg.Engine(path, max_gpt=8)
    a.forward(rand_tokens(8, 70), mode=0, want_logits=False)
    before = a.state_download(8)
    bad = [
        ([(1, [5]), (1, [6])], "appears twice"),
        ([(8, [5])], "slot 8 >= max_gpt"),
        ([(1, [5, 6]), (2, [])], "length 0"),
        ([(0, rand_tokens(9, 71))], "9 tokens > max_gpt"),
        ([(0, [5, 50277])], "out of range"),
    ]
    for streams, msg in bad:
        with pytest.raises(pkg.EngineError, match=msg):
            a.forward_streams(streams)
    toks = np.array([1, 2, 3], np.uint64)
    slots, lens = np.array([0, 1], np.uint64), np.array([1, 1], np.uint64)
    P = ctypes.POINTER(ctypes.c_ulonglong)
    rc = a.lib.rwkv_b200_forward_streams(a.h, toks.ctypes.data_as(P), 3, slots.ctypes.data_as(P), lens.ctypes.data_as(P), 2, None, None)
    assert rc != 0 and b"add up to 2" in a.lib.rwkv_b200_last_error()
    after = a.state_download(8)
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    a.forward([5])
    with pytest.raises(pkg.EngineError, match="no per-stream logits"):
        a.sample_typical_streams(1.0, [0.5])
    a.forward_streams([(0, [5]), (1, [6])], want_logits=False)
    with pytest.raises(pkg.EngineError, match="no per-stream logits"):
        a.sample_typical_streams(1.0, [0.5, 0.5])
    a.forward_streams([(0, [5]), (1, [6])])
    with pytest.raises(pkg.EngineError, match="3 rows asked"):
        a.sample_typical_streams(1.0, [0.5, 0.5, 0.5])
    for call in (lambda: a.slot_zero(8), lambda: a.slot_copy(0, 8), lambda: a.slot_download(9)):
        with pytest.raises(pkg.EngineError, match="max_gpt"):
            call()
    a.close()
    # a tensor-parallel rank (never wired, so no forward runs) refuses every multi-stream entry point
    t = pkg.Engine(path, max_gpt=4, tp_rank=0, tp_size=2)
    for call in (lambda: t.forward_streams([(0, [5])]), lambda: t.sample_typical_streams(1.0, [0.5]), lambda: t.slot_zero(0),
                 lambda: t.slot_copy(0, 1), lambda: t.slot_download(0), lambda: t.slot_upload(0, {})):
        with pytest.raises(pkg.EngineError, match="not supported with tensor parallelism"):
            call()
    t.close()


def test_multi_stream_decode_step_is_faster_than_single_forwards(pkg, make_model):
    """One 16-stream decode step through forward_streams (weights read once) against 16 single-token forwards."""
    path = make_model(2, 4096)
    S = 16
    a = pkg.Engine(path, max_gpt=S)
    toks = rand_tokens(S, 80)
    streams = [(s, [t]) for s, t in enumerate(toks)]
    a.forward_streams(streams, want_logits=False, want_next=True)  # records the graph of the shape
    t0 = time.perf_counter()
    for _ in range(5):
        a.forward_streams(streams, want_logits=False, want_next=True)
    batched = (time.perf_counter() - t0) / 5
    for t in toks:
        a.forward([t], want_logits=False)
    t0 = time.perf_counter()
    for _ in range(5):
        for t in toks:
            a.forward([t], want_logits=False)
    single = (time.perf_counter() - t0) / 5
    print("L=2 E=4096, %d streams: one forward_streams step %.2f ms, %d single-token forwards %.2f ms: %.1fx"
          % (S, batched * 1e3, S, single * 1e3, single / batched))
    assert batched < single
    a.close()
