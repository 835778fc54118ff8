"""Stop strings on the device (rwkv_b200_generate_streams_stop, the speculative call and the batcher).

The oracle is the host rule (engine.stop_match) applied to engine b's run of the same call without stop sets, from the
same state on the same forward path: it gives each stream's stop token j, hit, tail and match state. Engine b then
reruns from that state with every budget cut to min(budget, j + 1), and engine a's tokens, lengths, hit, tail, state,
log-probabilities, automaton states and named slots must equal b's bit for bit; every other slot must be untouched. The
stop strings are cut from b's own output, so matches are certain on a random synthetic model."""
import ctypes

import numpy as np
import pytest

from decoding import OVERRIDES, REGEXES, SHAPES, V, check_slots, engine_pair, mixed_samplers, rand_tokens, stops_at

pytestmark = pytest.mark.gpu

MAX_GPT = 12
FIELDS = ("logprobs", "ranks", "top_tokens", "top_logprobs", "state")


@pytest.fixture(scope="module")
def tbytes(pkg):
    return pkg.constrain.token_bytes()


@pytest.fixture(scope="module")
def number(pkg, tbytes):
    C = pkg.constrain
    return C.token_automaton(C.compile_regex(REGEXES["number"]), tbytes, eos=0)


def toks(r):
    return [int(x) for x in (r["tokens"] if isinstance(r, dict) else r)]


def strings_for(kind, chunks):
    """Stop strings cut from one stream's output bytes (chunks: the bytes of each token), or None."""
    n = len(chunks)
    mid = n // 2
    ok = lambda k, m: 0 <= k < n and len(chunks[k]) >= m
    if kind == "span2":  # two tokens, ending inside the second: tail > 0
        for k in list(range(mid, n - 1)) + list(range(0, mid)):
            if ok(k, 2) and ok(k + 1, 2):
                return [chunks[k][1:] + chunks[k + 1][:1]]
    if kind == "span3":  # three tokens
        for k in list(range(mid, n - 2)) + list(range(0, mid)):
            if ok(k, 1) and ok(k + 1, 1) and ok(k + 2, 1):
                return [chunks[k][-1:] + chunks[k + 1] + chunks[k + 2][:1]]
    if kind == "first" and ok(0, 1):  # a match in the first emitted token
        return [b"\x01never\x02", chunks[0][:1]]
    if kind == "multi":  # the earlier-ending string wins, whatever its index
        late = b"".join(chunks[mid:mid + 2])
        early = b"".join(chunks[max(mid - 3, 0):mid - 1])
        if late and early:
            return [late, early, late[-1:] + b"\x03"]
    if kind == "absent":
        return [b"\x01\x02\x03never"]
    if kind is None:
        return None
    whole = [c for c in chunks if c]
    return [whole[len(whole) // 2]] if whole else [b"\x01"]


KINDS = ["span2", None, "span3", "first", "multi", "absent", "span2"]


def expect(pkg, sets, outs, tbytes, starts=None):
    """Per stream (j or None, hit, tail, state) by the host rule; None for a stream without a set."""
    res = []
    for s, (st, out) in enumerate(zip(sets, outs)):
        if st is None:
            res.append(None)
            continue
        res.append(pkg.engine.stop_match(st, [tbytes[t] for t in out], starts[s] if starts else 0))
    return res


def add_sets(eng, sets):
    return [eng.add_stop_set(st) if st is not None else None for st in sets]


VARIANTS = ["argmax", "nucleus", "overrides", "logprobs_raw", "logprobs_processed", "constrained"]


def variant_kwargs(pkg, variant, S, max_new, number, eng):
    u = np.random.default_rng(31).random((max_new, S))
    if variant == "argmax":
        return {}
    if variant == "nucleus":
        return dict(sampling=mixed_samplers(pkg, S), u=u)
    if variant == "overrides":
        return dict(sampling=mixed_samplers(pkg, S), u=u, overrides=OVERRIDES)
    if variant == "logprobs_raw":
        return dict(sampling=mixed_samplers(pkg, S), u=u, overrides=OVERRIDES, logprobs="raw", top_n=3)
    if variant == "logprobs_processed":
        return dict(sampling=mixed_samplers(pkg, S), u=u, logprobs="processed", top_n=2)
    cid = eng.add_constraint(number)
    return dict(sampling=mixed_samplers(pkg, S, [(0.0,), (1.0, 0.9)]), u=u, constraints=[cid, None, cid] + [None] * (S - 3))


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("tc", [False, True])
@pytest.mark.parametrize("L,E", SHAPES)
def test_against_the_host_rule(pkg, make_model, tbytes, number, L, E, tc, variant):
    """Seven streams: strings spanning two and three tokens, ending mid-token, matching in the first token, several
    strings where the earlier end wins, one that never matches, and a stream without a set; budgets and a stop token."""
    S, max_new = 7, 28
    a, b = engine_pair(pkg, make_model(L, E), MAX_GPT, tc=tc, a_prefill_min=True)
    before = a.state_download(MAX_GPT)
    streams = [(s + 1, t) for s, t in enumerate(rand_tokens(S, 17))]
    budgets = [max_new - (3 * s) % 7 for s in range(S)]
    kw_a = variant_kwargs(pkg, variant, S, max_new, number, a)
    kw_b = variant_kwargs(pkg, variant, S, max_new, number, b)
    run0 = b.generate_streams(streams, max_new, budgets=budgets, **kw_b)
    stop = stops_at([toks(r) for r in run0], {5: 10})  # the never-matching stream ends on a stop token
    b.state_upload(before, MAX_GPT)
    full = [toks(r) for r in b.generate_streams(streams, max_new, budgets=budgets, stop=stop, **kw_b)]
    sets = [strings_for(KINDS[s], [tbytes[t] for t in full[s]]) for s in range(S)]
    rule = expect(pkg, sets, full, tbytes)
    cut = [min(budgets[s], r[0] + 1) if r and r[0] is not None else budgets[s] for s, r in enumerate(rule)]
    b.state_upload(before, MAX_GPT)
    want = b.generate_streams(streams, max_new, budgets=cut, stop=stop, **kw_b)
    got = a.generate_streams(streams, max_new, budgets=budgets, stop=stop, stop_strings=add_sets(a, sets), **kw_a)
    for s in range(S):
        assert toks(got[s]) == toks(want[s]), "stream %d: tokens" % s
        r = rule[s]
        if r is None:
            assert (got[s]["stop_hit"], got[s]["stop_tail"], got[s]["stop_state"]) == (None, 0, None), s
        else:
            assert (got[s]["stop_hit"], got[s]["stop_tail"], got[s]["stop_state"]) == (r[1], r[2], r[3]), s
        for f in FIELDS:
            if isinstance(want[s], dict) and f in want[s]:
                assert np.asarray(got[s][f]).tobytes() == np.asarray(want[s][f]).tobytes(), (s, f)
    check_slots(a, b, before, MAX_GPT, {slot for slot, _ in streams}, what=variant)
    hits = [r for r in rule if r and r[0] is not None]
    assert len(hits) >= 4, "too few matches: %s" % rule
    assert rule[3][0] == 0, "no match in the first token"
    assert any(r[2] > 0 for r in hits), "no match ending mid-token"
    a.close()
    b.close()


@pytest.mark.parametrize("tc", [False, True])
def test_two_calls_continued_equal_one(pkg, make_model, tbytes, tc):
    """start_states = states_out of a first call: the second call gives the tokens and hits of one call."""
    S, n1, n2 = 4, 10, 14
    a, b = engine_pair(pkg, make_model(3, 768), MAX_GPT, tc=tc, a_prefill_min=True)
    before = a.state_download(MAX_GPT)
    streams = [(s + 2, t) for s, t in enumerate(rand_tokens(S, 41))]
    full = [toks(r) for r in b.generate_streams(streams, n1 + n2)]
    sets = []
    for s in range(S):  # strings across the call boundary (tokens n1 - 1 .. n1 + s % 3)
        ch = [tbytes[t] for t in full[s]]
        sets.append([b"".join(ch[n1 - 1:n1 + 1 + s % 3])[-(3 + s):] or b"\x01"])
    one = a.generate_streams(streams, n1 + n2, stop_strings=add_sets(a, sets))
    a.state_upload(before, MAX_GPT)
    ids = add_sets(a, sets)
    first = a.generate_streams(streams, n1, stop_strings=ids)
    cont = [s for s in range(S) if first[s]["stop_hit"] is None]
    assert cont, "every stream matched inside the first call"
    second = a.generate_streams([(streams[s][0], int(first[s]["tokens"][-1])) for s in cont], n2,
                                stop_strings=[(ids[s], first[s]["stop_state"]) for s in cont])
    for s in range(S):
        got = toks(first[s]) + (toks(second[cont.index(s)]) if s in cont else [])
        last = second[cont.index(s)] if s in cont else first[s]
        assert got == toks(one[s]), s
        assert (last["stop_hit"], last["stop_tail"], last["stop_state"]) == \
            (one[s]["stop_hit"], one[s]["stop_tail"], one[s]["stop_state"]), s
    assert any(one[s]["stop_hit"] is not None for s in cont)
    a.close()
    b.close()


SPEC_GPT = 70
PAD = SPEC_GPT - 1


@pytest.mark.parametrize("L,E", SHAPES)
def test_speculative_equals_generate(pkg, make_model, tbytes, L, E):
    """Drafts from the greedy continuation run through the stop strings: tokens, lengths, first slots and hit, tail
    and state equal generate_streams(stop_strings=..., sampling=...) on the tensor cores."""
    S, k, max_new = 5, 7, 30
    a, b = engine_pair(pkg, make_model(L, E), SPEC_GPT, tc=True, seed=5, one_draw=True)
    before = a.state_download(SPEC_GPT)
    slot_lists = [[s * (k + 1) + i for i in range(k + 1)] for s in range(S)]
    firsts = [(sl[0], t) for sl, t in zip(slot_lists, rand_tokens(S, 8))]
    samp = [pkg.Sampler(temperature=0.0)] * S
    ceil = [toks(r) for r in b.generate_streams(firsts, max_new + 8, sampling=samp)]
    b.state_upload(before, SPEC_GPT)
    context = [[f] + c for (_, f), c in zip(firsts, ceil)]
    sets = [strings_for(KINDS[s], [tbytes[t] for t in ceil[s][:max_new]]) for s in range(S)]
    want = b.generate_streams(firsts, max_new, sampling=samp, stop_strings=add_sets(b, sets))
    got = a.generate_speculative([(sl, f) for sl, (_, f) in zip(slot_lists, firsts)], max_new, draft=k, context=context,
                                 stop_strings=add_sets(a, sets))
    for s in range(S):
        assert toks(got[s]) == toks(want[s]), s
        for f in ("stop_hit", "stop_tail", "stop_state"):
            assert got[s][f] == want[s][f], (s, f)
    assert any(g["steps"] < len(g["tokens"]) for g in got), "no step accepted a draft"
    assert sum(w["stop_hit"] is not None for w in want) >= 3
    spares = {x for sl in slot_lists for x in sl[1:]}
    check_slots(a, b, before, SPEC_GPT, {sl[0] for sl in slot_lists}, skip=spares)
    a.close()
    b.close()


BAT_GPT = 40


def bat_oracle(pkg, b, r, sid):
    """The batcher rule for one request on engine b: forward_streams(prompt[:-1]), then generate_streams_stop of the one
    stream (and a pad stream on a slot no request names)."""
    slot, prompt = r["slot"], r["prompt"]
    if len(prompt) > 1:
        b.forward_streams([(slot, prompt[:-1]), (BAT_GPT - 1, prompt[:1])], want_logits=False)
    us = None if r["u"] is None else np.stack([r["u"], np.full(r["max_new"], 0.5)], axis=1)
    out = b.generate_streams([(slot, prompt[-1]), (BAT_GPT - 1, prompt[-1])], r["max_new"], stop=r["stop"],
                             sampling=[r["sampling"], pkg.Sampler(temperature=0.0)], u=us,
                             stop_strings=[sid, None])
    return out[0]


def test_batcher_requests_equal_one_shot_calls(pkg, make_model, tbytes):
    """Mixed traffic (sets and no sets, greedy and sampled, prompts of several lengths) through rows = 3, with one
    cancellation: each request equals its one-shot generate_streams_stop; removing a set that an unfinished request
    names is refused."""
    a, b = engine_pair(pkg, make_model(3, 768), BAT_GPT, tc=True, seed=3, one_draw=True)
    before = a.state_download(BAT_GPT)
    rng = np.random.default_rng(12)
    reqs = []
    for i in range(8):
        mn = int(rng.integers(8, 30))
        samp = pkg.Sampler(temperature=0.0) if i % 2 else pkg.Sampler(temperature=0.9, top_p=0.9)
        reqs.append(dict(slot=i + 1, prompt=rand_tokens(1 + (7 * i) % 20, 50 + i), max_new=mn, sampling=samp,
                         u=rng.random(mn) if i % 2 == 0 else None, stop=()))
    sets = []
    for i, r in enumerate(reqs):  # strings from each request's own run
        out = toks(bat_oracle(pkg, b, r, None))
        b.state_upload(before, BAT_GPT)
        sets.append(None if i % 4 == 3 else strings_for(KINDS[i % 7], [tbytes[t] for t in out]))
    ids_a, ids_b = add_sets(a, sets), add_sets(b, sets)
    want = []
    for r, sid in zip(reqs, ids_b):
        want.append(bat_oracle(pkg, b, r, sid))
    with a.batcher(3, 16) as bat:
        rids = [bat.submit(r["slot"], r["prompt"], r["max_new"], sampling=r["sampling"], u=r["u"],
                           stop_strings=sid) if sid is not None else
                bat.submit(r["slot"], r["prompt"], r["max_new"], sampling=r["sampling"], u=r["u"])
                for r, sid in zip(reqs, ids_a)]
        bat.run(16)
        held = [i for i, rid in enumerate(rids) if ids_a[i] is not None and bat.result(rid)["status"] != "done"]
        assert held, "every request with a set finished in the first group"
        with pytest.raises(pkg.EngineError, match="unfinished request"):
            a.remove_stop_set(ids_a[held[0]])
        live = [i for i, rid in enumerate(rids) if bat.result(rid)["status"] in ("prefilling", "generating")]
        cancelled = live[-1] if live else None
        if cancelled is not None:
            bat.cancel(rids[cancelled])
        while bat.run(16):
            pass
        res = [bat.result(rid) for rid in rids]
    for i, (g, w) in enumerate(zip(res, want)):
        if i == cancelled:
            assert toks(g) == toks(w)[:len(g["tokens"])], i
            continue
        assert toks(g) == toks(w), i
        if ids_a[i] is not None:
            assert (g["stop_hit"], g["stop_tail"], g["stop_state"]) == (w["stop_hit"], w["stop_tail"], w["stop_state"]), i
    assert sum(w["stop_hit"] is not None for w in want) >= 3
    a.remove_stop_set(ids_a[0])  # every request has ended
    a.close()
    b.close()


def test_refusals_leave_every_slot_untouched(pkg, make_model, tbytes):
    a = pkg.Engine(make_model(3, 768), max_gpt=MAX_GPT)
    a.forward_streams([(j, [t]) for j, t in enumerate(rand_tokens(MAX_GPT, 9))], want_logits=False)
    before = a.state_download(MAX_GPT)
    lib, P, B = a.lib, ctypes.c_ulonglong, ctypes.c_ubyte
    streams = [(1, 11), (2, 12)]

    def add_raw(strings):
        start, data = pkg.engine.stop_set_bytes(strings)
        sid = P()
        rc = lib.rwkv_b200_stop_set_add(a.h, len(start) - 1, start.ctypes.data_as(ctypes.POINTER(P)),
                                        data.ctypes.data_as(ctypes.POINTER(B)), ctypes.byref(sid))
        return rc, int(sid.value)

    rc, early = add_raw(["ab"])  # before the model has token bytes
    assert rc == 0
    with pytest.raises(pkg.EngineError, match="before the model has a token-bytes table"):
        a.generate_streams(streams, 4, stop_strings=early)
    sid = a.add_stop_set(["ab", "abc"])
    with pytest.raises(pkg.EngineError, match="out of range"):
        a.generate_streams(streams, 4, stop_strings=[(sid, 4), None])
    with pytest.raises(pkg.EngineError, match="unknown or removed"):
        a.generate_streams(streams, 4, stop_strings=sid + 100)
    a.remove_stop_set(sid)
    with pytest.raises(pkg.EngineError, match="unknown or removed"):
        a.generate_streams(streams, 4, stop_strings=sid)
    with pytest.raises(pkg.EngineError, match="unknown or removed"):
        a.remove_stop_set(sid)
    for bad, msg in (([], "no strings"), (["a", ""], "empty"), (["x" * 4000, "y" * 97], "4097 bytes")):
        with pytest.raises(pkg.EngineError, match=msg):
            a.add_stop_set(bad)
    with pytest.raises(pkg.EngineError, match="stop_strings need sampling"):
        a.generate_streams(streams, 4, u=np.zeros((4, 2)), stop_strings=early)
    tb = np.zeros(V + 1, np.uint64)
    tb[5] = 3  # decreasing afterwards
    assert lib.rwkv_b200_token_bytes_set(a.h, tb.ctypes.data_as(ctypes.POINTER(P)), None) != 0
    after = a.state_download(MAX_GPT)
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    # the table is still the one add_stop_set uploaded
    sid = a.add_stop_set(tbytes[11][:1] or b"\x01")
    got = a.generate_streams([(1, 11), (2, 12)], 3, stop_strings=[sid, None])
    assert got[1]["stop_hit"] is None
    a.close()
