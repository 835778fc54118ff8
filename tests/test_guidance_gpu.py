"""Classifier-free guidance on the device (rwkv_b200_generate_streams_guided) against a host loop on engine b from the
same state and on the same path: each step one forward_streams call over every live stream's slot and every live
guidance slot, engine.guide_rows, then the host pick chain of decoding.host_decode (penalties in f32, overrides, the
automaton mask, sample_streams(logits=...) with the same u), the stop strings by engine.stop_match and the
log-probabilities by decoding.logprob_rule. Tokens, automaton and stop states and the slots the call names are bit for
bit b's; every other slot is untouched. Also: scale 1 is the unguided call bit for bit, guidance=None enqueues what
generate_streams_stop enqueues, and every refusal leaves every slot untouched."""
import ctypes

import numpy as np
import pytest

import decoding as dc

pytestmark = pytest.mark.gpu

M = 24  # slots of the engines of a case


def host_guided(pkg, eng, streams, guidance, max_new, samplers, u=None, budgets=None, stop=(), overrides=None,
                constraints=None, stop_sets=None, tbytes=None, logprobs=None, top_n=0, pad_slot=None):
    """The guided call as a host loop on eng (module docstring). guidance[s]: None or (slot, first token, scale);
    constraints[s]: (automaton, start state) or None; stop_sets[s]: the strings of its stop set or None. Returns
    (tokens, automaton states, stop results (j, hit, tail, state) or None, per stream the (logprob, rank, top tokens,
    top logprobs) of each emitted token in the mode `logprobs`)."""
    S = len(streams)
    budgets = list(budgets) if budgets is not None else [max_new] * S
    cons = constraints if constraints is not None else [None] * S
    sets = stop_sets if stop_sets is not None else [None] * S
    V = dc.V
    cnt = [np.zeros(V, np.float32) for _ in range(S)]
    seen = [np.zeros(V, bool) for _ in range(S)]
    pen = [sp.presence_penalty != 0 or sp.frequency_penalty != 0 for sp in samplers]
    cur = [int(t) for _, t in streams]
    gcur = [int(g[1]) if g is not None else None for g in guidance]
    state = [c[1] if c else None for c in cons]
    stop_res = [None] * S
    out = [[] for _ in range(S)]
    lps = [[] for _ in range(S)]
    live = list(range(S))
    for step in range(max_new):
        if not live:
            break
        gl = [s for s in live if guidance[s] is not None]
        call = [(streams[s][0], [cur[s]]) for s in live] + [(guidance[s][0], [gcur[s]]) for s in gl]
        if pad_slot is not None and len(call) == 1:
            call.append((pad_slot, [cur[live[0]]]))
        logits, _ = eng.forward_streams(call)
        raws, rows, ps, us = [], [], [], []
        for i, s in enumerate(live):
            sp, raw = samplers[s], logits[i].copy()
            row = raw.copy()
            if guidance[s] is not None:
                row = pkg.engine.guide_rows(raw, logits[len(live) + gl.index(s)], guidance[s][2])
            if pen[s]:
                k = seen[s]
                row[k] = row[k] - (np.float32(sp.presence_penalty) + np.float32(sp.frequency_penalty) * cnt[s][k])
            for tok, val in (overrides or {}).items():
                row[tok] = val
            if cons[s]:
                row[~dc.allowed(cons[s][0], state[s])] = -np.inf
            raws.append(raw)
            rows.append(row)
            ps.append(pkg.Sampler(sp.temperature, sp.top_p, sp.top_k))
            us.append(float(u[step][s]) if u is not None else 0.0)
        toks, _ = eng.sample_streams(ps, us, logits=np.stack(rows))
        ended = set()
        for i, s in enumerate(live):
            x = int(toks[i])
            if logprobs == "raw":
                lps[s].append(dc.logprob_rule(raws[i], x, top_n))
            elif logprobs == "processed":
                t = samplers[s].temperature
                lps[s].append(dc.logprob_rule(rows[i], x, top_n, float(np.float32(t)) if t > 0 else 1.0))
            out[s].append(x)
            cur[s] = x
            if guidance[s] is not None:
                gcur[s] = x
            if pen[s]:
                cnt[s] = cnt[s] * np.float32(samplers[s].penalty_decay)
                cnt[s][x] += np.float32(1.0)
                seen[s][x] = True
            if cons[s]:
                state[s] = cons[s][0].walk([x], state[s])
                assert state[s] is not None, "the host loop picked a masked token"
                if cons[s][0].complete(state[s]):
                    ended.add(s)
            if sets[s] is not None:
                stop_res[s] = pkg.engine.stop_match(sets[s], [tbytes[t] for t in out[s]])
                if stop_res[s][0] is not None:
                    ended.add(s)
        live = [s for s in live if len(out[s]) < budgets[s] and out[s][-1] not in stop and s not in ended]
    return out, state, stop_res, lps


def named_slots(streams, guidance):
    return {slot for slot, _ in streams} | {g[0] for g in guidance if g is not None}


def check_case(pkg, a, b, streams, guidance, max_new, samplers, what, u=None, tbytes=None, constraints=None,
               stop_sets=None, logprobs=None, top_n=0, m=M, **kw):
    """The guided call on a against host_guided on b (engines of m slots; the last is b's pad): tokens, states of the
    named slots, every other slot untouched, and, where asked for, automaton states, stop results and
    log-probabilities."""
    before = a.state_download(m)
    dev_kw = dict(kw)
    if constraints is not None:
        ids = {}
        dev_kw["constraints"] = [None if c is None else (ids.setdefault(id(c[0]), a.add_constraint(c[0])), c[1])
                                 for c in constraints]
    if stop_sets is not None:
        dev_kw["stop_strings"] = [None if st is None else a.add_stop_set(st) for st in stop_sets]
    if logprobs is not None:
        dev_kw.update(logprobs=logprobs, top_n=top_n)
    got = a.generate_streams(streams, max_new, sampling=samplers, u=u, guidance=guidance, **dev_kw)
    want, states, stops, lps = host_guided(pkg, b, streams, guidance, max_new, samplers, u=u, constraints=constraints,
                                           stop_sets=stop_sets, tbytes=tbytes, logprobs=logprobs, top_n=top_n,
                                           pad_slot=m - 1, **kw)
    dicts = constraints is not None or stop_sets is not None or logprobs is not None
    for s in range(len(streams)):
        g = got[s] if dicts else {"tokens": got[s]}
        assert [int(x) for x in g["tokens"]] == want[s], what + ": tokens of stream %d" % s
        if constraints is not None:
            assert g["state"] == (states[s] if constraints[s] else None), what + ": automaton state of stream %d" % s
        if stop_sets is not None and stop_sets[s] is not None:
            j, hit, tail, q = stops[s]
            assert (g["stop_hit"], g["stop_tail"], g["stop_state"]) == (hit, tail if j is not None else 0, q), (what, s)
        if logprobs is not None:
            for k, (lp, rank, top, top_lp) in enumerate(lps[s]):
                assert int(g["ranks"][k]) == rank, (what, s, k)
                assert abs(g["logprobs"][k] - lp) <= 1e-9, (what, s, k, g["logprobs"][k], lp)
                if top_n:
                    assert [int(x) for x in g["top_tokens"][k]] == [int(x) for x in top], (what, s, k)
                    assert dc.close(g["top_logprobs"][k], top_lp), (what, s, k)
    dc.check_slots(a, b, before, m, named_slots(streams, guidance), skip={m - 1}, what=what)
    return got


def pair(pkg, make_model, L, E, tc, max_gpt=M):
    return dc.engine_pair(pkg, make_model(L, E), max_gpt, tc, a_prefill_min=True)


PATHS = [False, True]  # the decode kernel (prefill 0 on both engines), the tensor cores (prefill_min 2 on both)


@pytest.mark.parametrize("tc", PATHS)
@pytest.mark.parametrize("L,E", dc.SHAPES)
def test_guided_streams(pkg, make_model, L, E, tc):
    """One guided arg-max stream; three sampled streams at gamma 0, 0.5, 1.5 and 3 with penalties; guided and unguided
    streams in one call; penalties with overrides."""
    a, b = pair(pkg, make_model, L, E, tc)
    check_case(pkg, a, b, [(1, 11)], [(9, 500, 1.5)], 12, [pkg.Sampler(0.0)], "arg-max")
    samplers = dc.mixed_samplers(pkg, 4)
    u = np.random.default_rng(3).random((14, 4))
    check_case(pkg, a, b, [(0, 11), (2, 500), (4, 4118), (6, 7)], [(10, 3, 0.0), (12, 500, 0.5), (14, 0, 1.5), (16, 9, 3.0)],
               14, samplers, "mixed samplers", u=u)
    check_case(pkg, a, b, [(3, 187), (5, 11), (7, 4118)], [(11, 187, 2.0), None, (13, 0, 0.5)], 10,
               dc.mixed_samplers(pkg, 3), "guided and unguided", u=u[:10, :3])
    pens = [pkg.Sampler(0.0, 1.0, 0, 0.7, 0.4, 0.95), pkg.Sampler(1.0, 0.9, 40, 0.3, 0.6, 1.0)]
    check_case(pkg, a, b, [(8, 11), (15, 500)], [(17, 11, 1.5), (18, 4118, 3.0)], 12, pens, "penalties and overrides",
               u=u[:12, :2], overrides=dc.OVERRIDES)
    a.close()
    b.close()


@pytest.mark.parametrize("mode", ["raw", "processed"])
@pytest.mark.parametrize("tc", PATHS)
@pytest.mark.parametrize("L,E", dc.SHAPES)
def test_automaton_stop_strings_logprobs(pkg, make_model, L, E, tc, mode):
    """A regex automaton, a stop set and top_n = 5 log-probabilities in one guided call."""
    C = pkg.constrain
    tbytes = C.token_bytes()
    au, _ = dc.regex_automata(C, ("date", "number"))
    a, b = pair(pkg, make_model, L, E, tc)
    samplers = dc.mixed_samplers(pkg, 3)
    u = np.random.default_rng(8).random((16, 3))
    check_case(pkg, a, b, [(0, 11), (2, 500), (4, 4118)], [(6, 11, 1.5), None, (8, 0, 3.0)], 16, samplers, mode, u=u,
               tbytes=tbytes, constraints=[(au["number"], 0), None, None], stop_sets=[None, ["e", "\n"], ["the"]],
               logprobs=mode, top_n=5)
    a.close()
    b.close()


@pytest.mark.parametrize("tc", PATHS)
@pytest.mark.parametrize("L,E", dc.SHAPES)
def test_stops_and_budgets_inside_groups(pkg, make_model, L, E, tc):
    """Stop tokens and budgets that end streams inside a group, max_new = 40 (three groups)."""
    a, b = pair(pkg, make_model, L, E, tc)
    streams = [(0, 11), (1, 500), (2, 4118), (3, 7)]
    guidance = [(4, 11, 1.5), (5, 500, 2.0), None, (6, 9, 0.5)]
    samplers = [pkg.Sampler(0.0)] * 4
    st = a.state_download(M)
    free = a.generate_streams(streams, 40, sampling=samplers, guidance=guidance)
    a.state_upload(st, M)
    stop = dc.stops_at(free, {0: 5, 3: 21}, prefer_unique=True)
    check_case(pkg, a, b, streams, guidance, 40, samplers, "stops and budgets", stop=stop, budgets=[40, 9, 27, 40])
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", dc.SHAPES)
def test_more_than_one_pass(pkg, make_model, L, E):
    """S + G = 140 rows: two tensor-core passes per step."""
    a, b = pair(pkg, make_model, L, E, True, max_gpt=160)
    streams = [(s, (s * 37) % dc.V) for s in range(70)]
    guidance = [(70 + s, (s * 11) % dc.V, (0.5, 1.5, 3.0)[s % 3]) for s in range(70)]
    samplers = dc.mixed_samplers(pkg, 70)
    u = np.random.default_rng(5).random((6, 70))
    check_case(pkg, a, b, streams, guidance, 6, samplers, "two passes", u=u, m=160)
    a.close()
    b.close()


def make_adapter(pkg, L, E, rank, seed):
    """A LoRA state dict of `rank` on every projection whose deltas move the projections by a few per cent."""
    rng = np.random.default_rng(seed)
    w = {}
    for l in range(L):
        for name in pkg.engine.ADAPTER_MATRICES:
            n_in, n_out = pkg.engine.adapter_dims(name, E)
            w["blocks.%d.%s.lora_A" % (l, name)] = (rng.standard_normal((rank, n_in)) * n_in ** -0.5).astype(np.float32)
            w["blocks.%d.%s.lora_B" % (l, name)] = (rng.standard_normal((n_out, rank)) * 0.1 / rank ** 0.5).astype(np.float32)
    return w


@pytest.mark.parametrize("L,E", dc.SHAPES)
def test_adapter_contrast(pkg, make_model, L, E):
    """A conditional slot bound to an adapter with an unbound guidance slot, and the reverse: the call takes the tensor
    cores, and each row runs under its own slot's binding."""
    a, b = pair(pkg, make_model, L, E, True)
    w = make_adapter(pkg, L, E, 8, 21)
    for e in (a, b):
        aid = e.add_adapter(w, 16.0)
        e.bind_adapter(1, aid)
        e.bind_adapter(12, aid)
    samplers = dc.mixed_samplers(pkg, 2)
    u = np.random.default_rng(6).random((12, 2))
    check_case(pkg, a, b, [(1, 11), (2, 500)], [(11, 11, 2.0), (12, 500, 1.5)], 12, samplers, "adapter contrast", u=u)
    a.close()
    b.close()


@pytest.mark.parametrize("tc", PATHS)
def test_scale_one_is_the_unguided_call(pkg, make_model, tc):
    """gamma = 1 on every stream: tokens, stream slots, log-probabilities, automaton and stop states bit for bit those of
    generate_streams(stop_strings=..., constraints=..., logprobs=...) on the same slots."""
    C = pkg.constrain
    au, _ = dc.regex_automata(C, ("date", "number"))
    a, _b = pair(pkg, make_model, 3, 768, tc)
    _b.close()
    cid, sid = a.add_constraint(au["number"]), a.add_stop_set(["e", "\n"])
    streams = [(0, 11), (1, 500), (2, 4118)]
    samplers = dc.mixed_samplers(pkg, 3)
    u = np.random.default_rng(2).random((20, 3))
    kw = dict(sampling=samplers, u=u, constraints=[cid, None, None], stop_strings=[None, sid, None], top_n=3)
    for mode in ("raw", "processed"):
        st = a.state_download(M)
        want = a.generate_streams(streams, 20, logprobs=mode, **kw)
        ref = a.state_download(M)
        a.state_upload(st, M)
        got = a.generate_streams(streams, 20, logprobs=mode, guidance=[(5, 9, 1.0), (6, 0, 1.0), (7, 500, 1.0)], **kw)
        sa = a.state_download(M)
        for s in range(3):
            for f in ("tokens", "state", "stop_hit", "stop_tail", "stop_state"):
                assert dc.bits(np.asarray(got[s][f])) == dc.bits(np.asarray(want[s][f])), (mode, s, f)
            for f in dc.FIELDS:
                assert dc.bits(got[s][f]) == dc.bits(want[s][f]), (mode, s, f)
        n = a.n_layers * a.n_embed
        for slot in range(3):
            for k in dc.KEYS5:
                assert np.array_equal(dc.slot_of(sa, slot, n)[k], dc.slot_of(ref, slot, n)[k]), (mode, slot, k)
        a.state_upload(st, M)
    a.close()


def c_call(pkg, eng, slots, first, max_new, guidance):
    """rwkv_b200_generate_streams_guided, arg-max, with a Guidance struct or NULL: (rc, tokens, lengths)."""
    P = ctypes.c_ulonglong
    sl = np.ascontiguousarray(slots, np.uint64)
    ft = np.ascontiguousarray(first, np.uint64)
    out, lens = np.zeros((len(slots), max_new), np.uint64), np.zeros(len(slots), np.uint64)
    pp = pkg.engine._ptr
    rc = eng.lib.rwkv_b200_generate_streams_guided(eng.h, pp(sl, P), pp(ft, P), len(slots), max_new, None, None, 0, None,
                                                   None, 0, None, None, pp(out, P), pp(lens, P), 0, 0, None, None, None,
                                                   None, None, None, None, None, guidance)
    return rc, out, lens


def test_null_guidance_is_generate_streams_stop(pkg, make_model):
    """guidance == NULL through the new entry point: the tokens, states and launch_count delta of generate_streams_stop
    (here through generate_streams_constrained, its stop == NULL form)."""
    a, _b = pair(pkg, make_model, 3, 768, True)
    _b.close()
    st = a.state_download(M)
    n0 = a.launch_count
    want = a.generate_streams([(0, 11), (1, 500)], 20, sampling=[pkg.Sampler(0.0)] * 2, constraints=[None, None])
    d_want = a.launch_count - n0
    ref = a.state_download(M)
    a.state_upload(st, M)
    n0 = a.launch_count
    rc, out, lens = c_call(pkg, a, [0, 1], [11, 500], 20, None)
    assert rc == 0
    assert a.launch_count - n0 == d_want
    for s in range(2):
        assert [int(x) for x in out[s, :int(lens[s])]] == [int(x) for x in want[s]["tokens"]]
    sa = a.state_download(M)
    for k in dc.KEYS5:
        assert np.array_equal(sa[k], ref[k])
    a.close()


def test_refusals_leave_every_slot_untouched(pkg, make_model):
    a, _b = pair(pkg, make_model, 2, 2048, True)
    _b.close()
    before = a.state_download(M)
    E = pkg.engine
    P, F = ctypes.c_ulonglong, ctypes.c_float

    def gd(slots, first=(0, 0), scales=(1.5, 1.5), null_first=False, null_scales=False):
        s = np.ascontiguousarray(slots, np.uint64)
        f = np.ascontiguousarray(first, np.uint64)
        w = np.ascontiguousarray(scales, np.float32)
        g = E.Guidance(E._ptr(s, P), None if null_first else E._ptr(f, P), None if null_scales else E._ptr(w, F))
        g._keep = (s, f, w)
        return g

    NG = E.NO_GUIDANCE
    cases = [
        (E.Guidance(None, None, None), "NULL slots"),
        (gd([NG, 5], null_first=True), "stream 1"),
        (gd([5, NG], null_scales=True), "stream 0"),
        (gd([NG, M]), "stream 1"),
        (gd([5, 5]), "stream 1"),
        (gd([5, 1]), "stream 1"),
        (gd([0, NG]), "stream 0"),
        (gd([5, 6], first=(0, 50277)), "stream 1"),
        (gd([5, 6], scales=(1.5, float("nan"))), "stream 1"),
        (gd([5, 6], scales=(float("inf"), 1.5)), "stream 0"),
        (gd([5, 6], scales=(-0.5, 1.5)), "stream 0"),
        (gd([5, 6], scales=(1.5, 100.5)), "stream 1"),
    ]
    for g, msg in cases:
        rc, _, _ = c_call(pkg, a, [0, 1], [11, 500], 8, ctypes.byref(g))
        err = a.lib.rwkv_b200_last_error().decode()
        assert rc != 0, msg
        assert "generate_streams_guided" in err and msg in err, (msg, err)
    # the refusals of generate_streams_stop come first and name that call's checks
    rc, _, _ = c_call(pkg, a, [0, 0], [11, 500], 8, ctypes.byref(gd([5, 6])))
    assert rc != 0 and b"appears twice" in a.lib.rwkv_b200_last_error()
    after = a.state_download(M)
    for k in dc.KEYS5:
        assert np.array_equal(after[k], before[k])
    with pytest.raises(E.EngineError, match="guidance needs sampling"):
        a.generate_streams([(0, 11)], 4, u=np.zeros((4, 1)), guidance=[(5, 0, 1.5)])
    with pytest.raises(E.EngineError, match="1 guidance entries for 2 streams"):
        a.generate_streams([(0, 11), (1, 3)], 4, guidance=[(5, 0, 1.5)])
    a.close()
