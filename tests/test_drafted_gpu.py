"""Speculative generation with a draft model (rwkv_b200_generate_streams_drafted) against generate_streams on the tensor
cores, and its steps and draft state against a host restatement on the draft model.

Target engine a runs the call; its oracle b (prefill_min = 2, same state of every slot) runs generate_streams with the
same features on the first slots. The draft engine da runs the call's drafts; its oracle db (prefill_min = 2, same
state) restates them: per step forward_streams of the input and then of each draft on a copy of D0, the host pick
chain (overrides, the row's automaton mask, sample_streams on the host rows with the uniform of target row i - 1), the
accepted prefix against the emitted tokens, and forward_streams of the absorbed tokens into D0. Tokens, feature results
and first slots must be bit-equal to b's, steps_out equal to the restatement, D0 bit-equal to db's D0, and every other
slot of both models but the scratch slots unchanged. A perfect drafter is a second handle on the target's own file."""
import numpy as np
import pytest

from decoding import KEYS4, KEYS5, V, allowed, bits, check_slots, engine_pair, regex_automata, slot_of

pytestmark = pytest.mark.gpu

MAX_GPT = 160      # S = 9 streams with k = 15 name 144 target slots
PAD = MAX_GPT - 1  # the oracles' pad stream; never named by a stream
# (target L, E, seed), (draft L, E, seed)
PAIRS = [((3, 768, 20240924), (2, 768, 7)), ((2, 2048, 20240924), (3, 768, 20240924))]


@pytest.fixture(scope="module", params=PAIRS, ids=["3x768+2x768", "2x2048+3x768"])
def setup(request, pkg, make_model):
    (tl, te, ts), (dl, de, ds) = request.param
    tpath, dpath = make_model(tl, te, ts), make_model(dl, de, ds)
    a, b = engine_pair(pkg, tpath, MAX_GPT, tc=True, seed=5, one_draw=True)
    da, db = engine_pair(pkg, dpath, MAX_GPT, tc=True, seed=11, one_draw=True)
    env = dict(pkg=pkg, a=a, b=b, da=da, db=db, before=a.state_download(MAX_GPT), dbefore=da.state_download(MAX_GPT),
               tpath=tpath, te=te, tl=tl)
    yield env
    for e in (a, b, da, db):
        e.close()


@pytest.fixture(scope="module")
def perfect(setup):
    """A second handle on the target's file (pa) and its oracle (pb), from the target's state of every slot."""
    pkg = setup["pkg"]
    pa = pkg.Engine(setup["tpath"], max_gpt=MAX_GPT)
    pb = pkg.Engine(setup["tpath"], max_gpt=MAX_GPT)
    pb.set_option("prefill_min", 2)
    yield pa, pb
    pa.close()
    pb.close()


def slots_of(S, k):
    """Stream s: target slots s (k + 1) + i, draft slots (D0, D1) = (s (k + 1), s (k + 1) + 1)."""
    sl = [[s * (k + 1) + i for i in range(k + 1)] for s in range(S)]
    return sl, [(x[0], x[0] + 1) for x in sl]


def oracle(pkg, b, firsts, max_new, sampling=None, u=None, budgets=None, stop=(), overrides=None, **features):
    """generate_streams on engine b (a pad stream joins a lone stream): one dict per stream with "tokens"."""
    S = len(firsts)
    streams = list(firsts)
    samp = list(sampling) if sampling is not None else [pkg.Sampler(temperature=0.0)] * S
    if S < 2:
        streams.append((PAD, firsts[0][1]))
        samp.append(pkg.Sampler(temperature=0.0))
        budgets = None if budgets is None else list(budgets) + [max_new]
        u = None if u is None else np.concatenate([u, np.full((max_new, 1), 0.5)], axis=1)
        for key in ("constraints", "stop_strings"):
            if features.get(key) is not None:
                features[key] = list(features[key]) + [None]
    out = b.generate_streams(streams, max_new, budgets=budgets, stop=stop, overrides=overrides, sampling=samp, u=u,
                             **features)
    return [dict(x) if isinstance(x, dict) else {"tokens": x} for x in out[:S]]


def restate(pkg, db, pairs, firsts, toks, k, max_new, sampling=None, u=None, budgets=None, overrides=None, cons=None):
    """The drafted call's steps per stream, by the rule, on the draft oracle db; db's D0 ends with the absorbed tokens."""
    S = len(firsts)
    budgets = list(budgets) if budgets is not None else [max_new] * S
    cons = cons if cons is not None else [None] * S
    pos, steps, x = [0] * S, [0] * S, [int(f) for _, f in firsts]
    state = [c[1] if c else None for c in cons]
    while True:
        live = [s for s in range(S) if pos[s] < len(toks[s])]
        if not live:
            return steps
        for s in live:
            db.slot_copy(pairs[s][0], pairs[s][1])
        d = {s: [] for s in live}
        q = {s: state[s] for s in live}
        cur = {s: x[s] for s in live}
        for i in range(1, k + 1):
            call = [(pairs[s][1], [cur[s]]) for s in live]
            if len(call) == 1:
                call.append((PAD, [cur[live[0]]]))
            logits, _ = db.forward_streams(call)
            ps, us = [], []
            for j, s in enumerate(live):
                row = logits[j]
                for tok, val in (overrides or {}).items():
                    row[tok] = val
                if q[s] is not None:
                    row[~allowed(cons[s][0], q[s])] = -np.inf
                sp = sampling[s] if sampling is not None else pkg.Sampler(temperature=0.0)
                ps.append(pkg.Sampler(sp.temperature, sp.top_p, sp.top_k))
                p = pos[s] + i - 1
                us.append(float(u[p][s]) if u is not None and p < budgets[s] else 0.0)
            if len(call) > len(live):
                ps.append(pkg.Sampler(temperature=0.0))
                us.append(0.0)
            picks, _ = db.sample_streams(ps, us, logits=logits)
            for j, s in enumerate(live):
                cur[s] = int(picks[j])
                d[s].append(cur[s])
                if q[s] is not None:
                    q2 = cons[s][0].walk([cur[s]], q[s])
                    q[s] = None if q2 is None or cons[s][0].complete(q2) else q2
        absorb = []
        for s in live:
            t, c = toks[s], 1
            while c <= k and pos[s] + c < len(t) and d[s][c - 1] == t[pos[s] + c - 1]:
                c += 1
            absorb.append((pairs[s][0], [x[s]] + t[pos[s]:pos[s] + c - 1]))
            if cons[s]:
                state[s] = cons[s][0].walk(t[pos[s]:pos[s] + c], state[s])
            x[s] = t[pos[s] + c - 1]
            pos[s] += c
            steps[s] += 1
        if sum(len(t) for _, t in absorb) < 2:
            absorb.append((PAD, [x[live[0]]]))
        db.forward_streams(absorb, want_logits=False)


def reset(env, draft_engines=None):
    for e in (env["a"], env["b"]):
        e.state_upload(env["before"], MAX_GPT)
    for e in (env["da"], env["db"]):
        e.state_upload(env["dbefore"], MAX_GPT)
    for e in draft_engines or ():
        e.state_upload(env["before"], MAX_GPT)


def check_target(env, slot_lists):
    a, b, before = env["a"], env["b"], env["before"]
    first = {sl[0] for sl in slot_lists}
    spares = {s for sl in slot_lists for s in sl[1:]}
    sa = check_slots(a, b, before, MAX_GPT, first, keys=KEYS5, skip=spares, what="target")
    n = a.n_layers * a.n_embed
    for f in first:
        assert np.array_equal(slot_of(sa, f, n)["pp"], slot_of(before, f, n)["pp"]), "first slot %d: pp" % f
    return sa


def check_draft(dut, ref, dbefore, pairs, what="draft"):
    """D0 of every stream equals the oracle's in xy, aa, bb, dd (pp untouched); every unnamed draft slot unchanged."""
    check_slots(dut, ref, dbefore, MAX_GPT, {p[0] for p in pairs}, skip={p[1] for p in pairs}, what=what)
    n = dut.n_layers * dut.n_embed
    sa = dut.state_download(MAX_GPT)
    for d0, _ in pairs:
        assert np.array_equal(slot_of(sa, d0, n)["pp"], slot_of(dbefore, d0, n)["pp"]), "D0 %d: pp" % d0


def run_case(env, S, k, max_new, seed, sampling=None, budgets=None, stop=(), overrides=None, stop_from_run=False,
             cons=None, **features):
    """One drafted call on (a, da), checked against b, db and the restatement; returns the results."""
    pkg, a, b, da, db = env["pkg"], env["a"], env["b"], env["da"], env["db"]
    reset(env)
    rng = np.random.default_rng(seed)
    slot_lists, pairs = slots_of(S, k)
    firsts = [(sl[0], int(rng.integers(0, V))) for sl in slot_lists]
    u = rng.random((max_new, S)) if sampling is not None and any(x.temperature > 0 for x in sampling) else None
    if cons is not None:
        features["constraints"] = [None if c is None else (c[2], c[1]) for c in cons]
    kw = dict(sampling=sampling, u=u, budgets=budgets, overrides=overrides)
    if stop_from_run:
        want = oracle(pkg, b, firsts, max_new, stop=(), **kw, **features)
        b.state_upload(env["before"], MAX_GPT)
        stop = tuple({int(w["tokens"][len(w["tokens"]) // 2]) for w in want if len(w["tokens"]) > 4})
    want = oracle(pkg, b, firsts, max_new, stop=stop, **kw, **features)
    got = a.generate_speculative([(sl, f) for sl, (_, f) in zip(slot_lists, firsts)], max_new, draft=k, stop=stop,
                                 drafter=(da, pairs), **kw, **features)
    toks = []
    for s in range(S):
        assert bits(got[s]["tokens"]) == bits(want[s]["tokens"]), "stream %d: tokens" % s
        for f in set(want[s]) - {"tokens"}:
            assert bits(np.asarray(got[s][f])) == bits(np.asarray(want[s][f])), "stream %d: %s" % (s, f)
        toks.append([int(x) for x in got[s]["tokens"]])
    check_target(env, slot_lists)
    steps = restate(pkg, db, pairs, firsts, toks, k, max_new, sampling, u, budgets, overrides,
                    None if cons is None else [None if c is None else (c[0], c[1]) for c in cons])
    assert [g["steps"] for g in got] == steps, "steps_out differs from the restatement"
    check_draft(da, db, env["dbefore"], pairs)
    return got


def mixed(pkg, S):
    sp = [pkg.Sampler(temperature=0.0), pkg.Sampler(temperature=0.8, top_p=0.9), pkg.Sampler(temperature=1.0, top_k=40),
          pkg.Sampler(temperature=0.7)]
    return [sp[i % len(sp)] for i in range(S)]


def test_one_stream_with_pad(setup):
    run_case(setup, 1, 3, 24, 1)


def test_three_streams_mixed_samplers(setup):
    run_case(setup, 3, 3, 24, 2, sampling=mixed(setup["pkg"], 3))


def test_eight_streams_k7(setup):
    run_case(setup, 8, 7, 20, 3, sampling=mixed(setup["pkg"], 8))


def test_two_first_passes(setup):
    # k = 3: 25 streams per first pass, so 30 streams take two
    run_case(setup, 30, 3, 12, 4, sampling=mixed(setup["pkg"], 30))


@pytest.mark.parametrize("k", [1, 15])
def test_extreme_drafts(setup, k):
    run_case(setup, 9 if k == 15 else 5, k, 16, 5 + k)


def test_stops_budgets_overrides(setup):
    pkg = setup["pkg"]
    run_case(setup, 6, 3, 24, 8, sampling=[pkg.Sampler(temperature=0.0)] * 6, stop_from_run=True)
    run_case(setup, 6, 3, 24, 9, budgets=[1, 2, 3, 4, 5, 24], overrides={0: -99.0, 11: 5.0, 187: -np.inf},
             sampling=mixed(pkg, 6))


def perfect_call(env, pa, S, k, max_new, seed, sampling=None, budgets=None, stop=(), firsts=None):
    """A drafted call with the perfect drafter pa (its state left as it is); returns (results, firsts)."""
    pkg, a, b = env["pkg"], env["a"], env["b"]
    rng = np.random.default_rng(seed)
    slot_lists, pairs = slots_of(S, k)
    firsts = firsts or [(sl[0], int(rng.integers(0, V))) for sl in slot_lists]
    u = rng.random((max_new, S)) if sampling is not None else None
    want = oracle(pkg, b, firsts, max_new, sampling=sampling, u=u, budgets=budgets, stop=stop)
    got = a.generate_speculative([(sl, f) for sl, (_, f) in zip(slot_lists, firsts)], max_new, draft=k, stop=stop,
                                 drafter=(pa, pairs), sampling=sampling, u=u, budgets=budgets)
    for s in range(S):
        assert bits(got[s]["tokens"]) == bits(want[s]["tokens"]), "stream %d: tokens" % s
    check_target(env, slot_lists)
    return got, u, firsts


def minimal(got, k):
    return [-(-len(g["tokens"]) // (k + 1)) for g in got]


@pytest.mark.parametrize("sampled", [False, True], ids=["argmax", "sampled"])
def test_perfect_drafter_accepts_everything(setup, perfect, sampled):
    pkg, a = setup["pkg"], setup["a"]
    pa, _ = perfect
    S, k = 6, 4
    reset(setup, [pa])
    sampling = mixed(pkg, S) if sampled else None
    got, _, firsts = perfect_call(setup, pa, S, k, 30, 21, sampling=sampling, budgets=[30, 7, 5, 30, 1, 12])
    assert [g["steps"] for g in got] == minimal(got, k)
    # D0 holds what the first slot holds: the same model over the same tokens
    n = a.n_layers * a.n_embed
    sa, sp = a.state_download(MAX_GPT), pa.state_download(MAX_GPT)
    slot_lists, pairs = slots_of(S, k)
    for sl, (d0, _) in zip(slot_lists, pairs):
        for key in KEYS4:
            assert np.array_equal(slot_of(sp, d0, n)[key], slot_of(sa, sl[0], n)[key]), "D0 %d: %s" % (d0, key)
    # the next turn continues from (first slot, D0): every draft is accepted again
    nxt = [(sl[0], int(g["tokens"][-1])) for sl, g in zip(slot_lists, got)]
    setup["b"].state_upload(sa, MAX_GPT)
    got2, _, _ = perfect_call(dict(setup, before=sa), pa, S, k, 20, 22, sampling=sampling, firsts=nxt)
    assert [g["steps"] for g in got2] == minimal(got2, k)


def test_partial_acceptance_with_adapter(setup, perfect):
    from importlib import import_module
    adims = import_module("rwkv-cpp-accelerated_b200").engine.adapter_dims
    pkg, L, E = setup["pkg"], setup["tl"], setup["te"]
    pa, pb = perfect
    S, k, max_new = 4, 3, 32
    rng = np.random.default_rng(3)
    w = {}
    for l in range(L):
        for name in ("att.key", "ffn.value"):
            n_in, n_out = adims(name, E)
            w["blocks.%d.%s.lora_A" % (l, name)] = (rng.standard_normal((8, n_in)) * n_in ** -0.5).astype(np.float32)
            w["blocks.%d.%s.lora_B" % (l, name)] = (rng.standard_normal((n_out, 8)) * 0.3).astype(np.float32)
    _, pairs = slots_of(S, k)
    ids = [e.add_adapter(w, 8.0) for e in (pa, pb)]
    try:
        for e, aid in zip((pa, pb), ids):
            for p in pairs:
                e.bind_adapter(p[0], aid)
                e.bind_adapter(p[1], aid)
        reset(setup, [pa, pb])
        got, u, firsts = perfect_call(setup, pa, S, k, max_new, 31)
        toks = [[int(x) for x in g["tokens"]] for g in got]
        steps = [g["steps"] for g in got]
        assert sum(minimal(got, k)) < sum(steps) < sum(len(t) for t in toks), steps
        assert steps == restate(pkg, pb, pairs, firsts, toks, k, max_new)
        check_draft(pa, pb, setup["before"], pairs, what="adapted draft")
    finally:
        for e, aid in zip((pa, pb), ids):
            for p in pairs:
                e.bind_adapter(p[0], None)
                e.bind_adapter(p[1], None)
            e.remove_adapter(aid)


@pytest.fixture(scope="module")
def automata(setup):
    from importlib import import_module
    C = import_module("rwkv-cpp-accelerated_b200.constrain")
    au, states = regex_automata(C, ("date", "labels", "number"))
    ids = {k: (setup["a"].add_constraint(t), setup["b"].add_constraint(t)) for k, t in au.items()}
    return au, states, ids


def test_logprobs(setup):
    pkg = setup["pkg"]
    run_case(setup, 3, 3, 16, 41, sampling=mixed(pkg, 3), logprobs="processed", top_n=3)
    run_case(setup, 4, 2, 16, 42, sampling=mixed(pkg, 4), logprobs="raw", top_n=2, overrides={11: 3.0})


def test_automata(setup, automata):
    pkg = setup["pkg"]
    au, states, ids = automata
    # (automaton, start state, id on a); the oracle's ids equal a's (both engines add them in the same order)
    cons = [(au["date"], states["date+"], ids["date"][0]), None, (au["labels"], 0, ids["labels"][0]),
            (au["number"], 0, ids["number"][0])]
    assert all(x == y for x, y in ids.values())
    run_case(setup, 4, 3, 20, 51, sampling=mixed(pkg, 4), cons=cons, logprobs="raw", top_n=2)


def test_stop_strings(setup):
    pkg, a, b = setup["pkg"], setup["a"], setup["b"]
    from importlib import import_module
    tb = import_module("rwkv-cpp-accelerated_b200.constrain").token_bytes()
    reset(setup)
    S, k, max_new = 3, 3, 24
    rng = np.random.default_rng(61)
    slot_lists, _ = slots_of(S, k)
    firsts = [(sl[0], int(rng.integers(0, V))) for sl in slot_lists]
    free = oracle(pkg, b, firsts, max_new)
    strings = [tb[int(f["tokens"][len(f["tokens"]) // 2])] or b"x" for f in free]
    sid_a, sid_b = a.add_stop_set(strings), b.add_stop_set(strings)
    assert sid_a == sid_b
    try:
        got = run_case(setup, S, k, max_new, 61, stop_strings=sid_a)
        assert any(g["stop_hit"] is not None for g in got), "no stop string fired"
    finally:
        a.remove_stop_set(sid_a)
        b.remove_stop_set(sid_b)


def test_refusals(setup, pkg, make_model):
    a, da = setup["a"], setup["da"]
    E = pkg.EngineError
    streams = [([0, 1, 2, 3], 5), ([4, 5, 6, 7], 6)]
    good = [(0, 1), (4, 5)]
    alias = object.__new__(pkg.Engine)
    alias.lib, alias.h = a.lib, a.h
    small = pkg.Engine(make_model(2, 768, 7), max_gpt=3)
    aid = da.add_adapter({"blocks.0.att.key.lora_A": np.zeros((4, setup["da"].n_embed), np.float32),
                          "blocks.0.att.key.lora_B": np.zeros((setup["da"].n_embed, 4), np.float32)}, 4.0)
    reset(setup)
    try:
        bad = [
            (dict(drafter=(alias, good)), "the draft model is the target model"),
            (dict(drafter=(small, good)), "draft model's max_gpt"),
            (dict(drafter=(da, [(0, 1), (4, MAX_GPT)])), "draft model: slot %d >= max_gpt" % MAX_GPT),
            (dict(drafter=(da, [(0, 1), (4, 0)])), "draft model: slot 0 appears twice"),
            (dict(drafter=(da, [(0, 1), (4, 7)]), sampling=pkg.Sampler(temperature=0.0, presence_penalty=0.5)),
             "penalties"),
            (dict(drafter=(da, [(0, 1), (4, 7)]), budgets=[0, 3]), "budget 0"),
        ]
        for kw, msg in bad:
            with pytest.raises(E, match=msg):
                a.generate_speculative(streams, 8, 3, **kw)
        da.bind_adapter(1, aid)
        with pytest.raises(E, match="not bound to the same adapter"):
            a.generate_speculative(streams, 8, 3, drafter=(da, good))
        da.bind_adapter(1, None)
        da.set_option("prefill", 0)
        with pytest.raises(E, match="prefill"):
            a.generate_speculative(streams, 8, 3, drafter=(da, good))
    finally:
        alias.h = None  # the handle is a's: the alias must not free it
        da.set_option("prefill", 1)
        da.bind_adapter(1, None)
        da.remove_adapter(aid)
        small.close()
    for eng, ref in ((a, setup["before"]), (da, setup["dbefore"])):
        st = eng.state_download(MAX_GPT)
        assert all(np.array_equal(st[k], ref[k]) for k in KEYS5), "a refused call changed a slot"
