"""Speculative generation with log-probabilities and token automata (rwkv_b200_generate_streams_speculative_constrained)
against generate_streams on the tensor cores.

The oracle is a second engine with prefill_min = 2, started from the same state of every slot, which runs
generate_streams(sampling=..., logprobs=..., constraints=..., stop_strings=...) on the streams' first slots with the same
arguments (a lone stream gets a pad stream on a slot nobody names). Tokens, the bits of the log-probabilities, ranks and
top entries (NaN by bits), the automaton and stop-string results and every first slot's five state arrays must equal the
oracle's (pp: untouched), every slot no stream names must be unchanged, and steps must equal the host restatement of the
draft rule (engine.speculative_steps)."""
import ctypes
import importlib

import numpy as np
import pytest

from decoding import KEYS5, OVERRIDES, SHAPES, V, check_slots, engine_pair, mixed_samplers, slot_of

pytestmark = pytest.mark.gpu

eng_mod = importlib.import_module("rwkv-cpp-accelerated_b200.engine")

MAX_GPT = 160      # S = 9 streams with k = 15 name 144 slots
PAD = MAX_GPT - 1  # the oracle's pad stream; never named by a speculative stream
FIELDS = ("logprobs", "ranks", "top_tokens", "top_logprobs", "state", "stop_hit", "stop_tail", "stop_state")
# "text" never completes (eos None, always extendable); "short" completes after 10 bytes
PATTERNS = {"text": r"[a-z ,.]+", "short": r"[a-z ,.]{4,10}"}
SAMPLERS = [(0.0,), (0.8, 0.9), (1.0, 1.0, 40), (0.7,)]  # mixed_samplers kinds without penalties (refused here)


@pytest.fixture(scope="module")
def automata(pkg):
    C = pkg.constrain
    tb = C.token_bytes()
    return {k: C.token_automaton(C.compile_regex(p), tb, eos=None) for k, p in PATTERNS.items()}, tb


@pytest.fixture(scope="module", params=SHAPES, ids=["3x768", "2x2048"])
def setup(request, pkg, make_model, automata):
    L, E = request.param
    a, b = engine_pair(pkg, make_model(L, E), MAX_GPT, tc=True, seed=5, one_draw=True)
    ids = [{k: e.add_constraint(ta) for k, ta in automata[0].items()} for e in (a, b)]
    before = a.state_download(MAX_GPT)
    yield pkg, a, b, before, ids, automata
    a.close()
    b.close()


def reset(a, b, before):
    a.state_upload(before, MAX_GPT)
    b.state_upload(before, MAX_GPT)


def toks(r):
    return [int(x) for x in r["tokens"]]


def features(eng, ids, cons, sets):
    """generate_* keywords of one engine: cons[s] = None, an automaton name or (name, start state); sets[s] = None, a
    list of stop strings or (set id, start state) of this engine."""
    kw = {}
    if cons is not None:
        kw["constraints"] = [None if c is None else (ids[c], 0) if isinstance(c, str) else (ids[c[0]], c[1]) for c in cons]
    if sets is not None:
        kw["stop_strings"] = [None if x is None else x if isinstance(x, tuple) else eng.add_stop_set(x) for x in sets]
    return kw


def oracle(pkg, b, firsts, max_new, sampling=None, u=None, budgets=None, **kw):
    """generate_streams on engine b, on the tensor cores; the result dicts of the first len(firsts) streams."""
    S = len(firsts)
    streams = list(firsts)
    samp = list(sampling) if sampling is not None else [pkg.Sampler(temperature=0.0)] * S
    if S < 2:
        streams.append((PAD, firsts[0][1]))
        samp.append(pkg.Sampler(temperature=0.0))
        budgets = None if budgets is None else list(budgets) + [max_new]
        u = None if u is None else np.concatenate([u, np.full((max_new, 1), 0.5)], axis=1)
        kw = {k: (v + [None] if k in ("constraints", "stop_strings") else v) for k, v in kw.items()}
    out = b.generate_streams(streams, max_new, budgets=budgets, sampling=samp, u=u, **kw)
    return [r if isinstance(r, dict) else {"tokens": r} for r in out[:S]]


def same(x, y):
    if isinstance(y, np.ndarray):
        return isinstance(x, np.ndarray) and x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()
    return x == y


def run_case(setup, S, k, max_new, seed, ctx="none", ngram=3, sampling=None, budgets=None, stop=(), overrides=None,
             logprobs=None, top_n=0, cons=None, sets=None, firsts=None):
    """One call from the saved state checked against the oracle; returns (results, oracle results, firsts). ctx
    "ceiling" is each stream's greedy run under the call's automata and overrides."""
    pkg, a, b, before, ids, _ = setup
    reset(a, b, before)
    rng = np.random.default_rng(seed)
    slot_lists = [[s * (k + 1) + i for i in range(k + 1)] for s in range(S)]
    firsts = firsts or [(sl[0], int(rng.integers(0, V))) for sl in slot_lists]
    u = rng.random((max_new, S)) if sampling is not None and any(x.temperature > 0 for x in sampling) else None
    if ctx == "ceiling":
        st = b.state_download(MAX_GPT)
        run = oracle(pkg, b, firsts, max_new + 8, overrides=overrides, **features(b, ids[1], cons, None))
        b.state_upload(st, MAX_GPT)
        context = [[f] + toks(r) for (_, f), r in zip(firsts, run)]
    elif ctx == "floor":
        context = [[int(x) for x in rng.integers(0, V, size=200)] for _ in range(S)]
    else:
        context = None
    kw = dict(budgets=budgets, stop=stop, overrides=overrides, sampling=sampling, u=u)
    if logprobs is not None:
        kw.update(logprobs=logprobs, top_n=top_n)
    want = oracle(pkg, b, firsts, max_new, **kw, **features(b, ids[1], cons, sets))
    got = a.generate_speculative([(sl, f) for sl, (_, f) in zip(slot_lists, firsts)], max_new, draft=k, ngram=ngram,
                                 context=context, **kw, **features(a, ids[0], cons, sets))
    for s in range(S):
        assert toks(got[s]) == toks(want[s]), "stream %d: tokens differ" % s
        for f in FIELDS:
            assert (f in got[s]) == (f in want[s]), (s, f)
            if f in want[s]:
                assert same(got[s][f], want[s][f]), "stream %d: %s differs" % (s, f)
        c = context[s] if context is not None else []
        assert got[s]["steps"] == eng_mod.speculative_steps(c, firsts[s][1], toks(got[s]), k, ngram), "stream %d: steps" % s
    first_slots = {sl[0] for sl in slot_lists}
    spares = {x for sl in slot_lists for x in sl[1:]}
    sa = check_slots(a, b, before, MAX_GPT, first_slots, keys=KEYS5, skip=spares)
    n = a.n_layers * a.n_embed
    for first in first_slots:
        assert np.array_equal(slot_of(sa, first, n)["pp"], slot_of(before, first, n)["pp"]), "first slot %d: pp" % first
    return got, want, firsts


def accepted(got):
    return sum(len(g["tokens"]) for g in got) > sum(g["steps"] for g in got)


@pytest.mark.parametrize("ctx,top_n", [("none", 0), ("floor", 5), ("ceiling", 20)])
@pytest.mark.parametrize("mode", ["raw", "processed"])
def test_logprobs_mixed_samplers(setup, mode, ctx, top_n):
    pkg = setup[0]
    got, _, _ = run_case(setup, 4, 3, 40, 3, ctx=ctx, sampling=mixed_samplers(pkg, 4, SAMPLERS),
                         logprobs=mode, top_n=top_n)
    if ctx == "ceiling":  # the greedy stream copies its own greedy run
        assert got[0]["steps"] < len(got[0]["tokens"])


def test_raw_logprobs_with_overrides(setup):
    """The overrides edit the rows in place, so raw mode scores the copy taken before them."""
    got, _, _ = run_case(setup, 3, 4, 40, 4, ctx="ceiling", overrides=OVERRIDES, logprobs="raw", top_n=3)
    assert accepted(got)


def test_constraint_never_completes_accepts_masked_drafts(setup):
    got, _, _ = run_case(setup, 3, 4, 40, 5, ctx="ceiling", cons=["text"] * 3)
    assert all(g["steps"] < len(g["tokens"]) for g in got), "a stream accepted no draft"
    assert all(len(g["tokens"]) == 40 for g in got)


def test_constraint_completes_inside_an_accepted_run(setup):
    got, _, _ = run_case(setup, 4, 4, 40, 6, ctx="ceiling", cons=["short"] * 4, logprobs="processed", top_n=2)
    assert any(len(g["tokens"]) < 40 and g["steps"] < len(g["tokens"]) for g in got), "no stream completed in a run"


def test_constraint_floor_context_rows_die(setup):
    pkg = setup[0]
    run_case(setup, 4, 7, 32, 7, ctx="floor", cons=["text", "short", "text", "short"],
             sampling=mixed_samplers(pkg, 4, SAMPLERS))


def test_constrained_and_unconstrained_mixed(setup):
    pkg = setup[0]
    got, _, _ = run_case(setup, 6, 3, 36, 8, ctx="ceiling", cons=["text", None, "short", None, "text", None],
                         sampling=[pkg.Sampler(temperature=0.0)] * 6, logprobs="processed", top_n=5)
    assert accepted(got)


def test_second_call_continues_from_states(setup):
    pkg, a, b, before, ids, _ = setup
    S, k, n1, n2 = 4, 3, 12, 20
    sets = [[b"e"], None, [b"th"], [b"\x01never"]]
    got, want, firsts = run_case(setup, S, k, n1, 9, ctx="ceiling", cons=["text", "text", None, "short"], sets=sets,
                                 logprobs="raw", top_n=1)
    cont = [s for s in range(S) if len(got[s]["tokens"]) == n1 and got[s].get("stop_hit") is None]
    assert cont, "every stream ended in the first call"
    slot_lists = [[firsts[s][0]] + [firsts[s][0] + 1 + i for i in range(k)] for s in cont]
    cons = [("text", int(got[s]["state"])) if s in (0, 1) else None if s == 2 else ("short", int(got[s]["state"]))
            for s in cont]
    # the stop sets continue too: the same strings added again, from each stream's match state
    sa = [None if sets[s] is None else (a.add_stop_set(sets[s]), got[s]["stop_state"]) for s in cont]
    sb = [None if sets[s] is None else (b.add_stop_set(sets[s]), want[s]["stop_state"]) for s in cont]
    first2 = [(firsts[s][0], int(got[s]["tokens"][-1])) for s in cont]
    want2 = oracle(pkg, b, first2, n2, logprobs="raw", top_n=1, **features(b, ids[1], cons, sb))
    got2 = a.generate_speculative([(sl, f) for sl, (_, f) in zip(slot_lists, first2)], n2, draft=k, logprobs="raw",
                                  top_n=1, **features(a, ids[0], cons, sa))
    for i in range(len(cont)):
        assert toks(got2[i]) == toks(want2[i]), i
        for f in FIELDS:
            if f in want2[i]:
                assert same(got2[i][f], want2[i][f]), (i, f)
    spares = {x for s in range(S) for x in range(firsts[s][0] + 1, firsts[s][0] + k + 1)}
    check_slots(a, b, before, MAX_GPT, {f[0] for f in firsts}, keys=KEYS5, skip=spares)


@pytest.mark.parametrize("k", [1, 15])
def test_extreme_drafts(setup, k):
    S = 9 if k == 15 else 5  # S = 9 with k = 15: two passes of 8 and 1 streams
    got, _, _ = run_case(setup, S, k, 40, 10 + k, ctx="ceiling", ngram=2, cons=["text", None] * (S // 2) + ["short"],
                         logprobs="processed", top_n=3)
    assert accepted(got)


def test_33_streams_two_passes(setup):
    pkg = setup[0]
    run_case(setup, 33, 3, 24, 11, ctx="floor", sampling=mixed_samplers(pkg, 33, SAMPLERS),
             cons=["text", None, "short"] * 11, logprobs="raw", top_n=2)


def test_everything_at_once(setup):
    pkg, a, b, before, ids, (_, tb) = setup
    S, k, max_new = 6, 4, 40
    cons = ["text", "short", None, "text", None, "text"]
    # stop strings and stop tokens cut from the oracle's own run, so that they fire
    reset(a, b, before)
    rng = np.random.default_rng(12)
    firsts = [(s * (k + 1), int(rng.integers(0, V))) for s in range(S)]
    run = oracle(pkg, b, firsts, max_new, overrides=OVERRIDES, **features(b, ids[1], cons, None))
    sets = [None] * S
    for s in (0, 3, 4):
        chunks = [tb[t] for t in toks(run[s])[len(run[s]["tokens"]) // 2:] if len(tb[t]) >= 2]
        sets[s] = [chunks[0][:2]] if chunks else [b"\x01never"]
    stop = tuple(toks(run[5])[len(run[5]["tokens"]) // 2:][:1])
    got, _, _ = run_case(setup, S, k, max_new, 12, ctx="ceiling", sampling=[pkg.Sampler(temperature=0.0)] * S,
                         budgets=[max_new, 30, 25, max_new, 7, max_new], stop=stop, overrides=OVERRIDES,
                         logprobs="processed", top_n=4, cons=cons, sets=sets, firsts=firsts)
    assert any(g.get("stop_hit") is not None for g in got), "no stop string fired"
    assert accepted(got)


def spec_args(a, streams, max_new, k):
    S, lead, tail, out, lens = eng_mod._gen_args(streams, max_new, None, (), None, None,
                                                  slots=[int(x) for sl, _ in streams for x in sl])
    steps = np.zeros(S, np.uint64)
    P = ctypes.c_ulonglong
    return (a.h, *lead, None, *tail, k, 3, None, None, steps.ctypes.data_as(ctypes.POINTER(P))), out


def test_null_features_launch_like_speculative_stop(setup):
    pkg, a, b, before, ids, _ = setup
    k = 3
    streams = [([s * (k + 1) + i for i in range(k + 1)], 100 + s) for s in range(5)]
    counts, outs = [], []
    for fn, extra in (("rwkv_b200_generate_streams_speculative_stop", (None,)),
                      ("rwkv_b200_generate_streams_speculative_constrained", (0, 0) + (None,) * 8)):
        a.state_upload(before, MAX_GPT)
        args, out = spec_args(a, streams, 24, k)
        n0 = a.launch_count
        assert getattr(a.lib, fn)(*args, *extra) == 0, a._err()
        counts.append(a.launch_count - n0)
        outs.append(out.copy())
    assert counts[0] == counts[1] > 0
    assert np.array_equal(outs[0], outs[1])


def test_refusals(setup):
    pkg, a, b, before, ids, (au, _) = setup
    E = pkg.EngineError
    short = au["short"]
    counts = [len(short.edges(q)[0]) for q in range(short.n_states)]
    complete = [q for q in range(short.n_states) if counts[q] == 0]
    narrow = min((q for q in range(short.n_states) if counts[q]), key=lambda q: counts[q])
    close_all = {int(t): -np.inf for t in short.edges(narrow)[0]}
    two = [([0, 1, 2, 3], 5), ([4, 5, 6, 7], 6)]
    cid = ids[0]["short"]
    bad = [
        (dict(logprobs="raw", top_n=21), "top_n 21"),
        (dict(constraints=[cid, 10 ** 6]), "unknown or removed"),
        (dict(constraints=[(cid, short.n_states + 3), None]), "out of range"),
        (dict(constraints=[(cid, complete[0]), None]), "has no edges"),
        (dict(constraints=[cid, None], overrides=close_all), "every edge token"),
        (dict(constraints=[cid, None], sampling=pkg.Sampler(temperature=0.0, frequency_penalty=0.5)), "penalties"),
        (dict(logprobs="processed", sampling=pkg.Sampler(temperature=0.0, presence_penalty=0.5)), "penalties"),
    ]
    reset(a, b, before)
    for kw, msg in bad:
        with pytest.raises(E, match=msg):
            a.generate_speculative(two, 8, 3, **kw)
    # a mode the Python layer does not produce, and top_n without its arrays, straight through the C entry point
    args, _ = spec_args(a, two, 8, 3)
    lp = np.zeros(16)
    pd = lp.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    fn = a.lib.rwkv_b200_generate_streams_speculative_constrained
    assert fn(*args, 7, 0, pd, None, None, None, None, None, None, None) != 0
    assert "logprob_mode 7" in a._err()
    assert fn(*args, 0, 3, pd, None, None, None, None, None, None, None) != 0
    assert "top_tokens_out" in a._err()
    assert all(np.array_equal(x, y) for x, y in ((a.state_download(MAX_GPT)[key], before[key]) for key in KEYS5)), \
        "a refused call changed a slot"
