"""Speculative generation (rwkv_b200_generate_streams_speculative) against generate_streams_ex on the tensor cores.

The oracle is a second engine with prefill_min = 2, started from the same state of every slot, which runs
generate_streams(sampling=...) on the streams' first slots with the same first tokens, budgets, stops, overrides,
samplers and uniforms (a lone stream gets a pad stream on a slot nobody names, as the batcher's oracle does). Tokens,
lengths and every first slot's five state arrays must be bit-equal to the oracle's (pp: untouched), every slot no stream
names must be unchanged, and steps_out must equal the host restatement of the draft rule (engine.speculative_steps)."""
import importlib

import numpy as np
import pytest

from decoding import KEYS5, SHAPES, V, check_slots, engine_pair, slot_of

pytestmark = pytest.mark.gpu

eng_mod = importlib.import_module("rwkv-cpp-accelerated_b200.engine")

MAX_GPT = 160      # S = 9 streams with k = 15 name 144 slots
PAD = MAX_GPT - 1  # the oracle's pad stream; never named by a speculative stream


@pytest.fixture(scope="module", params=SHAPES, ids=["3x768", "2x2048"])
def setup(request, pkg, make_model):
    L, E = request.param
    a, b = engine_pair(pkg, make_model(L, E), MAX_GPT, tc=True, seed=5, one_draw=True)
    before = a.state_download(MAX_GPT)
    yield pkg, a, b, before
    a.close()
    b.close()


def reset(a, b, before):
    a.state_upload(before, MAX_GPT)
    b.state_upload(before, MAX_GPT)


def oracle(pkg, b, firsts, max_new, budgets=None, stop=(), overrides=None, sampling=None, u=None):
    """generate_streams_ex on engine b, on the tensor cores; returns the tokens of the first len(firsts) streams."""
    S = len(firsts)
    streams = list(firsts)
    samp = list(sampling) if sampling is not None else [pkg.Sampler(temperature=0.0)] * S
    if S < 2:
        streams.append((PAD, firsts[0][1]))
        samp.append(pkg.Sampler(temperature=0.0))
        budgets = None if budgets is None else list(budgets) + [max_new]
        u = None if u is None else np.concatenate([u, np.full((max_new, 1), 0.5)], axis=1)
    out = b.generate_streams(streams, max_new, budgets=budgets, stop=stop, overrides=overrides, sampling=samp, u=u)
    return [[int(x) for x in t] for t in out[:S]]


def greedy_context(pkg, b, before, firsts, n):
    """The ceiling context of each stream: its first token and its own greedy continuation of n tokens."""
    toks = oracle(pkg, b, firsts, n)
    b.state_upload(before, MAX_GPT)
    return [[f] + t for (_, f), t in zip(firsts, toks)]


def step_counts(context, first, tokens, k, ngram):
    """Tokens emitted by each step, by the rule (engine.speculative_steps counts these steps)."""
    h, t, pos, counts = list(context) + [first], list(tokens), 0, []
    while pos < len(t):
        d = eng_mod.lookup_drafts(h, k, ngram)
        c = 1
        while c <= k and pos + c < len(t) and d[c - 1] == t[pos + c - 1]:
            c += 1
        h += t[pos:pos + c]
        pos += c
        counts.append(c)
    return counts


def run_case(setup, S, k, max_new, seed, ctx_kind="none", ngram=3, sampling=None, budgets=None, stop=(), overrides=None,
             stop_from_run=False):
    """One call checked against the oracle; returns (results, home per stream)."""
    pkg, a, b, before = setup
    reset(a, b, before)
    rng = np.random.default_rng(seed)
    slot_lists = [[s * (k + 1) + i for i in range(k + 1)] for s in range(S)]
    firsts = [(sl[0], int(rng.integers(0, V))) for sl in slot_lists]
    u = rng.random((max_new, S)) if sampling is not None and any(x.temperature > 0 for x in sampling) else None
    if ctx_kind == "ceiling":
        context = greedy_context(pkg, b, before, firsts, max_new + 8)
    elif ctx_kind == "floor":
        context = [[int(x) for x in rng.integers(0, V, size=200)] for _ in range(S)]
    else:
        context = None
    if stop_from_run:  # a token from the middle of an unstopped run, so that it falls inside an accepted step
        want = oracle(pkg, b, firsts, max_new, budgets, (), overrides, sampling, u)
        b.state_upload(before, MAX_GPT)
        stop = tuple({w[len(w) // 2] for w in want if len(w) > 4})
    want = oracle(pkg, b, firsts, max_new, budgets, stop, overrides, sampling, u)
    got = a.generate_speculative([(sl, f) for sl, (_, f) in zip(slot_lists, firsts)], max_new, draft=k, ngram=ngram,
                                 context=context, budgets=budgets, stop=stop, overrides=overrides, sampling=sampling, u=u)
    homes = []
    for s in range(S):
        toks = [int(x) for x in got[s]["tokens"]]
        assert toks == want[s], "stream %d: tokens differ" % s
        ctx = context[s] if context is not None else []
        counts = step_counts(ctx, firsts[s][1], toks, k, ngram)
        assert got[s]["steps"] == len(counts) == eng_mod.speculative_steps(ctx, firsts[s][1], toks, k, ngram), \
            "stream %d: steps" % s
        homes.append(sum(c - 1 for c in counts) % (k + 1))
    first_slots = {sl[0] for sl in slot_lists}
    spares = {s for sl in slot_lists for s in sl[1:]}
    sa = check_slots(a, b, before, MAX_GPT, first_slots, keys=KEYS5, skip=spares)
    n = a.n_layers * a.n_embed
    for first in first_slots:
        assert np.array_equal(slot_of(sa, first, n)["pp"], slot_of(before, first, n)["pp"]), "first slot %d: pp" % first
    return got, homes


def mixed(pkg, S):
    sp = [pkg.Sampler(temperature=0.0), pkg.Sampler(temperature=0.8, top_p=0.9), pkg.Sampler(temperature=1.0, top_k=40),
          pkg.Sampler(temperature=0.7)]
    return [sp[i % len(sp)] for i in range(S)]


def test_one_stream_with_pad(setup):
    run_case(setup, 1, 3, 40, 1)


def test_one_stream_ceiling_accepts_drafts(setup):
    got, homes = run_case(setup, 1, 3, 48, 2, ctx_kind="ceiling")
    assert got[0]["steps"] < len(got[0]["tokens"])


@pytest.mark.parametrize("ctx_kind", ["none", "floor", "ceiling"])
def test_three_streams_mixed_samplers(setup, ctx_kind):
    pkg = setup[0]
    got, homes = run_case(setup, 3, 3, 40, 3, ctx_kind=ctx_kind, sampling=mixed(pkg, 3))
    if ctx_kind == "ceiling":  # the greedy stream copies its own greedy run
        assert got[0]["steps"] < len(got[0]["tokens"])


def test_eight_streams_k7_ceiling_copy_back(setup):
    # 60 tokens: a stream that accepts every draft ends after 7 steps of 8 and one of 4, its home on slot 4 of 8
    got, homes = run_case(setup, 8, 7, 60, 4, ctx_kind="ceiling")
    assert all(g["steps"] < len(g["tokens"]) for g in got)
    assert any(h != 0 for h in homes), "no stream ended with its home on a spare slot"


def test_33_streams_two_passes(setup):
    pkg = setup[0]
    run_case(setup, 33, 3, 24, 5, ctx_kind="floor", sampling=mixed(pkg, 33))


@pytest.mark.parametrize("k", [1, 15])
def test_extreme_drafts(setup, k):
    S = 9 if k == 15 else 5  # S = 9 with k = 15: two passes of 8 and 1 streams
    got, homes = run_case(setup, S, k, 40, 6 + k, ctx_kind="ceiling", ngram=2)
    assert sum(len(g["tokens"]) for g in got) > sum(g["steps"] for g in got)


def test_stops_inside_accepted_drafts(setup):
    pkg = setup[0]
    got, _ = run_case(setup, 8, 3, 48, 8, ctx_kind="ceiling", sampling=[pkg.Sampler(temperature=0.0)] * 8,
                      stop_from_run=True)
    assert any(len(g["tokens"]) < 48 for g in got), "no stop token fired"


def test_budgets_below_k_and_overrides(setup):
    pkg = setup[0]
    S, k = 6, 3
    budgets = [1, 2, 3, 4, 5, 40]
    run_case(setup, S, k, 40, 9, ctx_kind="ceiling", budgets=budgets, overrides={0: -99.0, 11: 5.0, 187: -np.inf},
             sampling=mixed(pkg, S))


def test_refusals(setup):
    pkg, a, b, before = setup
    E = pkg.EngineError
    two = [([0, 1, 2, 3], 5), ([4, 5, 6, 7], 6)]
    bad = [
        (dict(streams=[([0, 1], 5)], draft=1, ngram=0), "ngram 0"),
        (dict(streams=[([0, 1], 5)], draft=1, ngram=9), "ngram 9"),
        (dict(streams=[([0] + list(range(1, 17)), 5)], draft=16), "draft 16"),
        (dict(streams=[([s * 4 + i for i in range(4)], 5) for s in range(41)], draft=3), "max_gpt"),
        (dict(streams=[([0, 1, 2, 3], 5), ([4, 5, 6, 0], 6)], draft=3), "appears twice"),
        (dict(streams=[([0, 1, 2, MAX_GPT], 5)], draft=3), ">= max_gpt"),
        (dict(streams=two, draft=3, context=[[1], [V]]), "context token"),
        (dict(streams=two, draft=3, sampling=pkg.Sampler(temperature=0.0, presence_penalty=0.5)), "penalties"),
        (dict(streams=two, draft=3, sampling=pkg.Sampler(temperature=0.5)), "u is NULL"),
        (dict(streams=two, draft=3, budgets=[0, 3]), "budget 0"),
    ]
    reset(a, b, before)
    for kw, msg in bad:
        streams, draft = kw.pop("streams"), kw.pop("draft")
        kw.setdefault("ngram", 3)
        with pytest.raises(E, match=msg):
            a.generate_speculative(streams, 8, draft, **kw)
    a.set_option("prefill", 0)
    try:
        with pytest.raises(E, match="prefill"):
            a.generate_speculative(two, 8, 3)
    finally:
        a.set_option("prefill", 1)
    assert all(np.array_equal(x, y) for x, y in ((a.state_download(MAX_GPT)[k], before[k]) for k in KEYS5)), \
        "a refused call changed a slot"
