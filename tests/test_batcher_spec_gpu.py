"""Speculative batcher requests (rwkv_b200_batcher_submit_spec) against each request run alone through the existing API.

The oracle is the plain batcher tests' (decoding.batcher_oracle): speculation changes only the number of steps, so a
speculative request's tokens, log-probabilities, ranks, top entries (NaN and -inf compared as bits), automaton state and
slot must equal the oracle exactly as a plain request's do. Its steps must equal engine.speculative_steps of the lookup
context ++ prompt[:-1], first token prompt[-1] and the emitted tokens, and for some requests the one-shot
generate_speculative call's steps. Spare slots are scratch and are not compared; every slot that no request names must
be unchanged. The engines have 1024 slots so that 64 rows of k = 15 fit max_gpt."""
import ctypes

import numpy as np
import pytest

from decoding import (KEYS4, KEYS5, PAD, SHAPES, V, add_stops, batcher_oracle, check_slots, engine_pair, finish, slot_of)
from test_batcher_ext_gpu import check_result, make_mixed_requests, register

pytestmark = pytest.mark.gpu

MG = 1024
KS = (1, 2, 4, 7, 15)
NGRAMS = (1, 3, 8)
CONTEXTS = ("none", "floor", "ceiling")


@pytest.fixture(scope="module")
def autos(pkg):
    from decoding import regex_automata
    return regex_automata(pkg.constrain, ("date", "labels", "json"))


def spares_from(pool, k):
    return [pool.pop() for _ in range(k)]


def speculate(reqs, want, pool, every=3, ks=KS, seed=3):
    """Give every request without penalties but every `every`-th a draft k, an n-gram, spare slots and a context: none,
    floor (random tokens) or ceiling (the request's own output, from the oracle)."""
    rng = np.random.default_rng(seed)
    j = 0
    for i, (r, w) in enumerate(zip(reqs, want)):
        s = r["sampling"]
        if i % every == every - 1 or s.presence_penalty or s.frequency_penalty:
            continue
        k = ks[j % len(ks)]
        kind = CONTEXTS[j % len(CONTEXTS)]
        r.update(draft=k, ngram=NGRAMS[j % len(NGRAMS)], spares=spares_from(pool, k),
                 context=None if kind == "none" else [int(x) for x in w["tokens"]] if kind == "ceiling"
                 else [int(x) for x in rng.integers(0, V, size=64)])
        j += 1


def submit(bat, r):
    kw = dict(sampling=r["sampling"], u=r["u"], stop=r["stop"])
    for k in ("overrides", "constraint", "logprobs"):
        if r.get(k) is not None:
            kw[k] = r[k]
    if r.get("logprobs") is not None:
        kw["top_n"] = r["top_n"]
    if r.get("draft"):
        kw.update(draft=r["draft"], spare_slots=r["spares"], ngram=r["ngram"], context=r["context"])
    return bat.submit(r["slot"], r["prompt"], r["max_new"], **kw)


def want_steps(pkg, r, toks):
    return pkg.engine.speculative_steps(list(r["context"] or []) + list(r["prompt"][:-1]), r["prompt"][-1], toks,
                                        r["draft"], r["ngram"])


def check_all(pkg, a, b, before, bat, rids, reqs, want, what):
    spares = set()
    for i, (rid, r, w) in enumerate(zip(rids, reqs, want)):
        got = bat.result(rid)
        assert got["status"] == "done", (what, i, got["status"])
        g = {k: v for k, v in got.items() if k != "steps"}
        check_result(g, w, "%s request %d" % (what, i))
        if r.get("draft"):
            assert got["steps"] == want_steps(pkg, r, [int(x) for x in got["tokens"]]), (what, i)
            spares |= set(r["spares"])
        else:
            assert "steps" not in got
    check_slots(a, b, before, MG, {r["slot"] for r in reqs}, skip=spares, what=what)


@pytest.fixture(scope="module", params=SHAPES, ids=["3x768", "2x2048"])
def setup(request, pkg, make_model, autos):
    """The engines with the automata, 30 mixed requests with stops, their oracle results, then speculation on most."""
    L, E = request.param
    a, b = engine_pair(pkg, make_model(L, E), MG, tc=True, one_draw=True)
    ids = register((a, b), autos)
    before = a.state_download(MG)
    reqs = make_mixed_requests(pkg, 30, 11, list(range(30)), ids, autos)
    add_stops(pkg, b, reqs)
    b.state_upload(before, MG)
    want = [batcher_oracle(pkg, b, r) for r in reqs]
    final = b.state_download(MG)  # the oracle's slot states after every request
    pool = [s for s in range(40, MG) if s != PAD]
    speculate(reqs, want, pool)
    assert sum(1 for r in reqs if r.get("draft")) >= 10
    yield pkg, a, b, before, reqs, want, pool, final
    a.close()
    b.close()


@pytest.mark.parametrize("rows,prefill", [(4, 1), (4, 17), (64, 300)])
def test_waves_equal_oracle(setup, rows, prefill):
    """Three waves of mixed speculative and plain requests submitted between runs of 5, 16 and 40 steps."""
    pkg, a, b, before, reqs, want, _, final = setup
    if rows == 64:  # rows x (k + 1) <= max_gpt: k <= 15 at 64 rows of 1024
        assert all(64 * (r.get("draft", 0) + 1) <= MG for r in reqs)
    b.state_upload(final, MG)
    a.state_upload(before, MG)
    with a.batcher(rows, prefill) as bat:
        rids = []
        for wave, steps in ((reqs[:10], 5), (reqs[10:20], 16), (reqs[20:], 40)):
            rids += [submit(bat, r) for r in wave]
            bat.run(steps)
        finish(bat)
        check_all(pkg, a, b, before, bat, rids, reqs, want, "rows %d prefill %d" % (rows, prefill))


def test_steps_equal_one_shot(setup):
    """For a few requests, steps equal the one-shot generate_speculative call's on the same slots and context."""
    pkg, a, b, before, reqs, want, _, final = setup
    picked = [r for r in reqs if r.get("draft") and r.get("constraint") is None and r.get("logprobs") is None][:4]
    assert picked
    a.state_upload(before, MG)
    with a.batcher(8, 64) as bat:
        rids = [submit(bat, r) for r in picked]
        finish(bat)
        got = [bat.result(i) for i in rids]
    b.state_upload(before, MG)
    for r, g in zip(picked, got):
        if len(r["prompt"]) > 1:
            call = [(r["slot"], r["prompt"][:-1])] + ([(PAD, r["prompt"][:1])] if len(r["prompt"]) == 2 else [])
            b.forward_streams(call, want_logits=False)
        one = b.generate_speculative([([r["slot"]] + r["spares"], r["prompt"][-1])], r["max_new"], r["draft"],
                                     ngram=r["ngram"], context=[list(r["context"] or []) + list(r["prompt"][:-1])],
                                     stop=r["stop"], overrides=r.get("overrides"), sampling=[r["sampling"]],
                                     u=None if r["u"] is None else np.asarray(r["u"]).reshape(-1, 1))[0]
        assert [int(x) for x in one["tokens"]] == [int(x) for x in g["tokens"]]
        assert one["steps"] == g["steps"]


def test_ceiling_runs_many_tokens_per_step(setup):
    """Requests whose context is their own output take far fewer steps than tokens; one with k = 15 and max_new = 300
    emits more than 16 tokens inside one group (the ring)."""
    pkg, a, b, before, reqs, want, pool, final = setup
    rng = np.random.default_rng(17)
    cs = []
    for i, k in enumerate((15, 4, 7)):
        prompt = [int(x) for x in rng.integers(0, V, size=40 + 30 * i)]
        cs.append(dict(slot=30 + i, prompt=prompt, max_new=300 if k == 15 else 80, sampling=pkg.Sampler(temperature=0.0),
                       u=None, stop=(), draft=k, ngram=3))
    b.state_upload(before, MG)
    w = [batcher_oracle(pkg, b, r) for r in cs]
    for r, x in zip(cs, w):
        r.update(spares=spares_from(pool, r["draft"]), context=[int(t) for t in x["tokens"]])
    a.state_upload(before, MG)
    with a.batcher(4, 32) as bat:
        rids = [submit(bat, r) for r in cs]
        grew, n = [], 0
        while bat.run(16):  # a run of 16 steps is one group
            m = len(bat.read(rids[0])[0])
            grew.append(m - n)
            n = m
        check_all(pkg, a, b, before, bat, rids, cs, w, "ceiling")
        for r, rid in zip(cs, rids):
            g = bat.result(rid)
            assert g["steps"] < len(g["tokens"]), (r["draft"], g["steps"], len(g["tokens"]))
        assert len(bat.result(rids[0])["tokens"]) == 300
        assert max(grew) > 16, grew


def test_two_passes_with_prefill(setup):
    """30 speculative lanes of k = 4 (150 decode rows: two passes) run with prefill segments in the same steps."""
    pkg, a, b, before, reqs, want, pool, final = setup
    rng = np.random.default_rng(23)
    rs = []
    for i in range(32):
        rs.append(dict(slot=100 + i, prompt=[int(x) for x in rng.integers(0, V, size=(2 if i < 30 else 200))], max_new=24,
                       sampling=pkg.Sampler(temperature=0.8, top_p=0.9), u=rng.random(24), stop=()))
    b.state_upload(before, MG)
    w = [batcher_oracle(pkg, b, r) for r in rs]
    free = [s for s in pool if s >= 400]
    for r in rs[:30]:
        r.update(draft=4, ngram=2, spares=spares_from(free, 4), context=None)
    a.state_upload(before, MG)
    with a.batcher(32, 64) as bat:
        rids = [submit(bat, r) for r in rs]
        finish(bat)
        check_all(pkg, a, b, before, bat, rids, rs, w, "two passes")


def test_streaming_and_cancel(setup):
    """Reads between runs give growing prefixes; a request cancelled mid-group, with its conversation on a spare slot
    (own-output context, so drafts are accepted), keeps a prefix of the oracle's tokens and its slot holds the oracle's
    state for a budget of its emitted length."""
    pkg, a, b, before, reqs, want, pool, final = setup
    rng = np.random.default_rng(41)
    rs = [dict(slot=150 + i, prompt=[int(x) for x in rng.integers(0, V, size=8)], max_new=60,
               sampling=pkg.Sampler(temperature=0.0), u=None, stop=(), draft=2, ngram=2, spares=spares_from(pool, 2))
          for i in range(3)]
    b.state_upload(before, MG)
    w = [batcher_oracle(pkg, b, r) for r in rs]
    for r, x in zip(rs, w):
        r["context"] = [int(t) for t in x["tokens"]]
    a.state_upload(before, MG)
    with a.batcher(4, 300) as bat:
        rids = [submit(bat, r) for r in rs]
        seen = [[] for _ in rids]
        for _ in range(3):
            bat.run(5)
            for j, rid in enumerate(rids):
                t = [int(x) for x in bat.read(rid)[0]]
                assert t[:len(seen[j])] == seen[j]
                assert t == [int(x) for x in w[j]["tokens"][:len(t)]]
                seen[j] = t
        # home moves by the tokens a step emits beyond its first, modulo k + 1 = 3: one-step runs until it is a spare
        for _ in range(6):
            n, steps = len(bat.read(rids[0])[0]), bat.result(rids[0])["steps"]
            if (n - steps) % 3:
                break
            bat.run(1)
        assert steps < n and (n - steps) % 3, (n, steps)
        assert n < 60  # at most 3 tokens in each of at most 21 steps
        assert [int(x) for x in bat.read(rids[0])[0]] == [int(x) for x in w[0]["tokens"][:n]]
        bat.cancel(rids[0])
        finish(bat)
        assert bat.result(rids[0])["status"] == "cancelled"
        assert [int(x) for x in bat.read(rids[0])[0]] == [int(x) for x in w[0]["tokens"][:n]]
        for rid, ww in zip(rids[1:], w[1:]):
            assert [int(x) for x in bat.read(rid)[0]] == [int(x) for x in ww["tokens"]]
    got = a.state_download(MG)
    b.state_upload(before, MG)
    batcher_oracle(pkg, b, dict(rs[0], max_new=n))
    ref = b.state_download(MG)
    E = a.n_layers * a.n_embed
    for k in KEYS4:
        assert np.array_equal(slot_of(got, rs[0]["slot"], E)[k], slot_of(ref, rs[0]["slot"], E)[k]), k


def step_starts(pkg, r, toks):
    """The position of the first token of each step, by the steps rule (engine.speculative_steps restated per step)."""
    h = list(r["context"] or []) + list(r["prompt"])
    pos, starts = 0, []
    while pos < len(toks):
        d = pkg.engine.lookup_drafts(h, r["draft"], r["ngram"])
        c = 1
        while c <= r["draft"] and pos + c < len(toks) and d[c - 1] == toks[pos + c - 1]:
            c += 1
        starts.append(pos)
        h += toks[pos:pos + c]
        pos += c
    return starts


def stop_oracle(pkg, b, r, sid):
    """batcher_oracle with a stop set: forward_streams of prompt[:-1], then generate_streams_stop of (slot, prompt[-1])
    and a pad stream."""
    slot, prompt = r["slot"], r["prompt"]
    b.forward_streams([(slot, prompt[:-1])] + ([(PAD, prompt[:1])] if len(prompt) == 2 else []), want_logits=False)
    return b.generate_streams([(slot, prompt[-1]), (PAD, prompt[-1])], r["max_new"], stop=r["stop"],
                              sampling=[r["sampling"], pkg.Sampler(temperature=0.0)], stop_strings=[sid, None])[0]


def test_stops_and_automata_inside_accepted_runs(setup, autos):
    """Own-output contexts, so that the token that ends a request lies inside an accepted run of drafts: a stop token, a
    stop string (hit, tail and state compared with generate_streams_stop) and token automata that complete (some of
    them inside an accepted run). Every result and named slot equals the oracle."""
    pkg, a, b, before, reqs, want, pool, final = setup
    ids = register((a, b), autos)
    tb = pkg.constrain.token_bytes()
    rng = np.random.default_rng(53)
    G = pkg.Sampler(temperature=0.0)
    base = lambda slot, extra=None: dict(dict(slot=slot, prompt=[int(x) for x in rng.integers(0, V, size=24)], max_new=48,
                                              sampling=G, u=None, stop=(), draft=4, ngram=3, overrides=None,
                                              constraint=None, logprobs=None, top_n=0), **(extra or {}))
    # stop token and stop string: from runs without them, a position inside an accepted run that ends the request
    stop_tok = stop_str = None
    for slot in range(33, 45):
        r = base(slot)
        b.state_upload(before, MG)
        full = [int(t) for t in batcher_oracle(pkg, b, r)["tokens"]]
        r["context"] = full
        starts = set(step_starts(pkg, r, full))
        inside = [p for p in range(1, len(full)) if p not in starts]
        if stop_tok is None:
            p = next((p for p in inside if full[p] not in full[:p]), None)
            if p is not None:
                stop_tok = dict(r, stop=(full[p],))
                continue
        if stop_str is None:
            chunks = [tb[t] for t in full]
            for p in inside:
                strings = [chunks[p][-2:]] if len(chunks[p]) else []
                if strings and pkg.engine.stop_match(strings, chunks)[0] == p:
                    stop_str = dict(r, strings=strings)
                    break
        if stop_tok is not None and stop_str is not None:
            break
    assert stop_tok is not None and stop_str is not None
    autom = []
    for slot in range(45, 49):
        r = base(slot, dict(constraint=(ids["json"], 0), overrides={0: 50.0}, max_new=64))
        b.state_upload(before, MG)
        r["context"] = [int(t) for t in batcher_oracle(pkg, b, r)["tokens"]]
        autom.append(r)
    rs = [stop_tok, stop_str] + autom
    for r in rs:
        r["spares"] = spares_from(pool, r["draft"])
    sid_a, sid_b = a.add_stop_set(stop_str["strings"]), b.add_stop_set(stop_str["strings"])
    b.state_upload(before, MG)
    w = [stop_oracle(pkg, b, r, sid_b) if "strings" in r else batcher_oracle(pkg, b, r) for r in rs]
    a.state_upload(before, MG)
    with a.batcher(8, 64) as bat:
        rids = []
        for r in rs:
            if "strings" in r:
                rids.append(bat.submit(r["slot"], r["prompt"], r["max_new"], sampling=G, draft=r["draft"],
                                       spare_slots=r["spares"], ngram=r["ngram"], context=r["context"], stop_strings=sid_a))
            else:
                rids.append(submit(bat, r))
        finish(bat)
        got = [bat.result(i) for i in rids]
    for i, (r, g, x) in enumerate(zip(rs, got, w)):
        assert g["status"] == "done", i
        assert [int(t) for t in g["tokens"]] == [int(t) for t in x["tokens"]], i
        toks = [int(t) for t in g["tokens"]]
        assert g["steps"] == want_steps(pkg, r, toks), i
        if "strings" in r:
            assert x["stop_hit"] is not None
            assert (g["stop_hit"], g["stop_tail"], g["stop_state"]) == (x["stop_hit"], x["stop_tail"], x["stop_state"])
        if r["constraint"] is not None:
            assert g["state"] == x["state"], i
            assert len(toks) < r["max_new"], i
    # the last token of the stop requests was emitted inside an accepted run: the step before it emitted it too
    for r, g in zip(rs[:2], got[:2]):
        toks = [int(t) for t in g["tokens"]]
        assert len(toks) < r["max_new"] and (len(toks) - 1) not in step_starts(pkg, r, toks)
    assert any(len(g["tokens"]) - 1 not in step_starts(pkg, r, [int(t) for t in g["tokens"]])
               for r, g in zip(autom, got[2:])), "no automaton completed inside an accepted run"
    check_slots(a, b, before, MG, {r["slot"] for r in rs}, skip={z for r in rs for z in r["spares"]})


def test_lane_and_slot_reuse(setup):
    """One lane: a speculative request, then a plain one, then a speculative one that names the first one's spare slots
    again (released when it finished)."""
    pkg, a, b, before, reqs, want, _, final = setup
    rng = np.random.default_rng(31)
    rs = [dict(slot=200 + i, prompt=[int(x) for x in rng.integers(0, V, size=20)], max_new=40,
               sampling=pkg.Sampler(temperature=0.0), u=None, stop=()) for i in range(3)]
    b.state_upload(before, MG)
    w = [batcher_oracle(pkg, b, r) for r in rs]
    rs[0].update(draft=3, ngram=3, spares=[300, 301, 302], context=[int(t) for t in w[0]["tokens"]])
    rs[2].update(draft=3, ngram=2, spares=[302, 300, 301], context=None)
    a.state_upload(before, MG)
    with a.batcher(1, 16) as bat:
        rids = []
        for r in rs:
            rids.append(submit(bat, r))
            finish(bat)
        check_all(pkg, a, b, before, bat, rids, rs, w, "reuse")


def trace_launches(pkg, a, before, plain, via_spec_null=False, warm=None):
    a.state_upload(before, MG)
    with a.batcher(4, 17) as bat:
        if warm:
            for r in warm:
                submit(bat, r)
            finish(bat)
        n0 = a.launch_count
        for r in plain:
            if not via_spec_null:
                submit(bat, r)
                continue
            P = ctypes.c_ulonglong
            pr = np.ascontiguousarray(r["prompt"], np.uint64)
            us = np.ascontiguousarray(r["u"], np.float64) if r["u"] is not None else None
            req = pkg.engine.Request(r["slot"], pr.ctypes.data_as(ctypes.POINTER(P)), len(pr), r["max_new"], r["sampling"],
                                     us.ctypes.data_as(ctypes.POINTER(ctypes.c_double)) if us is not None else None, None, 0)
            rid = P()
            assert a.lib.rwkv_b200_batcher_submit_spec(bat.h, ctypes.byref(req), None, pkg.engine.NO_STOP_SET, 0, None,
                                                       ctypes.byref(rid)) == 0
        finish(bat)
        return a.launch_count - n0


def test_cost_when_unused(setup):
    """A plain trace launches the same kernels through submit, through submit_spec(spec = NULL), and after a speculative
    batch has finished."""
    pkg, a, b, before, reqs, want, _, final = setup
    plain = [dict(r, stop=()) for r in reqs if not r.get("draft") and r.get("overrides") is None
             and r.get("constraint") is None and r.get("logprobs") is None][:6]
    warm = [r for r in reqs if r.get("draft")][:6]
    assert plain and warm
    n1 = trace_launches(pkg, a, before, plain)
    n2 = trace_launches(pkg, a, before, plain, via_spec_null=True)
    n3 = trace_launches(pkg, a, before, plain, warm=warm)
    assert n1 > 0 and n1 == n2 == n3, (n1, n2, n3)


def test_refusals(pkg, make_model):
    """Every refusal of submit_spec leaves every slot untouched, queues nothing and uses no id."""
    a, _ = engine_pair(pkg, make_model(3, 768), 64, tc=True, one_draw=True)
    before = a.state_download(64)
    E = pkg.EngineError
    lib = a.lib
    P = ctypes.c_ulonglong
    with a.batcher(4, 16) as bat:
        first = bat.submit(3, [1, 2, 3], 8, draft=2, spare_slots=[10, 11])
        bad = [dict(draft=16, spare_slots=list(range(20, 36))), dict(draft=1, spare_slots=[20], ngram=0),
               dict(draft=1, spare_slots=[20], ngram=9), dict(draft=2, spare_slots=[20, 20]),
               dict(draft=1, spare_slots=[64]), dict(draft=1, spare_slots=[4]), dict(draft=1, spare_slots=[3]),
               dict(draft=1, spare_slots=[11]), dict(draft=1, spare_slots=[20], context=[1, V]),
               dict(draft=1, spare_slots=[20], sampling=pkg.Sampler(temperature=0.0, presence_penalty=0.5)),
               dict(draft=1, spare_slots=[20], sampling=pkg.Sampler(temperature=0.0, frequency_penalty=0.5)),
               dict(draft=15, spare_slots=list(range(20, 35)))]  # 4 rows x 16 = 64 <= 64: accepted below
        for kw in bad[:-1]:
            with pytest.raises(E):
                bat.submit(4, [1, 2], 8, **kw)
        with pytest.raises(E, match="held by unfinished request"):  # a plain request on another's spare slot
            bat.submit(10, [1, 2], 8)
        pr = np.array([1, 2], np.uint64)
        req = pkg.engine.Request(4, pr.ctypes.data_as(ctypes.POINTER(P)), 2, 8, pkg.Sampler(temperature=0.0), None, None, 0)
        rid = P()
        spec = pkg.engine.RequestSpec(None, 1, 3, None, 0)
        assert lib.rwkv_b200_batcher_submit_spec(bat.h, ctypes.byref(req), None, pkg.engine.NO_STOP_SET, 0,
                                                 ctypes.byref(spec), ctypes.byref(rid)) != 0
        assert b"spare_slots is NULL" in lib.rwkv_b200_last_error()
        sp = np.array([20], np.uint64)
        spec = pkg.engine.RequestSpec(sp.ctypes.data_as(ctypes.POINTER(P)), 1, 3, None, 2)
        assert lib.rwkv_b200_batcher_submit_spec(bat.h, ctypes.byref(req), None, pkg.engine.NO_STOP_SET, 0,
                                                 ctypes.byref(spec), ctypes.byref(rid)) != 0
        ok = bat.submit(4, [1, 2], 8, **bad[-1])
        assert ok == first + 1, "a refusal used an id"
        bat.cancel(first)
        bat.cancel(ok)
        assert bat.run(16) == 0, "a refused request was queued"
        after = a.state_download(64)
        for k in KEYS5:
            assert np.array_equal(before[k], after[k]), k
    with a.batcher(5, 16) as bat:  # 5 rows x 16 > 64
        with pytest.raises(E, match="max_gpt"):
            bat.submit(4, [1, 2], 8, draft=15, spare_slots=list(range(20, 35)))
    a.close()
