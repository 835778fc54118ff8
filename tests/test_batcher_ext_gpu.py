"""Batcher requests with logit overrides, token automata and log-probabilities (rwkv_b200_batcher_submit_ex) against
each request run alone through the existing API.

The oracle is the plain batcher tests' (decoding.batcher_oracle): a second engine from the same state, prefill_min = 2,
forward_streams of prompt[:-1] (state only) and then one generate_streams call of (slot, prompt[-1]) plus a pad stream on
a spare slot. Here that call also carries the request's overrides, its automaton (the pad has none) and its
log-probability mode and top_n, so it is generate_streams_constrained, generate_streams_logprobs or generate_streams_ex.
The pad gets the call-wide overrides, mode and stops, which is harmless: rows are independent. Tokens, log-probabilities,
ranks, top entries (NaN and -inf compared as bits), final automaton states and every named slot must equal the oracle;
unnamed slots must not change."""
import ctypes

import numpy as np
import pytest

from decoding import (FIELDS, KEYS5, LENGTHS, MAX_GPT, OVERRIDES, PAD, SHAPES, V, add_stops, batcher_oracle,
                      batcher_samplers, bits, check_slots, engine_pair, ext, finish, regex_automata, run_schedule,
                      submit)

pytestmark = pytest.mark.gpu

RESULT_FIELDS = ("tokens",) + FIELDS
BIAS = {11: 1e3, 187: -99.0, 50: -np.inf}  # token 11 wins every unmasked pick
EOS = {0: 50.0}                            # the automata's eos (token 0) wins wherever a state allows it
# per request i, kind i % 10: (overrides, automaton, logprobs, top_n); automaton "date+" starts after "2024-"
KINDS = [
    (None, None, None, 0),
    (OVERRIDES, None, None, 0),
    ({**OVERRIDES, **EOS}, "date", "raw", 5),
    (None, None, "processed", 20),
    (None, "labels", "processed", 0),
    (BIAS, None, "raw", 0),
    ({**OVERRIDES, **EOS}, "json", "raw", 20),
    (None, None, None, 0),
    (EOS, "date+", None, 0),
    (OVERRIDES, None, "raw", 5),
]


@pytest.fixture(scope="module")
def autos(pkg):
    return regex_automata(pkg.constrain, ("date", "labels", "json"))


def register(engs, autos):
    """The automata on every engine, in the same order, so that their ids agree: {name: id}."""
    au, _ = autos
    ids = {}
    for k in sorted(au):
        got = {e.add_constraint(au[k]) for e in engs}
        assert len(got) == 1
        ids[k] = got.pop()
    return ids


def make_mixed_requests(pkg, n, seed, slots, ids, autos, kinds=None):
    rng = np.random.default_rng(seed)
    sp = batcher_samplers(pkg)
    reqs = []
    for i in range(n):
        ovr, auto, lp, top = KINDS[(kinds[i] if kinds else i) % len(KINDS)]
        L = LENGTHS[i % len(LENGTHS)] if i < 2 * len(LENGTHS) else int(rng.integers(1, 200))
        s = sp[i % len(sp)]
        max_new = 64 if auto else int(rng.integers(3, 40))
        cons = None
        if auto:
            cons = (ids[auto.rstrip("+")], autos[1][auto] if auto.endswith("+") else 0)
        reqs.append(dict(slot=slots[i], prompt=[int(x) for x in rng.integers(0, V, size=L)], max_new=max_new, sampling=s,
                         u=rng.random(max_new) if s.temperature > 0 else None, stop=(), overrides=ovr, constraint=cons,
                         auto=auto.rstrip("+") if auto else None, logprobs=lp, top_n=top))
    return reqs


def check_result(got, want, what, prefix=False):
    """got (Batcher.result) equals want (oracle) in every field, bit for bit; prefix: got is a prefix of want."""
    assert set(got) - {"status"} == set(want), (what, sorted(got), sorted(want))
    n = len(got["tokens"])
    assert n == len(want["tokens"]) or (prefix and n <= len(want["tokens"])), (what, n, len(want["tokens"]))
    for k in RESULT_FIELDS:
        if k in want:
            assert bits(got[k]) == bits(want[k][:n]), (what, k)
    if "state" in want and not prefix:
        assert got["state"] == want["state"], (what, "state")


@pytest.fixture(scope="module", params=SHAPES, ids=["3x768", "2x2048"])
def setup(request, pkg, make_model, autos):
    """The engines with the automata, ~40 mixed requests with stops, and their oracle results."""
    L, E = request.param
    a, b = engine_pair(pkg, make_model(L, E), MAX_GPT, tc=True, one_draw=True)
    ids = register((a, b), autos)
    before = a.state_download(MAX_GPT)
    reqs = make_mixed_requests(pkg, 40, 7, list(range(40)), ids, autos)
    add_stops(pkg, b, reqs)
    want = [batcher_oracle(pkg, b, r) for r in reqs]
    assert any(len(w["tokens"]) < r["max_new"] for w, r in zip(want, reqs) if r["constraint"] is None), "no stop fired"
    yield pkg, a, b, before, reqs, want, ids
    a.close()
    b.close()


@pytest.mark.parametrize("rows,prefill", [(4, 1), (4, 17), (64, 300)])
def test_mixed_waves_equal_oracle(setup, autos, rows, prefill):
    """Three waves of mixed requests submitted between runs of 5, 16 and 40 steps: every field and every named slot
    equals the oracle; constrained requests complete before max_new in a state without edges."""
    pkg, a, b, before, reqs, want, ids = setup
    a.state_upload(before, MAX_GPT)
    with a.batcher(rows, prefill) as bat:
        rids = []
        for wave, steps in ((reqs[:14], 5), (reqs[14:27], 16), (reqs[27:], 40)):
            rids += [submit(bat, r) for r in wave]
            bat.run(steps)
        finish(bat)
        for i, (rid, w) in enumerate(zip(rids, want)):
            got = bat.result(rid)
            assert got["status"] == "done", (i, got["status"])
            check_result(got, w, "request %d" % i)
            r = reqs[i]
            if r["constraint"] is not None:
                assert len(got["tokens"]) < r["max_new"], i
                assert autos[0][r["auto"]].complete(got["state"]), i
            tokens, status = bat.read(rid)
            assert status == "done" and np.array_equal(tokens, got["tokens"])
    check_slots(a, b, before, MAX_GPT, {r["slot"] for r in reqs}, keys=KEYS5, skip=(PAD,),
                what="rows=%d prefill=%d" % (rows, prefill))


def test_two_schedules_identical(setup):
    pkg, a, b, before, reqs, want, ids = setup
    result = lambda bat, rid: bat.result(rid)
    r1, s1 = run_schedule(a, before, reqs[:14], 8, 64, 1000, result)
    r2, s2 = run_schedule(a, before, reqs[:14], 3, 5, 7, result)
    for i, (x, y) in enumerate(zip(r1, r2)):
        assert set(x) == set(y)
        for k in x:
            assert bits(x[k]) == bits(y[k]) if k in RESULT_FIELDS else x[k] == y[k], (i, k)
    for k in KEYS5:
        assert np.array_equal(s1[k], s2[k]), k


def test_streaming_prefix(setup):
    """After each run(16), result() is a prefix of the final result in every field."""
    pkg, a, b, before, reqs, want, ids = setup
    a.state_upload(before, MAX_GPT)
    seen = {}
    with a.batcher(6, 40) as bat:
        rids = [submit(bat, r) for r in reqs[:12]]
        while bat.run(16):
            for i, rid in enumerate(rids):
                seen.setdefault(i, []).append(bat.result(rid))
        for i, rid in enumerate(rids):
            check_result(bat.result(rid), want[i], "request %d" % i)
            for p in seen[i]:
                check_result(p, want[i], "request %d, streamed" % i, prefix=True)
    assert any(0 < len(p["tokens"]) < len(want[i]["tokens"]) for i in seen for p in seen[i]), "nothing streamed"


def test_cancel_constrained_scored(setup, autos):
    """Cancelling generating constrained requests with log-probabilities leaves prefixes of the oracle's results, and
    their automaton states are the states after their emitted tokens; the other requests are unchanged."""
    pkg, a, b, before, reqs, want, ids = setup
    a.state_upload(before, MAX_GPT)
    pick = [2, 6, 12, 16]  # date and json, raw, top 5 and 20
    others = [0, 1, 3, 5]
    with a.batcher(8, 64) as bat:
        rids = {i: submit(bat, reqs[i]) for i in pick + others}
        left = set(pick)
        for _ in range(400):  # one-step groups; each picked request is cancelled once it has emitted 2 tokens
            if not left or not bat.run(1):
                break
            for i in sorted(left):
                x = bat.result(rids[i])
                if x["status"] == "generating" and len(x["tokens"]) >= 2:
                    bat.cancel(rids[i])
                    left.discard(i)
        assert not left, "never cancelled while generating: %s" % sorted(left)
        finish(bat)
        for i in pick:
            got = bat.result(rids[i])
            assert got["status"] == "cancelled"
            check_result(got, want[i], "cancelled request %d" % i, prefix=True)
            assert autos[0][reqs[i]["auto"]].walk([int(x) for x in got["tokens"]]) == got["state"], i
        for i in others:
            check_result(bat.result(rids[i]), want[i], "request %d" % i)


def test_lane_reuse(setup, autos):
    """One lane, three requests in turn: overridden + constrained + raw, plain, processed. Each equals its oracle, so
    no overrides, mask or ring of an earlier request reaches a later one."""
    pkg, a, b, before, reqs, want, ids = setup
    a.state_upload(before, MAX_GPT)
    held = b.state_download(MAX_GPT)
    b.state_upload(before, MAX_GPT)
    trio = make_mixed_requests(pkg, 3, 21, [100, 101, 102], ids, autos, kinds=[6, 0, 3])
    assert trio[0]["overrides"] and trio[0]["constraint"] and trio[0]["logprobs"] == "raw"
    with a.batcher(1, 32) as bat:
        rids = [submit(bat, r) for r in trio]
        finish(bat)
        got = [bat.result(i) for i in rids]
    for i, r in enumerate(trio):
        check_result(got[i], batcher_oracle(pkg, b, r), "lane reuse %d" % i)
    check_slots(a, b, before, MAX_GPT, {100, 101, 102}, keys=KEYS5, skip=(PAD,), what="lane reuse")
    b.state_upload(held, MAX_GPT)


def plain_trace_launches(pkg, a, before, reqs, via_ex_null=False, warm=None):
    a.state_upload(before, MAX_GPT)
    with a.batcher(4, 17) as bat:
        if warm:
            for r in warm:
                submit(bat, r)
            finish(bat)
        n0 = a.launch_count
        for r in reqs:
            if not via_ex_null:
                submit(bat, r)
                continue
            P = ctypes.c_ulonglong
            pr = np.ascontiguousarray(r["prompt"], np.uint64)
            us = np.ascontiguousarray(r["u"], np.float64) if r["u"] is not None else None
            req = pkg.engine.Request(r["slot"], pr.ctypes.data_as(ctypes.POINTER(P)), len(pr), r["max_new"], r["sampling"],
                                     us.ctypes.data_as(ctypes.POINTER(ctypes.c_double)) if us is not None else None, None, 0)
            rid = P()
            assert a.lib.rwkv_b200_batcher_submit_ex(bat.h, ctypes.byref(req), None, ctypes.byref(rid)) == 0
        finish(bat)
        return a.launch_count - n0


def test_cost_when_unused(setup):
    """A plain trace launches the same kernels through submit, through submit_ex with no extension, and after a batch
    that used every feature has finished."""
    pkg, a, b, before, reqs, want, ids = setup
    plain = [dict(r, stop=()) for r in reqs if not ext(r)][:8]
    featured = [r for r in reqs if ext(r)][:8]
    n1 = plain_trace_launches(pkg, a, before, plain)
    n2 = plain_trace_launches(pkg, a, before, plain, via_ex_null=True)
    n3 = plain_trace_launches(pkg, a, before, plain, warm=featured)
    assert n1 > 0 and n1 == n2 == n3, (n1, n2, n3)


def test_refusals(pkg, make_model, autos):
    """Every refusal of submit_ex leaves every slot untouched, queues nothing and uses no id; remove_constraint is refused
    while a queued or running request names the id, and succeeds once that request is done or cancelled."""
    a, _ = engine_pair(pkg, make_model(3, 768), MAX_GPT, tc=True, one_draw=True)
    ids = register((a,), autos)
    au, starts = autos
    before = a.state_download(MAX_GPT)
    E = pkg.EngineError
    labels = au["labels"]
    q_open = next(q for q in range(labels.n_states) if len(labels.edges(q)[0]) > 0)
    gone = a.add_constraint(au["date"])
    a.remove_constraint(gone)
    sink = next(q for q in range(labels.n_states) if labels.complete(q))
    with a.batcher(4, 16) as bat:
        first = bat.submit(3, [1, 2, 3], 8, logprobs="raw")
        bad = [dict(overrides={V: 1.0}), dict(overrides={5: float("nan")}), dict(overrides={5: float("inf")}),
               dict(overrides={t: -np.inf for t in range(V)}), dict(constraint=12345), dict(constraint=gone),
               dict(constraint=(ids["labels"], labels.n_states)), dict(constraint=(ids["labels"], sink)),
               dict(constraint=(ids["labels"], 0), overrides={int(t): -np.inf for t in labels.edges(q_open)[0]}),
               dict(logprobs="raw", top_n=21)]
        for kw in bad:
            with pytest.raises(E):
                bat.submit(4, [1, 2], 8, **kw)
        P = ctypes.c_ulonglong
        pr = np.array([1, 2], np.uint64)
        req = pkg.engine.Request(4, pr.ctypes.data_as(ctypes.POINTER(P)), 2, 8, pkg.Sampler(temperature=0.0), None, None, 0)
        for x in (pkg.engine.RequestEx(None, None, 2, pkg.engine.NO_CONSTRAINT, 0, 0, 0, 0),
                  pkg.engine.RequestEx(None, None, 0, pkg.engine.NO_CONSTRAINT, 0, 1, 2, 0)):
            rid = P()
            assert a.lib.rwkv_b200_batcher_submit_ex(bat.h, ctypes.byref(req), ctypes.byref(x), ctypes.byref(rid)) != 0
        lp = np.zeros(4, np.float64)
        plain = bat.submit(5, [1, 2], 4)
        assert plain == first + 1, "a refusal used an id"
        n = P()
        assert a.lib.rwkv_b200_batcher_read_ex(bat.h, plain, 4, None, lp.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                               None, None, None, None, ctypes.byref(n), None) != 0
        assert b"no log-probabilities" in a.lib.rwkv_b200_last_error()
        bat.cancel(first)
        bat.cancel(plain)
        assert bat.run(16) == 0, "a refused request was queued"
        after = a.state_download(MAX_GPT)
        for k in KEYS5:
            assert np.array_equal(before[k], after[k]), k
        # the automaton of an unfinished request cannot be removed
        q = bat.submit(6, [1, 2, 3], 64, constraint=ids["json"])
        with pytest.raises(E, match="unfinished request %d" % q):
            a.remove_constraint(ids["json"])
        bat.run(1)
        assert bat.result(q)["status"] in ("prefilling", "generating")
        with pytest.raises(E, match="unfinished request"):
            a.remove_constraint(ids["json"])
        bat.cancel(q)
        a.remove_constraint(ids["json"])
        d = bat.submit(7, [1, 2, 3], 64, constraint=ids["date"], overrides=EOS)
        with pytest.raises(E, match="unfinished request"):
            a.remove_constraint(ids["date"])
        finish(bat)
        assert bat.result(d)["status"] == "done"
        a.remove_constraint(ids["date"])
    a.close()
