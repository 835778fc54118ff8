"""Continuous batching (rwkv_b200_batcher_*) against each request run alone through the existing API.

The oracle is a second engine that starts from the same state and runs, per request, the two calls the batcher's rule
names, both on the tensor cores (prefill_min = 2): forward_streams of prompt[:-1] (state only), then
generate_streams_ex of (slot, prompt[-1]) with the request's max_new, stop tokens, sampler and uniforms. A call that
would have fewer than 2 tokens gets a pad stream on a spare slot; rows are independent, so the pad changes nothing (the
call-wide stop tokens apply to the pad too, which is harmless). Tokens and every named slot must be bit-equal to the
oracle whatever the schedule, and slots no request names must not change at all."""
import numpy as np
import pytest

from decoding import (KEYS5, LENGTHS, MAX_GPT, PAD, SHAPES, V, add_stops, batcher_oracle, batcher_samplers, check_slots,
                      engine_pair, finish, run_schedule, slot_of, submit)

pytestmark = pytest.mark.gpu


def make_requests(pkg, n, seed, slots):
    """n requests on the given distinct slots: every prompt length of LENGTHS, a mix of samplers."""
    rng = np.random.default_rng(seed)
    sp = batcher_samplers(pkg)
    reqs = []
    for i in range(n):
        L = LENGTHS[i % len(LENGTHS)] if i < 2 * len(LENGTHS) else int(rng.integers(1, 200))
        s = sp[i % len(sp)]
        max_new = int(rng.integers(3, 40))
        u = rng.random(max_new) if s.temperature > 0 else None
        reqs.append(dict(slot=slots[i], prompt=[int(x) for x in rng.integers(0, V, size=L)], max_new=max_new, sampling=s,
                         u=u, stop=()))
    return reqs


def oracle_tokens(pkg, b, r):
    """The rule's two calls for one request on engine b (decoding.batcher_oracle); returns its tokens."""
    return [int(x) for x in batcher_oracle(pkg, b, r)["tokens"]]


@pytest.fixture(scope="module", params=SHAPES, ids=["3x768", "2x2048"])
def setup(request, pkg, make_model):
    """The engines, the ~40 requests with stops, and their oracle tokens (b holds every request's final state)."""
    L, E = request.param
    a, b = engine_pair(pkg, make_model(L, E), MAX_GPT, tc=True, one_draw=True)
    before = a.state_download(MAX_GPT)
    reqs = make_requests(pkg, 40, 7, list(range(40)))
    add_stops(pkg, b, reqs)
    want = [oracle_tokens(pkg, b, r) for r in reqs]
    assert any(len(w) < r["max_new"] for w, r in zip(want, reqs)), "no stop token fired"
    yield pkg, a, b, before, reqs, want
    a.close()
    b.close()


@pytest.mark.parametrize("rows,prefill", [(4, 1), (4, 17), (64, 128), (64, 300)])
def test_waves_equal_oracle(setup, rows, prefill):
    """Three waves submitted between runs of 5, 16 and 40 steps: tokens and slots equal the oracle, bit for bit."""
    pkg, a, b, before, reqs, want = setup
    a.state_upload(before, MAX_GPT)
    with a.batcher(rows, prefill) as bat:
        ids = []
        for wave, steps in ((reqs[:14], 5), (reqs[14:27], 16), (reqs[27:], 40)):
            ids += [submit(bat, r) for r in wave]
            bat.run(steps)
        finish(bat)
        for i, (rid, w) in enumerate(zip(ids, want)):
            toks, status = bat.read(rid)
            assert status == "done", "request %d: %s" % (i, status)
            assert [int(x) for x in toks] == w, "request %d (prompt %d tokens): tokens" % (i, len(reqs[i]["prompt"]))
    check_slots(a, b, before, MAX_GPT, {r["slot"] for r in reqs}, keys=KEYS5, skip=(PAD,),
                what="rows=%d prefill=%d" % (rows, prefill))


def test_two_schedules_identical(setup):
    pkg, a, b, before, reqs, want = setup
    tokens = lambda bat, rid: [int(x) for x in bat.read(rid)[0]]
    t1, s1 = run_schedule(a, before, reqs[:12], 8, 64, 1000, tokens)
    t2, s2 = run_schedule(a, before, reqs[:12], 3, 5, 7, tokens)
    assert t1 == t2
    for k in KEYS5:
        assert np.array_equal(s1[k], s2[k]), k


def test_streaming_prefix(setup):
    """After each run(16), read is a prefix of the final tokens."""
    pkg, a, b, before, reqs, want = setup
    a.state_upload(before, MAX_GPT)
    seen = {}
    with a.batcher(6, 40) as bat:
        ids = [submit(bat, r) for r in reqs[:10]]
        while bat.run(16):
            for i, rid in enumerate(ids):
                toks, _ = bat.read(rid)
                seen.setdefault(i, []).append([int(x) for x in toks])
        for i, rid in enumerate(ids):
            final = [int(x) for x in bat.read(rid)[0]]
            assert final == want[i]
            for p in seen[i]:
                assert final[:len(p)] == p
        assert any(0 < len(p) < len(want[i]) for i in seen for p in seen[i]), "nothing streamed"


def test_release_between_runs(setup):
    """Done requests released between runs, while others still run and new ones arrive, change nothing in the rest."""
    pkg, a, b, before, reqs, want = setup
    a.state_upload(before, MAX_GPT)
    with a.batcher(3, 24) as bat:
        ids = {submit(bat, r): i for i, r in enumerate(reqs[:6])}
        got = {}
        pending = list(range(6, 12))
        while bat.run(16) or pending:
            for rid, i in list(ids.items()):
                toks, st = bat.read(rid)
                if st == "done":
                    got[i] = [int(x) for x in toks]
                    bat.release(rid)
                    del ids[rid]
            if pending:
                i = pending.pop(0)
                ids[submit(bat, reqs[i])] = i
        for rid, i in ids.items():
            got[i] = [int(x) for x in bat.read(rid)[0]]
    assert [got[i] for i in range(12)] == want[:12]


def test_cancel(setup):
    """Cancel a queued, a prefilling and a generating request: their tokens are prefixes of the oracle's, the queued
    request's slot is untouched, and every other request equals the run without the cancels."""
    pkg, a, b, before, reqs, want = setup
    a.state_upload(before, MAX_GPT)
    n = a.n_layers * a.n_embed
    sel = reqs[:12]
    with a.batcher(4, 3) as bat:
        ids = [submit(bat, r) for r in sel]
        for _ in range(20):  # group ends until one request of each kind is seen
            bat.run(16)
            status = {i: bat.read(rid)[1] for i, rid in enumerate(ids)}
            gen = [i for i in status if status[i] == "generating"]
            pre = [i for i in status if status[i] == "prefilling"]
            que = [i for i in status if status[i] == "queued"]
            if gen and pre and que:
                break
        assert gen and pre and que, status
        cancelled = {gen[0], pre[0], que[-1]}
        for i in cancelled:
            bat.cancel(ids[i])
        finish(bat)
        for i, rid in enumerate(ids):
            toks, st = bat.read(rid)
            toks = [int(x) for x in toks]
            if i in cancelled:
                assert st == "cancelled" and toks == want[i][:len(toks)], i
            else:
                assert st == "done" and toks == want[i], i
        sa = a.state_download(MAX_GPT)
        q = sel[que[-1]]["slot"]
        for k in KEYS5:
            assert np.array_equal(slot_of(sa, q, n)[k], slot_of(before, q, n)[k]), "queued slot touched"
    sb = b.state_download(MAX_GPT)
    for i, r in enumerate(sel):
        if i not in cancelled:
            for k in KEYS5:
                assert np.array_equal(slot_of(sa, r["slot"], n)[k], slot_of(sb, r["slot"], n)[k]), (i, k)


def test_next_turn_and_unrelated_forward(pkg, make_model):
    """A second request on a finished request's slot equals the oracle chained on that slot, and a forward_streams on an
    unrelated slot between runs changes nothing in the batcher's results."""
    a, b = engine_pair(pkg, make_model(3, 768), MAX_GPT, tc=True, one_draw=True)
    before = a.state_download(MAX_GPT)
    reqs = make_requests(pkg, 6, 11, [40, 41, 42, 43, 44, 45])
    turn2 = make_requests(pkg, 2, 12, [40, 41])
    with a.batcher(4, 20) as bat:
        ids = [submit(bat, r) for r in reqs]
        bat.run(5)
        a.forward_streams([(50, [1, 2, 3, 4, 5, 6, 7, 8, 9])], want_logits=False)
        b.forward_streams([(50, [1, 2, 3, 4, 5, 6, 7, 8, 9])], want_logits=False)
        finish(bat)
        for rid in ids[:2]:
            bat.release(rid)
        ids2 = [submit(bat, r) for r in turn2]
        finish(bat)
        got = [[int(x) for x in bat.read(i)[0]] for i in ids[2:] + ids2]
    want = [oracle_tokens(pkg, b, r) for r in reqs]
    want2 = [oracle_tokens(pkg, b, r) for r in turn2]
    assert got == want[2:] + want2
    named = {r["slot"] for r in reqs} | {50}
    check_slots(a, b, before, MAX_GPT, named, keys=KEYS5, skip=(PAD,), what="next turn")
    a.close()
    b.close()


def test_refusals(pkg, make_model):
    """Every refusal leaves every slot untouched; unknown ids are refused."""
    a, _ = engine_pair(pkg, make_model(3, 768), MAX_GPT, tc=True, one_draw=True)
    before = a.state_download(MAX_GPT)
    E = pkg.EngineError
    for rows, pf in ((0, 16), (MAX_GPT + 1, 16), (4, 0), (4, 2049)):
        with pytest.raises(E):
            a.batcher(rows, pf)
    a.set_option("prefill", 0)
    with pytest.raises(E, match="prefill"):
        a.batcher(4, 16)
    a.set_option("prefill", 1)
    with a.batcher(4, 16) as bat:
        with pytest.raises(E, match="already has an open batcher"):
            a.batcher(4, 16)
        rid = bat.submit(3, [1, 2, 3], 8)
        S = pkg.Sampler
        bad = [dict(slot=MAX_GPT, prompt=[1], max_new=4), dict(slot=3, prompt=[1], max_new=4),
               dict(slot=4, prompt=[V], max_new=4), dict(slot=4, prompt=[], max_new=4), dict(slot=4, prompt=[1], max_new=0),
               dict(slot=4, prompt=[1], max_new=4, stop=(V,)), dict(slot=4, prompt=[1], max_new=4, sampling=S(top_p=0.0)),
               dict(slot=4, prompt=[1], max_new=4, sampling=S(temperature=1.0)),
               dict(slot=4, prompt=[1], max_new=2, sampling=S(temperature=1.0), u=[0.5, 1.0])]
        for kw in bad:
            with pytest.raises(E):
                bat.submit(**kw)
        for call in (bat.read, bat.cancel, bat.release):
            with pytest.raises(E, match="unknown"):
                call(rid + 100)
        with pytest.raises(E, match="not ended"):
            bat.release(rid)
        bat.cancel(rid)  # queued: its slot stays untouched
        with pytest.raises(E, match="already ended"):
            bat.cancel(rid)
        bat.release(rid)
        assert bat.run(16) == 0
    after = a.state_download(MAX_GPT)
    for k in KEYS5:
        assert np.array_equal(before[k], after[k]), k
    a.close()
