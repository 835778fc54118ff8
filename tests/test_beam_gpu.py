"""Device-resident beam search (rwkv_b200_beam_search) against the host loop of its rule.

The oracle is a second engine that starts from the same state and runs, through the existing API and on the same forward
path, the rule of include/rwkv_b200.h: per step, score_streams on every live beam's one token with top_n = B + n_stop
(the top entries are bit for bit what logprob_row gives the device), the sort, the walk, the hypothesis list and the done
bound in Python floats with the device's operation order, and slot_copy for each fork by the slot rule. Hypotheses and
every named slot must match bit for bit; slots the call does not name must not change at all."""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

V = 50277
KEYS = ("xy", "aa", "bb", "pp", "dd")
SHAPES = [(3, 768), (2, 2048)]


def rand_tokens(n, seed):
    return [int(x) for x in np.random.default_rng(seed).integers(0, V, size=n)]


def slot_of(state, slot, n):
    return {k: state[k][slot * n:(slot + 1) * n] for k in state}


def engines(pkg, path, max_gpt, tc, seed=99):
    """(a, b): a runs beam_search, b the host loop on the same path, both from the same non-trivial state. tc: both take
    the tensor cores down to 2 rows (the loop's pad keeps a lone row there), else both the decode kernel."""
    a = pkg.Engine(path, max_gpt=max_gpt)
    b = pkg.Engine(path, max_gpt=max_gpt)
    for e in (a, b):
        e.set_option("prefill_min", 2) if tc else e.set_option("prefill", 0)
    for i in range(0, max_gpt, 128):
        n = min(128, max_gpt - i)
        a.forward_streams([(i + j, [t]) for j, t in enumerate(rand_tokens(n, seed + i))], want_logits=False)
    b.state_upload(a.state_download(max_gpt), max_gpt)
    return a, b


def offer(hyps, K, h):
    """The hypothesis list: K best by (score descending, offer order ascending); strictly above the worst to enter."""
    if len(hyps) == K and not h["score"] > hyps[-1]["score"]:
        return
    if len(hyps) == K:
        hyps.pop()
    i = len(hyps)
    while i > 0 and hyps[i - 1]["score"] < h["score"]:
        i -= 1
    hyps.insert(i, h)


def host_beam(eng, groups, max_new, B, stop=(), alpha=1.0, K=1, pad_slot=None, log=None):
    """The rule of rwkv_b200_beam_search as a host loop on `eng`. log: a dict that receives the steps at which finished
    hypotheses were offered ("offers") and the step after which each group was done ("done_at")."""
    N, C, stops = max_new, B + len(stop), set(int(s) for s in stop)
    P = [0.0] + [math.pow(float(n), alpha) for n in range(1, N + 1)]
    offers = []
    st = [dict(slots=[int(s) for s in slots], beams=[dict(slot=int(slots[0]), tok=int(first), cum=0.0, toks=[], lps=[])],
               hyps=[], done=False) for slots, first in groups]
    for step in range(N):
        live = [g for g in st if not g["done"]]
        if not live:
            break
        call = [(bm["slot"], [bm["tok"]]) for g in live for bm in g["beams"]]
        if pad_slot is not None and len(call) == 1:
            call.append((pad_slot, [call[0][1][0]]))
        res = eng.score_streams(call, targets=[[0]] * len(call), top_n=C)
        r = 0
        for g in live:
            cands = []
            for b, bm in enumerate(g["beams"]):
                tt, tl = res[r]["top_tokens"][0], res[r]["top_logprobs"][0]
                r += 1
                for i in range(C):
                    cands.append((bm["cum"] + float(tl[i]), b, i, int(tt[i]), float(tl[i])))
            cands.sort(key=lambda x: (-x[0], x[1], x[2]))
            prev, new = g["beams"], []
            for pos, (c, b, i, tok, lp) in enumerate(cands):
                if len(new) == B:
                    break
                if tok in stops:
                    if pos < B:
                        offers.append(step)
                        offer(g["hyps"], K, dict(score=c / P[step + 1], cum=c, toks=prev[b]["toks"] + [tok],
                                                 lps=prev[b]["lps"] + [lp], finished=True))
                    continue
                new.append((b, tok, lp, c))
            if step + 1 == N:
                for b, tok, lp, c in new:
                    offer(g["hyps"], K, dict(score=c / P[N], cum=c, toks=prev[b]["toks"] + [tok], lps=prev[b]["lps"] + [lp],
                                             finished=False))
                done = True
            else:
                Pb = P[step + 2] if alpha < 0 else P[N]
                done = len(g["hyps"]) == K and all(c / Pb <= g["hyps"][-1]["score"] for _, _, _, c in new)
            prev_slots = [bm["slot"] for bm in prev] if step > 0 else g["slots"]
            child = {b for b, _, _, _ in new}
            free = [p for p in range(B) if p not in child]
            taken, beams = set(), []
            for b, tok, lp, c in new:
                if b not in taken:
                    taken.add(b)
                    slot = prev_slots[b]
                else:
                    slot = prev_slots[free.pop(0)]
                    if not done:
                        eng.slot_copy(prev_slots[b], slot)
                beams.append(dict(slot=slot, tok=tok, cum=c, toks=prev[b]["toks"] + [tok], lps=prev[b]["lps"] + [lp]))
            g["beams"], g["done"], g["done_at"] = beams, done, step
    if log is not None:
        log["offers"], log["done_at"] = offers, [g["done_at"] for g in st]
    return [g["hyps"] for g in st]


def check(a, b, before, groups, got, want, max_gpt, what=""):
    assert len(got) == len(want)
    for gi, (gh, wh) in enumerate(zip(got, want)):
        assert len(gh) == len(wh), what + ": group %d holds %d hypotheses, expected %d" % (gi, len(gh), len(wh))
        for i, (x, y) in enumerate(zip(gh, wh)):
            tag = what + ": group %d hypothesis %d" % (gi, i)
            assert [int(t) for t in x["tokens"]] == y["toks"], tag + ": tokens"
            assert x["logprob"] == y["cum"] and x["score"] == y["score"], tag + ": logprob / score"
            assert x["finished"] == y["finished"], tag + ": finished"
            assert [float(v) for v in x["token_logprobs"]] == y["lps"], tag + ": token logprobs"
    n = a.n_layers * a.n_embed
    sa, sb = a.state_download(max_gpt), b.state_download(max_gpt)
    named = {int(s) for slots, _ in groups for s in slots}
    for slot in range(max_gpt):
        for k in KEYS:
            if slot in named:
                assert np.array_equal(slot_of(sa, slot, n)[k], slot_of(sb, slot, n)[k]), what + ": slot %d state %s" % (slot, k)
            else:
                assert np.array_equal(slot_of(sa, slot, n)[k], slot_of(before, slot, n)[k]), what + ": slot %d was touched" % slot


def make_groups(G, B, max_gpt, seed):
    perm = [int(x) for x in np.random.default_rng(seed).permutation(max_gpt)]
    return [(perm[g * B:(g + 1) * B], t) for g, t in zip(range(G), rand_tokens(G, seed + 1))], perm[G * B:]


def stops_from(hyps, at):
    """Stop tokens from a run without stops: the token of group j's best hypothesis at position at[j] (a token that
    hypothesis has not emitted before), so that groups finish near different steps."""
    stop = []
    for j, t in at.items():
        toks = [int(x) for x in hyps[j][0]["tokens"]]
        fresh = [i for i in range(t, len(toks)) if toks[i] not in toks[:i] and toks[i] not in stop]
        if fresh:
            stop.append(toks[fresh[0]])
    return stop


def scored_like_hypotheses(eng, prompt, spare, first, hyps, n):
    """score_streams of first + each hypothesis from the prompt state on a spare slot, the whole text in one call."""
    for h in hyps:
        eng.slot_upload(spare, prompt)
        text = [int(first)] + [int(t) for t in h["tokens"]]
        got = eng.score_streams([(spare, text)])[0]["logprobs"][:-1]
        assert [float(v) for v in got] == [float(v) for v in h["token_logprobs"]], "scoring differs from the beam's logprobs"
        s = 0.0
        for v in got:
            s += float(v)
        assert s == h["logprob"], "the left-to-right sum of the token logprobs is not the hypothesis' logprob"


# (G, B, K, alpha, stops, tc)
CASES = [
    (1, 4, 1, 1.0, False, False),
    (5, 4, 4, 2.0, True, True),
    (33, 4, 2, -0.5, True, True),
    (3, 2, 2, 0.0, True, False),
    (2, 8, 8, 1.0, False, True),
    (6, 1, 1, 1.0, True, True),
]


@pytest.mark.parametrize("L,E", SHAPES)
@pytest.mark.parametrize("G,B,K,alpha,with_stops,tc", CASES)
def test_bit_exact_against_the_host_loop(pkg, make_model, L, E, G, B, K, alpha, with_stops, tc):
    """Hypotheses, their per-token logprobs and every named slot bit for bit against the host loop; unnamed slots
    untouched. Stop tokens come from a run without them, so that groups finish at different steps, across the 16-step
    host groups (max_new = 40)."""
    max_new = 40
    max_gpt = max(G * B + 2, max_new + 1)  # a spare slot pads the loop's lone rows, another scores whole texts
    a, b = engines(pkg, make_model(L, E), max_gpt, tc)
    groups, spare = make_groups(G, B, max_gpt, seed=G * 10 + B)
    stop = []
    if with_stops:
        st = a.state_download(max_gpt)
        free_run = a.beam_search(groups, max_new, B, length_penalty=alpha, n_best=1)
        a.state_upload(st, max_gpt)
        stop = stops_from(free_run, {j % G: t for j, t in enumerate([4, 18, 33])})[:20 - B]
    before = a.state_download(max_gpt)
    got = a.beam_search(groups, max_new, B, stop=stop, length_penalty=alpha, n_best=K, token_logprobs=True)
    log = {}
    want = host_beam(b, groups, max_new, B, stop=stop, alpha=alpha, K=K, pad_slot=spare[0] if tc else None, log=log)
    if with_stops:
        assert log["offers"], "no stop token was offered as a finished hypothesis"
    print("G=%d B=%d K=%d alpha=%g: finished offers at steps %s, groups done after steps %s"
          % (G, B, K, alpha, sorted(set(log["offers"])), log["done_at"]))
    check(a, b, before, groups, got, want, max_gpt, "G=%d B=%d K=%d alpha=%g" % (G, B, K, alpha))
    # every hypothesis is what score_streams reports for its text from the prompt state
    n = a.n_layers * a.n_embed
    for (slots, first), hyps in zip(groups, got):
        scored_like_hypotheses(a, slot_of(before, slots[0], n), spare[1], first, hyps, n)
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", SHAPES)
@pytest.mark.parametrize("tc", [False, True])
def test_one_beam_without_penalty_is_greedy_generation(pkg, make_model, L, E, tc):
    """B = 1 with alpha = 0 emits generate_streams' arg-max tokens, stop tokens included, and leaves the slots where it
    does."""
    max_new, G = 40, 4
    max_gpt = G + 1
    a, b = engines(pkg, make_model(L, E), max_gpt, tc)
    groups = [([s], t) for s, t in zip([3, 0, 2, 1], rand_tokens(G, 5))]
    streams = [(slots[0], t) for slots, t in groups]
    st = a.state_download(max_gpt)
    seqs = [[int(x) for x in s] for s in a.generate_streams(streams, max_new)]
    a.state_upload(st, max_gpt)
    stop = []
    for j, at in enumerate([3, 17, 30]):
        fresh = [i for i in range(at, max_new) if seqs[j][i] not in seqs[j][:i] and seqs[j][i] not in stop]
        stop.append(seqs[j][fresh[0]])
    got = a.beam_search(groups, max_new, 1, stop=stop, length_penalty=0.0)
    want = b.generate_streams(streams, max_new, stop=stop)
    assert [[int(t) for t in hs[0]["tokens"]] for hs in got] == [[int(t) for t in w] for w in want]
    assert [hs[0]["finished"] for hs in got] == [int(w[-1]) in stop for w in want]
    n = a.n_layers * a.n_embed
    sa, sb = a.state_download(max_gpt), b.state_download(max_gpt)
    for slots, _ in groups:
        for k in KEYS:
            assert np.array_equal(slot_of(sa, slots[0], n)[k], slot_of(sb, slots[0], n)[k]), "slot %d %s" % (slots[0], k)
    a.close()
    b.close()


def test_groups_are_independent(pkg, make_model):
    """A group's hypotheses are the same alone as among 32 other groups (both on the tensor cores)."""
    G, B, max_new = 33, 4, 24
    max_gpt = G * B
    a, _ = engines(pkg, make_model(3, 768), max_gpt, tc=True)
    groups, _ = make_groups(G, B, max_gpt, seed=5)
    st = a.state_download(max_gpt)
    seen = a.beam_search(groups, max_new, B, stop=[0, 11], length_penalty=1.0, n_best=3, token_logprobs=True)
    for j in (0, 17, 32):
        a.state_upload(st, max_gpt)
        alone = a.beam_search([groups[j]], max_new, B, stop=[0, 11], length_penalty=1.0, n_best=3, token_logprobs=True)[0]
        for x, y in zip(alone, seen[j]):
            assert [int(t) for t in x["tokens"]] == [int(t) for t in y["tokens"]], "group %d" % j
            assert (x["logprob"], x["score"], x["finished"]) == (y["logprob"], y["score"], y["finished"]), "group %d" % j
            assert np.array_equal(x["token_logprobs"], y["token_logprobs"]), "group %d" % j
    a.close()


def test_rejected_inputs_leave_the_state_untouched(pkg, make_model):
    import ctypes
    path = make_model(2, 768)
    a = pkg.Engine(path, max_gpt=8)
    a.forward(rand_tokens(8, 70), mode=0, want_logits=False)
    before = a.state_download(8)
    ok = [([0, 1], 5), ([2, 3], 6)]
    bad = [
        (dict(groups=[], max_new=4, beams=2), "no groups"),
        (dict(groups=[([], 5)], max_new=4, beams=0), "beams is 0"),
        (dict(groups=ok, max_new=4, beams=2, stop=list(range(19))), r"beams \+ n_stop = 2 \+ 19 > 20"),
        (dict(groups=ok, max_new=4, beams=2, n_best=0), "n_best 0 is outside 1..beams = 2"),
        (dict(groups=ok, max_new=4, beams=2, n_best=3), "n_best 3 is outside 1..beams = 2"),
        (dict(groups=ok, max_new=0, beams=2), "max_new is 0"),
        (dict(groups=[([0, 8], 5)], max_new=4, beams=2), "slot 8 >= max_gpt"),
        (dict(groups=[([0, 1], 5), ([2, 1], 6)], max_new=4, beams=2), "slot 1 appears twice"),
        (dict(groups=[([0, 1], 50277)], max_new=4, beams=2), "first token 50277"),
        (dict(groups=ok, max_new=4, beams=2, stop=[3, 50277]), "stop token 50277"),
        (dict(groups=ok, max_new=4, beams=2, length_penalty=float("nan")), "length_penalty nan is not finite"),
        (dict(groups=ok, max_new=4, beams=2, length_penalty=float("inf")), "length_penalty inf is not finite"),
    ]
    for kw, msg in bad:
        with pytest.raises(pkg.EngineError, match=msg):
            a.beam_search(**kw)
    P = ctypes.POINTER(ctypes.c_ulonglong)
    D = ctypes.POINTER(ctypes.c_double)
    U = ctypes.POINTER(ctypes.c_ubyte)
    slots, first = np.array([0, 1], np.uint64), np.array([5], np.uint64)
    toks, lens = np.zeros(4, np.uint64), np.zeros(1, np.uint64)
    lp, sc, fin = np.zeros(1), np.zeros(1), np.zeros(1, np.uint8)
    args = [slots.ctypes.data_as(P), first.ctypes.data_as(P), 1, 2, 4, None, 0, 1.0, 1, toks.ctypes.data_as(P),
            lens.ctypes.data_as(P), lp.ctypes.data_as(D), sc.ctypes.data_as(D), fin.ctypes.data_as(U), None]
    for i in (0, 1, 9, 10, 11, 12, 13):
        call = list(args)
        call[i] = None
        assert a.lib.rwkv_b200_beam_search(a.h, *call) != 0 and b"null argument" in a.lib.rwkv_b200_last_error()
    call = list(args)
    call[6] = 1  # n_stop = 1, stop_tokens NULL
    assert a.lib.rwkv_b200_beam_search(a.h, *call) != 0 and b"n_stop = 1" in a.lib.rwkv_b200_last_error()
    after = a.state_download(8)
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    # a successful call leaves no per-stream logits behind
    a.forward_streams([(0, [5]), (1, [6])], want_next=True)
    a.beam_search(ok, 3, 2, n_best=2)
    with pytest.raises(pkg.EngineError, match="no per-stream logits"):
        a.sample_typical_streams(1.0, [0.5, 0.5])
    a.close()
    t = pkg.Engine(path, max_gpt=4, tp_rank=0, tp_size=2)
    with pytest.raises(pkg.EngineError, match="not supported with tensor parallelism"):
        t.beam_search([([0, 1], 5)], 4, 2)
    t.close()
