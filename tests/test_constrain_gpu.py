"""rwkv_b200_generate_streams_constrained: token automata mask every step's logits on the device and end streams on
completion.

Generation is compared with the host loop it replaces, on a second engine from the same state and on the same forward
path: forward_streams logits, the penalties in numpy float32, the overrides, then the numpy mask row[~allowed] = -inf,
sample_streams(logits=...) with the same u, append, the automaton advance, and the stop on a stop token, the budget or
a state without edges. That loop is exact, so tokens, lengths, final states and every named slot must match bit for
bit, and slots the call does not name must not change."""
import ctypes
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

V = 50277
KEYS = ("xy", "aa", "bb", "dd")
SHAPES = [(3, 768), (2, 2048)]
FIELDS = ("logprobs", "ranks", "top_tokens", "top_logprobs")
REGEXES = {
    "date": r"\d{4}-\d{2}-\d{2}",
    "labels": r"positive|negative|neutral",
    "json": r'\{"name": "[a-z]{1,12}", "age": \d{1,3}\}',
    "number": r"-?\d+(\.\d+)?",
}
OVERRIDES = {11: 3.0, 187: -99.0, 50: -np.inf}


@pytest.fixture(scope="module")
def C(pkg):
    return pkg.constrain


@pytest.fixture(scope="module")
def tbytes(C):
    return C.token_bytes()


@pytest.fixture(scope="module")
def autos(C, tbytes):
    return {k: C.token_automaton(C.compile_regex(p), tbytes, eos=0) for k, p in REGEXES.items()}


_ALLOWED = {}


def allowed(ta, q):
    key = (id(ta), q)
    if key not in _ALLOWED:
        a = np.zeros(V, bool)
        a[ta.edges(q)[0].astype(np.int64)] = True
        _ALLOWED[key] = a
    return _ALLOWED[key]


def rand_tokens(n, seed):
    return [int(x) for x in np.random.default_rng(seed).integers(0, V, size=n)]


def slot_of(state, slot, n):
    return {k: state[k][slot * n:(slot + 1) * n] for k in state}


def engines(pkg, path, max_gpt, tc, seed=99):
    """(a, b): a generates, b runs the host loop on the same forward path, both from the same non-trivial state."""
    a = pkg.Engine(path, max_gpt=max_gpt)
    b = pkg.Engine(path, max_gpt=max_gpt)
    if tc:
        b.set_option("prefill_min", 2)  # the loop's calls shrink below 8 streams as streams finish
    else:
        a.set_option("prefill", 0)
        b.set_option("prefill", 0)
    for i in range(0, max_gpt, 128):
        n = min(128, max_gpt - i)
        a.forward_streams([(i + j, [t]) for j, t in enumerate(rand_tokens(n, seed + i))], want_logits=False)
    b.state_upload(a.state_download(max_gpt), max_gpt)
    return a, b


def check_slots(a, b, before, streams, max_gpt):
    n = a.n_layers * a.n_embed
    sa, sb = a.state_download(max_gpt), b.state_download(max_gpt)
    named = {slot for slot, _ in streams}
    for slot in range(max_gpt):
        if slot in named:
            for k in KEYS:
                assert np.array_equal(slot_of(sa, slot, n)[k], slot_of(sb, slot, n)[k]), "slot %d state %s" % (slot, k)
        else:
            for k in ("xy", "aa", "bb", "pp", "dd"):
                assert np.array_equal(slot_of(sa, slot, n)[k], slot_of(before, slot, n)[k]), "slot %d was touched" % slot


def mixed_samplers(pkg, S):
    """Greedy and sampled streams, penalties with decay < 1 and = 1, cuts by top-p and top-k."""
    Sm = pkg.Sampler
    kinds = [Sm(1.0, 0.85, 0, 0.2, 0.2, 0.996), Sm(0.0), Sm(0.8, 1.0, 40, 0.5, 0.0, 1.0), Sm(1.0, 0.85),
             Sm(0.0, 1.0, 0, 1.0, 0.3, 0.9), Sm(1.2, 0.95, 100, 0.0, 0.4, 1.0), Sm(0.0, 1.0, 0, 0.3, 0.0, 1.0)]
    return [kinds[s % len(kinds)] for s in range(S)]


def host_loop(pkg, eng, streams, max_new, samplers, u, budgets, stop, overrides, cons, pad_slot=None, rows_out=None):
    """The exact host loop; cons[s] = (automaton, start state) or None. Returns (tokens, final states). rows_out, when
    given, receives every (stream, masked row) in step order."""
    S = len(streams)
    budgets = list(budgets) if budgets is not None else [max_new] * S
    cnt = [np.zeros(V, np.float32) for _ in range(S)]
    seen = [np.zeros(V, bool) for _ in range(S)]
    pen = [sp.presence_penalty != 0 or sp.frequency_penalty != 0 for sp in samplers]
    cur = [int(t) for _, t in streams]
    state = [c[1] if c else None for c in cons]
    out = [[] for _ in range(S)]
    live = list(range(S))
    for step in range(max_new):
        if not live:
            break
        call = [(streams[s][0], [cur[s]]) for s in live]
        if pad_slot is not None and len(call) == 1:
            call.append((pad_slot, [cur[live[0]]]))
        logits, _ = eng.forward_streams(call)
        ps, us = [], []
        for i, s in enumerate(live):
            sp, row = samplers[s], logits[i]
            if pen[s]:
                k = seen[s]
                row[k] = row[k] - (np.float32(sp.presence_penalty) + np.float32(sp.frequency_penalty) * cnt[s][k])
            for tok, val in (overrides or {}).items():
                row[tok] = val
            if cons[s]:
                row[~allowed(cons[s][0], state[s])] = -np.inf
            if rows_out is not None:
                rows_out.append((s, row.copy()))
            ps.append(pkg.Sampler(sp.temperature, sp.top_p, sp.top_k))
            us.append(float(u[step][s]) if u is not None else 0.0)
        if len(call) > len(live):
            ps.append(pkg.Sampler(0.0))
            us.append(0.0)
        toks, _ = eng.sample_streams(ps, us, logits=logits)
        ended = set()
        for i, s in enumerate(live):
            x = int(toks[i])
            out[s].append(x)
            cur[s] = x
            if pen[s]:
                cnt[s] = cnt[s] * np.float32(samplers[s].penalty_decay)
                cnt[s][x] += np.float32(1.0)
                seen[s][x] = True
            if cons[s]:
                state[s] = cons[s][0].walk([x], state[s])
                assert state[s] is not None, "the host loop picked a masked token"
                if cons[s][0].complete(state[s]):
                    ended.add(s)
        live = [s for s in live if len(out[s]) < budgets[s] and out[s][-1] not in stop and s not in ended]
    return out, state


def stops_at(seqs, targets):
    stop = []
    for j, t in targets.items():
        seq = seqs[j]
        fresh = [i for i in range(t, len(seq)) if seq[i] not in seq[:i]]
        if fresh:
            stop.append(seq[fresh[0]])
    return stop


def prefix_state(ta, tbytes, text):
    """The state after the shortest token spelling of `text` (one token per byte where needed)."""
    ids = []
    for ch in text.encode():
        ids.append([t for t in range(2, V) if tbytes[t] == bytes([ch])][0])
    q = ta.walk(ids)
    assert q is not None
    return q


# -- 1. bit for bit against the host loop ----------------------------------------------------------------------------

def spec_for(autos, tbytes, S):
    """Per stream: date / unconstrained / labels / json / date from a non-zero start / number, in turn."""
    kinds = ["date", None, "labels", "json", "date+", "number"]
    cons, ids_key = [], []
    for s in range(S):
        k = kinds[s % len(kinds)]
        if k is None:
            cons.append(None)
        elif k == "date+":
            cons.append((autos["date"], prefix_state(autos["date"], tbytes, "2024-")))
        else:
            cons.append((autos[k], 0))
        ids_key.append(k)
    return cons, ids_key


def ids_of(eng, autos, cons):
    reg = {}
    out = []
    for c in cons:
        if c is None:
            out.append(None)
            continue
        key = id(c[0])
        if key not in reg:
            reg[key] = eng.add_constraint(c[0])
        out.append((reg[key], c[1]))
    return out


def against_host_loop(pkg, make_model, autos, tbytes, L, E, S, max_gpt, max_new, tc, greedy_only=False):
    a, b = engines(pkg, make_model(L, E), max_gpt, tc=tc)
    streams = [(s, t) for s, t in zip([(7 * i + 2) % (max_gpt - 1) for i in range(S)], rand_tokens(S, 21))]  # pad: max_gpt - 1
    samplers = [pkg.Sampler(0.0)] * S if greedy_only else mixed_samplers(pkg, S)
    u = np.random.default_rng(22).random((max_new, S))
    budgets = [max_new - (5 * i) % 23 for i in range(S)]
    cons, _ = spec_for(autos, tbytes, S)
    ids = ids_of(a, autos, cons)
    st = a.state_download(max_gpt)
    first = a.generate_streams(streams, max_new, overrides=OVERRIDES, u=u, sampling=samplers, constraints=ids)
    a.state_upload(st, max_gpt)
    stop = stops_at([[int(x) for x in r["tokens"]] for r in first], {1: 9})  # a stop in an unconstrained stream
    got = a.generate_streams(streams, max_new, budgets=budgets, stop=stop, overrides=OVERRIDES, u=u, sampling=samplers,
                             constraints=ids)
    want, states = host_loop(pkg, b, streams, max_new, samplers, u, budgets, stop, OVERRIDES, cons,
                             pad_slot=max_gpt - 1 if tc else None)
    assert [len(g["tokens"]) for g in got] == [len(w) for w in want], "lengths"
    for s, (g, w) in enumerate(zip(got, want)):
        assert [int(x) for x in g["tokens"]] == w, "tokens of stream %d" % s
        assert g["state"] == states[s], "state of stream %d" % s
    check_slots(a, b, st, streams, max_gpt)
    completed = [s for s in range(S) if cons[s] and cons[s][0].complete(states[s])]
    assert completed and any(len(want[s]) % 16 for s in completed), "no stream completed mid-group"
    a.close()
    b.close()
    return got


@pytest.mark.parametrize("L,E", SHAPES)
@pytest.mark.parametrize("tc", [False, True])
def test_against_the_host_loop(pkg, make_model, autos, tbytes, L, E, tc):
    """Mixed samplers with penalties, overrides, constrained and unconstrained streams, four automata, a non-zero start
    state, budgets and a stop token. S = 6 on the decode kernel, S = 12 on the tensor cores."""
    against_host_loop(pkg, make_model, autos, tbytes, L, E, 12 if tc else 6, 16, 40, tc)


def test_150_streams(pkg, make_model, autos, tbytes):
    against_host_loop(pkg, make_model, autos, tbytes, 3, 768, 150, 256, 24, True)


# -- 2. validity -----------------------------------------------------------------------------------------------------

def test_every_sequence_walks_and_completed_ones_match(pkg, make_model, autos, tbytes):
    S, max_new = 32, 64
    a = pkg.Engine(make_model(3, 768), max_gpt=S)
    names = list(REGEXES)
    ids = {k: a.add_constraint(autos[k]) for k in names}
    streams = list(zip(range(S), rand_tokens(S, 5)))
    samplers = [pkg.Sampler(0.0) if s % 3 == 0 else pkg.Sampler(1.0, 0.9) for s in range(S)]
    u = np.random.default_rng(6).random((max_new, S))
    got = a.generate_streams(streams, max_new, u=u, sampling=samplers, constraints=[ids[names[s % 4]] for s in range(S)])
    done = 0
    for s, g in enumerate(got):
        name = names[s % 4]
        ta, toks = autos[name], [int(x) for x in g["tokens"]]
        q = ta.walk(toks)
        assert q is not None and q == g["state"], (name, toks)
        if ta.complete(q):
            assert toks[-1] == 0 and q == ta.sink
            text = b"".join(tbytes[t] for t in toks[:-1])
            assert re.fullmatch(REGEXES[name].encode(), text), (name, text)
            done += 1
        else:
            assert len(toks) == max_new
    assert done >= 8
    a.close()


# -- 3. no side effects ----------------------------------------------------------------------------------------------

def raw_call(eng, streams, max_new, samplers, u, ids=None, starts=None):
    """rwkv_b200_generate_streams_constrained with no log-probabilities: (tokens, lengths, states)."""
    P, D = ctypes.POINTER(ctypes.c_ulonglong), ctypes.POINTER(ctypes.c_double)
    S = len(streams)
    arr = lambda a: np.ascontiguousarray(a, np.uint64)
    slots, first = arr([s for s, _ in streams]), arr([t for _, t in streams])
    sp = (type(samplers[0]) * S)(*samplers)
    us = np.ascontiguousarray(u, np.float64)
    out, lens, states = np.zeros((S, max_new), np.uint64), np.zeros(S, np.uint64), np.zeros(S, np.uint64)
    ptr = lambda a, t=P: a.ctypes.data_as(t) if a is not None else None
    rc = eng.lib.rwkv_b200_generate_streams_constrained(
        eng.h, ptr(slots), ptr(first), S, max_new, None, None, 0, None, None, 0, sp, ptr(us, D), ptr(out), ptr(lens),
        7, 99, None, None, None, None, ptr(arr(ids) if ids is not None else None),
        ptr(arr(starts) if starts is not None else None), ptr(states))
    assert rc == 0, eng.lib.rwkv_b200_last_error()
    return out, lens, states


@pytest.mark.parametrize("tc", [False, True])
def test_no_side_effects(pkg, make_model, C, tc):
    """NULL constraints without log-probabilities (logprob_mode and top_n are not read then), and a one-state automaton
    that allows every token, are generate_streams_ex: the same tokens and slot states."""
    max_gpt, max_new = 12, 32
    S = 10 if tc else 3
    a, b = engines(pkg, make_model(3, 768), max_gpt, tc=tc)
    streams = list(zip(range(S), rand_tokens(S, 31)))
    samplers = mixed_samplers(pkg, S)
    u = np.random.default_rng(32).random((max_new, S))
    st = a.state_download(max_gpt)
    want = b.generate_streams(streams, max_new, u=u, sampling=samplers)
    cid = a.add_constraint(C.allow_all())
    for ids in (None, [cid] * S):
        a.state_upload(st, max_gpt)
        out, lens, states = raw_call(a, streams, max_new, samplers, u, ids=ids)
        assert [int(x) for x in lens] == [len(w) for w in want]
        for s, w in enumerate(want):
            assert np.array_equal(out[s, :len(w)], w) and not out[s, len(w):].any()
        assert not states.any()
        check_slots(a, b, st, streams, max_gpt)
    a.close()
    b.close()


def test_two_calls_continued_equal_one(pkg, make_model, autos):
    """Without penalties, a call of 5 steps continued by one of 27 from each stream's last token and final state equals
    one call of 32 steps."""
    S, n1, n2 = 10, 5, 27
    a = pkg.Engine(make_model(2, 2048), max_gpt=S)
    a.set_option("prefill", 0)  # the continuing call has fewer streams: keep both on one forward path
    Sm = pkg.Sampler
    samplers = [Sm(0.0) if s % 2 else Sm(1.0, 0.9, 50) for s in range(S)]
    streams = list(zip(range(S), rand_tokens(S, 41)))
    u = np.random.default_rng(42).random((n1 + n2, S))
    cid = a.add_constraint(autos["json"])
    st = a.state_download(S)
    one = a.generate_streams(streams, n1 + n2, u=u, sampling=samplers, constraints=cid)
    s_one = a.state_download(S)
    a.state_upload(st, S)
    part = a.generate_streams(streams, n1, u=u[:n1], sampling=samplers, constraints=cid)
    cont = [s for s in range(S) if len(part[s]["tokens"]) == n1 and not autos["json"].complete(part[s]["state"])]
    assert len(cont) >= 5
    rest = a.generate_streams([(s, int(part[s]["tokens"][-1])) for s in cont], n2, u=u[n1:, cont],
                              sampling=[samplers[s] for s in cont], constraints=[(cid, part[s]["state"]) for s in cont])
    for s in range(S):
        toks = [int(x) for x in part[s]["tokens"]]
        state = part[s]["state"]
        if s in cont:
            r = rest[cont.index(s)]
            toks += [int(x) for x in r["tokens"]]
            state = r["state"]
        assert toks == [int(x) for x in one[s]["tokens"]] and state == one[s]["state"], s
    s_two = a.state_download(S)
    for k in s_one:
        assert np.array_equal(s_one[k], s_two[k]), k
    a.close()


# -- 4. log-probabilities --------------------------------------------------------------------------------------------

def bits(x):
    return np.ascontiguousarray(x).tobytes()


@pytest.mark.parametrize("tc", [False, True])
def test_raw_logprobs_equal_score_streams(pkg, make_model, autos, tbytes, tc):
    max_gpt, max_new = 12, 32
    S = 10 if tc else 3
    a, b = engines(pkg, make_model(3, 768), max_gpt, tc=tc)
    streams = list(zip([(5 * i + 2) % (max_gpt - 1) for i in range(S)], rand_tokens(S, 51)))
    samplers = mixed_samplers(pkg, S)
    u = np.random.default_rng(52).random((max_new, S))
    cons, _ = spec_for(autos, tbytes, S)
    st = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, overrides=OVERRIDES, u=u, sampling=samplers, constraints=ids_of(a, autos, cons),
                             logprobs="raw", top_n=20)
    pad = max_gpt - 1 if tc else None
    cur = [t for _, t in streams]
    lens = [len(g["tokens"]) for g in got]
    for k in range(max(lens)):
        live = [s for s in range(S) if lens[s] > k]
        call = [(streams[s][0], [cur[s]]) for s in live]
        tg = [[int(got[s]["tokens"][k])] for s in live]
        if pad is not None and len(call) == 1:
            call.append((pad, [cur[live[0]]]))
            tg.append([None])
        res = b.score_streams(call, tg, top_n=20)
        for i, s in enumerate(live):
            for f in FIELDS:
                assert bits(res[i][f][0]) == bits(got[s][f][k]), (s, k, f)
            cur[s] = int(got[s]["tokens"][k])
    check_slots(a, b, st, streams, max_gpt)
    a.close()
    b.close()


def rule(row, y, tau, top_n):
    l = np.asarray(row, np.float32).astype(np.float64)
    with np.errstate(invalid="ignore"):
        z = (l - l.max()) / tau
    log_s = np.log(np.exp(z).sum())
    order = np.lexsort((np.arange(V), -l))
    rank = int(np.nonzero(order == y)[0][0])
    top = order[:top_n]
    return z[y] - log_s, rank, top, z[top] - log_s


def close(a, b):
    a, b = np.asarray(a), np.asarray(b)
    inf = np.isinf(b)
    return np.array_equal(a[inf], b[inf]) and (not (~inf).any() or np.max(np.abs(a[~inf] - b[~inf])) <= 1e-9)


@pytest.mark.parametrize("tc", [False, True])
def test_processed_logprobs_on_the_masked_rows(pkg, make_model, autos, tbytes, tc):
    max_gpt, max_new, top_n = 12, 24, 20
    S = 9 if tc else 4
    a, b = engines(pkg, make_model(2, 2048), max_gpt, tc=tc)
    streams = list(zip([(3 * i + 1) % (max_gpt - 1) for i in range(S)], rand_tokens(S, 61)))
    samplers = mixed_samplers(pkg, S)
    u = np.random.default_rng(62).random((max_new, S))
    cons = [(autos["labels"], 0) if s % 2 else (autos["date"], 0) for s in range(S)]
    cons[-1] = None
    got = a.generate_streams(streams, max_new, overrides=OVERRIDES, u=u, sampling=samplers,
                             constraints=ids_of(a, autos, cons), logprobs="processed", top_n=top_n)
    rows = []
    want, _ = host_loop(pkg, b, streams, max_new, samplers, u, None, (), OVERRIDES, cons,
                        pad_slot=max_gpt - 1 if tc else None, rows_out=rows)
    assert [[int(x) for x in g["tokens"]] for g in got] == want
    k_of = [0] * S
    masked_tops = 0
    for s, row in rows:
        k = k_of[s]
        k_of[s] += 1
        g, sp = got[s], samplers[s]
        y = int(g["tokens"][k])
        tau = float(np.float32(sp.temperature)) if sp.temperature > 0 else 1.0
        lp, rank, top, top_lp = rule(row, y, tau, top_n)
        assert int(g["ranks"][k]) == rank, (s, k)
        assert abs(g["logprobs"][k] - lp) <= 1e-9, (s, k)
        assert [int(x) for x in g["top_tokens"][k]] == [int(x) for x in top], (s, k)
        assert close(g["top_logprobs"][k], top_lp), (s, k)
        masked_tops += int(np.sum(g["top_logprobs"][k] == -np.inf))
    assert masked_tops > 0  # the labels' first states allow fewer than 20 tokens
    a.close()
    b.close()


# -- 5. refusals -----------------------------------------------------------------------------------------------------

def test_refusals_leave_every_slot_untouched(pkg, make_model, autos, C):
    path = make_model(2, 768)
    a = pkg.Engine(path, max_gpt=8)
    a.forward_streams([(s, [5 + s]) for s in range(8)], want_logits=False)
    before = a.state_download(8)
    T = C.TokenAutomaton
    bad_add = [
        (T([0], [], []), "n_states = 0 is outside 1..65536"),
        (T(np.zeros(65538, np.int64), [], []), "n_states = 65537 is outside"),
        (T([1, 1], [], []), "edge_start[0] = 1, not 0"),
        (T([0, 2, 1], [3, 4], [0, 1]), "edge_start decreases from state 1 to 2"),
        (T([0, 1], [V], [0]), "state 0: edge token 50277 out of range"),
        (T([0, 2], [7, 5], [0, 0]), "state 0: edge tokens are not strictly ascending (5 after 7)"),
        (T([0, 2], [5, 5], [0, 0]), "not strictly ascending (5 after 5)"),
        (T([0, 1, 1], [5], [2]), "edge of token 5 leads to state 2 >= n_states 2"),
    ]
    for ta, msg in bad_add:
        with pytest.raises(pkg.EngineError, match=re.escape(msg)):
            a.add_constraint(ta)
    labels = a.add_constraint(autos["labels"])
    gone = a.add_constraint(autos["date"])
    a.remove_constraint(gone)
    with pytest.raises(pkg.EngineError, match="constraint id %d is unknown or removed" % gone):
        a.remove_constraint(gone)
    ok = [(0, 5), (3, 6)]
    Sm = pkg.Sampler
    sink = autos["labels"].sink
    first_edges = {int(t): -np.inf for t in autos["labels"].edges(0)[0]}
    bad_gen = [
        (dict(constraints=[labels, 999]), "stream 1: constraint id 999 is unknown or removed"),
        (dict(constraints=[gone, labels]), "stream 0: constraint id %d is unknown or removed" % gone),
        (dict(constraints=[(labels, autos["labels"].n_states), None]), "stream 0: start state %d of constraint %d is out of range"
         % (autos["labels"].n_states, labels)),
        (dict(constraints=[None, (labels, sink)]), "stream 1: start state %d of constraint %d has no edges" % (sink, labels)),
        (dict(constraints=labels, overrides=first_edges), "the overrides set every edge token of state 0 of constraint %d to -inf"
         % labels),
        (dict(constraints=labels, logprobs="raw", top_n=21), "generate_streams_constrained: top_n 21 > 20"),
        (dict(constraints=labels, budgets=[4, 0]), "generate_streams_constrained: budget 0 of stream 1"),
        (dict(constraints=labels, sampling=[Sm(0.0), Sm(1.0)]), "u is NULL but stream 1 samples"),
        (dict(constraints=[labels] * 3), "3 constraints for 2 streams"),
        (dict(constraints=labels, u=[[0.5, 0.5]] * 4, sampling=None), "constraints need sampling"),
        (dict(constraints=labels, temp=0.7, sampling=None), "constraints need sampling"),
    ]
    for kw, msg in bad_gen:
        args = dict(sampling=Sm(0.0))
        args.update(kw)
        with pytest.raises(pkg.EngineError, match=re.escape(msg)):
            a.generate_streams(ok, 4, **args)
    after = a.state_download(8)
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    # the refusals changed nothing: the same call now runs
    res = a.generate_streams(ok, 4, sampling=Sm(0.0), constraints=[labels, None])
    assert autos["labels"].walk([int(x) for x in res[0]["tokens"]]) == res[0]["state"]
    a.close()
    t = pkg.Engine(path, max_gpt=4, tp_rank=0, tp_size=2)
    with pytest.raises(pkg.EngineError, match="constraint_add: not supported with tensor parallelism"):
        t.add_constraint(autos["labels"])
    with pytest.raises(pkg.EngineError, match="not supported with tensor parallelism"):
        t.generate_streams([(0, 5)], 4, sampling=Sm(0.0), constraints=[None])
    t.close()
