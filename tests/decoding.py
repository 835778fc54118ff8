"""What the GPU decoding tests share: engine pairs from one state, the slot check, the host references of the decoding
calls (the pick chain, the legacy generate loop, the log-probability rule, the score_streams replay), the batcher's
per-request oracle and the regex automata.

A decoding test runs the call under test on engine a and its host reference on engine b, both started from the same
non-trivial state of every slot and on the same forward path. The references are exact, so tokens and named slots
compare bit for bit."""
import numpy as np

from util import REL_TOL, SEED_TOKEN, margin, rel_err

V = 50277
SHAPES = [(3, 768), (2, 2048)]
KEYS4 = ("xy", "aa", "bb", "dd")        # the recurrent state a forward writes
KEYS5 = ("xy", "aa", "bb", "pp", "dd")  # every array of a slot
FIELDS = ("logprobs", "ranks", "top_tokens", "top_logprobs")
NO_TARGET = 2 ** 64 - 1


def rand_tokens(n, seed):
    return [int(x) for x in np.random.default_rng(seed).integers(0, V, size=n)]


def slot_of(state, slot, n):
    return {k: state[k][slot * n:(slot + 1) * n] for k in state}


def bits(x):
    return np.ascontiguousarray(x).tobytes()


def close(a, b):
    """Equal where b is infinite, within 1e-9 elsewhere."""
    a, b = np.asarray(a), np.asarray(b)
    inf = np.isinf(b)
    return np.array_equal(a[inf], b[inf]) and (not (~inf).any() or np.max(np.abs(a[~inf] - b[~inf])) <= 1e-9)


# -- engine pairs and the slot check ---------------------------------------------------------------------------------

def engine_pair(pkg, path, max_gpt, tc, seed=99, a_prefill_min=False, one_draw=False):
    """(a, b): a runs the call under test, b its host reference, both from the same non-trivial state of every slot.
    tc: b takes the tensor cores down to 2 rows, as the reference's calls shrink below 8 streams when streams finish
    (a_prefill_min: a too); else both take the decode kernel. The state is one token per slot, from rand_tokens(n,
    seed + i) per 128 slots i.., or, with one_draw, from one generator of `seed` drawing slot by slot in one call."""
    a = pkg.Engine(path, max_gpt=max_gpt)
    b = pkg.Engine(path, max_gpt=max_gpt)
    if tc:
        for e in (a, b) if a_prefill_min else (b,):
            e.set_option("prefill_min", 2)
    else:
        a.set_option("prefill", 0)
        b.set_option("prefill", 0)
    if one_draw:
        rng = np.random.default_rng(seed)
        a.forward_streams([(j, [int(rng.integers(0, V))]) for j in range(max_gpt)], want_logits=False)
    else:
        for i in range(0, max_gpt, 128):
            n = min(128, max_gpt - i)
            a.forward_streams([(i + j, [t]) for j, t in enumerate(rand_tokens(n, seed + i))], want_logits=False)
    b.state_upload(a.state_download(max_gpt), max_gpt)
    return a, b


def check_slots(a, b, before, max_gpt, named, keys=KEYS4, untouched=KEYS5, skip=(), what=""):
    """Every slot below max_gpt but those in `skip`: a named slot equals b's in `keys`, any other slot equals `before`
    in `untouched`. Returns a's state."""
    n = a.n_layers * a.n_embed
    sa, sb = a.state_download(max_gpt), b.state_download(max_gpt)
    for slot in range(max_gpt):
        if slot in skip:
            continue
        if slot in named:
            for k in keys:
                assert np.array_equal(slot_of(sa, slot, n)[k], slot_of(sb, slot, n)[k]), what + ": slot %d state %s" % (slot, k)
        else:
            for k in untouched:
                assert np.array_equal(slot_of(sa, slot, n)[k], slot_of(before, slot, n)[k]), what + ": slot %d was touched" % slot
    return sa


def check_generated(a, b, before, streams, got, want, max_gpt, what=""):
    """Tokens equal the reference's, named slots b's state, every other slot untouched."""
    assert [len(x) for x in got] == [len(x) for x in want], what + ": lengths"
    for s, (g, w) in enumerate(zip(got, want)):
        assert [int(x) for x in g] == [int(x) for x in w], what + ": tokens of stream %d" % s
    check_slots(a, b, before, max_gpt, {slot for slot, _ in streams}, what=what)


# -- host references of generation -----------------------------------------------------------------------------------

def host_loop(eng, streams, max_new, budgets=None, stop=(), overrides=None, temp=1.0, u=None, pad_slot=None, greedy_api=False):
    """The loop generate_streams stands for, one forward_streams call per step over the live streams, picking through
    forward_greedy (greedy_api), np.argmax of the overridden logits, the device arg-max (want_next) or
    sample_typical_streams with the uniforms u. pad_slot: a spare slot that keeps a lone live stream on the tensor cores
    (rows are independent, so the pad changes nothing)."""
    S = len(streams)
    budgets = list(budgets) if budgets is not None else [max_new] * S
    cur = [int(t) for _, t in streams]
    out = [[] for _ in range(S)]
    live = list(range(S))
    for step in range(max_new):
        if not live:
            break
        call = [(streams[s][0], [cur[s]]) for s in live]
        us = [float(u[step][s]) for s in live] if u is not None else None
        if pad_slot is not None and len(call) == 1:
            call.append((pad_slot, [cur[live[0]]]))
            us = us + [0.5] if us is not None else None
        if greedy_api:
            picks = [int(eng.forward_greedy(cur[live[0]]))]
        elif overrides:
            logits, _ = eng.forward_streams(call)
            for tok, val in overrides.items():
                logits[:, tok] = val
            picks = [int(np.argmax(r)) for r in logits]
        elif u is None:
            _, nxt = eng.forward_streams(call, want_logits=False, want_next=True)
            picks = [int(x) for x in nxt]
        else:
            eng.forward_streams(call, want_logits=False, want_next=True)
            toks, _ = eng.sample_typical_streams(temp, us)
            picks = [int(x) for x in toks]
        for i, s in enumerate(live):
            out[s].append(picks[i])
            cur[s] = picks[i]
        live = [s for s in live if len(out[s]) < budgets[s] and out[s][-1] not in stop]
    return out


_ALLOWED = {}


def allowed(ta, q):
    """The tokens automaton ta allows in state q, as a boolean row."""
    key = (id(ta), q)
    if key not in _ALLOWED:
        a = np.zeros(V, bool)
        a[ta.edges(q)[0].astype(np.int64)] = True
        _ALLOWED[key] = a
    return _ALLOWED[key]


def host_decode(pkg, eng, streams, max_new, samplers, u=None, budgets=None, stop=(), overrides=None, constraints=None,
                pad_slot=None, rows_out=None):
    """The pick chain of the per-stream decoding calls as a host loop: forward_streams logits, the penalties in numpy
    float32, the overrides, the automaton mask row[~allowed] = -inf, sample_streams(logits=...) with the same u, append,
    the automaton advance, and the stop on a stop token, the budget or a state without edges. constraints[s] =
    (automaton, start state) or None. Returns (tokens, final automaton states). rows_out, when given, receives every
    (stream, processed row) in step order."""
    S = len(streams)
    budgets = list(budgets) if budgets is not None else [max_new] * S
    cons = constraints if constraints is not None else [None] * S
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


def stops_at(seqs, targets, prefer_unique=False):
    """A stop token per stream j near step targets[j]: the first token at or after the target that the stream has not
    emitted before; prefer_unique: preferring one that no other stream emits."""
    stop = []
    for j, t in targets.items():
        seq = seqs[j]
        fresh = [i for i in range(t, len(seq)) if seq[i] not in seq[:i]]
        alone = [i for i in fresh if all(seq[i] not in other for k, other in enumerate(seqs) if k != j)] if prefer_unique else []
        if alone or fresh:
            stop.append(seq[(alone or fresh)[0]])
    return stop


# Sampler arguments: greedy and sampled streams, penalties with decay < 1 and = 1, cuts by top-p and top-k
MIXED = [(1.0, 0.85, 0, 0.2, 0.2, 0.996), (0.0,), (0.8, 1.0, 40, 0.5, 0.0, 1.0), (1.0, 0.85), (0.0, 1.0, 0, 1.0, 0.3, 0.9),
         (1.2, 0.95, 100, 0.0, 0.4, 1.0), (0.0, 1.0, 0, 0.3, 0.0, 1.0)]


def mixed_samplers(pkg, S, kinds=MIXED):
    """Stream s samples with kinds[s % len(kinds)]."""
    sp = [pkg.Sampler(*k) for k in kinds]
    return [sp[s % len(sp)] for s in range(S)]


# -- log-probabilities -----------------------------------------------------------------------------------------------

def logprob_rule(row, y, top_n, tau=1.0):
    """(logprob, rank, top tokens, top logprobs) of target y on one f32 logits row divided by tau, in float64: ranks
    by logit descending, ties by lower index."""
    l = np.asarray(row, np.float32).astype(np.float64)
    with np.errstate(invalid="ignore"):  # rows masked to -inf
        z = (l - l.max()) / tau
    log_s = np.log(np.exp(z).sum())
    order = np.lexsort((np.arange(V), -l))
    rank = int(np.nonzero(order == y)[0][0])
    top = order[:top_n]
    return z[y] - log_s, rank, top, z[top] - log_s


def check_processed_rows(got, rows, samplers, top_n):
    """Processed log-probabilities of every step against logprob_rule on the host row (rows: host_decode's rows_out),
    divided by the stream's temperature (1 when greedy). Returns the number of -inf top entries."""
    k_of = [0] * len(got)
    masked_tops = 0
    for s, row in rows:
        k = k_of[s]
        k_of[s] += 1
        g, sp = got[s], samplers[s]
        y = int(g["tokens"][k])
        tau = float(np.float32(sp.temperature)) if sp.temperature > 0 else 1.0
        lp, rank, top, top_lp = logprob_rule(row, y, top_n, tau)
        assert int(g["ranks"][k]) == rank, (s, k)
        assert abs(g["logprobs"][k] - lp) <= 1e-9, (s, k, g["logprobs"][k], lp)
        assert [int(x) for x in g["top_tokens"][k]] == [int(x) for x in top], (s, k)
        assert close(g["top_logprobs"][k], top_lp), (s, k)
        masked_tops += int(np.sum(g["top_logprobs"][k] == -np.inf))
    return masked_tops


def replay_with_score(b, streams, got, top_n, pad_slot):
    """Per step one score_streams call on b: every live stream's current token, its emitted token as target."""
    cur = [t for _, t in streams]
    lens = [len(g["tokens"]) for g in got]
    for k in range(max(lens)):
        live = [s for s in range(len(streams)) if lens[s] > k]
        call = [(streams[s][0], [cur[s]]) for s in live]
        tg = [[int(got[s]["tokens"][k])] for s in live]
        if pad_slot is not None and len(call) == 1:  # one token alone would take the decode kernel
            call.append((pad_slot, [cur[live[0]]]))
            tg.append([None])
        res = b.score_streams(call, tg, top_n=top_n)
        for i, s in enumerate(live):
            for f in FIELDS:
                assert bits(res[i][f][0]) == bits(got[s][f][k]), (s, k, f)
            cur[s] = int(got[s]["tokens"][k])


# -- continuous batching ---------------------------------------------------------------------------------------------

MAX_GPT = 320      # batcher engines: the longest prompt (300 tokens) is one forward_streams call of the oracle
PAD = MAX_GPT - 1  # the batcher oracle's pad stream; never named by a request
LENGTHS = (1, 2, 31, 32, 33, 127, 128, 129, 300)


def batcher_samplers(pkg):
    S = pkg.Sampler
    return [S(temperature=0.0), S(temperature=0.8, top_p=0.9), S(temperature=1.0, top_k=40, presence_penalty=0.6,
            frequency_penalty=0.3, penalty_decay=0.95), S(temperature=0.0, presence_penalty=2.0, frequency_penalty=1.0)]


def ext(r):
    """The request uses overrides, an automaton or log-probabilities."""
    return r.get("overrides") is not None or r.get("constraint") is not None or r.get("logprobs") is not None


def batcher_oracle(pkg, b, r):
    """The batcher rule's two calls for one request on engine b: forward_streams of prompt[:-1] (state only), then one
    generate_streams call of (slot, prompt[-1]) and a pad stream, with the request's max_new, stops, sampler, uniforms,
    overrides, automaton and log-probabilities. Returns the result dict as Batcher.result gives it (no status)."""
    slot, prompt = r["slot"], r["prompt"]
    if len(prompt) > 1:
        call = [(slot, prompt[:-1])]
        if len(prompt) - 1 < 2:
            call.append((PAD, prompt[:1]))
        b.forward_streams(call, want_logits=False)
    us = None if r["u"] is None else np.stack([r["u"], np.full(r["max_new"], 0.5)], axis=1)
    kw = dict(stop=r["stop"], sampling=[r["sampling"], pkg.Sampler(temperature=0.0)], u=us, overrides=r.get("overrides"))
    if r.get("logprobs") is not None or r.get("constraint") is not None:
        kw.update(logprobs=r["logprobs"], top_n=r["top_n"],
                  constraints=[r["constraint"], None] if r["constraint"] is not None else None)
    out = b.generate_streams([(slot, prompt[-1]), (PAD, prompt[-1])], r["max_new"], **kw)[0]
    d = dict(out) if isinstance(out, dict) else {"tokens": out}
    if d.get("state", 0) is None:
        del d["state"]
    return d


def add_stops(pkg, b, reqs):
    """Every other unconstrained request gets a stop token from its own run, so that it fires mid-way."""
    st = b.state_download(MAX_GPT)
    for i, r in enumerate(reqs):
        if i % 2 == 0 or r.get("constraint") is not None:
            continue
        toks = [int(x) for x in batcher_oracle(pkg, b, r)["tokens"]]
        fresh = [k for k in range(len(toks) // 2, len(toks)) if toks[k] not in toks[:k]]
        if fresh:
            r["stop"] = (toks[fresh[0]],)
    b.state_upload(st, MAX_GPT)


def submit(bat, r):
    if not ext(r):
        return bat.submit(r["slot"], r["prompt"], r["max_new"], sampling=r["sampling"], u=r["u"], stop=r["stop"])
    return bat.submit(r["slot"], r["prompt"], r["max_new"], sampling=r["sampling"], u=r["u"], stop=r["stop"],
                      overrides=r["overrides"], constraint=r["constraint"], logprobs=r["logprobs"], top_n=r["top_n"])


def finish(bat):
    while bat.run(1000):
        pass


def run_schedule(a, before, reqs, rows, prefill, steps, read):
    """Every request of reqs through one batcher (rows, prefill) from state `before`, run(steps) until it is idle:
    ([read(batcher, id) per request], the final state)."""
    a.state_upload(before, MAX_GPT)
    with a.batcher(rows, prefill) as bat:
        rids = [submit(bat, r) for r in reqs]
        while bat.run(steps):
            pass
        res = [read(bat, i) for i in rids]
    return res, a.state_download(MAX_GPT)


# -- token automata --------------------------------------------------------------------------------------------------

REGEXES = {
    "date": r"\d{4}-\d{2}-\d{2}",
    "labels": r"positive|negative|neutral",
    "json": r'\{"name": "[a-z]{1,12}", "age": \d{1,3}\}',
    "number": r"-?\d+(\.\d+)?",
}
OVERRIDES = {11: 3.0, 187: -99.0, 50: -np.inf}


def prefix_state(ta, tbytes, text):
    """The state after the shortest token spelling of `text` (one token per byte where needed)."""
    ids = []
    for ch in text.encode():
        ids.append([t for t in range(2, V) if tbytes[t] == bytes([ch])][0])
    q = ta.walk(ids)
    assert q is not None
    return q


def regex_automata(C, names=tuple(REGEXES)):
    """The token automata of REGEXES (eos token 0) over C.token_bytes(): ({name: automaton}, {"date+": the state of
    "date" after "2024-"})."""
    tbytes = C.token_bytes()
    au = {k: C.token_automaton(C.compile_regex(REGEXES[k]), tbytes, eos=0) for k in names}
    return au, {"date+": prefix_state(au["date"], tbytes, "2024-")}


# -- forward passes --------------------------------------------------------------------------------------------------

def host_pick(logits, temp, u):
    """include/rwkv/sampler/typical.h restated in numpy (float64, sequential cumulative sum)."""
    p = np.exp(logits.astype(np.float64))
    p /= p.sum()
    e = int(np.uint8(int(1.0 / temp))) if temp != 1.0 else 1
    p = np.ones_like(p) if e == 0 else p ** e
    cp = np.cumsum(p / p.sum())
    cp[-1] = 1.0
    return int(np.searchsorted(cp, u, side="left")), cp


def run_pair(pkg, path, steps, threads=None):
    """`steps` tokens through the decode kernel against the CPU oracle, teacher-forced on the oracle's greedy stream:
    logits within REL_TOL, the arg-max wherever the oracle's margin exceeds 1e-3, and the final state.
    Returns (worst logits error, steps whose arg-max was checked)."""
    from oracle.oracle import Oracle
    eng = pkg.Engine(path)
    orc = Oracle(path, threads=threads)
    tok, worst, checked_argmax = SEED_TOKEN, 0.0, 0
    for step in range(steps):
        got = eng.forward([tok])[0]
        ref = orc.forward(tok)
        e = rel_err(got, ref)
        worst = max(worst, e)
        assert e < REL_TOL, "step %d: logits rel err %.3g" % (step, e)
        if margin(ref) > 1e-3:
            assert int(got.argmax()) == int(ref.argmax()), "step %d argmax" % step
            checked_argmax += 1
        tok = int(ref.argmax())  # teacher forcing on the oracle's greedy stream
    st = eng.state_download()
    for k in KEYS4:
        ref = orc.state[k]
        scale = max(np.abs(ref).max(), 1e-6)
        assert np.abs(st[k] - ref).max() / scale < REL_TOL, "state %s" % k
    assert np.all(st["pp"] == 0.0)
    eng.close()
    orc.close()
    return worst, checked_argmax


def solo(eng, toks, start=None):
    """Logits of the last token and the state after running `toks` alone in GPT mode on slot 0 from `start`."""
    if start is None:
        eng.state_zero()
    else:
        eng.state_upload(start)
    last = eng.forward(toks, mode=1)[-1]
    return last, eng.state_download()


def check_against_solo(got_logits, got_state, ref_logits, ref_state, length, what):
    """Bit for bit against the solo run on the tensor cores; a one-token stream (the decode kernel) within 2e-5."""
    n = ref_state["xy"].size
    if length > 1:
        assert np.array_equal(got_logits, ref_logits), what + ": logits differ from the solo run"
        for k in KEYS4:
            assert np.array_equal(got_state[k], ref_state[k][:n]), what + ": state " + k
    else:
        assert rel_err(got_logits, ref_logits) < 2e-5, what
        for k in KEYS4:
            assert rel_err(got_state[k], ref_state[k][:n]) < 2e-5, what + ": state " + k


def run_ragged_vs_solo(pkg, path, max_gpt, streams):
    """One ragged forward_streams pass on slots that hold state against each stream alone (prefill_min = 2); slots the
    pass does not name must not change, and the device arg-max is np.argmax of each row."""
    a = pkg.Engine(path, max_gpt=max_gpt)
    n = a.n_layers * a.n_embed
    a.forward(rand_tokens(min(max_gpt, 128), 99), mode=0, want_logits=False)  # every slot holds some state
    before = a.state_download(max_gpt)
    logits, nxt = a.forward_streams(streams, want_next=True)
    after = a.state_download(max_gpt)
    named = {s for s, _ in streams}
    for slot in range(max_gpt):
        if slot not in named:
            for k in KEYS5:
                assert np.array_equal(slot_of(after, slot, n)[k], slot_of(before, slot, n)[k]), "slot %d was touched" % slot
    assert [int(x) for x in nxt] == [int(np.argmax(r)) for r in logits]
    b = pkg.Engine(path, max_gpt=max(len(t) for _, t in streams))
    b.set_option("prefill_min", 2)
    for i, (slot, toks) in enumerate(streams):
        ref, sb = solo(b, toks, slot_of(before, slot, n))
        check_against_solo(logits[i], slot_of(after, slot, n), ref, sb, len(toks), "stream %d (slot %d, %d tokens)" % (i, slot, len(toks)))
    a.close()
    b.close()
