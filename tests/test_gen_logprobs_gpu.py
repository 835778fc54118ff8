"""rwkv_b200_generate_streams_logprobs: the log-probability, rank and top alternatives of every token device-resident
generation emits.

Asking for log-probabilities must not change generation: tokens, lengths and every slot are compared bit for bit with
generate_streams_ex on a second engine from the same state. Raw mode scores the model's row of each step with
score_streams' device function, so a replay of the generation through score_streams (one call per step, or the whole
emitted text at once on the tensor cores) must give identical bits. Processed mode is checked against a numpy float64
restatement of the rule (include/rwkv_b200.h) on the rows the host loop builds: forward_streams logits, float32
penalties, overrides, divided by the stream's temperature. Ranks and top tokens must match exactly, log-probabilities
within 1e-9 (the device sums in another order)."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

V = 50277
KEYS = ("xy", "aa", "bb", "dd")
SHAPES = [(3, 768), (2, 2048)]
NO_TARGET = 2 ** 64 - 1
FIELDS = ("logprobs", "ranks", "top_tokens", "top_logprobs")


def rand_tokens(n, seed):
    return [int(x) for x in np.random.default_rng(seed).integers(0, V, size=n)]


def slot_of(state, slot, n):
    return {k: state[k][slot * n:(slot + 1) * n] for k in state}


def engines(pkg, path, max_gpt, tc, seed=99):
    """(a, b) from the same non-trivial state on the same forward path; b replays calls that shrink below 8 streams."""
    a = pkg.Engine(path, max_gpt=max_gpt)
    b = pkg.Engine(path, max_gpt=max_gpt)
    if tc:
        b.set_option("prefill_min", 2)
    else:
        a.set_option("prefill", 0)
        b.set_option("prefill", 0)
    for i in range(0, max_gpt, 128):
        n = min(128, max_gpt - i)
        a.forward_streams([(i + j, [t]) for j, t in enumerate(rand_tokens(n, seed + i))], want_logits=False)
    b.state_upload(a.state_download(max_gpt), max_gpt)
    return a, b


def mixed_samplers(pkg, S):
    """Greedy and sampled streams, penalties with decay < 1 and = 1, cuts by top-p and top-k."""
    Sm = pkg.Sampler
    kinds = [Sm(1.0, 0.85, 0, 0.2, 0.2, 0.996), Sm(0.0), Sm(0.8, 1.0, 40, 0.5, 0.0, 1.0), Sm(1.0, 0.85),
             Sm(0.0, 1.0, 0, 1.0, 0.3, 0.9), Sm(1.2, 0.95, 100, 0.0, 0.4, 1.0), Sm(0.0, 1.0, 0, 0.3, 0.0, 1.0),
             Sm(0.6, 1.0, 5, 0.0, 0.0, 1.0)]
    return [kinds[s % len(kinds)] for s in range(S)]


def stops_at(seqs, targets):
    """A stop token per stream j near step targets[j]: the first token there that the stream has not emitted before."""
    stop = []
    for j, t in targets.items():
        seq = seqs[j]
        fresh = [i for i in range(t, len(seq)) if seq[i] not in seq[:i]]
        if fresh:
            stop.append(seq[fresh[0]])
    return stop


def full_call(eng, streams, max_new, samplers=None, u=None, budgets=None, stop=(), overrides=None, mode=0, top_n=0,
              lp=True, top=True):
    """rwkv_b200_generate_streams_logprobs with full [S][max_new] outputs (any result array may be left NULL):
    (rc, error, tokens, lengths, logprobs, ranks, top_tokens, top_logprobs)."""
    P, D = ctypes.POINTER(ctypes.c_ulonglong), ctypes.POINTER(ctypes.c_double)
    S = len(streams)
    arr = lambda a, t: np.ascontiguousarray(a, t)
    slots, first = arr([s for s, _ in streams], np.uint64), arr([t for _, t in streams], np.uint64)
    bud = arr(budgets, np.uint64) if budgets is not None else None
    stops = arr(list(stop), np.uint64)
    ovr = dict(overrides or {})
    otok, oval = arr(list(ovr.keys()), np.uint64), arr(list(ovr.values()), np.float32)
    us = arr(u, np.float64) if u is not None else None
    sp = (type(samplers[0]) * S)(*samplers) if samplers is not None else None
    out, lens = np.zeros((S, max_new), np.uint64), np.zeros(S, np.uint64)
    o_lp, o_rank = np.empty((S, max_new)), np.empty((S, max_new), np.uint64)
    o_tt, o_tl = np.empty((S, max_new, max(1, top_n)), np.uint64), np.empty((S, max_new, max(1, top_n)))
    ptr = lambda a, t: a.ctypes.data_as(t) if a is not None else None
    rc = eng.lib.rwkv_b200_generate_streams_logprobs(
        eng.h, ptr(slots, P), ptr(first, P), S, max_new, ptr(bud, P), ptr(stops, P), len(stops), ptr(otok, P),
        ptr(oval, ctypes.POINTER(ctypes.c_float)), len(otok), sp, ptr(us, D), ptr(out, P), ptr(lens, P), mode, top_n,
        ptr(o_lp, D) if lp else None, ptr(o_rank, P), ptr(o_tt, P) if top else None, ptr(o_tl, D) if top else None)
    return rc, eng.lib.rwkv_b200_last_error().decode(), out, lens, o_lp, o_rank, o_tt[:, :, :top_n], o_tl[:, :, :top_n]


def bits(x):
    return np.ascontiguousarray(x).tobytes()


def check_state(a, b, before, streams, max_gpt):
    """Named slots equal on a and b; slots not named are where `before` left them on a."""
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


def check_tail(lens, lp, rank, tt, tl):
    """Entries at or beyond each length: NaN and NO_TARGET; entries inside: finite logprob, a real rank."""
    for s, n in enumerate(int(x) for x in lens):
        assert np.all(np.isnan(lp[s, n:])) and np.all(rank[s, n:] == np.uint64(NO_TARGET)), s
        assert np.all(tt[s, n:] == np.uint64(NO_TARGET)) and np.all(np.isnan(tl[s, n:])), s
        assert np.all(np.isfinite(lp[s, :n])) and np.all(rank[s, :n] < V), s


# -- 1. nothing changes when log-probabilities are asked for ---------------------------------------------------------

def unchanged_case(pkg, path, max_gpt, S, max_new, tc, budgets, stop_targets, top_n):
    a, b = engines(pkg, path, max_gpt, tc=tc)
    perm = [int(x) for x in np.random.default_rng(S).permutation(max_gpt)]
    streams = list(zip(perm[:S], rand_tokens(S, 7 + S)))
    samplers = mixed_samplers(pkg, S)
    u = np.random.default_rng(22 + S).random((max_new, S))
    overrides = {0: -np.inf, 11: 3.0, 187: -99.0}
    st = a.state_download(max_gpt)
    seqs = [[int(x) for x in q] for q in a.generate_streams(streams, max_new, overrides=overrides, u=u, sampling=samplers)]
    stop = stops_at(seqs, stop_targets)
    kw = dict(budgets=budgets, stop=stop, overrides=overrides, u=u, sampling=samplers)
    want = b.generate_streams(streams, max_new, **kw)
    assert len({len(w) for w in want}) >= 2
    for mode in ("raw", "processed"):
        a.state_upload(st, max_gpt)
        got = a.generate_streams(streams, max_new, logprobs=mode, top_n=top_n, **kw)
        assert [len(g["tokens"]) for g in got] == [len(w) for w in want], mode
        for g, w in zip(got, want):
            assert bits(g["tokens"]) == bits(w), mode
            assert np.all(np.isfinite(g["logprobs"])) and np.all(g["ranks"] < V)
        check_state(a, b, st, streams, max_gpt)
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", SHAPES)
def test_unchanged_decode_kernel(pkg, make_model, L, E):
    unchanged_case(pkg, make_model(L, E), 6, 3, 36, False, [20, 36, 36], {1: 5}, 4)


@pytest.mark.parametrize("L,E", SHAPES)
def test_unchanged_tensor_cores(pkg, make_model, L, E):
    budgets = [40, 7, 40, 16, 33, 17, 1, 40, 25, 40, 9, 40]
    unchanged_case(pkg, make_model(L, E), 16, 12, 40, True, budgets, {0: 0, 2: 20, 3: 35}, 20)


def test_unchanged_150_streams(pkg, make_model):
    budgets = [20 if i % 5 == 0 else 1 + (7 * i) % 16 for i in range(150)]
    unchanged_case(pkg, make_model(3, 768), 256, 150, 20, True, budgets, {0: 3, 7: 10}, 3)


# -- 2. raw mode is score_streams, bit for bit -----------------------------------------------------------------------

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


@pytest.mark.parametrize("L,E", SHAPES)
@pytest.mark.parametrize("tc", [False, True])
def test_raw_equals_score_streams(pkg, make_model, L, E, tc):
    """Penalties and overrides are on, so the scored row must be the copy taken before they apply."""
    max_gpt, max_new = 12, 32
    S = 10 if tc else 3
    path = make_model(L, E)
    a, b = engines(pkg, path, max_gpt, tc=tc)
    streams = list(zip([(5 * i + 2) % (max_gpt - 1) for i in range(S)], rand_tokens(S, 21)))
    samplers = mixed_samplers(pkg, S)
    u = np.random.default_rng(23).random((max_new, S))
    overrides = {0: -np.inf, 11: 3.0, 187: -99.0}
    budgets = [max_new - (5 * i) % 23 for i in range(S)]
    st = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, budgets=budgets, overrides=overrides, u=u, sampling=samplers,
                             logprobs="raw", top_n=20)
    replay_with_score(b, streams, got, 20, max_gpt - 1 if tc else None)
    check_state(a, b, st, streams, max_gpt)
    if tc:
        # each whole emitted text in one score_streams call from the stream's starting state, on slot 0 of an engine
        # that takes max_new tokens in one call
        c = pkg.Engine(path, max_gpt=64)
        c.set_option("prefill_min", 2)
        for (slot, first), g in zip(streams, got):
            toks = [int(x) for x in g["tokens"]]
            c.slot_upload(0, slot_of(st, slot, a.n_layers * a.n_embed))
            seq = [first] + toks[:-1]
            call, tg = [(0, seq)], [toks]
            if len(seq) == 1:
                call.append((1, [first]))
                tg.append([None])
            res = c.score_streams(call, tg, top_n=20)[0]
            for f in FIELDS:
                assert bits(res[f]) == bits(g[f]), (slot, f)
        c.close()
    a.close()
    b.close()


# -- 3. processed mode against the rule ------------------------------------------------------------------------------

def rule(row, y, tau, top_n):
    l = np.asarray(row, np.float32).astype(np.float64)
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


@pytest.mark.parametrize("L,E", SHAPES)
@pytest.mark.parametrize("tc", [False, True])
def test_processed_against_the_rule(pkg, make_model, L, E, tc):
    max_gpt, max_new, top_n = 12, 24, 8
    S = 9 if tc else 4
    a, b = engines(pkg, make_model(L, E), max_gpt, tc=tc)
    streams = list(zip([(3 * i + 1) % (max_gpt - 1) for i in range(S)], rand_tokens(S, 41)))
    samplers = mixed_samplers(pkg, S)
    u = np.random.default_rng(42).random((max_new, S))
    overrides = {0: -np.inf, 11: 3.0, 187: -99.0}
    budgets = [max_new - (7 * i) % 19 for i in range(S)]
    got = a.generate_streams(streams, max_new, budgets=budgets, overrides=overrides, u=u, sampling=samplers,
                             logprobs="processed", top_n=top_n)
    # the host loop, teacher-forced with the emitted tokens: forward_streams logits, f32 penalties, overrides
    cnt = [np.zeros(V, np.float32) for _ in range(S)]
    seen = [np.zeros(V, bool) for _ in range(S)]
    cur = [t for _, t in streams]
    lens = [len(g["tokens"]) for g in got]
    for k in range(max(lens)):
        live = [s for s in range(S) if lens[s] > k]
        call = [(streams[s][0], [cur[s]]) for s in live]
        if tc and len(call) == 1:
            call.append((max_gpt - 1, [cur[live[0]]]))
        logits, _ = b.forward_streams(call)
        for i, s in enumerate(live):
            sp, row = samplers[s], logits[i]
            if sp.presence_penalty != 0 or sp.frequency_penalty != 0:
                m = seen[s]
                row[m] = row[m] - (np.float32(sp.presence_penalty) + np.float32(sp.frequency_penalty) * cnt[s][m])
            for tok, val in overrides.items():
                row[tok] = val
            y = int(got[s]["tokens"][k])
            tau = float(np.float32(sp.temperature)) if sp.temperature > 0 else 1.0
            lp, rank, top, top_lp = rule(row, y, tau, top_n)
            assert int(got[s]["ranks"][k]) == rank, (s, k)
            assert abs(got[s]["logprobs"][k] - lp) <= 1e-9, (s, k, got[s]["logprobs"][k], lp)
            assert [int(x) for x in got[s]["top_tokens"][k]] == [int(x) for x in top], (s, k)
            assert close(got[s]["top_logprobs"][k], top_lp), (s, k)
            if sp.presence_penalty != 0 or sp.frequency_penalty != 0:
                cnt[s] = cnt[s] * np.float32(sp.penalty_decay)
                cnt[s][y] += np.float32(1.0)
                seen[s][y] = True
            cur[s] = y
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", SHAPES)
def test_processed_equals_raw_at_unit_temperature(pkg, make_model, L, E):
    """Temperature 1 or 0, no penalties, no overrides: the processed row is the raw row and tau = 1."""
    max_gpt, max_new, S = 12, 20, 10
    a = pkg.Engine(make_model(L, E), max_gpt=max_gpt)
    streams = list(zip(range(S), rand_tokens(S, 51)))
    samplers = [pkg.Sampler(1.0, 0.9) if s % 2 else pkg.Sampler(0.0) for s in range(S)]
    u = np.random.default_rng(52).random((max_new, S))
    st = a.state_download(max_gpt)
    out = {}
    for mode in ("raw", "processed"):
        a.state_upload(st, max_gpt)
        out[mode] = a.generate_streams(streams, max_new, u=u, sampling=samplers, logprobs=mode, top_n=5)
    a.state_upload(st, max_gpt)
    out["greedy"] = a.generate_streams(streams, max_new, logprobs="processed", top_n=5)  # sampling=None: arg-max
    a.state_upload(st, max_gpt)
    out["greedy_raw"] = a.generate_streams(streams, max_new, logprobs="raw", top_n=5)
    for x, y in (("raw", "processed"), ("greedy", "greedy_raw")):
        for gx, gy in zip(out[x], out[y]):
            for f in ("tokens",) + FIELDS:
                assert bits(gx[f]) == bits(gy[f]), (x, f)
    a.close()


# -- 4. consistency --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("L,E", SHAPES)
def test_consistency(pkg, make_model, L, E):
    max_gpt, max_new, S = 16, 24, 14
    a = pkg.Engine(make_model(L, E), max_gpt=max_gpt)
    streams = list(zip(range(S), rand_tokens(S, 61)))
    samplers = mixed_samplers(pkg, S)
    u = np.random.default_rng(62).random((max_new, S))
    st = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, u=u, sampling=samplers, overrides={0: -np.inf, 11: 3.0},
                             logprobs="processed", top_n=20)
    hits = 0
    for sp, g in zip(samplers, got):
        toks = [int(x) for x in g["tokens"]]
        if sp.temperature == 0:
            assert np.all(g["ranks"] == 0)
            assert [int(x) for x in g["top_tokens"][:, 0]] == toks
        elif sp.top_k:
            assert np.all(g["ranks"] < sp.top_k)
        for k, y in enumerate(toks):
            at = np.nonzero(g["top_tokens"][k] == np.uint64(y))[0]
            if len(at):
                hits += 1
                assert bits(g["top_logprobs"][k][at[0]]) == bits(g["logprobs"][k])
                assert int(at[0]) == int(g["ranks"][k])
    assert hits > 0
    # overrides that mask all but 3 tokens: entries 4 and 5 are -inf, the lowest masked indices in order
    keep = (100, 200, 300)
    mask = {t: -np.inf for t in range(V) if t not in keep}
    a.state_upload(st, max_gpt)
    got = a.generate_streams(streams[:4], 3, u=u[:3, :4], sampling=samplers[:4], overrides=mask, logprobs="processed",
                             top_n=5)
    for g in got:
        assert set(int(x) for x in g["tokens"]) <= set(keep)
        for k in range(len(g["tokens"])):
            assert sorted(int(x) for x in g["top_tokens"][k][:3]) == list(keep)
            assert np.all(np.isfinite(g["top_logprobs"][k][:3]))
            assert [int(x) for x in g["top_tokens"][k][3:]] == [0, 1]
            assert np.all(g["top_logprobs"][k][3:] == -np.inf)
    a.close()


# -- 5. boundaries ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("tc", [False, True])
def test_boundaries(pkg, make_model, tc):
    """max_new a multiple of 16; streams end mid-group by budget and by stop token, at the last step, and in the first
    step. A finished stream keeps its row until the group ends: it must write nothing, neither past its own length
    nor into its neighbour's first entry."""
    max_gpt, max_new = 12, 32
    S = 9 if tc else 4
    a, b = engines(pkg, make_model(3, 768), max_gpt, tc=tc)
    streams = list(zip(range(S), rand_tokens(S, 71)))
    samplers = [pkg.Sampler(0.0)] * S
    budgets = [32, 5, 21, 32, 1, 16, 30, 17, 32][:S]
    st = a.state_download(max_gpt)
    seqs = [[int(x) for x in q] for q in a.generate_streams(streams, max_new, sampling=samplers)]
    stop = stops_at(seqs, {S - 1: 9})
    before = a.state_download(max_gpt)
    for mode in (0, 1):
        for top_n in (0, 3):
            a.state_upload(st, max_gpt)
            rc, err, out, lens, lp, rank, tt, tl = full_call(a, streams, max_new, samplers, None, budgets, stop, None,
                                                             mode, top_n)
            assert rc == 0, err
            assert len(set(int(x) for x in lens)) >= 3 and any(int(x) % 16 for x in lens)
            check_tail(lens, lp, rank, tt, tl)
            for s in range(S):  # greedy without penalties or overrides: every entry is its own stream's arg-max
                assert np.all(rank[s, :int(lens[s])] == 0), s
    got = [{"tokens": out[s, :int(lens[s])], "logprobs": lp[s, :int(lens[s])], "ranks": rank[s, :int(lens[s])],
            "top_tokens": tt[s, :int(lens[s])], "top_logprobs": tl[s, :int(lens[s])]} for s in range(S)]
    replay_with_score(b, streams, got, 3, max_gpt - 1 if tc else None)
    check_state(a, b, before, streams, max_gpt)
    a.close()
    b.close()


# -- 6. launches -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("tc", [False, True])
def test_one_launch_per_step(pkg, make_model, tc):
    max_gpt, max_new = 12, 40
    S = 9 if tc else 3
    a = pkg.Engine(make_model(3, 768), max_gpt=max_gpt)
    if not tc:
        a.set_option("prefill", 0)
    streams = list(zip(range(S), rand_tokens(S, 81)))
    budgets = [20, 3, 17] + [9] * (S - 3)  # the call ends after two groups, 32 steps
    st = a.state_download(max_gpt)
    counts = {}
    for name in ("warm", "ex", "raw", "raw_top"):
        a.state_upload(st, max_gpt)
        c0 = a.launch_count
        if name in ("warm", "ex"):
            a.generate_streams(streams, max_new, budgets=budgets, sampling=pkg.Sampler(0.0))
        else:
            a.generate_streams(streams, max_new, budgets=budgets, sampling=pkg.Sampler(0.0), logprobs="raw",
                               top_n=20 if name == "raw_top" else 0)
        counts[name] = a.launch_count - c0
    steps = min(max_new, 16 * -(-max(budgets) // 16))
    assert counts["raw"] - counts["ex"] == steps
    assert counts["raw_top"] == counts["raw"]
    a.close()


# -- 7. refusals -----------------------------------------------------------------------------------------------------

def test_refusals_leave_the_state_untouched(pkg, make_model):
    Sm = pkg.Sampler
    path = make_model(2, 768)
    a = pkg.Engine(path, max_gpt=8)
    a.forward_streams([(s, [5 + s]) for s in range(8)], want_logits=False)
    before = a.state_download(8)
    ok = [(0, 5), (3, 6)]
    sp = [Sm(0.0), Sm(0.0)]
    cases = [
        (dict(mode=2), "generate_streams_logprobs: logprob_mode 2 is neither RWKV_B200_LOGPROBS_RAW"),
        (dict(mode=-1), "logprob_mode -1 is neither"),
        (dict(top_n=21), "generate_streams_logprobs: top_n 21 > 20"),
        (dict(lp=False), "generate_streams_logprobs: logprobs_out is NULL"),
        (dict(top_n=3, top=False), "generate_streams_logprobs: top_n = 3 needs top_tokens_out and top_logprobs_out"),
        (dict(budgets=[4, 0]), "generate_streams_logprobs: budget 0 of stream 1"),
        (dict(samplers=[Sm(0.0), Sm(1.0)]), "generate_streams_logprobs: u is NULL but stream 1 samples"),
        (dict(samplers=[Sm(0.0), Sm(0.0, penalty_decay=0.0)]), r"stream 1: penalty_decay 0 is outside"),
        (dict(overrides={5: float("nan")}), "override value nan of token 5"),
    ]
    for kw, msg in cases:
        args = dict(samplers=sp, budgets=None, mode=0, top_n=0, overrides=None, lp=True, top=True)
        args.update(kw)
        rc, err, *_ = full_call(a, ok, 4, args["samplers"], None, args["budgets"], (), args["overrides"], args["mode"],
                                args["top_n"], lp=args["lp"], top=args["top"])
        assert rc != 0 and msg in err, (msg, err)
    for kw, msg in [(dict(logprobs="raw", u=[[0.5, 0.5]] * 4), "logprobs need sampling"),
                    (dict(logprobs="raw", temp=0.7), "logprobs need sampling"),
                    (dict(logprobs="sampled", sampling=Sm(0.0)), "logprobs must be 'raw' or 'processed'")]:
        with pytest.raises(pkg.EngineError, match=msg):
            a.generate_streams(ok, 4, **kw)
    after = a.state_download(8)
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    a.close()
    t = pkg.Engine(path, max_gpt=4, tp_rank=0, tp_size=2)
    with pytest.raises(pkg.EngineError, match="not supported with tensor parallelism"):
        t.generate_streams([(0, 5)], 4, sampling=Sm(0.0), logprobs="raw")
    t.close()
