"""Per-stream sampling (rwkv_b200_sample_streams, rwkv_b200_generate_streams_ex) against a numpy restatement of its rule.

The rule (include/rwkv_b200.h, rwkv_b200_sampler): rank by logit descending, ties by lower index; temperature 0 is the
arg-max; otherwise p = exp((l - max) / T) in double, keep the first min(n_p, top_k) tokens of the ranking, n_p the
smallest count whose mass reaches top_p * sum(p), and walk the kept tokens in vocabulary order to the first one with
p > 0 whose cumulative share reaches u. The device sums in another order than numpy, so a pick is only compared when
u is at least 1e-9 from its interval's edges (the returned margin) and the top-p target at least 1e-9 (relative) from a
token boundary; the number of such unsure picks is bounded.

Generation is compared with the host loop it stands for, on a second engine from the same state and on the same forward
path: forward_streams logits, the penalties in numpy float32, the overrides, sample_streams(logits=...) with the same u,
append, stop check. That loop is exact, so tokens and every named slot must match bit for bit, and slots the call does
not name must not change."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

V = 50277
KEYS = ("xy", "aa", "bb", "dd")
SHAPES = [(3, 768), (2, 2048)]


def rule(l, sp, u):
    """The sampling rule on one row of (already penalised and overridden) logits: (token, top-p cut gap)."""
    l = np.asarray(l, np.float32)
    T = float(np.float32(sp.temperature))
    if T == 0.0:
        return int(np.argmax(l)), np.inf
    l64 = l.astype(np.float64)
    p = np.exp((l64 - l64.max()) / T)
    order = np.lexsort((np.arange(V), -l64))
    n_keep, gap = V, np.inf
    if sp.top_p < 1.0:
        cs = np.cumsum(p[order])
        target = float(np.float32(sp.top_p)) * cs[-1]
        n_keep = int(np.searchsorted(cs, target, side="left")) + 1
        gap = min(cs[n_keep - 1] - target, target - cs[n_keep - 2] if n_keep >= 2 else np.inf) / cs[-1]
    if sp.top_k and sp.top_k < n_keep:
        n_keep = sp.top_k
    kept = np.zeros(V, bool)
    kept[order[:n_keep]] = True
    pk = np.where(kept, p, 0.0)
    c = np.cumsum(pk) / pk.sum()
    hit = np.nonzero(kept & (p > 0) & (c >= u))[0]
    return (int(hit[0]) if len(hit) else int(np.nonzero(kept & (p > 0))[0][-1])), gap


def compare(pkg, eng, rows, params, us):
    """sample_streams(logits=rows) against the rule, in calls of at most max_gpt rows; returns the unsure rows."""
    unsure = []
    for i in range(0, len(rows), eng.max_gpt):
        sl = slice(i, i + eng.max_gpt)
        toks, margins = eng.sample_streams(params[sl], us[sl], logits=np.asarray(rows[sl], np.float32))
        for j, (row, sp, u) in enumerate(zip(rows[sl], params[sl], us[sl])):
            want, gap = rule(row, sp, u)
            if margins[j] >= 1e-9 and gap >= 1e-9:
                assert int(toks[j]) == want, "T %g top_p %g top_k %d u %.17g: device %d rule %d (margin %g gap %g)" % (
                    sp.temperature, sp.top_p, sp.top_k, u, toks[j], want, margins[j], gap)
            else:
                unsure.append(i + j)
    return unsure


def model_rows(eng, n, seed):
    rng = np.random.default_rng(seed)
    logits, _ = eng.forward_streams([(s, [int(t)]) for s, t in enumerate(rng.integers(0, V, n))])
    return list(logits)


@pytest.mark.parametrize("L,E", SHAPES)
def test_kernel_against_the_rule(pkg, make_model, L, E):
    S = pkg.Sampler
    eng = pkg.Engine(make_model(L, E), max_gpt=16)
    rng = np.random.default_rng(L * 1000 + E)
    real = model_rows(eng, 8, 5)
    params = [S(T, p, k) for T in (1e-3, 1.0, 100.0) for p in (1e-6, 0.3, 0.9, 1.0) for k in (0, 1, 40, V)]
    rows, ps, us = [], [], []
    for i, sp in enumerate(params):
        for r in (real[i % 8], real[(i + 3) % 8]):
            rows.append(r)
            ps.append(sp)
            us.append(float(rng.random()))
    # synthetic rows: all equal (ties at the top-k and top-p cut), -inf masks, one dominant token, mixed signs of zero
    flat = np.zeros(V, np.float32)
    masked = np.where(rng.random(V) < 0.9, -np.inf, rng.normal(0, 2, V)).astype(np.float32)
    dominant = rng.normal(0, 1, V).astype(np.float32)
    dominant[31337] = 40.0
    zeros = np.where(rng.random(V) < 0.5, np.float32(-0.0), np.float32(0.0)).astype(np.float32)
    zeros[:100] = rng.normal(0, 1, 100)
    for row in (flat, masked, dominant, zeros):
        for sp in (S(1.0, 0.3), S(1.0, 1.0, 100), S(2.0, 0.5, 1000), S(1e-3, 1e-6), S(100.0, 1.0), S(1.0, 1.0, V),
                   S(0.0), S(1.0, 0.999, 7)):
            for u in (0.0, float(rng.random()), 0.5, 1.0 - 2 ** -53):
                rows.append(row)
                ps.append(sp)
                us.append(u)
    unsure = compare(pkg, eng, rows, ps, us)
    # u = 0 and u = 1 - 2^-53 sit on an interval edge by construction, and so does u = 0.5 on the all-equal row when
    # an even number of tokens is kept; any other draw is unsure with probability ~1e-9
    edge = [i for i in unsure if us[i] in (0.0, 1.0 - 2 ** -53) or (us[i] == 0.5 and rows[i] is flat)]
    assert len(unsure) - len(edge) <= 2, [(ps[i].temperature, ps[i].top_p, ps[i].top_k, us[i]) for i in unsure if i not in edge]
    # a mass cut that falls inside a run of equal logits: all-equal row, top_p * V not an integer
    toks, _ = eng.sample_streams([S(1.0, 0.5)] * 2, [0.25, 1.0 - 2 ** -53], logits=np.stack([flat, flat]))
    assert [int(x) for x in toks] == [int(0.25 * 25139), 25138]
    eng.close()


def test_greedy_rows_equal_the_device_argmax(pkg, make_model):
    eng = pkg.Engine(make_model(3, 768), max_gpt=128)
    rng = np.random.default_rng(1)
    _, nxt = eng.forward_streams([(s, [int(t)]) for s, t in enumerate(rng.integers(0, V, 128))], want_logits=False, want_next=True)
    toks, margins = eng.sample_streams([pkg.Sampler(0.0)] * 128, None)
    assert np.array_equal(toks, nxt)
    assert np.all(margins == 1.0)
    eng.close()


@pytest.mark.parametrize("L,E", SHAPES)
def test_deterministic_and_same_bits_from_host_logits(pkg, make_model, L, E):
    S = pkg.Sampler
    eng = pkg.Engine(make_model(L, E), max_gpt=12)
    rng = np.random.default_rng(2)
    logits, _ = eng.forward_streams([(s, [int(t)]) for s, t in enumerate(rng.integers(0, V, 12))])
    ps = [S(1.0, 0.85), S(0.7, 0.95, 50), S(0.0), S(1.3), S(1.0, 1.0, 3), S(1e-3), S(100.0, 0.5), S(1.0, 1e-6),
          S(0.9, 0.6, 1000), S(1.0), S(2.0, 0.99), S(0.5, 1.0, 1)]
    us = rng.random(12)
    a = eng.sample_streams(ps, us)
    b = eng.sample_streams(ps, us)
    c = eng.sample_streams(ps, us, logits=logits)
    d = eng.sample_streams(ps, us, logits=logits)
    for x in (b, c, d):
        assert np.array_equal(a[0], x[0]) and np.array_equal(a[1].view(np.uint64), x[1].view(np.uint64))
    eng.close()


# -- generation ------------------------------------------------------------------------------------------------------

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


def check(a, b, before, streams, got, want, max_gpt):
    n = a.n_layers * a.n_embed
    assert [len(x) for x in got] == [len(x) for x in want], "lengths"
    for s, (g, w) in enumerate(zip(got, want)):
        assert [int(x) for x in g] == [int(x) for x in w], "tokens of stream %d" % s
    sa, sb = a.state_download(max_gpt), b.state_download(max_gpt)
    named = {slot for slot, _ in streams}
    for slot in range(max_gpt):
        if slot in named:
            for k in KEYS:
                assert np.array_equal(slot_of(sa, slot, n)[k], slot_of(sb, slot, n)[k]), "slot %d state %s" % (slot, k)
        else:
            for k in ("xy", "aa", "bb", "pp", "dd"):
                assert np.array_equal(slot_of(sa, slot, n)[k], slot_of(before, slot, n)[k]), "slot %d was touched" % slot


def host_loop(pkg, eng, streams, max_new, samplers, u=None, budgets=None, stop=(), overrides=None, pad_slot=None):
    """forward_streams logits, float32 penalties, overrides, sample_streams(logits=...) with the same u, append, stop."""
    S = len(streams)
    budgets = list(budgets) if budgets is not None else [max_new] * S
    cnt = [np.zeros(V, np.float32) for _ in range(S)]
    seen = [np.zeros(V, bool) for _ in range(S)]
    pen = [sp.presence_penalty != 0 or sp.frequency_penalty != 0 for sp in samplers]
    cur = [int(t) for _, t in streams]
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
            ps.append(pkg.Sampler(sp.temperature, sp.top_p, sp.top_k))
            us.append(float(u[step][s]) if u is not None else 0.0)
        if len(call) > len(live):
            ps.append(pkg.Sampler(0.0))
            us.append(0.0)
        toks, _ = eng.sample_streams(ps, us, logits=logits)
        for i, s in enumerate(live):
            x = int(toks[i])
            out[s].append(x)
            cur[s] = x
            if pen[s]:
                cnt[s] = cnt[s] * np.float32(samplers[s].penalty_decay)
                cnt[s][x] += np.float32(1.0)
                seen[s][x] = True
        live = [s for s in live if len(out[s]) < budgets[s] and out[s][-1] not in stop]
    return out


def stops_at(seqs, targets):
    """A stop token per stream j near step targets[j]: the first token there that the stream has not emitted before."""
    stop = []
    for j, t in targets.items():
        seq = seqs[j]
        fresh = [i for i in range(t, len(seq)) if seq[i] not in seq[:i]]
        alone = [i for i in fresh if all(seq[i] not in other for k, other in enumerate(seqs) if k != j)]
        if alone or fresh:
            stop.append(seq[(alone or fresh)[0]])
    return stop


def greedy_case(pkg, make_model, L, E, max_gpt, S, max_new, tc, stop_targets=None, budgets=None):
    a, b = engines(pkg, make_model(L, E), max_gpt, tc=tc)
    perm = [int(x) for x in np.random.default_rng(S).permutation(max_gpt)]
    streams = [(s, t) for s, t in zip(perm[:S], rand_tokens(S, 7 + S))]
    stop = []
    if stop_targets:
        st = a.state_download(max_gpt)
        stop = stops_at([[int(x) for x in q] for q in a.generate_streams(streams, max_new)], stop_targets)
        a.state_upload(st, max_gpt)
    before = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, budgets=budgets, stop=stop, sampling=pkg.Sampler(0.0, 0.5, 3))
    want = b.generate_streams(streams, max_new, budgets=budgets, stop=stop)
    check(a, b, before, streams, got, want, max_gpt)
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", SHAPES)
def test_greedy_generation_decode_kernel(pkg, make_model, L, E):
    greedy_case(pkg, make_model, L, E, max_gpt=6, S=3, max_new=36, tc=False, stop_targets={1: 5}, budgets=[20, 36, 36])


@pytest.mark.parametrize("L,E", SHAPES)
def test_greedy_generation_tensor_cores(pkg, make_model, L, E):
    budgets = [40, 7, 40, 16, 33, 17, 1, 40, 25, 40, 9, 40]
    greedy_case(pkg, make_model, L, E, max_gpt=16, S=12, max_new=40, tc=True, stop_targets={0: 0, 2: 20, 3: 35}, budgets=budgets)


def test_greedy_generation_150_streams(pkg, make_model):
    budgets = [20 if i % 5 == 0 else 1 + (7 * i) % 16 for i in range(150)]
    greedy_case(pkg, make_model, 3, 768, max_gpt=256, S=150, max_new=20, tc=True, budgets=budgets)


def mixed_samplers(pkg, S):
    """Greedy and sampled streams, penalties with decay < 1 and = 1, cuts by top-p and top-k."""
    Sm = pkg.Sampler
    kinds = [Sm(1.0, 0.85, 0, 0.2, 0.2, 0.996), Sm(0.0), Sm(0.8, 1.0, 40, 0.5, 0.0, 1.0), Sm(1.0, 0.85),
             Sm(0.0, 1.0, 0, 1.0, 0.3, 0.9), Sm(1.2, 0.95, 100, 0.0, 0.4, 1.0), Sm(0.0, 1.0, 0, 0.3, 0.0, 1.0)]
    return [kinds[s % len(kinds)] for s in range(S)]


@pytest.mark.parametrize("L,E", SHAPES)
@pytest.mark.parametrize("S", [3, 10])
def test_sampled_generation_against_the_host_loop(pkg, make_model, L, E, S):
    """S = 3 on the decode kernel, S = 10 on the tensor cores; per-stream samplers, overrides, stops and budgets."""
    max_gpt, max_new = 12, 40
    tc = S >= 8
    a, b = engines(pkg, make_model(L, E), max_gpt, tc=tc)
    streams = [(s, t) for s, t in zip([(5 * i + 2) % (max_gpt - 1) for i in range(S)], rand_tokens(S, 21))]  # max_gpt - 1: pad
    samplers = mixed_samplers(pkg, S)
    u = np.random.default_rng(22).random((max_new, S))
    overrides = {0: -np.inf, 11: 3.0, 187: -99.0}
    budgets = [max_new - (5 * i) % 23 for i in range(S)]
    st = a.state_download(max_gpt)
    seqs = [[int(x) for x in q] for q in a.generate_streams(streams, max_new, overrides=overrides, u=u, sampling=samplers)]
    a.state_upload(st, max_gpt)
    stop = stops_at(seqs, {0: 9, S - 1: 25})
    before = a.state_download(max_gpt)
    got = a.generate_streams(streams, max_new, budgets=budgets, stop=stop, overrides=overrides, u=u, sampling=samplers)
    want = host_loop(pkg, b, streams, max_new, samplers, u=u, budgets=budgets, stop=stop, overrides=overrides,
                     pad_slot=max_gpt - 1 if tc else None)
    assert len({len(w) for w in want}) >= 2
    assert all(0 not in w for w in want)
    check(a, b, before, streams, got, want, max_gpt)
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", SHAPES)
def test_presence_penalty_takes_effect(pkg, make_model, L, E):
    max_gpt, max_new, S = 12, 256, 10  # long enough for greedy chains to revisit a token
    eng = pkg.Engine(make_model(L, E), max_gpt=max_gpt)
    streams = [(s, t) for s, t in zip(range(S), rand_tokens(S, 31))]
    st = eng.state_download(max_gpt)
    plain = eng.generate_streams(streams, max_new)
    eng.state_upload(st, max_gpt)
    pen = eng.generate_streams(streams, max_new, sampling=pkg.Sampler(0.0, presence_penalty=1e4))
    assert any(len(set(int(x) for x in q)) < len(q) for q in plain)
    for q in pen:
        assert len(q) == max_new and len(set(int(x) for x in q)) == max_new
    eng.close()


def test_rejected_inputs_leave_the_state_untouched(pkg, make_model):
    Sm = pkg.Sampler
    path = make_model(2, 768)
    a = pkg.Engine(path, max_gpt=8)
    good = np.zeros((2, V), np.float32)
    with pytest.raises(pkg.EngineError, match="no per-stream logits"):
        a.sample_streams([Sm(0.0)] * 2, None)
    a.forward(rand_tokens(8, 70), mode=0, want_logits=False)
    a.forward_streams([(0, [5]), (1, [6])], want_next=True)
    before = a.state_download(8)
    nan_row, inf_row, dead = good.copy(), good.copy(), good.copy()
    nan_row[0, 7] = np.nan
    inf_row[1, 9] = np.inf
    dead[1, :] = -np.inf
    bad_sample = [
        (dict(params=[Sm(0.0)] * 3, us=None), "3 rows asked, the last forward_streams produced 2"),
        (dict(params=Sm(0.0), us=None, logits=np.zeros((0, V), np.float32)), "no streams"),
        (dict(params=Sm(0.0), us=None, logits=np.zeros((9, V), np.float32)), "9 rows of logits > max_gpt 8"),
        (dict(params=[Sm(1.0), Sm(-1.0)], us=[0.5, 0.5]), "stream 1: temperature -1 is not a finite value"),
        (dict(params=[Sm(float("nan")), Sm()], us=[0.5, 0.5]), "stream 0: temperature nan"),
        (dict(params=[Sm(float("inf")), Sm()], us=[0.5, 0.5]), "stream 0: temperature inf"),
        (dict(params=[Sm(1.0, 0.0), Sm()], us=[0.5, 0.5]), r"stream 0: top_p 0 is outside \(0, 1\]"),
        (dict(params=[Sm(), Sm(1.0, 1.5)], us=[0.5, 0.5]), r"stream 1: top_p 1.5 is outside"),
        (dict(params=[Sm(), Sm(1.0, 1.0, V + 1)], us=[0.5, 0.5]), "stream 1: top_k 50278 > 50277"),
        (dict(params=[Sm(presence_penalty=0.5), Sm()], us=[0.5, 0.5]), "presence_penalty and frequency_penalty must be 0"),
        (dict(params=[Sm(), Sm(frequency_penalty=0.5)], us=[0.5, 0.5]), "stream 1: presence_penalty and frequency_penalty"),
        (dict(params=[Sm(0.0), Sm(1.0)], us=None, logits=good), "u is NULL but stream 1 samples"),
        (dict(params=Sm(), us=[0.5, 1.0]), r"u\[1\] = 1 is outside \[0, 1\)"),
        (dict(params=Sm(), us=[float("nan"), 0.5]), r"u\[0\] = nan"),
        (dict(params=Sm(), us=[0.5, 0.5], logits=nan_row), r"logits\[0\]\[7\] = nan"),
        (dict(params=Sm(), us=[0.5, 0.5], logits=inf_row), r"logits\[1\]\[9\] = inf"),
        (dict(params=Sm(), us=[0.5, 0.5], logits=dead), "row 1 of the logits has no finite value"),
    ]
    for kw, msg in bad_sample:
        with pytest.raises(pkg.EngineError, match=msg):
            a.sample_streams(**kw)
    P = ctypes.POINTER(ctypes.c_ulonglong)
    toks = np.zeros(2, np.uint64)
    assert a.lib.rwkv_b200_sample_streams(a.h, 2, None, None, None, toks.ctypes.data_as(P), None) != 0
    assert b"null argument" in a.lib.rwkv_b200_last_error()
    # nothing was replaced: the rows of the last forward_streams are still there
    a.sample_typical_streams(1.0, [0.5, 0.5])
    ok = [(0, 5), (1, 6)]
    allmask = {t: -np.inf for t in range(V)}
    bad_gen = [
        (dict(sampling=Sm(), u=None), "u is NULL but stream 0 samples"),
        (dict(sampling=[Sm(0.0), Sm(1.0, 2.0)], u=None), "generate_streams_ex: stream 1: top_p 2 is outside"),
        (dict(sampling=[Sm(0.0, presence_penalty=float("inf")), Sm(0.0)]), "stream 0: presence_penalty inf is not finite"),
        (dict(sampling=[Sm(0.0), Sm(0.0, frequency_penalty=2e6)]), "stream 1: frequency_penalty 2e\\+06 is not finite or exceeds"),
        (dict(sampling=[Sm(0.0), Sm(0.0, penalty_decay=0.0)]), r"stream 1: penalty_decay 0 is outside \(0, 1\]"),
        (dict(sampling=[Sm(0.0), Sm(0.0, penalty_decay=1.5)]), r"stream 1: penalty_decay 1.5"),
        (dict(sampling=[Sm(0.0), Sm(0.0, top_k=V + 1)]), "stream 1: top_k 50278"),
        (dict(sampling=Sm(0.0), overrides={5: float("nan")}), "override value nan of token 5 is neither finite nor -inf"),
        (dict(sampling=Sm(0.0), overrides={9: float("inf")}), "override value inf of token 9"),
        (dict(sampling=Sm(0.0), overrides=allmask), "the overrides set every token to -inf"),
        (dict(sampling=Sm(), u=[[0.5, 1.0]] * 4), r"u\[1\] = 1 is outside"),
        (dict(sampling=[Sm(0.0)] * 3), "3 samplers for 2 streams"),
        (dict(sampling=Sm(0.0), budgets=[4, 0]), "generate_streams_ex: budget 0 of stream 1"),
    ]
    for kw, msg in bad_gen:
        with pytest.raises(pkg.EngineError, match=msg):
            a.generate_streams(ok, 4, **kw)
    after = a.state_download(8)
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    a.close()
    t = pkg.Engine(path, max_gpt=4, tp_rank=0, tp_size=2)
    with pytest.raises(pkg.EngineError, match="not supported with tensor parallelism"):
        t.generate_streams([(0, 5)], 4, sampling=Sm(0.0))
    with pytest.raises(pkg.EngineError, match="not supported with tensor parallelism"):
        t.sample_streams(Sm(0.0), None, logits=np.zeros((1, V), np.float32))
    t.close()
