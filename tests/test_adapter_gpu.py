"""LoRA adapters bound to state slots (include/rwkv_b200.h, "adapters") on the GPU.

- Numerics: forward_streams on bound slots against the float64 restatement with each stream's delta
  (lora_numerics.py, "engine" mode), logits and state per layer within numerics.TOL, on both decoding SHAPES and a width with a K tail,
  at ranks 1, 16 and 64 and with an adapter of only some projections.
- Isolation: one pass of unbound streams, two adapters and a stream across the 128-token cut; unbound streams are bit
  for bit an engine without adapters, bound streams bit for bit themselves alone, and a call without a bound slot
  enqueues exactly the launches of an engine without adapters.
- Path: a bound call under prefill_min tokens is bit for bit the same call with prefill_min = 2.
- Entry points on bound slots, each bit for bit its oracle on an engine with the same bindings: generate_streams with a
  sampler and log-probabilities against the host pick chain, generate_speculative against generate_streams, batcher
  requests against forward_streams + generate_streams, beam_search against itself on a fresh engine and score_streams
  against the log-softmax of forward_streams' logits.
- Refusals, each leaving every slot untouched."""
import numpy as np
import pytest

import decoding as dc
import lora_numerics as lm
import numerics as nm

pytestmark = pytest.mark.gpu

NAMES = {"att.key": "k", "att.value": "v", "att.receptance": "r", "att.output": "out", "ffn.key": "ffn_k",
         "ffn.value": "ffn_v", "ffn.receptance": "ffn_r"}


def make_adapter(L, E, rank, seed, names=tuple(NAMES)):
    """A LoRA state dict of `rank` over `names` whose deltas move the projections by a few per cent."""
    from importlib import import_module
    adims = import_module("rwkv-cpp-accelerated_b200").engine.adapter_dims
    rng = np.random.default_rng(seed)
    w = {}
    for l in range(L):
        for name in names:
            n_in, n_out = adims(name, E)
            w["blocks.%d.%s.lora_A" % (l, name)] = (rng.standard_normal((rank, n_in)) * n_in ** -0.5).astype(np.float32)
            w["blocks.%d.%s.lora_B" % (l, name)] = (rng.standard_normal((n_out, rank)) * 0.1 / rank ** 0.5).astype(np.float32)
    return w


def restated(w, alpha, L, E):
    """The adapter of a state dict in lora_numerics' form."""
    from importlib import import_module
    rank, mats = import_module("rwkv-cpp-accelerated_b200").engine.parse_adapter(w, L, E)
    return {"scale": alpha / rank, "A": {NAMES[n]: m[0] for n, m in mats.items()}, "B": {NAMES[n]: m[1] for n, m in mats.items()}}


@pytest.mark.parametrize("L,E,rank,names", [
    (3, 768, 16, tuple(NAMES)), (2, 2048, 1, tuple(NAMES)), (2, 784, 64, tuple(NAMES)),
    (3, 768, 8, ("att.value", "att.output", "ffn.value")),
])
def test_numerics(pkg, make_model, L, E, rank, names):
    path = make_model(L, E)
    model = nm.Model(path)
    w = make_adapter(L, E, rank, seed=rank + E, names=names)
    alpha = 2.0 * rank
    ad = restated(w, alpha, L, E)
    streams = [dc.rand_tokens(n, seed=E + n) for n in (5, 40, 1)]
    slots = (2, 0, 5)
    eng = pkg.Engine(path, max_gpt=64)
    aid = eng.add_adapter(w, alpha)
    for s in slots[:2]:
        eng.bind_adapter(s, aid)            # the third stream stays unbound
    lg, _ = eng.forward_streams(list(zip(slots, streams)))
    sd = eng.state_download(6)
    n = L * E
    ref_l, ref_s = lm.forward(model, streams, [ad, ad, None])
    base_l, _ = nm.forward(model, streams)
    for i, s in enumerate(slots):
        got_s = dc.slot_of(sd, s, n)
        le = nm.logits_err(lg[i][None, :], ref_l[i][-1:])
        errs = nm.state_errs(got_s, ref_s[i], L, E)
        assert le <= nm.TOL and max(errs.values()) <= nm.TOL, (s, le, errs)
        if i < 2:   # the adapter moves the bound streams far beyond the tolerance
            assert nm.logits_err(ref_l[i][-1:], base_l[i][-1:]) > 100 * nm.TOL
    eng.close()


def test_isolation_and_launches(pkg, make_model):
    L, E = 3, 768
    path = make_model(L, E)
    w1, w2 = make_adapter(L, E, 16, 1), make_adapter(L, E, 4, 2, names=("att.key", "ffn.key"))
    lens = (30, 70, 3, 50, 20)      # 173 tokens: the 4th stream crosses the 128-token cut
    slots = (0, 1, 2, 3, 4)
    bind = {1: "a", 3: "b", 4: "a"}
    streams = [dc.rand_tokens(n, seed=n) for n in lens]
    a = pkg.Engine(path, max_gpt=256)
    plain = pkg.Engine(path, max_gpt=256)
    ids = {"a": a.add_adapter(w1, 16.0), "b": a.add_adapter(w2, 8.0)}
    # a call without a bound slot: same bits and same launches as an engine without adapters
    la0, lp0 = a.launch_count, plain.launch_count
    ga, _ = a.forward_streams([(10, streams[0])])
    gp, _ = plain.forward_streams([(10, streams[0])])
    assert dc.bits(ga) == dc.bits(gp)
    assert a.launch_count - la0 == plain.launch_count - lp0
    for s, k in bind.items():
        a.bind_adapter(s, ids[k])
    lg, _ = a.forward_streams(list(zip(slots, streams)))
    pl, _ = plain.forward_streams(list(zip(slots, streams)))
    sa, sp = a.state_download(5), plain.state_download(5)
    n = L * E
    for i, s in enumerate(slots):
        if s not in bind:
            assert dc.bits(lg[i]) == dc.bits(pl[i]), "unbound stream %d" % i
            for k in dc.KEYS5:
                assert dc.bits(dc.slot_of(sa, s, n)[k]) == dc.bits(dc.slot_of(sp, s, n)[k])
        else:
            solo = pkg.Engine(path, max_gpt=256)
            sid = solo.add_adapter(w1 if bind[s] == "a" else w2, 16.0 if bind[s] == "a" else 8.0)
            solo.bind_adapter(s, sid)
            ls, _ = solo.forward_streams([(s, streams[i])])
            ss = solo.state_download(5)
            assert dc.bits(lg[i]) == dc.bits(ls[0]), "bound stream %d" % i
            for k in dc.KEYS5:
                assert dc.bits(dc.slot_of(sa, s, n)[k]) == dc.bits(dc.slot_of(ss, s, n)[k])
            assert dc.bits(lg[i]) != dc.bits(pl[i])
            solo.close()
    a.close()
    plain.close()


def test_bound_call_takes_tensor_cores(pkg, make_model):
    L, E = 3, 768
    path = make_model(L, E)
    w = make_adapter(L, E, 8, 3)
    out = []
    for pmin in (None, 2):
        e = pkg.Engine(path, max_gpt=16)
        if pmin:
            e.set_option("prefill_min", pmin)
        e.bind_adapter(1, e.add_adapter(w, 8.0))
        lg, _ = e.forward_streams([(1, [11, 12, 13])])    # 3 tokens < prefill_min 8
        out.append((dc.bits(lg), dc.bits(e.state_download(2)["aa"])))
        e.close()
    assert out[0] == out[1]


def bound_pair(pkg, path, max_gpt, w, alpha, slots):
    """(a, b) as decoding.engine_pair on the tensor cores, each with the adapter bound to `slots`."""
    a, b = dc.engine_pair(pkg, path, max_gpt, tc=True, a_prefill_min=True)
    for e in (a, b):
        aid = e.add_adapter(w, alpha)
        for s in slots:
            e.bind_adapter(s, aid)
    return a, b


@pytest.mark.parametrize("L,E", dc.SHAPES)
def test_generate_with_logprobs(pkg, make_model, L, E):
    path = make_model(L, E)
    w = make_adapter(L, E, 16, 5)
    M = 16
    a, b = bound_pair(pkg, path, M, w, 32.0, (1, 3))
    streams = [(1, 11), (2, 500), (3, 4118)]
    samplers = dc.mixed_samplers(pkg, 3)
    u = np.random.default_rng(4).random((12, 3))
    before = a.state_download(M)
    got = a.generate_streams(streams, 12, sampling=samplers, u=u, logprobs="raw", top_n=3)
    want, _ = dc.host_decode(pkg, b, streams, 12, samplers, u=u, pad_slot=M - 1)
    dc.check_slots(a, b, before, M, {1, 2, 3}, skip={M - 1})
    for s in range(3):
        assert [int(x) for x in got[s]["tokens"]] == want[s]
        assert np.all(np.isfinite(got[s]["logprobs"]))
    a.close()
    b.close()


@pytest.mark.parametrize("L,E", dc.SHAPES)
def test_speculative_equals_generate(pkg, make_model, L, E):
    path = make_model(L, E)
    w = make_adapter(L, E, 16, 6)
    M = 16
    slots = (1, 4, 5, 6)
    a, b = bound_pair(pkg, path, M, w, 16.0, slots)
    before = a.state_download(M)
    got = a.generate_speculative([(slots, 11)], 20, 3, context=[[11, 12] * 8])
    want = b.generate_streams([(1, 11), (M - 1, 11)], 20)   # a pad stream keeps b on the tensor cores
    assert [int(x) for x in got[0]["tokens"]] == [int(x) for x in want[0]]
    dc.check_slots(a, b, before, M, {1}, skip=set(slots[1:]) | {M - 1})
    a.close()
    b.close()


def test_batcher_requests(pkg, make_model):
    L, E = 3, 768
    path = make_model(L, E)
    M = 80
    a, b = dc.engine_pair(pkg, path, M, tc=True, a_prefill_min=True)
    for e in (a, b):
        e.bind_adapter(1, e.add_adapter(make_adapter(L, E, 16, 7), 16.0))
        e.bind_adapter(2, e.add_adapter(make_adapter(L, E, 8, 8), 8.0))
    prompts = {1: dc.rand_tokens(40, 1), 2: dc.rand_tokens(7, 2), 3: dc.rand_tokens(20, 3)}
    with a.batcher(3, 32) as bat:
        rids = {s: bat.submit(s, p, 10) for s, p in prompts.items()}
        while any(bat.result(r)["status"] not in ("done", "cancelled") for r in rids.values()):
            bat.run(16)
        got = {s: [int(x) for x in bat.result(r)["tokens"]] for s, r in rids.items()}
    b.forward_streams([(s, p[:-1]) for s, p in prompts.items()], want_logits=False)
    want = b.generate_streams([(s, p[-1]) for s, p in prompts.items()], 10)
    for i, s in enumerate(prompts):
        assert got[s] == [int(x) for x in want[i]], "request on slot %d" % s
    a.close()
    b.close()


def test_beam_and_score(pkg, make_model):
    L, E = 2, 2048
    path = make_model(L, E)
    M = 16
    w = make_adapter(L, E, 16, 9)
    a, b = bound_pair(pkg, path, M, w, 16.0, (1, 2, 3, 4))
    st0 = b.state_download(M)
    hyps = [e.beam_search([((1, 2, 3), 11)], 6, 3, n_best=2, token_logprobs=True) for e in (a, b)]
    assert [list(h["tokens"]) for h in hyps[0][0]] == [list(h["tokens"]) for h in hyps[1][0]]
    assert dc.bits(hyps[0][0][0]["token_logprobs"]) == dc.bits(hyps[1][0][0]["token_logprobs"])
    # beam search on the bound group scores what forward_streams on the bound slot computes
    toks = [int(x) for x in hyps[0][0][0]["tokens"]]
    c = pkg.Engine(path, max_gpt=M)
    c.state_upload(st0, M)
    c.bind_adapter(1, c.add_adapter(w, 16.0))
    lg, _ = c.forward_streams([(1, [11])])
    row = lg[0].astype(np.float64)
    lsm = row - row.max() - np.log(np.exp(row - row.max()).sum())
    assert abs(hyps[0][0][0]["token_logprobs"][0] - lsm[toks[0]]) < 1e-9
    # score_streams on bound slots: the log-softmax of forward_streams' logits
    seq = dc.rand_tokens(12, 4)
    b.state_upload(a.state_download(M), M)
    sc = a.score_streams([(4, seq)], targets=[[None] * 11 + [77]])
    lg, _ = b.forward_streams([(4, seq)])
    row = lg[0].astype(np.float64)
    lsm = row - row.max() - np.log(np.exp(row - row.max()).sum())
    assert abs(sc[0]["logprobs"][-1] - lsm[77]) < 1e-9
    for e in (a, b, c):
        e.close()


def test_refusals(pkg, make_model):
    L, E = 3, 768
    path = make_model(L, E)
    e = pkg.Engine(path, max_gpt=32)
    e.forward_streams([(s, [s + 1]) for s in range(32)], want_logits=False)
    before = e.state_download(32)
    w = make_adapter(L, E, 4, 9)
    bad = dict(w)
    bad["blocks.0.att.key.lora_A"] = np.full_like(w["blocks.0.att.key.lora_A"], np.nan)
    with pytest.raises(pkg.EngineError, match="non-finite"):
        e.add_adapter(bad, 4.0)
    aid = e.add_adapter(w, 4.0)
    e.bind_adapter(0, aid)
    e.bind_adapter(1, aid)
    with pytest.raises(pkg.EngineError, match="still bound"):
        e.remove_adapter(aid)
    with pytest.raises(pkg.EngineError, match="unknown"):
        e.bind_adapter(2, aid + 100)
    with pytest.raises(pkg.EngineError, match="bound to an adapter"):
        e.forward([1, 2, 3])                    # the decode-kernel API on slot 0
    with pytest.raises(pkg.EngineError, match="bound to an adapter"):
        e.forward_greedy(5)
    with pytest.raises(pkg.EngineError, match="bound to an adapter"):
        e.decode_timed([1, 2])
    with pytest.raises(pkg.EngineError, match="same adapter"):
        e.generate_speculative([((0, 2), 5)], 4, 1)
    with pytest.raises(pkg.EngineError, match="same adapter"):
        e.beam_search([((1, 3), 5)], 4, 2)
    with pytest.raises(pkg.EngineError, match="same adapter"):
        with e.batcher(2, 16) as bat:
            bat.submit(0, [1, 2], 4, draft=1, spare_slots=(5,))
    with e.batcher(2, 16) as bat:
        bat.submit(3, [1, 2], 4)
        with pytest.raises(pkg.EngineError, match="held by batcher request"):
            e.bind_adapter(3, aid)
        with pytest.raises(pkg.EngineError, match="held by batcher request"):
            e.bind_adapter(3, None)
    e.set_option("prefill", 0)
    with pytest.raises(pkg.EngineError, match="needs the tensor cores"):
        e.forward_streams([(1, [7, 8])])
    with pytest.raises(pkg.EngineError, match="needs the tensor cores"):
        e.generate_streams([(1, 7)], 3)
    e.set_option("prefill", 1)
    after = e.state_download(32)
    for k in dc.KEYS5:
        assert dc.bits(after[k]) == dc.bits(before[k]), k
    e.bind_adapter(0, None)
    e.bind_adapter(1, None)
    e.remove_adapter(aid)
    with pytest.raises(pkg.EngineError, match="unknown"):
        e.remove_adapter(aid)
    e.close()
