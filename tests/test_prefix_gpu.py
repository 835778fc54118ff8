"""Prefix state cache (include/rwkv_b200.h, "Prefix state cache") on the GPU.

- prefix_forward bit for bit against slot_zero + forward_streams of the full tokens on the tensor cores (prefill_min 2):
  logits, arg-max and all five arrays of every named slot, every other slot untouched. On both decoding SHAPES and a
  width with a K tail (784), with hits of 0 tokens, inside a block, exactly a block and all but the last token, streams
  across the 128-token cut with snapshots at 127, 128 and their last tokens, streams of one call sharing a prefix, and a
  state-only call that is fully cached and runs no pass.
- Snapshot content: download(prefix) is bit for bit slot_download of forward_streams(prefix) from a zeroed slot.
- cached counts and stats() as the policy predicts, including eviction of a stream's own restore source and skipped
  snapshots at a small capacity, with exact results throughout.
- An open but unused cache changes no launch and no bit of forward_streams and generate_streams.
- Multi-turn chat: insert of a finished turn's state gives the next turn a hit, with exact results.
- Adapters: a bound stream never hits an unbound entry, and the reverse.
- Batcher: requests with the cache are bit for bit the same requests without it on zeroed slots (tokens,
  log-probabilities, final slot states), in mixed traffic with requests that do not use the cache, a speculative
  request, a small prefill budget so that snapshots fall inside split segments, and a cancelled request; a cache that an
  unfinished request names cannot be closed.
- Beam search on the tensor cores over more than 128 rows after a freed cache has dirtied device memory: the same
  results as an engine created before.
- Refusals, each leaving every slot untouched."""
import numpy as np
import pytest

import decoding as dc

pytestmark = pytest.mark.gpu

MAX_GPT = 512


def engines(pkg, path):
    a, b = dc.engine_pair(pkg, path, MAX_GPT, tc=True)
    return a, b


def check_call(a, b, cache, streams, head=True, what=""):
    """prefix_forward on a against slot_zero + forward_streams on b; returns the cached counts."""
    before = a.state_download(MAX_GPT)
    logits, nxt, cached = cache.forward(streams, want_logits=head, want_next=head)
    for slot, _ in streams:
        b.slot_zero(slot)
    ref_logits, ref_next = b.forward_streams(streams, want_logits=head, want_next=head)
    if head:
        assert dc.bits(logits) == dc.bits(ref_logits), what + ": logits"
        assert np.array_equal(nxt, ref_next), what + ": arg-max"
    dc.check_slots(a, b, before, MAX_GPT, {s for s, _ in streams}, keys=dc.KEYS5, what=what)
    return [int(x) for x in cached]


def zero_state_of(b, slot, tokens):
    b.slot_zero(slot)
    b.forward_streams([(slot, tokens)], want_logits=False)
    return b.slot_download(slot)


@pytest.mark.parametrize("L,E", dc.SHAPES + [(2, 784)])
def test_prefix_forward_bit_exact(pkg, make_model, L, E):
    a, b = engines(pkg, make_model(L, E))
    cache = a.prefix_cache(32, block=32)
    P, Q = dc.rand_tokens(150, seed=E), dc.rand_tokens(127, seed=E + 1)
    ta, tb, tc = dc.rand_tokens(10, E + 2), dc.rand_tokens(7, E + 3), dc.rand_tokens(3, E + 4)
    # three streams, two sharing P across the 128-token cut: snapshots at 32, 64, 96, 128, 160, 155 and 32, 64, 96, 127
    got = check_call(a, b, cache, [(0, P + ta), (1, P + tb[:5]), (2, Q)], what="first call")
    assert got == [0, 0, 0]
    assert cache.stats()["snapshots"] == 10
    # all but the last token, inside a block, exactly a block, nothing
    got = check_call(a, b, cache, [(3, P + ta + [5]), (4, P + tb), (5, P[:128] + tc), (6, dc.rand_tokens(20, E + 5))],
                     what="hits")
    assert got == [160, 155, 128, 0]
    for key in (P[:32], P[:64], P[:128], Q, P + ta):  # inside a segment, at the pass cut, at stream ends
        want = zero_state_of(b, 9, key)
        have = cache.download(key)
        for k in dc.KEYS4:
            assert dc.bits(have[k]) == dc.bits(want[k]), "snapshot after %d tokens: %s" % (len(key), k)
    assert cache.download(P[:129]) is None
    # state only: fully cached streams run no pass, only the restore copy
    n0 = a.launch_count
    got = check_call(a, b, cache, [(7, P + ta), (8, Q)], head=False, what="state only")
    assert got == [160, 127] and a.launch_count - n0 == 1
    st = cache.stats()
    assert st == dict(live=14, lookups=9, hit_tokens=730, prefilled_tokens=468, snapshots=14, skipped=0, evictions=0)
    cache.clear()
    assert cache.stats()["live"] == 0 and cache.download(Q) is None
    assert check_call(a, b, cache, [(0, Q + [1])], what="after clear") == [0]
    cache.close()


def test_eviction_and_skipped_snapshots(pkg, make_model):
    """Capacity 3, block 4. A stream evicts the entry it restores from (the restore runs first) and skips a snapshot
    when every other entry is extended or pinned; results stay exact."""
    a, b = engines(pkg, make_model(2, 768))
    cache = a.prefix_cache(3, block=4)
    T, U = dc.rand_tokens(10, 1), dc.rand_tokens(7, 2)
    assert check_call(a, b, cache, [(0, T)], what="fill") == [0]  # 4, 8, 10
    assert check_call(a, b, cache, [(1, T + U[:6])], what="evict own source") == [10]  # 12 replaces 10, 16 skipped
    assert cache.stats() == dict(live=3, lookups=2, hit_tokens=10, prefilled_tokens=16, snapshots=4, skipped=1, evictions=1)
    assert cache.download(T) is None and cache.download(T + U[:2]) is not None
    assert check_call(a, b, cache, [(2, T + U)], what="again") == [12]  # 16 replaces 12, 17 skipped
    assert cache.stats() == dict(live=3, lookups=3, hit_tokens=22, prefilled_tokens=21, snapshots=5, skipped=2, evictions=2)
    want = zero_state_of(b, 9, T + U[:6])
    have = cache.download(T + U[:6])
    for k in dc.KEYS4:
        assert dc.bits(have[k]) == dc.bits(want[k]), k


def test_unused_cache_changes_nothing(pkg, make_model):
    path = make_model(2, 768)
    a, b = dc.engine_pair(pkg, path, 64, tc=True, a_prefill_min=True)
    cache = a.prefix_cache(4)
    streams = [(s, dc.rand_tokens(9 + s, s)) for s in range(4)]
    counts = []
    for e in (a, b):
        n0 = e.launch_count
        lg, nx = e.forward_streams(streams, want_logits=True, want_next=True)
        gen = e.generate_streams([(s, 11 + s) for s in range(4)], 6)
        with e.batcher(2, 8) as bat:
            ids = [bat.submit(10 + s, dc.rand_tokens(12 + s, 40 + s), 5) for s in range(3)]
            bat.run(64)
            res = [bat.result(i)["tokens"].tolist() for i in ids]
        counts.append((e.launch_count - n0, dc.bits(lg), nx.tolist(), [g.tolist() for g in gen], res))
    assert counts[0] == counts[1]
    assert dc.bits(a.state_download(64)["xy"]) == dc.bits(b.state_download(64)["xy"])
    cache.close()


def test_multi_turn_insert(pkg, make_model):
    a, b = engines(pkg, make_model(2, 768))
    a.set_option("prefill_min", 2)  # the turn's generation on the tensor cores, like the reference forward
    cache = a.prefix_cache(8, block=16)
    p0, p1 = dc.rand_tokens(40, 7), dc.rand_tokens(30, 8)
    _, nxt, _ = cache.forward([(0, p0), (1, p1)], want_logits=False, want_next=True)
    gen = a.generate_streams([(0, int(nxt[0])), (1, int(nxt[1]))], 5)
    fed = p0 + [int(nxt[0])] + [int(x) for x in gen[0][:-1]]  # the last emitted token is not fed
    cache.insert(0, fed)
    want = zero_state_of(b, 9, fed)
    have = cache.download(fed)
    for k in dc.KEYS4:
        assert dc.bits(have[k]) == dc.bits(want[k]), k
    turn2 = fed + [int(gen[0][-1])] + dc.rand_tokens(12, 9)
    assert check_call(a, b, cache, [(2, turn2)], what="next turn") == [len(fed)]


def test_adapter_bindings_separate_entries(pkg, make_model):
    L, E = 2, 768
    a, b = engines(pkg, make_model(L, E))
    from importlib import import_module
    adims = import_module("rwkv-cpp-accelerated_b200").engine.adapter_dims
    rng = np.random.default_rng(4)
    w = {}
    for l in range(L):
        n_in, n_out = adims("att.value", E)
        w["blocks.%d.att.value.lora_A" % l] = (rng.standard_normal((2, n_in)) * n_in ** -0.5).astype(np.float32)
        w["blocks.%d.att.value.lora_B" % l] = (rng.standard_normal((n_out, 2)) * 0.05).astype(np.float32)
    for e in (a, b):
        aid = e.add_adapter(w, 4.0)
        for slot in (10, 11):
            e.bind_adapter(slot, aid)
    cache = a.prefix_cache(16, block=8)
    T = dc.rand_tokens(20, 3)
    assert check_call(a, b, cache, [(0, T)], what="unbound") == [0]
    assert check_call(a, b, cache, [(10, T + [1])], what="bound after unbound") == [0]
    assert check_call(a, b, cache, [(11, T + [1, 2])], what="bound after bound") == [21]
    assert check_call(a, b, cache, [(1, T + [1, 4])], what="unbound after bound") == [20]


def test_refusals(pkg, make_model):
    a, b = engines(pkg, make_model(2, 768))
    E = pkg.engine
    for cap, block in ((0, 64), (4, 0), (4, 2049)):
        with pytest.raises(E.EngineError):
            a.prefix_cache(cap, block)
    cache = a.prefix_cache(4, block=8)
    before = a.state_download(MAX_GPT)
    bad = [
        lambda: cache.forward([(0, [1, 2]), (0, [3])]),                 # a slot twice
        lambda: cache.forward([(0, [1, E.VOCAB])]),                     # a token out of range
        lambda: cache.forward([(MAX_GPT, [1, 2])]),                     # a slot out of range
        lambda: cache.forward([(0, [])]),                               # an empty stream
        lambda: cache.forward([(0, list(range(MAX_GPT + 1)))]),          # more than max_gpt tokens
        lambda: cache.insert(0, []),
        lambda: cache.insert(0, [5, E.VOCAB]),
        lambda: cache.insert(MAX_GPT, [5]),
    ]
    for call in bad:
        with pytest.raises(E.EngineError):
            call()
    after = a.state_download(MAX_GPT)
    for k in dc.KEYS5:
        assert dc.bits(after[k]) == dc.bits(before[k]), k
    assert cache.stats() == dict(live=0, lookups=0, hit_tokens=0, prefilled_tokens=0, snapshots=0, skipped=0, evictions=0)
    a.set_option("prefill", 0)
    with pytest.raises(E.EngineError, match="prefill"):
        cache.forward([(0, [1, 2])])
    with pytest.raises(E.EngineError, match="prefill"):
        a.prefix_cache(4)
    a.close()
    with pytest.raises(E.EngineError, match="closed"):
        cache.stats()


def test_batcher_requests_exact(pkg, make_model):
    """Requests with the cache on engine a against the same requests without it on zeroed slots of engine b."""
    path = make_model(2, 768)
    a, b = dc.engine_pair(pkg, path, 64, tc=True)
    cache = a.prefix_cache(32, block=8)
    system = dc.rand_tokens(40, 11)
    reqs = [  # slot, prompt, options, uses the cache
        (0, system + dc.rand_tokens(5, 12), {}, True),
        (1, dc.rand_tokens(20, 13), {}, False),
        (2, system + dc.rand_tokens(7, 14), dict(logprobs="raw", top_n=2), True),
        (3, system + dc.rand_tokens(3, 15), dict(draft=2, spare_slots=(20, 21)), True),
        (4, system[:30] + dc.rand_tokens(6, 16), dict(logprobs="processed"), True),
        (5, system + dc.rand_tokens(9, 17), {}, True),
    ]
    for slot, _, _, cached in reqs:
        if cached:
            b.slot_zero(slot)
    before = a.state_download(64)
    got, want = {}, {}
    for eng, use in ((a, True), (b, False)):
        with eng.batcher(3, 16) as bat:
            ids = [bat.submit(slot, prompt, 10, prefix_cache=cache if use and c else None, **opt)
                   for slot, prompt, opt, c in reqs]
            if use:
                bat.run(16)
                assert bat.result(ids[5])["status"] == "queued"
                with pytest.raises(pkg.engine.EngineError, match="unfinished batcher request"):
                    cache.close()
                while bat.result(ids[5])["status"] == "queued":
                    bat.run(1)
                bat.cancel(ids[5])  # admitted and restored, then cut short
            while bat.run(64):
                pass
            (got if use else want).update({i: bat.result(rid) for i, rid in enumerate(ids)})
    assert got[5]["status"] == "cancelled"
    n5 = len(got[5]["tokens"])
    assert got[5]["tokens"].tolist() == want[5]["tokens"][:n5].tolist()
    for i in range(5):
        for k, v in want[i].items():
            if k in ("status", "steps"):
                continue
            assert dc.bits(np.asarray(got[i][k])) == dc.bits(np.asarray(v)), "request %d: %s" % (i, k)
    assert [got[i].get("cached") for i in range(6)] == [0, None, 0, 40, 24, 40]
    skip = {5, 20, 21}
    dc.check_slots(a, b, before, 64, {r[0] for r in reqs}, keys=dc.KEYS5, skip=skip, what="batcher")
    st = cache.stats()
    assert st["lookups"] == 5 and st["hit_tokens"] == 104 and st["skipped"] == 0
    cache.close()


def test_beam_after_freed_cache(pkg, make_model):
    """A beam step fills tokens and descriptors of passes no upload reached (more rows than step 0's passes): those
    passes must take no snapshot whatever the memory held before."""
    path = make_model(2, 768)
    ref = pkg.Engine(path, max_gpt=200)
    dirty = pkg.Engine(path, max_gpt=200)
    with dirty.prefix_cache(64, block=1) as c:
        c.forward([(s, dc.rand_tokens(30, s)) for s in range(6)], want_logits=False)
    dirty.close()
    eng = pkg.Engine(path, max_gpt=200)
    out = []
    for e in (ref, eng):
        e.set_option("prefill_min", 2)
        e.forward_streams([(4 * g, [int(t)]) for g, t in enumerate(dc.rand_tokens(40, 5))], want_logits=False)
        res = e.beam_search([(list(range(4 * g, 4 * g + 4)), 100 + g) for g in range(40)], 4, 4, n_best=2)
        out.append([[(h["tokens"].tolist(), h["score"]) for h in grp] for grp in res])
    assert out[0] == out[1]
