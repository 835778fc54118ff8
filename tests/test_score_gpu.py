"""rwkv_b200_score_streams against its rule (include/rwkv_b200.h, DESIGN §4.3), restated in numpy float64 on the logits of
the same stream run alone from the same starting state on the same forward path.

rank and top-n tokens follow a stable sort on (-l, index) and must match exactly; log-probabilities are sums in another
order than numpy's, so they are compared within 1e-9. Everything the device computes twice (the same stream in another
call, a top entry and the same token as a target, chunked and whole documents) must agree bit for bit, and the slots
must end where forward_streams leaves them."""
import ctypes
import os
import shutil

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

V = 50277
KEYS = ("xy", "aa", "bb", "dd")
SHAPES = [(3, 768), (2, 2048)]


def rule(row, y, top_n):
    """(logprob, rank, top tokens, top logprobs) of target y on one f32 logits row."""
    l = np.asarray(row, np.float32).astype(np.float64)
    m = l.max()
    log_s = np.log(np.exp(l - m).sum())
    order = np.lexsort((np.arange(V), -l))
    lp = lambda v: (l[v] - m) - log_s
    rank = int(np.nonzero(order == y)[0][0])
    top = order[:top_n]
    return lp(y), rank, top, np.array([lp(v) for v in top])


def alone_logits(ref, state, seq, tc):
    """Logits after every token of `seq` run alone on slot 0 of `ref` from `state`, on the tensor cores (tc) or the
    decode kernel (ref has "prefill" = 0)."""
    ref.slot_upload(0, state)
    if tc and len(seq) == 1:  # one token alone would take the decode kernel: give it a companion stream
        lg, _ = ref.forward_streams([(0, list(seq)), (1, [0])])
        return lg[:1]
    return ref.forward(list(seq))


def check_against_rule(res, logits, targets, top_n):
    for t, y in enumerate(targets):
        if y is None:
            assert np.isnan(res["logprobs"][t]) and int(res["ranks"][t]) == 2 ** 64 - 1
            if top_n:
                assert np.all(res["top_tokens"][t] == np.uint64(2 ** 64 - 1)) and np.all(np.isnan(res["top_logprobs"][t]))
            continue
        lp, rank, top, top_lp = rule(logits[t], y, top_n)
        assert int(res["ranks"][t]) == rank, (t, y)
        assert abs(res["logprobs"][t] - lp) <= 1e-9, (t, res["logprobs"][t], lp)
        if top_n:
            assert [int(x) for x in res["top_tokens"][t]] == [int(x) for x in top], t
            assert np.max(np.abs(res["top_logprobs"][t] - top_lp)) <= 1e-9


def warm_slots(eng, slots, rng):
    eng.forward_streams([(s, [int(x) for x in rng.integers(0, V, 3)]) for s in slots], want_logits=False)
    return {s: eng.slot_download(s) for s in slots}


def random_targets(rng, seqs, p_none=0.2):
    return [[None if rng.random() < p_none else int(rng.integers(0, V)) for _ in s] for s in seqs]


def all_states(eng):
    return eng.state_download(eng.max_gpt)


def same_state(a, b):
    return all(np.array_equal(a[k], b[k]) for k in KEYS)


@pytest.mark.parametrize("L,E", SHAPES)
@pytest.mark.parametrize("path", ["tc", "decode", "short"])
def test_against_the_rule(pkg, make_model, L, E, path):
    """Ragged streams on non-contiguous slots that already hold state, each against the same stream run alone."""
    model = make_model(L, E)
    eng = pkg.Engine(model, max_gpt=128)
    ref = pkg.Engine(model, max_gpt=128)
    if path == "decode":
        eng.set_option("prefill", 0)
    if path in ("decode", "short"):
        ref.set_option("prefill", 0)
    else:
        ref.set_option("prefill_min", 2)
    rng = np.random.default_rng(L * 7 + E)
    lengths = [1, 3, 2] if path == "short" else [1, 7, 16, 33, 60]  # "short": 6 tokens, under prefill_min
    slots = [9, 2, 40, 17, 5][:len(lengths)]
    start = warm_slots(eng, slots, rng)
    seqs = [[int(x) for x in rng.integers(0, V, n)] for n in lengths]
    targets = random_targets(rng, seqs)
    for top_n in (0, 7, 20):
        for s in slots:
            eng.slot_upload(s, start[s])
        res = eng.score_streams(list(zip(slots, seqs)), targets, top_n=top_n)
        for s, seq, tg, r in zip(slots, seqs, targets, res):
            check_against_rule(r, alone_logits(ref, start[s], seq, path == "tc"), tg, top_n)
    # the default targets: each stream's own next tokens, the last position unscored
    for s in slots:
        eng.slot_upload(s, start[s])
    res = eng.score_streams(list(zip(slots, seqs)))
    for s, seq, r in zip(slots, seqs, res):
        check_against_rule(r, alone_logits(ref, start[s], seq, path == "tc"), seq[1:] + [None], 0)
    eng.close()
    ref.close()


def tied_model(src_path, dst_path, L, E, group, src_token):
    """A copy of the model whose head columns of every token in `group` equal the column of `src_token`, so their
    logits are exactly equal. HEAD (tensor 43, include/rwkv/rwkv/format.h) is u8 [E in][V out], followed by head_r and
    head_o (f32 [E] each), at the end of the file."""
    shutil.copyfile(src_path, dst_path)
    off = os.path.getsize(dst_path) - V * E - 8 * E
    head = np.memmap(dst_path, dtype=np.uint8, mode="r+", offset=off, shape=(E, V))
    col = np.array(head[:, src_token])
    for g in group:
        head[:, g] = col
    head.flush()
    del head
    return dst_path


def test_ties_follow_the_lower_index_rule(pkg, make_model, tmp_path):
    L, E = 3, 768
    base = make_model(L, E)
    rng = np.random.default_rng(3)
    seq = [int(x) for x in rng.integers(0, V, 96)]
    # the token most often among the top 5 of the unmodified model: its tied group lands at the top-n cut there
    ref = pkg.Engine(base, max_gpt=128)
    lg = ref.forward(seq)
    ref.close()
    top5 = np.argsort(-lg.astype(np.float64), axis=1, kind="stable")[:, :5]
    src = int(np.bincount(top5.ravel(), minlength=V).argmax())
    group = sorted(set([src] + [int(x) for x in rng.choice(V, 40, replace=False)]))[:30]
    if src not in group:
        group = sorted(group[:29] + [src])
    path = tied_model(base, str(tmp_path / "tied.bin"), L, E, group, src)
    eng = pkg.Engine(path, max_gpt=128)
    ref = pkg.Engine(path, max_gpt=128)
    ref.set_option("prefill_min", 2)
    start = eng.slot_download(0)
    # a member of the tied group is the target at every third position and wherever the group is near the top
    hot = (top5 == src).any(axis=1)
    inside = np.array([t % 3 == 0 or bool(hot[t]) for t in range(len(seq))])
    targets = [group[t % len(group)] if inside[t] else int(rng.integers(0, V)) for t in range(len(seq))]
    res = eng.score_streams([(0, seq)], [targets], top_n=20)[0]
    logits = alone_logits(ref, start, seq, True)
    check_against_rule(res, logits, targets, 20)
    gv = logits[:, group[0]].astype(np.float64)
    assert all(np.array_equal(logits[:, g], logits[:, group[0]]) for g in group)
    above = (logits.astype(np.float64) > gv[:, None]).sum(axis=1)
    straddle = above < 20  # 30 tied tokens with fewer than 20 above: the top-20 cut falls inside the group
    assert straddle.sum() >= 1, "no row with the tied group at the top-20 cut"
    assert (straddle & inside).sum() >= 1, "no row with the target inside a tied group at the cut"
    # the rank of a tied target counts the tied tokens of lower index
    for t in np.nonzero(straddle & inside)[0]:
        assert int(res["ranks"][t]) == int(above[t]) + group.index(targets[t])
    eng.close()
    ref.close()


@pytest.mark.parametrize("L,E", SHAPES)
def test_consistency_with_argmax_and_top_entries(pkg, make_model, L, E):
    eng = pkg.Engine(make_model(L, E), max_gpt=128)
    rng = np.random.default_rng(11)
    slots = [3, 0, 7, 12]
    start = warm_slots(eng, slots, rng)
    seqs = [[int(x) for x in rng.integers(0, V, n)] for n in (5, 20, 1, 30)]
    streams = list(zip(slots, seqs))
    _, nxt = eng.forward_streams(streams, want_logits=False, want_next=True)
    for s in slots:
        eng.slot_upload(s, start[s])
    ta = random_targets(rng, seqs, 0.0)
    a = eng.score_streams(streams, ta, top_n=20)
    for i, r in enumerate(a):
        assert int(r["top_tokens"][-1][0]) == int(nxt[i])  # the first top entry is the device arg-max
        for t in range(len(seqs[i])):
            assert (int(r["ranks"][t]) == 0) == (ta[i][t] == int(r["top_tokens"][t][0]))
    # each position targets its k-th top entry (k = t % 20): the rank is k and the logprob the top entry's, bit for bit
    tb = [[int(r["top_tokens"][t][t % 20]) for t in range(len(s))] for r, s in zip(a, seqs)]
    for s in slots:
        eng.slot_upload(s, start[s])
    b = eng.score_streams(streams, tb)
    hits = 0
    for i, (ra, rb) in enumerate(zip(a, b)):
        for t in range(len(seqs[i])):
            k = t % 20
            assert int(rb["ranks"][t]) == k
            assert rb["logprobs"][t].tobytes() == ra["top_logprobs"][t][k].tobytes()
        # rank 0 exactly when the target is forward_streams' arg-max of the row (both cases occur: k = 4, 19, 0, 9)
        assert (int(rb["ranks"][-1]) == 0) == (tb[i][-1] == int(nxt[i]))
        hits += tb[i][-1] == int(nxt[i])
    assert 0 < hits < len(seqs)
    eng.close()


def raw_score(eng, tokens, slots, lens, targets, top_n, lp=True, top=True, tg=True):
    """rwkv_b200_score_streams with any of its arrays left NULL: (rc, error message)."""
    P, D = ctypes.POINTER(ctypes.c_ulonglong), ctypes.POINTER(ctypes.c_double)
    arr = lambda a, t: np.ascontiguousarray(a, t)
    tok, sl, ln, tgt = arr(tokens, np.uint64), arr(slots, np.uint64), arr(lens, np.uint64), arr(targets, np.uint64)
    n = len(tok)
    out_lp, out_rank = np.empty(n), np.empty(n, np.uint64)
    out_tt, out_tl = np.empty(max(1, n * top_n), np.uint64), np.empty(max(1, n * top_n))
    rc = eng.lib.rwkv_b200_score_streams(eng.h, tok.ctypes.data_as(P), n, sl.ctypes.data_as(P), ln.ctypes.data_as(P), len(sl),
                                         tgt.ctypes.data_as(P) if tg else None, top_n, out_lp.ctypes.data_as(D) if lp else None,
                                         out_rank.ctypes.data_as(P), out_tt.ctypes.data_as(P) if top else None,
                                         out_tl.ctypes.data_as(D) if top else None)
    return rc, eng.lib.rwkv_b200_last_error().decode()


@pytest.mark.parametrize("L,E", SHAPES)
def test_state_slots_and_chunks(pkg, make_model, L, E):
    eng = pkg.Engine(make_model(L, E), max_gpt=300)
    rng = np.random.default_rng(21)
    slots = [4, 1, 30, 22]
    warm_slots(eng, list(range(0, 300, 7)), rng)
    before = all_states(eng)
    seqs = [[int(x) for x in rng.integers(0, V, n)] for n in (150, 9, 1, 40)]  # 200 tokens: passes of 128 and 72
    streams = list(zip(slots, seqs))
    tg = random_targets(rng, seqs)
    res = eng.score_streams(streams, tg, top_n=5)
    after_score = all_states(eng)
    eng.state_upload(before, eng.max_gpt)
    eng.forward_streams(streams, want_logits=False)
    after_fwd = all_states(eng)
    assert same_state(after_score, after_fwd)
    n = eng.n_layers * eng.n_embed
    for s in range(eng.max_gpt):
        if s not in slots:
            assert all(np.array_equal(after_score[k][s * n:(s + 1) * n], before[k][s * n:(s + 1) * n]) for k in KEYS), s
    # the 150-token stream across the pass boundary scores as it does alone
    eng.state_upload(before, eng.max_gpt)
    alone = eng.score_streams([streams[0]], [tg[0]], top_n=5)[0]
    for k in ("logprobs", "ranks", "top_tokens", "top_logprobs"):
        assert res[0][k].tobytes() == alone[k].tobytes(), k
    # a 300-token document in three chunks, targets linked across the cuts, equals one call
    doc = [int(x) for x in rng.integers(0, V, 300)]
    eng.slot_zero(0)
    whole = eng.score_streams([(0, doc)], top_n=3)[0]
    state_whole = eng.slot_download(0)
    eng.slot_zero(0)
    parts = []
    for c0 in (0, 100, 200):
        chunk = doc[c0:c0 + 100]
        nxt = doc[c0 + 1:c0 + 101] + ([None] if c0 == 200 else [])
        parts.append(eng.score_streams([(0, chunk)], [nxt], top_n=3)[0])
    state_chunks = eng.slot_download(0)
    for k in ("logprobs", "ranks", "top_tokens", "top_logprobs"):
        assert np.concatenate([p[k] for p in parts]).tobytes() == whole[k].tobytes(), k
    assert same_state(state_whole, state_chunks)
    eng.close()


def test_sparse_targets(pkg, make_model):
    eng = pkg.Engine(make_model(3, 768), max_gpt=300)
    rng = np.random.default_rng(8)
    seqs = [[int(x) for x in rng.integers(0, V, n)] for n in (60, 25, 3)]
    streams = list(zip([2, 5, 0], seqs))
    full = random_targets(rng, seqs, 0.0)
    some = [[y if rng.random() < 0.3 else None for y in row] for row in full]
    before = all_states(eng)
    a = eng.score_streams(streams, full, top_n=4)
    eng.state_upload(before, eng.max_gpt)
    b = eng.score_streams(streams, some, top_n=4)
    for ra, rb, row in zip(a, b, some):
        on = np.array([y is not None for y in row])
        for k in ("logprobs", "ranks", "top_tokens", "top_logprobs"):
            assert ra[k][on].tobytes() == rb[k][on].tobytes(), k
        assert np.all(np.isnan(rb["logprobs"][~on]))
    # no target at all: the state of a state-only forward_streams, with the same launches
    eng.state_upload(before, eng.max_gpt)
    c0 = eng.launch_count
    eng.score_streams(streams, [[None] * len(s) for s in seqs])
    c_none = eng.launch_count - c0
    st_none = all_states(eng)
    eng.state_upload(before, eng.max_gpt)
    c0 = eng.launch_count
    eng.forward_streams(streams, want_logits=False)
    c_fwd = eng.launch_count - c0
    assert same_state(st_none, all_states(eng))
    assert c_none == c_fwd
    # a long unscored prefix runs no head: 300 tokens are passes of 128, 128 and 44; scoring only the last 10 positions
    # adds one head (and the scoring kernel), scoring every position three heads
    doc = [int(x) for x in rng.integers(0, V, 300)]
    counts = {}
    for name, tg in (("none", [None] * 300), ("tail", [None] * 290 + doc[:10]), ("all", doc[1:] + [None])):
        eng.slot_zero(0)
        eng.score_streams([(0, doc)], [tg])  # the first call of a shape records its graph
        eng.slot_zero(0)
        c0 = eng.launch_count
        eng.score_streams([(0, doc)], [tg])
        counts[name] = eng.launch_count - c0
    head = counts["tail"] - counts["none"] - 1
    assert head > 0
    assert counts["all"] - counts["none"] - 1 == 3 * head
    eng.close()


def test_multiple_choice(pkg, make_model):
    """A context prefilled once and forked to four slots, four continuations scored in one call, against each
    context + continuation scored alone."""
    eng = pkg.Engine(make_model(2, 2048), max_gpt=128)
    rng = np.random.default_rng(13)
    ctx = [int(x) for x in rng.integers(0, V, 41)]
    conts = [[int(x) for x in rng.integers(0, V, n)] for n in (5, 9, 12, 3)]
    eng.slot_zero(0)
    eng.forward_streams([(0, ctx[:-1])], want_logits=False)
    for s in range(1, 5):
        eng.slot_copy(0, s)
    # stream i feeds the last context token and the continuation but its last token; it targets the continuation
    streams = [(i + 1, [ctx[-1]] + c[:-1]) for i, c in enumerate(conts)]
    got = eng.score_streams(streams, [c for c in conts], top_n=2)
    for i, c in enumerate(conts):
        eng.slot_zero(6)
        tg = [None] * (len(ctx) - 1) + c
        alone = eng.score_streams([(6, ctx + c[:-1])], [tg], top_n=2)[0]
        for k in ("logprobs", "ranks", "top_tokens", "top_logprobs"):
            assert got[i][k].tobytes() == alone[k][len(ctx) - 1:].tobytes(), (i, k)
        assert np.isfinite(got[i]["logprobs"]).all()
    eng.close()


def test_determinism_and_refusals(pkg, make_model):
    eng = pkg.Engine(make_model(3, 768), max_gpt=64)
    rng = np.random.default_rng(17)
    slots = [3, 9]
    warm_slots(eng, slots, rng)
    seqs = [[int(x) for x in rng.integers(0, V, n)] for n in (12, 20)]
    streams = list(zip(slots, seqs))
    tg = random_targets(rng, seqs)
    before = all_states(eng)
    a = eng.score_streams(streams, tg, top_n=20)
    eng.state_upload(before, eng.max_gpt)
    b = eng.score_streams(streams, tg, top_n=20)
    for ra, rb in zip(a, b):
        for k in ra:
            assert ra[k].tobytes() == rb[k].tobytes(), k
    # after scoring no per-stream logits are held
    with pytest.raises(pkg.EngineError, match="no per-stream logits"):
        eng.sample_typical_streams(1.0, [0.5, 0.5])
    with pytest.raises(pkg.EngineError, match="no per-stream logits"):
        eng.sample_streams([pkg.Sampler(0.0)] * 2, None)
    toks = seqs[0] + seqs[1]
    lens = [12, 20]
    ok = [y if y is not None else 2 ** 64 - 1 for row in tg for y in row]
    bad_tg = list(ok)
    bad_tg[15] = V
    st = all_states(eng)
    cases = [
        (dict(targets=bad_tg), "targets[15] = 50277 (stream 1, position 3)"),
        (dict(top_n=21), "top_n 21 > 20"),
        (dict(lp=False), "logprobs_out is NULL"),
        (dict(top_n=3, top=False), "top_n = 3 needs top_tokens_out and top_logprobs_out"),
        (dict(tg=False), "targets is NULL"),
        (dict(slots=[3, 3]), "slot 3 appears twice"),
        (dict(lens=[12, 19]), "the lengths add up to 31"),
    ]
    for kw, msg in cases:
        args = dict(tokens=toks, slots=slots, lens=lens, targets=ok, top_n=0)
        args.update({k: v for k, v in kw.items() if k in args})
        flags = {k: v for k, v in kw.items() if k in ("lp", "top", "tg")}
        rc, err = raw_score(eng, args["tokens"], args["slots"], args["lens"], args["targets"], args["top_n"], **flags)
        assert rc != 0 and msg in err and err.startswith("score_streams: "), (msg, err)
        assert same_state(st, all_states(eng)), msg
    eng.close()
