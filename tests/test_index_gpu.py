"""State indexes on the device (rwkv_b200_index_*, Engine.create_index, Engine.embed).

Entries are held bit for bit to slot_download's dd over the index's layers; distances to a float64 numpy restatement
of the rule (within 1e-10 relative) and, bit for bit, to themselves across query batches, index sizes and duplicate
uploads; rankings to numpy's wherever the k-th and (k+1)-th distances are apart by more than that tolerance; refusals
leave the index and every slot unchanged; and Engine.embed's entries equal each document run alone from a zeroed slot,
the ragged-pass invariant on the tensor cores."""
import ctypes

import numpy as np
import pytest

from decoding import KEYS5, SHAPES, bits, rand_tokens

pytestmark = pytest.mark.gpu

MAX_GPT = 8
QB = 8        # rk::kIdxQB: queries per scan
SEL = 4096    # rk::kIdxSelN: pairs one selection CTA sorts
TOL = 1e-10
WIDTHS = SHAPES + [(1, 5120)]


@pytest.fixture(scope="module", params=WIDTHS, ids=["%dx%d" % s for s in WIDTHS])
def eng(request, pkg, make_model):
    """An engine whose every slot holds the state after a few random tokens."""
    L, E = request.param
    e = pkg.Engine(make_model(L, E), max_gpt=MAX_GPT)
    for i in range(3):
        e.forward_streams([(s, rand_tokens(1, 7 + 10 * s + i)) for s in range(MAX_GPT)], want_logits=False)
    yield e
    e.close()


def host_dist(a, b, E):
    """(l1, l2) of query vector a against the rows of b, in float64."""
    d = np.atleast_2d(b) - a
    return np.abs(d).sum(axis=1) / E, np.sqrt((d * d).sum(axis=1) / E)


def set_query(eng, slot, vec, lb):
    """Slot `slot`'s dd holds `vec` over layers lb.. (the rest of the slot stays as it is)."""
    st = eng.slot_download(slot)
    dd = st["dd"].copy()
    dd[lb * eng.n_embed:lb * eng.n_embed + len(vec)] = vec
    eng.slot_upload(slot, {"dd": dd})


def check_search(idx, ent, l1, l2, found, qvecs, vecs, live_ids, k, metric, E):
    """Distances within TOL of numpy, each list sorted by (metric, id), ids numpy's where the cut is clear."""
    live_ids = np.asarray(live_ids)
    for q, a in enumerate(qvecs):
        h1, h2 = host_dist(a, vecs[live_ids], E)
        f = int(found[q])
        assert f == min(k, len(live_ids))
        assert np.all(ent[q, f:] == 2 ** 64 - 1) and np.all(np.isnan(l1[q, f:])) and np.all(np.isnan(l2[q, f:]))
        pos = {int(e): i for i, e in enumerate(live_ids)}
        got = [pos[int(e)] for e in ent[q, :f]]
        assert np.allclose(l1[q, :f], h1[got], rtol=TOL, atol=0) and np.allclose(l2[q, :f], h2[got], rtol=TOL, atol=0)
        key = l1[q, :f] if metric == "l1" else l2[q, :f]
        for i in range(f - 1):
            assert key[i] < key[i + 1] or (key[i] == key[i + 1] and ent[q, i] < ent[q, i + 1]), "query %d position %d" % (q, i)
        hk = h1 if metric == "l1" else h2
        order = np.lexsort((live_ids, hk))
        if f < len(live_ids):
            gap = hk[order[f]] - hk[order[f - 1]]
            if gap <= TOL * max(hk[order[f]], 1e-300):
                continue
        assert sorted(int(e) for e in ent[q, :f]) == sorted(int(live_ids[i]) for i in order[:f]), "query %d" % q


def test_add_matches_slot_download(pkg, eng):
    before = eng.state_download(MAX_GPT)
    E, L = eng.n_embed, eng.n_layers
    for layers in (None, range(L // 2, L // 2 + 1)):
        lb, nl = (0, L) if layers is None else (layers[0], len(layers))
        with eng.create_index(16, layers) as idx:
            slots = [3, 1, 5, 1]
            ids = idx.add(slots)
            assert [int(x) for x in ids] == [0, 1, 2, 3]
            got = idx.vectors(ids)
            for s, v in zip(slots, got):
                assert bits(v) == bits(eng.slot_download(s)["dd"][lb * E:(lb + nl) * E])
    after = eng.state_download(MAX_GPT)
    for k in KEYS5:
        assert bits(after[k]) == bits(before[k]), "state %s changed" % k


@pytest.mark.parametrize("metric", ["l1", "l2"])
def test_distances_and_ranking(pkg, eng, metric):
    E, L = eng.n_embed, eng.n_layers
    lb = L - 1
    D = E
    rng = np.random.default_rng(5)
    vecs = rng.normal(0.0, 1.0, (600, D)) * rng.uniform(0.2, 2.0, (600, 1))
    qvecs = [vecs[17] + rng.normal(0, 0.05, D), rng.normal(0.0, 1.0, D), vecs[400] * 1.01]
    for q, v in enumerate(qvecs):
        set_query(eng, q, v, lb)
    qvecs = [eng.slot_download(q)["dd"][lb * E:(lb + 1) * E] for q in range(3)]
    with eng.create_index(600, range(lb, L)) as idx:
        ids = idx.upload(vecs)
        assert [int(x) for x in ids] == list(range(600))
        assert bits(idx.vectors(ids)) == bits(vecs)
        for k in (1, 7, 256):
            ent, l1, l2, found = idx.search([0, 1, 2], k, metric)
            check_search(idx, ent, l1, l2, found, qvecs, vecs, ids, k, metric, E)


def test_independence_of_batch_size_and_duplicates(pkg, eng):
    E, L = eng.n_embed, eng.n_layers
    D = L * E
    rng = np.random.default_rng(11)
    n_max = 5000 if D <= 4096 else 2500
    vecs = rng.normal(0.0, 1.0, (n_max, D))
    qvecs = [eng.slot_download(q)["dd"] for q in range(MAX_GPT)]
    queries = [int(x) for x in rng.integers(0, MAX_GPT, 3 * QB + 1)]
    seen = {}  # (query slot, entry) -> (l1 bits, l2 bits) across every search below
    def record(qslots, ent, l1, l2, found):
        for i, q in enumerate(qslots):
            for j in range(int(found[i])):
                key, val = (q, int(ent[i, j])), (bits(l1[i, j]), bits(l2[i, j]))
                assert seen.setdefault(key, val) == val, "distance of entry %d to slot %d changed" % key[::-1]
    with eng.create_index(n_max, None) as idx:
        idx.upload(vecs)
        batch = idx.search(queries, 256, "l2")
        record(queries, *batch)
        for i, q in enumerate(queries[:QB + 2]):
            alone = idx.search([q], 256, "l2")
            for a, b in zip(alone, batch):
                assert bits(a[0]) == bits(b[i]), "query %d alone and in a batch" % i
        check_search(idx, *batch[:4], [qvecs[q] for q in queries], vecs, np.arange(n_max), 256, "l2", E)
    for n in (1, 2, 7, 8, 9, SEL - 1, SEL, SEL + 1, n_max):
        if n > n_max:
            continue
        with eng.create_index(n, None) as idx:
            idx.upload(vecs[:n])
            for metric in ("l1", "l2"):
                qs = list(range(MAX_GPT))
                res = idx.search(qs, 7, metric)
                record(qs, *res)
                assert [int(f) for f in res[3]] == [min(7, n)] * MAX_GPT
    # the same vector twice: the same bits, and distance exactly 0 to a query that equals it
    v = vecs[3]
    set_query(eng, 0, v, 0)
    with eng.create_index(8, None) as idx:
        ids = idx.upload(np.stack([vecs[1], v, vecs[2], v, v]))
        ent, l1, l2, found = idx.search([0], 5, "l1")
        assert [int(x) for x in ent[0, :3]] == [1, 3, 4]
        assert np.all(l1[0, :3] == 0.0) and np.all(l2[0, :3] == 0.0)
        assert bits(idx.vectors([1])) == bits(idx.vectors([3])) == bits(v)


def test_ties_and_nan(pkg, eng):
    E, L = eng.n_embed, eng.n_layers
    D = L * E
    rng = np.random.default_rng(3)
    w = rng.normal(0, 1, D)
    others = rng.normal(0, 1, (4, D)) * 3.0
    nan_slot = MAX_GPT - 1
    st = eng.slot_download(nan_slot)
    dd = st["dd"].copy()
    dd[D // 2] = np.nan
    eng.slot_upload(nan_slot, {"dd": dd})
    set_query(eng, 0, w + 0.01, 0)
    with eng.create_index(16, None) as idx:
        a = idx.add([nan_slot])
        b = idx.upload(np.stack([w, others[0], w, others[1], w]))
        c = idx.add([nan_slot])
        for metric in ("l1", "l2"):
            ent, l1, l2, found = idx.search([0], 16, metric)
            assert int(found[0]) == 7
            order = [int(x) for x in ent[0, :7]]
            assert order[:3] == [int(b[0]), int(b[2]), int(b[4])]
            assert order[5:] == [int(a[0]), int(c[0])]
            assert np.all(np.isnan(l1[0, 5:7])) and np.all(np.isnan(l2[0, 5:7]))
            assert bits(l1[0, 0]) == bits(l1[0, 1]) == bits(l1[0, 2])


def test_remove(pkg, eng):
    E, L = eng.n_embed, eng.n_layers
    D = L * E
    rng = np.random.default_rng(8)
    vecs = rng.normal(0, 1, (40, D))
    qvecs = [eng.slot_download(q)["dd"] for q in range(2)]
    with eng.create_index(40, None) as idx:
        ids = idx.upload(vecs)
        gone = [0, 5, 6, 7, 39, 20]
        idx.remove(gone)
        live = [i for i in range(40) if i not in gone]
        for k in (3, 34, 40, 256):
            ent, l1, l2, found = idx.search([0, 1], k, "l1")
            assert [int(f) for f in found] == [min(k, 34)] * 2
            assert not set(int(e) for e in ent.ravel()) & set(gone)
            check_search(idx, ent, l1, l2, found, qvecs, vecs, live, k, "l1", E)
        with pytest.raises(pkg.EngineError, match="entry 5 was removed"):
            idx.remove([5])
        with pytest.raises(pkg.EngineError, match="entry 5 was removed"):
            idx.vectors([5])
        idx.remove(live)
        ent, l1, l2, found = idx.search([0], 4, "l2")
        assert int(found[0]) == 0 and np.all(ent == 2 ** 64 - 1) and np.all(np.isnan(l1)) and np.all(np.isnan(l2))
        # capacity counts every add: the removed rows are not reclaimed
        with pytest.raises(pkg.EngineError, match="would pass the capacity"):
            idx.upload(vecs[:1])
        assert int(ids[-1]) == 39


def test_refusals_change_nothing(pkg, eng):
    E, L = eng.n_embed, eng.n_layers
    D = L * E
    lib = eng.lib
    P, Dp = ctypes.POINTER(ctypes.c_ulonglong), ctypes.POINTER(ctypes.c_double)
    rng = np.random.default_rng(2)
    vecs = rng.normal(0, 1, (6, D))
    idx = eng.create_index(8, None)
    ids = idx.upload(vecs[:3])
    ids = np.concatenate([ids, idx.add([2, 4])])
    idx.remove([1])
    keep = [0, 2, 3, 4]
    want_v = bits(idx.vectors(keep))
    want_s = [bits(x) for x in idx.search([0, 3], 8, "l1")]
    before = eng.state_download(MAX_GPT)
    err = pkg.EngineError
    iid = ctypes.c_ulonglong()
    a = np.array([0], np.uint64)
    out = np.zeros(8, np.uint64)
    f1, f2, fo = np.zeros(8), np.zeros(8), np.zeros(1, np.uint64)
    p, d = (lambda x: x.ctypes.data_as(P)), (lambda x: x.ctypes.data_as(Dp))

    def refused(rc, msg):
        assert rc != 0 and msg.encode() in lib.rwkv_b200_last_error(), lib.rwkv_b200_last_error()

    with pytest.raises(err, match="not a non-empty range"):
        eng.create_index(4, range(L, L + 1))
    refused(lib.rwkv_b200_index_create(eng.h, 0, 0, 4, ctypes.byref(iid)), "not a non-empty range")
    refused(lib.rwkv_b200_index_create(eng.h, 0, L + 1, 4, ctypes.byref(iid)), "not a non-empty range")
    with pytest.raises(err, match="capacity 0"):
        eng.create_index(0)
    with pytest.raises(err, match="index_create: .*entries of"):
        eng.create_index((2 ** 50) // (D * 8))  # about a petabyte: the allocation fails with a message
    with pytest.raises(err, match="would pass the capacity"):
        idx.upload(vecs[:4])
    with pytest.raises(err, match="would pass the capacity"):
        idx.add([0, 1, 2, 3])
    with pytest.raises(err, match="slot %d >= max_gpt" % MAX_GPT):
        idx.add([0, MAX_GPT])
    bad = vecs[:2].copy()
    bad[1, 7] = np.nan
    with pytest.raises(err, match="element 7 of vector 1 is not finite"):
        idx.upload(bad)
    bad[1, 7] = np.inf
    with pytest.raises(err, match="not finite"):
        idx.upload(bad)
    with pytest.raises(err, match="entry 9 was never added"):
        idx.vectors([0, 9])
    with pytest.raises(err, match="entry 9 was never added"):
        idx.remove([0, 9])
    with pytest.raises(err, match="entry 1 was removed"):
        idx.remove([0, 1])
    with pytest.raises(err, match="entry 0 appears twice"):
        idx.remove([0, 0])
    refused(lib.rwkv_b200_index_search(eng.h, idx.h, p(a), 1, 2, 4, p(out), d(f1), d(f2), p(fo)), "unknown metric 2")
    with pytest.raises(err, match="k = 0"):
        idx.search([0], 0)
    with pytest.raises(err, match="k = 257"):
        idx.search([0], 257)
    with pytest.raises(err, match="slot %d >= max_gpt" % MAX_GPT):
        idx.search([0, MAX_GPT], 4)
    refused(lib.rwkv_b200_index_search(eng.h, idx.h, p(a), 0, 0, 4, p(out), d(f1), d(f2), p(fo)), "no queries")
    refused(lib.rwkv_b200_index_search(eng.h, idx.h, p(a), 1, 0, 4, None, d(f1), d(f2), p(fo)), "null argument")
    refused(lib.rwkv_b200_index_add_slots(eng.h, idx.h, None, 1, p(out)), "no slots")
    refused(lib.rwkv_b200_index_upload(eng.h, idx.h, None, 1, p(out)), "no vectors")
    refused(lib.rwkv_b200_index_download(eng.h, idx.h, p(a), 1, None), "no entries")
    refused(lib.rwkv_b200_index_remove(eng.h, idx.h, None, 1), "no entries")
    refused(lib.rwkv_b200_index_search(eng.h, idx.h + 100, p(a), 1, 0, 4, p(out), d(f1), d(f2), p(fo)), "unknown or freed")
    assert bits(idx.vectors(keep)) == want_v
    assert [bits(x) for x in idx.search([0, 3], 8, "l1")] == want_s
    after = eng.state_download(MAX_GPT)
    for k in KEYS5:
        assert bits(after[k]) == bits(before[k]), "state %s changed" % k
    h = idx.h
    idx.close()
    refused(lib.rwkv_b200_index_search(eng.h, h, p(a), 1, 0, 4, p(out), d(f1), d(f2), p(fo)), "unknown or freed")
    refused(lib.rwkv_b200_index_free(eng.h, h), "unknown or freed")


# -- the vectordb workflow -------------------------------------------------------------------------------------------

DOC_LENGTHS = [5, 9, 2, 14, 3, 7, 11, 4, 6, 8, 2, 13]
QUERY_LENGTHS = [4, 6, 3]


@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%d" % s for s in SHAPES])
def test_embed_is_the_vectordb_loop(pkg, make_model, shape):
    L, E = shape
    path = make_model(L, E)
    max_gpt = 16
    a = pkg.Engine(path, max_gpt=max_gpt)
    a.set_option("prefill_min", 2)
    docs = [rand_tokens(n, 100 + i) for i, n in enumerate(DOC_LENGTHS)]
    queries = [list(docs[3][:4]), rand_tokens(6, 900), list(docs[7][:3])]
    calls = []
    orig = a.forward_streams
    a.forward_streams = lambda streams, **kw: (calls.append([len(t) for _, t in streams]), orig(streams, **kw))[1]
    with a.create_index(len(docs), None) as idx:
        ids = a.embed(docs, [0, 2, 5], idx)
        assert sorted(ids) == list(range(len(docs)))
        assert all(sum(c) >= 2 for c in calls), calls  # every packed call runs on the tensor cores
        assert any(len(c) > 1 for c in calls) and sum(map(sum, calls)) == sum(DOC_LENGTHS)
        # each document alone from a zeroed slot, on the tensor cores
        b = pkg.Engine(path, max_gpt=max_gpt)
        b.set_option("prefill_min", 2)
        ref = []
        for doc in docs:
            b.slot_zero(0)
            b.forward_streams([(0, doc)], want_logits=False)
            ref.append(b.slot_download(0)["dd"])
        for i, e in enumerate(ids):
            assert bits(idx.vectors([e])[0]) == bits(ref[i]), "document %d" % i
        # the queries on their own slots, ranked against the host's ranking of the downloaded states
        qslots = [8, 9, 10]
        for s in qslots:
            a.slot_zero(s)
        a.forward_streams(list(zip(qslots, queries)), want_logits=False)
        qref = []
        for q in queries:
            b.slot_zero(0)
            b.forward_streams([(0, q)], want_logits=False)
            qref.append(b.slot_download(0)["dd"])
        for s, r in zip(qslots, qref):
            assert bits(a.slot_download(s)["dd"]) == bits(r)
        vecs = np.stack([ref[ids.index(e)] for e in range(len(docs))])
        for metric in ("l1", "l2"):
            ent, l1, l2, found = idx.search(qslots, len(docs), metric)
            check_search(idx, ent, l1, l2, found, qref, vecs, np.arange(len(docs)), len(docs), metric, E)
            for q, r in enumerate(qref):
                h1, h2 = host_dist(r, vecs, E)
                hk = h1 if metric == "l1" else h2
                assert [int(x) for x in ent[q]] == [int(x) for x in np.lexsort((np.arange(len(docs)), hk))]
        b.close()
    a.close()
