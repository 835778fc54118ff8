"""The engine against the float64 restatement of its own arithmetic (tests/numerics.py, "engine" mode) at production
depth, width and length, held to numerics.case_tol as tests/test_numerics_gpu.py holds its small cases: logits at every
token (each stream's last row on the ragged path) and the state per layer and per array.

- The decode kernel over 3 layers at 4096, 5104 and 5120 (the 7B and 14B variants and the bounded one): the weight
  ring runs on from layer l's ffn-V into layer l+1's K and the exchange tags move on at every layer boundary.
- The tensor cores over 3 layers: 4096 x 128 tokens (Tp 128, split-K on the att and ffn-V GEMMs) and 5104 x 140 (two
  passes, a K tail); two ragged forward_streams calls at 3 x 4096 on 27 slots that hold state, 24 one-token rows and
  three streams filling each 128-token pass, the second call reading the state the first wrote.
- The bench models (bench.model_path): 7B through the decode kernel over 16 golden tokens and as one 64-token chunk,
  14B over 8 and 64; the 1.5B model over its 1024 golden tokens as one chunk (8 passes) and through the decode kernel,
  and one sequence switching paths on one state: 200 tokens on the tensor cores, 24 on the decode kernel, 40 again.
- Greedy feedback at 7B: 32 forward_greedy steps, each fed the device's choice, against the restatement teacher-forced
  on those tokens: each choice is the restatement's arg-max wherever its top-1 / top-2 margin exceeds twice the logits
  tolerance; then decode_timed without teacher forcing ends in the chain's logits and state bit for bit.
- LoRA adapters at production width against tests/lora_numerics.py within numerics.TOL, in one pass of bound and
  unbound slots: 3 x 4096 at rank 64 on all seven matrices (the ffn-V A matrix has 16384 inputs), 2 x 5120 at rank 16.

tests/test_depth_numerics_host.py proves on the CPU that a quantiser bug moves every case here by at least 4 times its
tolerance, including one that hits a single middle or last layer of the bench models. Each model's cases are restated
once per module, together in one pass; each case prints its worst error, its tolerance and the restatement's time."""
import time

import numpy as np
import pytest

import lora_numerics as lm
import numerics as nm
from test_adapter_gpu import make_adapter, restated
from util import ROOT, SEED_TOKEN, margin

pytestmark = pytest.mark.gpu

WIDE_CASES = [(E, path) for E in sorted(nm.WIDE) for path in nm.WIDE[E]]


def bench_path(pkg, workload):
    import sys
    sys.path.insert(0, ROOT)
    import bench
    return bench.model_path(workload, pkg)


def greedy_chain(pkg, path, n):
    """n forward_greedy steps from SEED_TOKEN, each fed the device's pick: (fed tokens, picks, logits [n][V], final
    state), then decode_timed over the same start without teacher forcing: (its last logits, its state)."""
    eng = pkg.Engine(path)
    fed, picks, rows, tok = [], [], [], SEED_TOKEN
    for _ in range(n):
        nxt, lg = eng.forward_greedy(tok, want_logits=True)
        fed.append(tok)
        picks.append(int(nxt))
        rows.append(lg.copy())
        tok = int(nxt)
    chain = eng.state_download()
    eng.state_zero()
    eng.decode_timed([SEED_TOKEN] * n, teacher_forced=False)
    timed = eng.debug_read("logits").copy(), eng.state_download()
    eng.close()
    return {"fed": fed, "picks": picks, "logits": np.stack(rows), "state": chain, "timed": timed}


@pytest.fixture(scope="module")
def groups(pkg, make_model):
    """group -> (model, restated passes of numerics.passes); the 7B group also holds the greedy chain it restates."""
    cache = {}

    def get(group):
        if group not in cache:
            path = make_model(nm.DEPTH_L, group) if group in nm.WIDE else bench_path(pkg, group)
            model = nm.Model(path)
            chain = greedy_chain(pkg, path, nm.BENCH_CASES["7b"]["greedy"]) if group == "7b" else None
            t0 = time.time()
            ps = nm.passes(group, model, greedy=chain and chain["fed"])
            print("\n%s (%d x %d): restated %s with tolerances in %.1f s" % (
                group, model.L, model.E, ", ".join(sorted(set(c for p in ps for c in p["ids"]))), time.time() - t0))
            cache[group] = (path, model, ps, chain)
        return cache[group]
    return get


def restated_case(ps, cid):
    """(streams, initial states, logits, final states, tolerances) of case cid, over the passes that hold it."""
    out = [[], [], [], [], []]
    for p in ps:
        for i, c in enumerate(p["ids"]):
            if c == cid:
                for lst, src in zip(out, (p["streams"], p["states"], p["logits"], p["final"], p["tols"])):
                    lst.append(src[i] if src is not None else None)
    assert out[0], cid
    return out


def layer_errs(got, ref, L, E):
    """Per array, the error of every layer as numerics.state_errs measures it, for a failure message."""
    out = []
    for k in nm.KEYS:
        g = np.asarray(got[k], np.float64)[:L * E].reshape(L, E)
        r = np.asarray(ref[k], np.float64)[:L * E].reshape(L, E)
        den = np.maximum(np.abs(r), 1e-300) if k == "bb" else np.maximum(np.abs(r).max(axis=1, keepdims=True), 1e-30)
        out.append("%s [%s]" % (k, " ".join("%.2g" % e for e in (np.abs(g - r) / den).max(axis=1))))
    return "; ".join(out)


def check(cid, model, got_l, ref_l, got_s, ref_s, tol):
    """One stream: logits row by row and the state per layer and per array within tol = (logits, state)."""
    L, E = model.L, model.E
    assert np.isfinite(got_l).all(), "%s: non-finite logits" % cid
    for k in nm.KEYS:
        assert np.isfinite(got_s[k][:L * E]).all(), "%s: non-finite state %s" % (cid, k)
    got_l, ref_l = np.asarray(got_l, np.float64), np.asarray(ref_l, np.float64)
    per_tok = np.abs(got_l - ref_l).max(axis=-1) / np.maximum(np.abs(ref_l).max(axis=-1), 1e-30)
    errs = nm.state_errs(got_s, ref_s, L, E)
    sk = max(errs, key=errs.get)
    print("%s: vs restatement logits %.3g (worst token %d of %d) state %.3g (%s); tolerance logits %.3g state %.3g"
          % (cid, per_tok.max(), int(per_tok.argmax()), len(per_tok), errs[sk], sk, tol[0], tol[1]))
    bad = np.flatnonzero(per_tok > tol[0])
    assert not bad.size, "%s: logits from the restatement at tokens %s: %s; state %s" % (
        cid, bad[:16].tolist(), " ".join("%.3g" % e for e in per_tok[bad[:16]]), layer_errs(got_s, ref_s, L, E))
    assert errs[sk] <= tol[1], "%s: state %s %.3g from the restatement; per layer %s" % (
        cid, sk, errs[sk], layer_errs(got_s, ref_s, L, E))


def single_stream(pkg, path, toks, path_kind):
    """Every token's logits and the final state of one stream from zeros, on the decode kernel or one GPT chunk."""
    eng = pkg.Engine(path, max_gpt=len(toks))
    eng.set_option("prefill", 0) if path_kind == "decode" else eng.set_option("prefill_min", 2)
    lg = eng.forward(toks, mode=1)
    st = eng.state_download()
    eng.close()
    return lg, st


@pytest.mark.parametrize("E,kind", WIDE_CASES, ids=["%s-%dx%d" % (k, nm.DEPTH_L, E) for E, k in WIDE_CASES])
def test_wide(pkg, groups, E, kind):
    path, model, ps, _ = groups(E)
    cid = "%s-%dx%d" % (kind, nm.DEPTH_L, E)
    streams, _, ref_l, ref_s, tols = restated_case(ps, cid)
    got_l, got_s = single_stream(pkg, path, streams[0], kind)
    check(cid, model, got_l, ref_l[0], got_s, ref_s[0], tols[0])


def test_wide_ragged_calls(pkg, groups):
    """Two forward_streams calls at 3 x 4096 on slots holding state; each stream's last row and its slot after each."""
    path, model, ps, _ = groups(4096)
    n, slots = model.L * model.E, max(nm.RAGGED_SLOTS) + 1
    eng = pkg.Engine(path, max_gpt=128)
    eng.set_option("prefill_min", 2)
    streams, states, _, _, _ = restated_case(ps, "ragged-1")
    up = {k: np.zeros(slots * n) for k in nm.KEYS}
    for slot, s in zip(nm.RAGGED_SLOTS, states):
        for k in nm.KEYS:
            up[k][slot * n:(slot + 1) * n] = s[k]
    eng.state_upload(up, slots)
    for cid in ("ragged-1", "ragged-2"):
        streams, _, ref_l, ref_s, tols = restated_case(ps, cid)
        assert sum(len(s) for s in streams) == 128
        lg, _ = eng.forward_streams(list(zip(nm.RAGGED_SLOTS, streams)))
        sd = eng.state_download(slots)
        for i, slot in enumerate(nm.RAGGED_SLOTS):
            got_s = {k: sd[k][slot * n:(slot + 1) * n] for k in sd}
            check("%s slot %d (%d tokens)" % (cid, slot, len(streams[i])), model, lg[i][None, :], ref_l[i][-1:],
                  got_s, ref_s[i], tols[i])
    eng.close()


@pytest.mark.parametrize("workload", ["7b", "14b"])
@pytest.mark.parametrize("kind", ["decode", "tc"])
def test_bench_model(pkg, groups, workload, kind):
    path, model, ps, _ = groups(workload)
    cid = "%s-%s" % (kind, workload)
    streams, _, ref_l, ref_s, tols = restated_case(ps, cid)
    got_l, got_s = single_stream(pkg, path, streams[0], kind)
    check(cid, model, got_l, ref_l[0], got_s, ref_s[0], tols[0])


@pytest.mark.parametrize("kind", ["decode", "tc"])
def test_long_run(pkg, groups, kind):
    """The 1.5B model over its 1024 golden tokens: one GPT chunk of 8 passes, or 1024 decode-kernel steps."""
    path, model, ps, _ = groups("1b5")
    streams, _, ref_l, ref_s, tols = restated_case(ps, "long-1b5")
    got_l, got_s = single_stream(pkg, path, streams[0], kind)
    check("long-1b5 %s" % kind, model, got_l, ref_l[0], got_s, ref_s[0], tols[0])


def test_path_switching(pkg, groups):
    """One state through the tensor cores, the decode kernel and the tensor cores again, against one restatement."""
    path, model, ps, _ = groups("1b5")
    streams, _, ref_l, ref_s, tols = restated_case(ps, "switch-1b5")
    toks = streams[0]
    a, b, _ = nm.SWITCH
    eng = pkg.Engine(path, max_gpt=a)
    eng.set_option("prefill_min", 2)
    parts = [eng.forward(toks[:a], mode=1)]
    eng.set_option("prefill", 0)
    parts.append(eng.forward(toks[a:a + b], mode=1))
    eng.set_option("prefill", 1)
    parts.append(eng.forward(toks[a + b:], mode=1))
    st = eng.state_download()
    eng.close()
    check("switch-1b5", model, np.concatenate(parts), ref_l[0], st, ref_s[0], tols[0])


def test_greedy_feedback(pkg, groups):
    path, model, ps, chain = groups("7b")
    streams, _, ref_l, ref_s, tols = restated_case(ps, "greedy-7b")
    assert streams[0] == chain["fed"]
    ref, tol = ref_l[0], tols[0]
    checked = 0
    for i, pick in enumerate(chain["picks"]):
        if margin(ref[i]) > 2 * tol[0]:
            assert pick == int(ref[i].argmax()), "step %d: the device picked %d, the restatement %d" % (
                i, pick, int(ref[i].argmax()))
            checked += 1
    print("greedy-7b: %d of %d picks checked against the restatement's arg-max" % (checked, len(chain["picks"])))
    check("greedy-7b", model, chain["logits"], ref, chain["state"], ref_s[0], tol)
    lg, st = chain["timed"]
    assert lg.tobytes() == chain["logits"][-1].tobytes(), "decode_timed's last logits differ from the chain's"
    for k in nm.KEYS:
        assert st[k].tobytes() == chain["state"][k].tobytes(), "decode_timed's state %s differs from the chain's" % k


@pytest.mark.parametrize("L,E,rank", [(3, 4096, 64), (2, 5120, 16)])
def test_lora_at_production_width(pkg, make_model, L, E, rank):
    """Bound and unbound slots in one pass, against the restatement with each stream's adapter."""
    path = make_model(L, E)
    model = nm.Model(path)
    w = make_adapter(L, E, rank, seed=rank + E)
    alpha = 2.0 * rank
    ad = restated(w, alpha, L, E)
    lens, slots, bound = (5, 40, 1, 17), (2, 0, 5, 3), (True, True, False, True)
    streams = [[int(t) for t in np.random.default_rng(E + n).integers(0, nm.V, size=n)] for n in lens]
    eng = pkg.Engine(path, max_gpt=64)
    aid = eng.add_adapter(w, alpha)
    for s, b in zip(slots, bound):
        if b:
            eng.bind_adapter(s, aid)
    lg, _ = eng.forward_streams(list(zip(slots, streams)))
    sd = eng.state_download(max(slots) + 1)
    eng.close()
    t0 = time.time()
    ref_l, ref_s = lm.forward(model, streams, [ad if b else None for b in bound])
    base_l, _ = nm.forward(model, streams)
    print("lora %d x %d rank %d: restated in %.1f s" % (L, E, rank, time.time() - t0))
    n = L * E
    for i, s in enumerate(slots):
        got_s = {k: sd[k][s * n:(s + 1) * n] for k in sd}
        check("lora-%dx%d-r%d slot %d%s" % (L, E, rank, s, "" if bound[i] else " unbound"), model, lg[i][None, :],
              ref_l[i][-1:], got_s, ref_s[i], (nm.TOL, nm.TOL))
        if bound[i]:   # the adapter moves the bound streams far beyond the tolerance
            assert nm.logits_err(ref_l[i][-1:], base_l[i][-1:]) > 100 * nm.TOL
