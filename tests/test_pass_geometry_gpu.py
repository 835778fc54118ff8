"""The tensor-core pass (csrc/prefill.cuh) at every launch geometry its GEMMs take, against the float64 restatement
(tests/numerics.py, "engine" mode) within numerics.case_tol: logits of every headed row and the four state arrays of
every layer.

A GEMM launch of a pass is decided by three numbers (pf_gemm): the split-K factor ks (1, 2, 4 or 8, from the matrix
shape), the token-block count NB = Tp / 32 (from the padded pass size) and whether K or M ends in a partial tile.
tests/test_pass_geometry_host.py restates that rule for every width the loader accepts and fails if the cases below miss
a reachable (GEMM, ks, NB) cell. The cases:

- Decode-step passes: S one-token rows on scattered slots that hold state, as one forward_streams call, the pass a
  generate_streams step runs. S = 1 (with a pad row), 2, 31, 32, 33, 64, 65, 96, 97 and 128 give NB = 1 to 4, at the
  widths that reach every split: 768 (ffn-V ks 4), 1024 (E x E ks 2, ffn-K 2, ffn-V 8), 2048 (E x E 4, ffn-V 8), 4096
  (E x E 4, ffn-V 4), 5120 (E x E 2, ffn-V 2), and 784, whose K and M end in partial tiles (ks 1 everywhere).
  Then two of those shapes again on other slots and tokens: the recorded CUDA graph is replayed, not recorded again.
- Multi-pass ragged calls of 530 and 600 tokens: streams cross the pass cuts, one spans three passes, one has exactly
  one token on each side of a cut, one pass ends no stream. Each runs with the head on each stream's last row
  (forward_streams, a head smaller than its pass), then again with prefill_graph 0 (the same bits), then with the head
  on every row (score_streams: log-probabilities of every position).
- The prefill_min boundary: 7 tokens run on the decode kernel and 8 on the tensor cores; both match the restatement.

Each width's cases are restated together, as independent streams of one restatement pass (numerics.forward runs
streams independently), so that the weights are converted once per width; each case prints its worst error."""
import ctypes
import time

import numpy as np
import pytest

import numerics as nm
from util import token_stream

pytestmark = pytest.mark.gpu

MAX_GPT = 640
NSLOTS = 131                      # slots that hold state (prime: row i of a case goes to slot (37 i + c) % 131)
STEP_WIDTHS = {768: 2, 784: 2, 1024: 2, 2048: 2, 4096: 1, 5120: 1}   # n_embed -> layers
STEP_ROWS = (1, 2, 31, 32, 33, 64, 65, 96, 97, 128)                  # 1: one stream and a pad row
REPLAY_ROWS = (32, 97)            # recorded by the step cases, replayed under another layout
# Stream lengths of the multi-pass ragged calls (pass cuts at 128, 256, 384, 512).
# 1024: stream 3 has tokens 127 and 128, stream 6 spans passes 1-3 (tokens 230-399; pass 2 ends no stream), stream 9
# crosses 512; the last pass has 18 tokens. 784: stream 1 crosses 128, stream 2 spans passes 1-3 (129-427), stream 5
# has tokens 511 and 512; the last pass has 88 tokens.
RAGGED = {1024: (9, 1, 117, 2, 1, 100, 170, 1, 3, 120, 6), 784: (64, 65, 299, 2, 81, 2, 87)}
BOUNDARY_E = 784
BOUNDARY = ((3, 4), (3, 5))       # at the default prefill_min of 8: 7 tokens (decode kernel), 8 (tensor cores)
PREFILL_MIN = 8
TOP_N = 20


def step_slots(S, c):
    return [(37 * i + c) % NSLOTS for i in range(S)]


def cases(E):
    """The cases of width E, in the order they run: dicts of id, kind (step, replay, ragged, boundary), slots and
    streams (token lists)."""
    rng = np.random.default_rng(E)
    toks = lambda n: [int(t) for t in rng.integers(0, nm.V, size=n)]
    out = []
    for k, S in enumerate(STEP_ROWS):
        n = max(S, 2)
        out.append({"id": "step-%dx%d-S%d%s" % (STEP_WIDTHS[E], E, S, "+pad" if S == 1 else ""), "kind": "step",
                    "slots": step_slots(n, 3 + 7 * k), "streams": [[t] for t in toks(n)]})
    for k, S in enumerate(REPLAY_ROWS):
        out.append({"id": "replay-%dx%d-S%d" % (STEP_WIDTHS[E], E, S), "kind": "replay",
                    "slots": step_slots(S, 90 + 11 * k)[::-1], "streams": [[t] for t in toks(S)]})
    if E in RAGGED:
        lens = RAGGED[E]
        out.append({"id": "ragged-%dx%d-n%d" % (STEP_WIDTHS[E], E, sum(lens)), "kind": "ragged",
                    "slots": [(13 * i + 5) % NSLOTS for i in range(len(lens))], "streams": [toks(n) for n in lens]})
    if E == BOUNDARY_E:
        for k, lens in enumerate(BOUNDARY):
            out.append({"id": "boundary-%dx%d-T%d" % (STEP_WIDTHS[E], E, sum(lens)), "kind": "boundary",
                        "slots": [20 + 40 * k, 60 + 40 * k], "streams": [toks(n) for n in lens]})
    return out


def slot_states(model):
    """The state each slot holds before every case: two tokens from the zero state, other tokens per slot."""
    return nm.forward(model, [token_stream(2, seed=3000 + s) for s in range(NSLOTS)])[1]


@pytest.fixture(scope="module")
def restated(make_model):
    """E -> (path, model, {case id: (case, initial states, logits, final states, tolerances)}), every case of the
    width restated in one pass (and twice more, nudged, for the tolerances of numerics.stream_tols)."""
    cache = {}

    def get(E):
        if E not in cache:
            path = make_model(STEP_WIDTHS[E], E)
            model = nm.Model(path)
            t0 = time.time()
            pre = slot_states(model)
            cs = cases(E)
            streams = [s for c in cs for s in c["streams"]]
            states = [pre[slot] for c in cs for slot in c["slots"]]
            logits, final = nm.forward(model, streams, states)
            tols = nm.stream_tols(model, streams, states, (logits, final))
            out, i = {}, 0
            for c in cs:
                j = i + len(c["streams"])
                out[c["id"]] = (c, states[i:j], logits[i:j], final[i:j], tols[i:j])
                i = j
            print("\n%d x %d: restated %d cases (%d streams, %d tokens) with tolerances in %.1f s" % (
                model.L, E, len(cs), len(streams), sum(len(s) for s in streams), time.time() - t0))
            cache[E] = (path, model, pre, out)
        return cache[E]
    return get


def upload(eng, model, pre):
    n = model.L * model.E
    eng.state_upload({k: np.concatenate([pre[s][k][:n] for s in range(NSLOTS)]) for k in nm.KEYS}, NSLOTS)


def slot_state(sd, slot, n):
    return {k: sd[k][slot * n:(slot + 1) * n] for k in sd}


def graph_records(eng):
    a = np.zeros(1, np.uint64)
    assert eng.lib.rwkv_b200_debug_read(eng.h, b"graph_records", a.ctypes.data_as(ctypes.c_void_p), 8) == 1
    return int(a[0])


def held(what, model, got, tols):
    """got: per stream (logits error, state error, state array); each within its stream's tolerance. Prints the
    case's worst errors and its tightest tolerances."""
    le = max(g[0] for g in got)
    k = max(range(len(got)), key=lambda i: got[i][1])
    tl, ts = min(t[0] for t in tols), min(t[1] for t in tols)
    print("%s: vs restatement logits %.3g state %.3g (%s); tolerance logits %.3g state %.3g"
          % (what, le, got[k][1], got[k][2], tl, ts))
    bad = ["stream %d: logits %.3g state %s %.3g" % (i, g[0], g[2], g[1]) for i, (g, t) in enumerate(zip(got, tols))
           if not (g[0] <= t[0] and g[1] <= t[1])]
    assert not bad, "%s from the restatement: %s" % (what, "; ".join(bad[:8]))


def streams_errs(model, lg, sd, rec):
    """Per stream of a forward_streams call: (logits error of its last row, state error, worst state array)."""
    c, _, ref_l, ref_s, _ = rec
    n = model.L * model.E
    out = []
    for i, slot in enumerate(c["slots"]):
        le, se, sk = nm.worst([lg[i][None, :]], [ref_l[i][-1:]], [slot_state(sd, slot, n)], [ref_s[i]], model.L, model.E)
        out.append((le, se, sk))
    return out


def run_streams(eng, model, pre, c):
    """(last-row logits, state of every slot, kernel launches) of the case's forward_streams call from the slot states."""
    upload(eng, model, pre)
    l0 = eng.launch_count
    lg, _ = eng.forward_streams(list(zip(c["slots"], c["streams"])))
    launches = eng.launch_count - l0
    assert np.isfinite(lg).all(), "%s: non-finite logits" % c["id"]
    return lg, eng.state_download(NSLOTS), launches


@pytest.mark.parametrize("E", sorted(STEP_WIDTHS))
def test_decode_step_passes(pkg, restated, E):
    path, model, pre, rec = restated(E)
    eng = pkg.Engine(path, max_gpt=MAX_GPT)
    eng.set_option("prefill_min", 2)   # every step on the tensor cores, the lone stream with its pad row too
    for cid, r in rec.items():
        c = r[0]
        if c["kind"] not in ("step", "replay"):
            continue
        before = graph_records(eng)
        lg, sd, _ = run_streams(eng, model, pre, c)
        if c["kind"] == "replay":
            assert graph_records(eng) == before, "%s: the graph of %d rows was recorded again" % (cid, len(c["slots"]))
        held(cid, model, streams_errs(model, lg, sd, r), r[4])
    eng.close()


@pytest.mark.parametrize("E", sorted(RAGGED))
def test_multi_pass_ragged_calls(pkg, restated, E):
    path, model, pre, rec = restated(E)
    (c, _, ref_l, ref_s, tols), = [r for r in rec.values() if r[0]["kind"] == "ragged"]
    n = model.L * model.E
    eng = pkg.Engine(path, max_gpt=MAX_GPT)
    # head on each stream's last row, the passes replayed from recorded graphs
    lg, sd, _ = run_streams(eng, model, pre, c)
    held(c["id"] + " head=2", model, streams_errs(model, lg, sd, rec[c["id"]]), tols)
    # the same call with every pass launched directly: the same bits
    eng.set_option("prefill_graph", 0)
    lg0, sd0, _ = run_streams(eng, model, pre, c)
    assert lg0.tobytes() == lg.tobytes(), "%s: prefill_graph 0 gives other logits" % c["id"]
    for k in sd:
        assert sd0[k].tobytes() == sd[k].tobytes(), "%s: prefill_graph 0 gives another state %s" % (c["id"], k)
    eng.set_option("prefill_graph", 1)
    # head on every row: score_streams' log-probabilities of each position's target and its top tokens, against the
    # restatement's log-softmax. |d log p| <= 2 max|d logits|, so the bound is twice the logits tolerance.
    upload(eng, model, pre)
    targets = [[int(t) for t in np.random.default_rng(E + i).integers(0, nm.V, size=len(s))] for i, s in enumerate(c["streams"])]
    sc = eng.score_streams(list(zip(c["slots"], c["streams"])), targets=targets, top_n=TOP_N)
    sd1 = eng.state_download(NSLOTS)
    for k in sd:
        assert sd1[k].tobytes() == sd[k].tobytes(), "%s: score_streams leaves another state %s" % (c["id"], k)
    got = []
    for i in range(len(c["streams"])):
        ref = np.asarray(ref_l[i], np.float64)
        m = ref.max(axis=1, keepdims=True)
        lp = ref - (m + np.log(np.exp(ref - m).sum(axis=1, keepdims=True)))
        rows = np.arange(len(ref))
        d = np.abs(sc[i]["logprobs"] - lp[rows, targets[i]])
        tt = sc[i]["top_tokens"].astype(np.int64)
        d = np.maximum(d, np.abs(sc[i]["top_logprobs"] - lp[rows[:, None], tt]).max(axis=1))
        scale = np.abs(ref).max(axis=1)
        got.append((float((d / (2 * scale)).max()), 0.0, "-"))
    held(c["id"] + " head=1", model, got, tols)
    eng.close()


def test_prefill_min_boundary(pkg, restated):
    """One token below prefill_min runs on the decode kernel (one launch per token), prefill_min tokens on the tensor
    cores; both match the restatement."""
    path, model, pre, rec = restated(BOUNDARY_E)
    eng = pkg.Engine(path, max_gpt=MAX_GPT)
    eng.set_option("prefill_min", PREFILL_MIN)
    for cid, r in rec.items():
        c = r[0]
        if c["kind"] != "boundary":
            continue
        T = sum(len(s) for s in c["streams"])
        lg, sd, launches = run_streams(eng, model, pre, c)
        assert (launches == T) == (T < PREFILL_MIN), "%s: %d launches for %d tokens" % (cid, launches, T)
        held("%s (%s)" % (cid, "decode kernel" if T < PREFILL_MIN else "tensor cores"), model,
             streams_errs(model, lg, sd, r), r[4])
    eng.close()
