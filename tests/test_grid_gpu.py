"""The decode kernel at every launch geometry and ring schedule the engine accepts, not only the default grid of one CTA
per SM (132 on an H100 SXM).

The grid decides how much of every matrix a CTA owns (csrc/token_kernel.cuh make_slices): at the smallest admitted
grid a CTA holds up to 1006 head rows and 159 ffn keys, at 132 at most 381 and 156. tests/test_grid_host.py derives the
grids each width must visit and fails if GRIDS below misses one.

- Grids against the float64 restatement (tests/numerics.py): the decode-<E> cases of numerics.cases() and the 3-layer
  decode cases of numerics.WIDE, whose mutation sensitivity tests/test_numerics_host.py and test_depth_numerics_host.py
  prove, held to numerics.case_tol at every grid (not to the default grid's bits: the f64 offset and layernorm
  statistic partial sums of the CTAs are added in another order). The restatement does not depend on the grid and is
  computed once per case.
- Greedy picks across CTA slices: forward_greedy, decode_timed without teacher forcing and the teacher-forced logits of
  the same chain agree; a head column copied onto a lower token of another CTA makes a tie that the in-kernel arg-max,
  k_argmax_rows (forward_streams want_next) and score_streams' rank all break towards the lower index.
- Ring depth ("stages"), L2 prefetch distance ("pf_dist") and the traced kernel ("trace") only decide when weight bytes
  arrive or add timestamps: they give the logits and state of the defaults bit for bit, as the copy schedule of
  tests/test_stream_budget_gpu.py does.
- Refusals: grids outside 1..SMs or too small for the slice capacities, ring depths outside 2..12 or above the shared
  memory limit, prefetch distances outside 0..64. A refused option launches nothing and changes nothing."""
import os
import shutil

import numpy as np
import pytest

import numerics as nm
from util import SEED_TOKEN, margin, token_stream

pytestmark = pytest.mark.gpu

KEYS = ("xy", "aa", "bb", "pp", "dd")
DEFAULT_GRID = 132
# Per width, ascending: the smallest admitted grid (which also gives a CTA the most residual elements, ffn keys and
# vocabulary rows), an odd grid with uneven slices, 114 (H100 PCIe) where admitted, and the default
# (tests/test_grid_host.py grids_to_visit).
GRIDS = {
    144: (50, 91, 114, 132), 256: (50, 91, 114, 132), 272: (50, 91, 114, 132), 768: (50, 91, 114, 132),
    784: (50, 91, 114, 132), 1024: (50, 91, 114, 132), 1040: (50, 91, 114, 132), 2048: (52, 91, 114, 132),
    2560: (65, 99, 114, 132), 3072: (78, 105, 114, 132), 3600: (91, 111, 114, 132), 4096: (104, 114, 117, 132),
    5104: (129, 131, 132), 5120: (129, 131, 132),
}
# (case id, L, E): the decode-<E> cases of numerics.cases() and the 3-layer decode cases of numerics.WIDE
CASES = [(c["id"], c["L"], c["E"]) for c in nm.cases() if c["path"] == "decode" and c["kind"] is None and c["edge"] is None]
CASES += [("decode-%dx%d" % (nm.DEPTH_L, E), nm.DEPTH_L, E) for E in sorted(nm.WIDE) if "decode" in nm.WIDE[E]]
DECODE_L = {E: L for cid, L, E in CASES if cid == "decode-%d" % E}

# The shapes of tests/test_stream_budget_gpu.py: the exact consume_sub path over three layers and a bounded one.
SHAPES = {"exact": (3, 4096), "bounded": (2, 784)}
# Ring depths. The deepest ring that fits (5 and 12) is also configure_ring's default, so that entry runs the defaults
# against themselves; 2, 3 and the middle depths are the ones that differ from them.
STAGES = {4096: (2, 3, 4, 5), 784: (2, 3, 7, 12)}
STAGES_OVER = {4096: 6}                             # the first ring depth above the shared-memory limit
PF_DISTS = (0, 1, 64)
GREEDY_STEPS = 32


def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def case_stream(cid, L, E):
    """The tokens of a case: numerics.inputs for decode-<E>; for the 3-layer cases the decode stream numerics.depth_passes
    restates (numerics.wide_streams)."""
    if cid != "decode-%d" % E:
        ids, streams = nm.wide_streams(E)
        return streams[ids.index(cid)]
    return token_stream(8, seed=E)


def run(eng, toks):
    """Every token's logits through the decode kernel from the zero state, and the state after the last."""
    eng.state_zero()
    return eng.forward(toks, mode=1), eng.state_download()


def assert_same(got, want, what):
    (gl, gs), (wl, ws) = got, want
    assert np.array_equal(gl, wl), "%s: logits differ" % what
    for k in KEYS:
        assert np.array_equal(gs[k], ws[k]), "%s: state %s differs" % (what, k)


# -- every grid against the restatement ------------------------------------------------------------------------------

@pytest.mark.parametrize("cid,L,E", CASES, ids=[c[0] for c in CASES])
def test_grid_matches_restatement(pkg, make_model, cid, L, E):
    path = make_model(L, E)
    model = nm.Model(path)
    toks = case_stream(cid, L, E)
    ref_l, ref_s = nm.forward(model, [toks])
    tol_l, tol_s = nm.stream_tols(model, [toks], None, (ref_l, ref_s))[0]
    n_sm = sms()
    grids = [g for g in GRIDS[E] if g <= n_sm]
    assert grids, "%s: no grid of GRIDS[%d] fits %d SMs" % (cid, E, n_sm)
    eng = pkg.Engine(path, max_gpt=len(toks))
    eng.set_option("prefill", 0)  # every token through the decode kernel
    bad = []
    for g in grids:
        eng.set_option("grid", g)
        lg, st = run(eng, toks)
        assert np.isfinite(lg).all(), "%s grid %d: non-finite logits" % (cid, g)
        le, se, sk = nm.worst([lg], ref_l, [st], ref_s, L, E)
        print("%s grid %d: vs restatement logits %.3g state %.3g (%s); tolerance logits %.3g state %.3g"
              % (cid, g, le, se, sk, tol_l, tol_s))
        if not (le <= tol_l and se <= tol_s):
            bad.append("grid %d: logits %.3g state %s %.3g" % (g, le, sk, se))
    eng.close()
    assert not bad, "%s from the restatement: %s" % (cid, "; ".join(bad))


# -- greedy picks across CTA slices ----------------------------------------------------------------------------------

def greedy_grids(E):
    return [g for g in (GRIDS[E][0], DEFAULT_GRID) if g <= sms()]


@pytest.mark.parametrize("E", sorted(DECODE_L))
def test_greedy_chain_across_grids(pkg, make_model, E):
    """forward_greedy for 32 steps from SEED_TOKEN: each pick is the arg-max (first index on ties) of the teacher-forced
    logits of the same engine on that chain, which equal the chain's bit for bit; decode_timed without teacher forcing
    ends in the chain's logits and state."""
    eng = pkg.Engine(make_model(DECODE_L[E], E), max_gpt=GREEDY_STEPS)
    eng.set_option("prefill", 0)
    for g in greedy_grids(E):
        eng.set_option("grid", g)
        eng.state_zero()
        fed, picks, rows, tok = [], [], [], SEED_TOKEN
        for _ in range(GREEDY_STEPS):
            nxt, lg = eng.forward_greedy(tok, want_logits=True)
            fed.append(tok)
            picks.append(int(nxt))
            rows.append(lg.copy())
            tok = int(nxt)
        chain = np.stack(rows), eng.state_download()
        forced = run(eng, fed)
        assert_same(forced, chain, "E=%d grid %d: teacher-forced on the greedy chain" % (E, g))
        argmax = [int(r.argmax()) for r in forced[0]]
        assert picks == argmax, "E=%d grid %d: in-kernel picks %s, arg-max %s" % (E, g, picks, argmax)
        eng.state_zero()
        eng.decode_timed([SEED_TOKEN] * GREEDY_STEPS, teacher_forced=False)
        assert_same((eng.debug_read("logits")[None, :], eng.state_download()), (chain[0][-1:], chain[1]),
                    "E=%d grid %d: decode_timed without teacher forcing" % (E, g))
        print("E=%d grid %d: %d greedy picks, %d distinct" % (E, g, len(picks), len(set(picks))))
    eng.close()


def cta_of(row, grid):
    """(CTA, its first row) that owns vocabulary row `row` at `grid` (single GPU)."""
    for b in range(grid):
        if (nm.V * (b + 1)) // grid > row:
            return b, (nm.V * b) // grid
    raise AssertionError(row)


@pytest.mark.parametrize("E", sorted(DECODE_L))
def test_greedy_tie_across_ctas(pkg, make_model, tmp_path, E):
    """Copy the head column of a prompt's arg-max token v1 onto v2 < v1, the row just below the first row of v1's CTA
    (the lower of that row at the smallest and at the default grid), so v2 lies in another CTA at both. Both logits are
    then the same bits (the head has a scale and an offset per input row), and the in-kernel greedy pick,
    k_argmax_rows and score_streams' rank name v2, the lower index."""
    src = make_model(DECODE_L[E], E)
    grids = greedy_grids(E)
    eng = pkg.Engine(src, max_gpt=8)
    eng.set_option("prefill", 0)
    for seed in range(E, E + 50):   # a prompt whose arg-max lies beyond CTA 0 at every grid, with a clear margin
        prompt = token_stream(8, seed=seed)
        last = run(eng, prompt)[0][-1]
        v1 = int(last.argmax())
        if all(cta_of(v1, g)[0] > 0 for g in grids) and margin(last) > 1e-4:
            break
    else:
        pytest.fail("E=%d: no prompt with an arg-max past CTA 0 and a margin" % E)
    eng.close()
    v2 = min(cta_of(v1, g)[1] for g in grids) - 1
    assert all(cta_of(v2, g)[0] != cta_of(v1, g)[0] for g in grids)
    tie = str(tmp_path / "tie.bin")
    shutil.copyfile(src, tie)
    _, _, t = nm.tensors(tie, mode="r+")
    head = t["head"].reshape(E, nm.V)
    head[:, v2] = head[:, v1]
    head.flush()
    del head, t

    eng = pkg.Engine(tie, max_gpt=2 * len(prompt))
    eng.set_option("prefill", 0)   # forward_streams and score_streams on the decode kernel too
    for g in grids:
        what = "E=%d grid %d: v1 %d (CTA %d), v2 %d (CTA %d)" % (E, g, v1, cta_of(v1, g)[0], v2, cta_of(v2, g)[0])
        eng.set_option("grid", g)
        eng.state_zero()
        for tok in prompt:
            nxt, lg = eng.forward_greedy(tok, want_logits=True)
        assert lg[v1].tobytes() == lg[v2].tobytes(), "%s: the copied column gives other logits" % what
        assert lg[v1] == lg.max() and int(lg.argmax()) == v2, "%s: the tie is not the maximum" % what
        assert int(nxt) == v2, "%s: the in-kernel greedy picks %d" % (what, nxt)
        eng.state_zero()
        lgs, nx = eng.forward_streams([(0, prompt)], want_next=True)
        assert lgs[0].tobytes() == lg.tobytes(), "%s: forward_streams logits differ from forward_greedy's" % what
        assert int(nx[0]) == v2, "%s: k_argmax_rows picks %d" % (what, nx[0])
        eng.state_zero()
        pad = [None] * (len(prompt) - 1)
        sc = eng.score_streams([(0, prompt), (1, prompt)], targets=[pad + [v2], pad + [v1]])
        assert int(sc[0]["ranks"][-1]) == 0 and int(sc[1]["ranks"][-1]) == 1, "%s: ranks %d, %d" % (
            what, sc[0]["ranks"][-1], sc[1]["ranks"][-1])
        print(what + ": tie broken towards v2 by all three")
    eng.close()
    os.remove(tie)


# -- ring depth, L2 prefetch distance and the traced kernel give the same bits ---------------------------------------

def option_sets(E):
    return [{"stages": s} for s in STAGES[E]] + [{"pf_dist": d} for d in PF_DISTS] + [{"trace": 1}]


def with_options(pkg, path, opts, toks):
    """(teacher-forced logits and state, decode_timed greedy logits and state) of one engine with `opts`, a dict of
    some of grid, stages, pf_dist and trace."""
    assert set(opts) <= {"grid", "stages", "pf_dist", "trace"}, opts
    eng = pkg.Engine(path, max_gpt=len(toks))
    eng.set_option("prefill", 0)
    if "grid" in opts:
        eng.set_option("grid", opts["grid"])
    if "stages" in opts:
        eng.set_option("stages", opts["stages"])
    if "pf_dist" in opts:
        eng.set_option("pf_dist", opts["pf_dist"])
    if "trace" in opts:
        eng.set_option("trace", opts["trace"])
    forced = run(eng, toks)
    eng.state_zero()
    eng.decode_timed([SEED_TOKEN] * 24, teacher_forced=False)
    timed = eng.debug_read("logits")[None, :].copy(), eng.state_download()
    eng.close()
    return forced, timed


@pytest.mark.parametrize("kind", sorted(SHAPES))
def test_ring_options_are_bit_identical(pkg, make_model, kind):
    L, E = SHAPES[kind]
    path = make_model(L, E)
    toks = token_stream(6, seed=E)
    want = with_options(pkg, path, {}, toks)
    for opts in option_sets(E):
        got = with_options(pkg, path, opts, toks)
        assert_same(got[0], want[0], "E=%d %s teacher-forced" % (E, opts))
        assert_same(got[1], want[1], "E=%d %s decode_timed" % (E, opts))
    # the smallest grid with the shallowest ring and no L2 prefetch, against that grid with default options
    g = GRIDS[E][0]
    want = with_options(pkg, path, {"grid": g}, toks)
    got = with_options(pkg, path, {"grid": g, "stages": 2, "pf_dist": 0}, toks)
    assert_same(got[0], want[0], "E=%d grid %d stages 2 pf_dist 0 teacher-forced" % (E, g))
    assert_same(got[1], want[1], "E=%d grid %d stages 2 pf_dist 0 decode_timed" % (E, g))


# -- refusals ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", sorted(SHAPES))
def test_refused_options_change_nothing(pkg, make_model, kind):
    L, E = SHAPES[kind]
    toks = token_stream(4, seed=E + 1)
    n_sm = sms()
    eng = pkg.Engine(make_model(L, E), max_gpt=len(toks))
    eng.set_option("prefill", 0)
    want = run(eng, toks)
    refused = [("grid", 0, r"grid=0 must be 1\.\.%d" % n_sm), ("grid", n_sm + 1, r"grid=%d must be 1\.\.%d" % (n_sm + 1, n_sm)),
               ("grid", GRIDS[E][0] - 1, r"a grid of %d CTAs does not fit n_embed=%d" % (GRIDS[E][0] - 1, E)),
               ("stages", 1, r"stages must be 2\.\.12"), ("stages", 13, r"stages must be 2\.\.12"),
               ("pf_dist", -1, r"pf_dist is 0\.\.64 tiles"), ("pf_dist", 65, r"pf_dist is 0\.\.64 tiles")]
    if E in STAGES_OVER:
        refused.append(("stages", STAGES_OVER[E], r"stages=%d needs \d+ bytes of shared memory" % STAGES_OVER[E]))
    for key, value, message in refused:
        launches = eng.launch_count
        with pytest.raises(pkg.EngineError, match=message):
            eng.set_option(key, value)
        assert eng.launch_count == launches, "set_option(%s, %d) launched a kernel" % (key, value)
        assert_same(run(eng, toks), want, "E=%d after the refused set_option(%s, %d)" % (E, key, value))
    eng.close()
